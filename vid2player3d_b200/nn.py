"""Host side of libb200nn.so (C ABI: include/b200nn.h): the low-level policy MLP and the MVAE mixture-of-experts decoder as
chains of hand-written sm_90a GEMM launches (csrc/b200nn.cu).  Mirrors, by name and argument meaning,

  * the actor of the reference's imitation network (embodied_pose/models/im_network_builder.py:191-230: RunningMeanStd
    normalisation, `actor_mlp` 734 -> 1024 -> 1024 -> 512 with ReLU, linear `mu`) as run by ImitatorPlayer.run_one_step
    (vid2player/players/im_player.py:187-202): `PolicyMLP`;
  * `MixedDecoder.forward(z, c)` (vid2player/motion_vae/model.py:186-252): `MixedDecoder`.

Operands are bf16 with fp32 accumulation (the reference runs the MVAE under autocast, motion_vae/base.py:390-406, and the policy
in fp32; tolerances are stated in tests/test_gpu_nn.py).  Every buffer is allocated once; `forward` is launches only, no
allocation and no host synchronisation, so it can be captured into the step's CUDA graph.  There is no fallback: without the
built library or a CUDA device the constructors raise.
"""
import ctypes as C
import os

import torch

from . import abi, native
from .build import LIB_NN

ACT = {None: 0, "none": 0, "relu": 1, "elu": 2}
_lib = None

ABI_VERSION = 2

LinearDesc = abi.LinearDesc   # b200nn_linear_desc_t, typed pointers: native.fill builds it


# name -> (restype, argtypes) of every function include/b200nn.h declares; lib() applies all of them when it loads the library, so an
# argument too many or too few, or one that does not convert to its C type, raises ctypes.ArgumentError at the call.  Pointers and
# opaque handles are c_void_p.  tests/test_host.py holds the table to the header.
_i32, _f32, _p = C.c_int32, C.c_float, C.c_void_p
SIGNATURES = {
    "b200nn_abi_version": (C.c_int, []),
    "b200nn_linear_desc_size": (C.c_int32, []),
    "b200nn_last_error": (C.c_char_p, []),
    "b200nn_linear_create": (C.c_int, [_p, _i32, _p]),
    "b200nn_linear_destroy": (C.c_int, [_p]),
    "b200nn_linear_run": (C.c_int, [_p, _p]),
    "b200nn_cast_rows": (C.c_int, [_p, _i32, _p, _i32, _i32, _i32, _p, _p, _f32, _f32, _p]),
    "b200nn_cast_rows_masked": (C.c_int, [_p, _i32, _p, _i32, _i32, _i32, _p, _f32, _f32, _p]),
    "b200nn_cast_rows3": (C.c_int, [_p, _i32, _p, _p, _p, _i32, _i32, _i32, _p]),
    "b200nn_gate_softmax": (C.c_int, [_p, _i32, _i32, _p, _p, _i32, _p, _i32, _p]),
}


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_NN):
            raise RuntimeError(f"{LIB_NN} not built - run `python -c 'import __graft_entry__ as g; g.build()'` (no fallback)")
        L = C.CDLL(LIB_NN)
        for name, (restype, argtypes) in SIGNATURES.items():
            try:
                fn = getattr(L, name)
            except AttributeError:
                raise RuntimeError(f"{LIB_NN} has no {name}: built from older sources - rebuild") from None
            fn.restype, fn.argtypes = restype, argtypes
        if L.b200nn_abi_version() != ABI_VERSION:
            raise RuntimeError("libb200nn.so ABI version mismatch - rebuild")
        if L.b200nn_linear_desc_size() != C.sizeof(LinearDesc):   # the descriptor grows by appended fields within one version
            raise RuntimeError(f"libb200nn.so takes a {L.b200nn_linear_desc_size()}-byte b200nn_linear_desc_t, the binding fills "
                               f"{C.sizeof(LinearDesc)} bytes - rebuild")
        _lib = L
    return _lib


def _check(rc):
    if rc != 0:
        raise RuntimeError(f"b200nn error {rc}: {lib().b200nn_last_error().decode()}")


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _up(x, m):
    return (x + m - 1) // m * m


def padded_rows(rows):
    return _up(rows, 128)


def padded_bf16(rows, cols, device):
    """zero-initialised bf16 operand buffer [rows padded to 128, cols padded to 64]: the pad stays zero for its lifetime"""
    return torch.zeros(padded_rows(rows), _up(cols, 64), device=device, dtype=torch.bfloat16)


class Linear:
    """out[:, col0:col0+N] = act(sum_e coef[:, e] (a W_e^T + b_e)); one launch.  weight [E, N, K] or [N, K] float (torch layout:
    out x in), bias [E, N] or [N]; `a` / `out` are buffers from padded_bf16 (out may also be a float [rows, N] tensor).  residual = (float
    tensor [rows, >= cols], cols): a single-expert layer with a float output adds resid[:, :cols] to its first cols outputs before the
    activation and the clamp.  noise = (sigma float [N], seed): the sampled action of the same kind of layer, out = clamp(act(x +
    sigma[col] * eps)) after the residual, eps the counter-based N(0, 1) draw (seed, noise_step, row * ldo + out_col0 + col); the layer
    owns its device step counter `noise_step`, which every launch advances."""

    def __init__(self, a, weight, bias, out, rows, act=None, coef=None, out_col0=0, out_clamp=None, residual=None, noise=None):
        dev = a.device
        if dev.type != "cuda":
            raise RuntimeError("b200nn runs on a CUDA device only (no CPU fallback)")
        w = weight.detach().to(dev, torch.float32)
        b = bias.detach().to(dev, torch.float32)
        if w.dim() == 2:
            w, b = w[None], b[None]
        E, N, K = w.shape
        bn = 128 if E == 1 else 32
        self.n_padded, self.k_padded = _up(N, bn), _up(K, 64)
        assert a.dtype == torch.bfloat16 and a.is_contiguous() and a.shape[1] >= self.k_padded and a.shape[0] >= padded_rows(rows)
        self.w = torch.zeros(E, self.n_padded, self.k_padded, device=dev, dtype=torch.bfloat16)
        self.w[:, :N, :K] = w.to(torch.bfloat16)
        self.b = torch.zeros(E, self.n_padded, device=dev, dtype=torch.float32)
        self.b[:, :N] = b
        self.a, self.out, self.coef = a, out, coef
        out_bf16 = out.dtype == torch.bfloat16
        assert out.is_contiguous() and out.shape[1] >= out_col0 + N and (out_bf16 or out.dtype == torch.float32)
        assert out.shape[0] >= (padded_rows(rows) if out_bf16 else rows)
        if E > 1:
            assert coef is not None and coef.dtype == torch.float32 and coef.is_contiguous() and tuple(coef.shape) == (rows, E)
        resid, cols = residual if residual is not None else (None, 0)
        if resid is not None:
            assert resid.dtype == torch.float32 and resid.stride(-1) == 1 and resid.device == dev and resid.shape[0] >= rows
        self.residual = residual
        self.noise_sigma = self.noise_step = self.noise_done = None
        seed = 0
        if noise is not None:
            sigma, seed = noise
            self.noise_sigma = sigma.detach().to(dev, torch.float32).reshape(-1).contiguous()
            if self.noise_sigma.shape[0] != N:
                raise ValueError(f"noise: {self.noise_sigma.shape[0]} sigmas for a layer of {N} outputs")
            self.noise_step = torch.zeros(1, device=dev, dtype=torch.int64)
            self.noise_done = torch.zeros(1, device=dev, dtype=torch.int32)
        d = native.fill(LinearDesc, dict(lda=a.shape[1], ldw=self.k_padded, ldo=out.shape[1], out_col0=out_col0, rows=rows, n=N,
                                          n_padded=self.n_padded, k_padded=self.k_padded, num_experts=E, act=ACT[act], out_bf16=int(out_bf16),
                                          out_min=out_clamp[0] if out_clamp else None, out_max=out_clamp[1] if out_clamp else None,
                                          ld_resid=resid.stride(0) if resid is not None else None, resid_cols=int(cols),
                                          noise_seed=int(seed) & (2 ** 64 - 1)),
                        dict(a=a, w=self.w, bias=self.b, coef=coef, out=out, resid=resid, noise_sigma=self.noise_sigma,
                             noise_step=self.noise_step, noise_done=self.noise_done))
        self._h = C.c_void_p()
        _check(lib().b200nn_linear_create(C.byref(d), dev.index or 0, C.byref(self._h)))
        self.flops = 2.0 * rows * N * K * E

    def run(self):
        _check(lib().b200nn_linear_run(self._h, _stream()))

    def __del__(self):
        try:
            if self._h:
                lib().b200nn_linear_destroy(self._h)
                self._h = C.c_void_p()
        except Exception:
            pass


def cast_rows(src, dst, cols, mean=None, rstd=None, lo=-3.0e38, hi=3.0e38):
    """dst[:, :cols] = bf16(clamp((src - mean) * rstd, lo, hi)); src float [rows, >= cols], dst bf16 buffer"""
    assert src.dtype == torch.float32 and src.stride(-1) == 1 and dst.dtype == torch.bfloat16
    _check(lib().b200nn_cast_rows(src.data_ptr(), src.stride(0), dst.data_ptr(), dst.shape[1], src.shape[0], cols,
                                  mean.data_ptr() if mean is not None else None, rstd.data_ptr() if rstd is not None else None, lo, hi,
                                  _stream()))


class PolicyMLP:
    """mu = W4 relu(W3 relu(W2 relu(W1 x + b1) + b2) + b3) + b4 with x = clamp((obs - mean) / sqrt(var + eps), -5, 5)
    (im_network_builder.py:191-230 `actor_mlp` + `mu`, RunningMeanStd; im_player.py:187-202).  `layers` = [(weight [out, in],
    bias [out]), ...] in torch nn.Linear layout; the last layer has no activation.  clamp_actions = 1.0 folds
    ImitatorPlayer's `torch.clamp(action, -1, 1)` (im_player.py:198) into the last layer's epilogue.  obs_rstd: the normaliser's
    1 / std given as it is (RunningNorm's 1 / (std + 1e-8)) instead of from obs_var.  residual = (float tensor [num_envs, >= cols], cols):
    the last layer adds it to its first cols outputs before the action clamp (the embodied_pose imitation policy's residual action,
    `mu[:, :69] += target_dof_pos`, im_network_builder.py:226-228).  noise_sigma (float [out_dim], the fixed sigma = exp(logstd)):
    the sampled action mu + sigma * N(0, 1) of a stochastic player (im_models.py:24-42 `distr.sample()`), drawn in the last layer's
    epilogue after the residual and before the action clamp from the counter-based generator under `seed`."""

    def __init__(self, layers, num_envs, device, obs_mean=None, obs_var=None, eps=1e-5, clamp_obs=5.0, activation="relu", clamp_actions=None,
                 obs_rstd=None, residual=None, noise_sigma=None, seed=0):
        self.rows, self.device = num_envs, torch.device(device)
        self.in_dim = layers[0][0].shape[1]
        self.out_dim = layers[-1][0].shape[0]
        self.clamp_obs = float(clamp_obs)
        self.clamp_actions = clamp_actions
        self.mean = obs_mean.to(self.device, torch.float32).contiguous() if obs_mean is not None else None
        self.rstd = (1.0 / torch.sqrt(obs_var.to(self.device, torch.float32) + eps)).contiguous() if obs_var is not None else None
        if obs_rstd is not None:
            if obs_var is not None:
                raise ValueError("obs_var and obs_rstd are two forms of the same statistic: give one")
            self.rstd = obs_rstd.to(self.device, torch.float32).contiguous()
        if (self.mean is None) != (self.rstd is None):
            raise ValueError("obs_mean and obs_var go together")
        self.x = padded_bf16(num_envs, self.in_dim, self.device)
        self.out = torch.zeros(num_envs, self.out_dim, device=self.device)
        self.layers, a = [], self.x
        for i, (w, b) in enumerate(layers):
            last = i == len(layers) - 1
            o = self.out if last else padded_bf16(num_envs, w.shape[0], self.device)
            self.layers.append(Linear(a, w, b, o, num_envs, act=None if last else activation,
                                      out_clamp=(-clamp_actions, clamp_actions) if (last and clamp_actions) else None,
                                      residual=residual if last else None,
                                      noise=(noise_sigma, seed) if (last and noise_sigma is not None) else None))
            a = o
        self.noise_step = self.layers[-1].noise_step     # None: the deterministic mu
        self.flops = sum(l.flops for l in self.layers)
        self.launches_per_forward = 1 + len(self.layers)

    def forward(self, obs):
        """obs float [rows, in_dim] -> mu float [rows, out_dim] (a static buffer, overwritten by the next call)"""
        cast_rows(obs, self.x, self.in_dim, self.mean, self.rstd, -self.clamp_obs, self.clamp_obs)
        for l in self.layers:
            l.run()
        return self.out

    __call__ = forward

    def forward_prepared(self):
        """the layers only: the normalised / clamped bf16 observation row is already in `self.x` (b200env_obs_imitation_rows writes it
        in the launch that computes the observation)"""
        for l in self.layers:
            l.run()
        return self.out

    @classmethod
    def random(cls, num_envs, device, in_dim=734, units=(1024, 1024, 512), out_dim=75, seed=0, out_gain=0.1, **kw):
        """random weights of the reference's shape (torch nn.Linear default init; the `mu` layer scaled by out_gain)"""
        g = torch.Generator().manual_seed(seed)
        dims = [in_dim, *units, out_dim]
        layers = []
        for i in range(len(dims) - 1):
            bound = 1.0 / dims[i] ** 0.5
            w = (torch.rand(dims[i + 1], dims[i], generator=g) * 2 - 1) * bound
            b = (torch.rand(dims[i + 1], generator=g) * 2 - 1) * bound
            if i == len(dims) - 2:
                w, b = w * out_gain, b * out_gain
            layers.append((w, b))
        return cls(layers, num_envs, device, **kw)


V2P_ACTOR_KEYS = ("actor_mlp.0", "actor_mlp.2", "actor_mlp.4", "mu")   # rl_games A2C actor: Linear / ReLU pairs, then the mu head


def _load(cp):
    return torch.load(cp, map_location="cpu", weights_only=False) if isinstance(cp, (str, os.PathLike)) else cp


def _pad_first(w, obs_dim):
    """the zero-padded first layer of V2PPlayer.restore / load_dual_cp when the network's obs dim is larger than the checkpoint's"""
    if obs_dim is None or w.shape[1] == obs_dim:
        return w
    if w.shape[1] > obs_dim:
        raise ValueError(f"the checkpoint's first layer takes {w.shape[1]} observations, the env has {obs_dim}")
    return torch.cat([w, w.new_zeros(w.shape[0], obs_dim - w.shape[1])], 1)


def _prefix(full, part):
    full[:part.shape[0]] = part.float()
    return full


def _fixed_sigma(model, what):
    """sigma = exp(a2c_network.sigma) of a checkpoint's actor (`fixed_sigma: True`: the model's `sigma_act(self.sigma)` is the log std,
    v2p_models.py:26 / im_models.py:24 take exp of it); refused with the reason for a learned sigma head or no sigma"""
    if "sigma.weight" in model:
        raise ValueError(f"{what}: the checkpoint has a learned sigma head (sigma.weight, fixed_sigma: False); the sampled action "
                         "serves the fixed sigma parameter only (every shipped cfg sets fixed_sigma: True)")
    if "sigma" not in model:
        raise ValueError(f"{what}: deterministic=False samples mu + sigma * N(0, 1), but the checkpoint has no fixed sigma "
                         "(a2c_network.sigma)")
    return torch.exp(model["sigma"].float())


def v2p_networks_from_checkpoint(checkpoint, obs_dim=None, normalize_input=True, dual=False, deterministic=True):
    """What V2PPlayer.restore (vid2player/players/v2p_player.py:71-111; dual: load_dual_cp :21-69) reads from the controller
    checkpoint(s), as one dict per network: `layers` [(weight, bias)] x 4 (actor_mlp.{0,2,4}, mu; the first zero-padded to obs_dim
    columns), `mean` / `rstd` [obs_dim] (None: no normaliser) and `clip` (the normaliser's clamp, inf for none).
      single (normalize_input): rl_games RunningMeanStd of `running_mean_std`, rstd = 1 / sqrt(var + 1e-5), clamp 5; with a padded
              first layer only the checkpoint's prefix is loaded, the rest keeps the fresh statistics (mean 0, var 1).
      dual:   each network's RunningNorm (running_obs_type 'ours'): `running_obs.{n,mean,std}` of the model, or else rl_games statistics
              of the checkpoint's `running_mean_std` or of the model's `running_obs.{running_mean,running_var,count}` with std = sqrt(var);
              a prefix leaves mean 0, std 0 behind it (rstd 1e8).  rstd = 1 / (std + 1e-8), clamp 5; identity while n == 0.
    deterministic=False (a stochastic player): also `sigma` [actions] = exp(a2c_network.sigma) of each checkpoint (see _fixed_sigma).
    checkpoint: a path or a loaded dict (dual: a pair).  CPU tensors, float32."""
    out = []
    for p, cp in enumerate(checkpoint if dual else [checkpoint]):
        ck = _load(cp)
        model = {k[len("a2c_network."):]: v for k, v in ck["model"].items() if k.startswith("a2c_network.")}
        sigma = None if deterministic else _fixed_sigma(model, f"checkpoint {p}" if dual else "checkpoint")
        layers = [(model[k + ".weight"].float(), model[k + ".bias"].float()) for k in V2P_ACTOR_KEYS]
        D = obs_dim or layers[0][0].shape[1]
        layers[0] = (_pad_first(layers[0][0], D), layers[0][1])
        net = dict(layers=layers, mean=None, rstd=None, clip=float("inf"))
        if sigma is not None:
            net["sigma"] = sigma
        if not dual:
            if normalize_input:
                rms = ck["running_mean_std"]
                net["mean"] = _prefix(torch.zeros(D), rms["running_mean"])
                var = _prefix(torch.ones(D), rms["running_var"])
                net["rstd"], net["clip"] = 1.0 / torch.sqrt(var + 1e-5), 5.0
        else:
            net.update(_running_norm(ck, model, D))
        out.append(net)
    return out


def _running_norm(ck, model, D, rlgame_fallback=True):
    """{mean, rstd, clip} of a RunningNorm (`running_obs_type: ours`, embodied_pose/models/running_norm.py: y = clamp((x - mean) /
    (std + 1e-8), -5, 5) while n > 0, the identity at n == 0), as the players load it: the model's `running_obs.{n,mean,std}`, or else
    (rlgame_fallback: the load_rlgame_norm branch of ImitatorPlayer.load_pretrained / V2PPlayer.load_dual_cp) rl_games statistics of
    the checkpoint's `running_mean_std` or of the model's `running_obs.{running_mean,running_var,count}` with std = sqrt(var).  A
    statistic shorter than D fills a prefix and leaves mean 0, std 0 behind it (rstd 1e8).  The identity: mean / rstd None, clip inf."""
    mean, std, n = torch.zeros(D), torch.zeros(D), 0
    if "running_obs.n" in model:
        n = int(model["running_obs.n"])
        _prefix(mean, model["running_obs.mean"])
        _prefix(std, model["running_obs.std"])
    elif rlgame_fallback and ("running_mean_std" in ck or "running_obs.running_mean" in model):
        rms = ck["running_mean_std"] if "running_mean_std" in ck else \
            {k: model["running_obs." + k] for k in ("running_mean", "running_var", "count")}
        n = int(rms["count"])
        _prefix(mean, rms["running_mean"])
        _prefix(std, torch.sqrt(rms["running_var"].float()))
    if n > 0:
        return dict(mean=mean, rstd=1.0 / (std + 1e-8), clip=5.0)
    return dict(mean=None, rstd=None, clip=float("inf"))


def im_networks_from_checkpoint(checkpoint, use_running_obs=True, running_obs_type="ours", normalize_input=False, use_ik=False,
                                deterministic=True, obs_dim=734):
    """What ImitatorPlayer.restore / load_pretrained (embodied_pose/players/im_player.py:43-94) read from an embodied_pose imitation
    checkpoint, as one network dict: `layers` [(weight, bias)] x 4 (actor_mlp.{0,2,4} and mu of `model`, or of a Lightning checkpoint's
    `state_dict`), `mean` / `rstd` [obs_dim] (None: no normaliser) and `clip` (the normaliser's clamp, inf for none).  The keyword
    arguments are the network / player cfg entries of the same names (cfg/amass_im.yaml: use_running_obs True, running_obs_type ours).
      running_obs_type ours:    RunningNorm (see _running_norm); a Lightning checkpoint loads only its own running_obs.* keys
      running_obs_type rl_game: RunningMeanStd, rstd = 1 / sqrt(var + 1e-5), clamp 5, always applied: the model's
                                running_obs.{running_mean,running_var}, else the fresh statistics (mean 0, var 1)
    deterministic=False (a stochastic player): also `sigma` [actions] = exp(sigma) of the actor (see _fixed_sigma), which
    HumanoidSMPLIMVis.run_test then samples with.  Refused, with the reason: normalize_input (the player's own RunningMeanStd over the
    raw obs), use_ik, and with deterministic=False a learned sigma head or a checkpoint without sigma.  checkpoint: a path or a loaded
    dict.  CPU tensors, float32."""
    if normalize_input:
        raise ValueError("normalize_input: True normalises the raw 461-wide observation before the network; the device operand launch "
                         "reads obs_buf as the wrapper clamps it and does not implement that normaliser (neither shipped cfg sets it)")
    if use_ik:
        raise ValueError("use_ik: the network's inverse kinematics of the context (perform_ik) needs the SMPL model files and is not "
                         "implemented on the device")
    ck = _load(checkpoint)
    lightning = "pytorch-lightning_version" in ck
    if lightning:
        model = dict(ck["state_dict"])
    else:
        model = {k[len("a2c_network."):]: v for k, v in ck["model"].items() if k.startswith("a2c_network.")}
    sigma = None if deterministic else _fixed_sigma(model, "imitation checkpoint")
    layers = [(model[k + ".weight"].float(), model[k + ".bias"].float()) for k in V2P_ACTOR_KEYS]
    net = dict(layers=layers, mean=None, rstd=None, clip=float("inf"))
    if sigma is not None:
        net["sigma"] = sigma
    if not use_running_obs:
        return net
    if running_obs_type == "rl_game":
        mean = model.get("running_obs.running_mean", torch.zeros(obs_dim)).float()
        var = model.get("running_obs.running_var", torch.ones(obs_dim)).float()
        net.update(mean=mean.clone(), rstd=1.0 / torch.sqrt(var + 1e-5), clip=5.0)
    else:
        net.update(_running_norm({} if lightning else ck, model, obs_dim, rlgame_fallback=not lightning))
    return net


def low_level_networks_from_cfg(physics, num_obs, num_actions, dual):
    """The tennis controller's trained low-level imitation policy, named by the controller cfg's `env.physics` block (PlayerBuilder,
    vid2player/env/utils/player_builder.py:142-161; ImitatorPlayer.__init__, vid2player/players/im_player.py:32-42), as the network
    dicts V2PPolicy takes; None when the block names no checkpoint.
      single (physics.pretrained_model_cp): ImitatorPlayer.load_pretrained (:92-133), im_networks_from_checkpoint with tennis_im.yaml's
              use_running_obs True, running_obs_type ours: one dict;
      dual   (physics.dual_model_cp, one checkpoint per player): ImitatorPlayer.load_dual_cp (:54-90): each network's actor layers and
              RunningNorm (see _running_norm) as they are - unlike V2PPlayer.load_dual_cp no zero-padded first layer, and the
              statistics fill the whole row: two dicts, player 0 (even envs) first.
    Refused with the reason (ValueError; nothing reaches the device): physics.checkpoint other than 'base' (the named restore reads
    rl_games' network_path), a list of pretrained_model_cp files, the key of the other mode, a dual_model_cp that is not two
    checkpoints, a first layer that does not take num_obs observations, a mu that does not give num_actions actions and (dual)
    statistics of another width than num_obs.  CPU tensors, float32."""
    single_cp, dual_cp = physics.get("pretrained_model_cp"), physics.get("dual_model_cp")
    if not single_cp and not dual_cp:
        return None
    if physics.get("checkpoint", "base") != "base":
        raise ValueError(f"physics.checkpoint = {physics['checkpoint']!r}: only 'base' (load the named pretrained_model_cp / "
                         "dual_model_cp) is implemented; the named restore reads rl_games' network_path")
    if dual and single_cp:
        raise ValueError("physics.pretrained_model_cp on a dual-player task: a rally loads one network per player from dual_model_cp")
    if not dual and dual_cp:
        raise ValueError("physics.dual_model_cp on a single-player task: it loads from pretrained_model_cp")
    if single_cp:
        if isinstance(single_cp, (list, tuple)):
            raise ValueError("physics.pretrained_model_cp is a list: loading several checkpoints in turn is not implemented "
                             "(no shipped cfg uses it)")
        nets = [im_networks_from_checkpoint(single_cp, use_running_obs=True, running_obs_type="ours", obs_dim=num_obs)]
    else:
        if not isinstance(dual_cp, (list, tuple)) or len(dual_cp) != 2:
            raise ValueError("physics.dual_model_cp must name exactly two checkpoints, one per player")
        nets = []
        for p, cp in enumerate(dual_cp):
            ck = _load(cp)
            model = {k[len("a2c_network."):]: v for k, v in ck["model"].items() if k.startswith("a2c_network.")}
            if "running_obs.n" in model:
                stat = model["running_obs.mean"]
            elif "running_mean_std" in ck:
                stat = ck["running_mean_std"]["running_mean"]
            else:
                stat = model.get("running_obs.running_mean")
            if stat is not None and stat.shape[0] != num_obs:
                raise ValueError(f"dual_model_cp[{p}]: the observation statistics are {stat.shape[0]} wide, the env's observation "
                                 f"{num_obs} (load_dual_cp fills the whole row)")
            net = dict(layers=[(model[k + ".weight"].float(), model[k + ".bias"].float()) for k in V2P_ACTOR_KEYS])
            net.update(_running_norm(ck, model, num_obs))
            nets.append(net)
    for p, net in enumerate(nets):
        w0, mu = net["layers"][0][0], net["layers"][-1][0]
        if w0.shape[1] != num_obs:
            raise ValueError(f"low-level network {p}: the first layer takes {w0.shape[1]} observations, the env has {num_obs}")
        if mu.shape[0] != num_actions:
            raise ValueError(f"low-level network {p}: mu gives {mu.shape[0]} actions, the env takes {num_actions}")
    return nets


class V2PPolicy:
    """The tennis controller's trained high-level policy at test time (V2PPlayer.get_action with the deterministic `mu`,
    players/v2p_player.py:113-131; V2PBuilder.Network.eval_actor, models/v2p_network_builder.py:52-81): per network
    mu = W4 relu(W3 relu(W2 relu(W1 x + b1) + b2) + b3) + b4, x = clamp((clamp(obs, -clip_obs, clip_obs) - mean) * rstd, -c, c),
    the wrapper's `clip_actions` folded into the last layer's clamp.  Single: one chain of four wgmma layers over all envs.  Dual
    (V2PBuilderDual.Network.eval_actor, models/v2p_network_builder_dual.py:39-47): network p acts for envs p, p + 2, ...; its operand
    rows are one contiguous block (env e at row (e & 1) * N/2 + (e >> 1)) and its last layer writes rows p, p + 2, ... of `out`
    (ldo = 2 * actions, first column p * actions), so `out` is [N, actions] in env order.
    It also serves the trained low-level imitation policy (low_level_networks_from_cfg; operand rows from b200env_obs_imitation_rows).

    The operand `x` is normally written by the controller's post launch (`operand()` gives it the fields of b200v2p_ctrl_t), and
    `forward_prepared()` runs the layers only; `forward(obs)` fills it from a float observation first.  bf16 operands, fp32 accumulation.

    deterministic=False: the sampled action of a stochastic player (V2PPlayer.get_action's `res_dict['actions']`, the `distr.sample()`
    of Normal(mu, sigma), v2p_models.py:26-43): every network dict carries `sigma` [actions] and network p's last layer adds
    sigma_p[col] * N(0, 1) to its rows before the action clamp.  The normals come from the counter-based generator under `seed`, keyed
    on the output element (env * actions + col) and each last layer's device step counter (`noise_steps`), so a graph replay draws
    afresh: the distribution of the reference's torch draws, not their stream."""

    def __init__(self, networks, num_envs, device, clip_obs=float("inf"), clip_actions=None, activation="relu", deterministic=True, seed=0):
        self.dual = len(networks) == 2
        if len(networks) not in (1, 2):
            raise ValueError("one network (single) or two (dual)")
        if self.dual and num_envs % 2:
            raise ValueError("dual mode needs an even number of envs")
        self.rows, self.device = num_envs, torch.device(device)
        self.in_dim = networks[0]["layers"][0][0].shape[1]
        self.out_dim = networks[0]["layers"][-1][0].shape[0]
        self.clip_obs, self.clip_actions = float(clip_obs), clip_actions
        P, dev = len(networks), self.device
        self.deterministic, self.seed = bool(deterministic), int(seed)
        if not deterministic and any(n.get("sigma") is None for n in networks):
            raise ValueError("deterministic=False needs every network's sigma (v2p_networks_from_checkpoint(..., deterministic=False))")
        if all(n["mean"] is None for n in networks):
            self.mean = self.rstd = None
        else:   # a network without a normaliser (RunningNorm with n == 0) is the identity: mean 0, rstd 1, no clamp
            self.mean = torch.stack([n["mean"] if n["mean"] is not None else torch.zeros(self.in_dim) for n in networks]).to(dev, torch.float32)
            self.rstd = torch.stack([n["rstd"] if n["rstd"] is not None else torch.ones(self.in_dim) for n in networks]).to(dev, torch.float32)
        self.clip = [float(n["clip"]) for n in networks]
        H = num_envs // P                                        # rows per chain
        self.x = torch.zeros(H * (P - 1) + padded_rows(H), _up(self.in_dim, 64), device=dev, dtype=torch.bfloat16)
        self.out = torch.zeros(num_envs, self.out_dim, device=dev)
        out_view = self.out.view(H, P * self.out_dim)
        self.layers = []
        for p, net in enumerate(networks):
            a = self.x[p * H:]
            for i, (w, b) in enumerate(net["layers"]):
                last = i == len(net["layers"]) - 1
                o = out_view if last else padded_bf16(H, w.shape[0], dev)
                noise = (net["sigma"], seed) if (last and not deterministic) else None
                self.layers.append(Linear(a, w, b, o, H, act=None if last else activation, out_col0=p * self.out_dim if last else 0,
                                          out_clamp=(-clip_actions, clip_actions) if (last and clip_actions) else None, noise=noise))
                a = o
        self.noise_steps = [l.noise_step for l in self.layers if l.noise_step is not None]   # one per network; [] when deterministic
        self.flops = sum(l.flops for l in self.layers)

    @classmethod
    def from_checkpoint(cls, checkpoint, num_envs, device, obs_dim=None, normalize_input=True, clip_obs=float("inf"), clip_actions=None,
                        deterministic=True, seed=0):
        """checkpoint: a path or loaded dict (single, V2PPlayer.restore), or a pair of them (dual, load_dual_cp); clip_obs / clip_actions:
        the wrapper's clamps (VecTaskPython.clip_obs / clip_actions); deterministic / seed: the player's `is_determenistic` and the
        cfg's params.seed (offset by rank like the task's cfg["seed"]) for the sampled action"""
        dual = isinstance(checkpoint, (list, tuple))
        nets = v2p_networks_from_checkpoint(checkpoint, obs_dim=obs_dim, normalize_input=normalize_input, dual=dual, deterministic=deterministic)
        return cls(nets, num_envs, device, clip_obs=clip_obs, clip_actions=clip_actions, deterministic=deterministic, seed=seed)

    def operand(self):
        """(scalars, tensors) of b200v2p_ctrl_t's policy fields for native_v2p.controller_post"""
        return (dict(policy_dual=int(self.dual), policy_clip_obs=self.clip_obs, policy_clip=self.clip * (1 if self.dual else 2)),
                dict(policy_x=self.x, policy_mean=self.mean, policy_rstd=self.rstd))

    def forward_prepared(self):
        """the layers only, on the operand rows the post launch wrote; -> float [N, actions] (a static buffer)"""
        for l in self.layers:
            l.run()
        return self.out

    def forward(self, obs):
        """obs float [N, >= in_dim] in env order -> the action (static buffer); the operand is cast from obs first"""
        obs = torch.clamp(obs, -self.clip_obs, self.clip_obs) if self.clip_obs != float("inf") else obs
        P, H = (2, self.rows // 2) if self.dual else (1, self.rows)
        for p in range(P):
            src = obs[p::P] if self.dual else obs
            mean = self.mean[p] if self.mean is not None else None
            rstd = self.rstd[p] if self.rstd is not None else None
            cast_rows(src, self.x[p * H:], self.in_dim, mean, rstd, -self.clip[p], self.clip[p])
        return self.forward_prepared()

    __call__ = forward


class MixedDecoder:
    """MixedDecoder.forward(z, c) (vid2player/motion_vae/model.py:237-252) with the reference's parameter layout:
    `weights[i]` [E, in_i, out_i], `biases[i]` [E, out_i] for the three decoder layers (input of every layer = cat(z, previous
    output)), `gate` = [(weight [out, in], bias [out])] x 3 (nn.Linear layout, ELU between).  The reference blends the expert weight
    matrices per env and runs a batched GEMV; here every layer is one launch: the E expert products of a 128 x 64 output tile are E
    register accumulators, the softmax coefficients blend them in the epilogue."""

    def __init__(self, weights, biases, gate, num_envs, device, latent_size=32):
        self.rows, self.device, self.L = num_envs, torch.device(device), latent_size
        E = weights[0].shape[0]
        self.E = E
        self.cond = weights[0].shape[1] - latent_size
        hid = weights[0].shape[2]
        self.out_dim = weights[2].shape[2]
        dev = self.device
        self.x0 = padded_bf16(num_envs, latent_size + self.cond, dev)     # [z | c]
        self.x1 = padded_bf16(num_envs, latent_size + hid, dev)           # [z | h1]
        self.x2 = padded_bf16(num_envs, latent_size + hid, dev)           # [z | h2]
        self.g1 = padded_bf16(num_envs, gate[0][0].shape[0], dev)
        self.g2 = padded_bf16(num_envs, gate[1][0].shape[0], dev)
        self.coef = torch.zeros(num_envs, E, device=dev)
        self.out = torch.zeros(num_envs, self.out_dim, device=dev)
        self.gate1 = Linear(self.x0, gate[0][0], gate[0][1], self.g1, num_envs, act="elu")
        self.gate2 = Linear(self.g1, gate[1][0], gate[1][1], self.g2, num_envs, act="elu")
        self.gw = gate[2][0].detach().to(dev, torch.float32).contiguous()
        self.gb = gate[2][1].detach().to(dev, torch.float32).contiguous()
        t = lambda w: w.detach().transpose(1, 2)   # noqa: E731   [E, in, out] -> [E, out, in]
        self.l1 = Linear(self.x0, t(weights[0]), biases[0], self.x1, num_envs, act="elu", coef=self.coef, out_col0=latent_size)
        self.l2 = Linear(self.x1, t(weights[1]), biases[1], self.x2, num_envs, act="elu", coef=self.coef, out_col0=latent_size)
        self.l3 = Linear(self.x2, t(weights[2]), biases[2], self.out, num_envs, act=None, coef=self.coef)
        self.flops = sum(l.flops for l in (self.gate1, self.gate2, self.l1, self.l2, self.l3))
        self.launches_per_forward = 1 + 1 + 2 + 1 + 3

    def forward(self, z, c=None, c_clamp=None):
        """z float [rows, latent], c float [rows, >= cond] -> float [rows, out_dim] (static buffer).  c = None: the condition block
        already sits in the first layer's operand buffer (`set_condition`, or the autoregressive `feed_back`)."""
        assert z.dtype == torch.float32 and z.stride(-1) == 1
        _check(lib().b200nn_cast_rows3(z.data_ptr(), z.stride(0), self.x0.data_ptr(), self.x1.data_ptr(), self.x2.data_ptr(), self.x0.shape[1],
                                       self.rows, self.L, _stream()))
        if c is not None:
            self.set_condition(c, c_clamp)
        self.gate1.run()
        self.gate2.run()
        _check(lib().b200nn_gate_softmax(self.g2.data_ptr(), self.g2.shape[1], self.gw.shape[1], self.gw.data_ptr(), self.gb.data_ptr(), self.E,
                                         self.coef.data_ptr(), self.rows, _stream()))
        self.l1.run()
        self.l2.run()
        self.l3.run()
        return self.out

    __call__ = forward

    def set_condition(self, c, clamp=None, row_mask=None):
        """condition block of the first layer's operand <- bf16(clamp(c[:, :cond])); row_mask (bool [rows]): those rows only"""
        lo, hi = (-clamp, clamp) if clamp else (-3.0e38, 3.0e38)
        _cast_cols(c, self.x0, self.L, self.cond, lo, hi, row_mask)

    def feed_back(self, clamp=3.0):
        """autoregression of MVAEPlayer (players/mvae_player.py:201-204): the predicted frame becomes the next condition - one cast
        launch from the output buffer straight into the operand buffer (kept inside the normalised range)"""
        self.set_condition(self.out, clamp)

    @classmethod
    def random(cls, num_envs, device, frame_size=288, latent_size=32, hidden_size=256, num_experts=6, out_extra=2, seed=0):
        """random parameters of the reference's shapes (motion_vae/config.py: latent 32, hidden 256, 6 experts; frame 6 + 24*6 +
        23*3 + 23*3 = 288, + 2 phase outputs): uniform expert weights, bias 0.01, nn.Linear default gate"""
        g = torch.Generator().manual_seed(seed)
        inp, inter, out = latent_size + frame_size, latent_size + hidden_size, frame_size + out_extra
        ws, bs = [], []
        for i, o in ((inp, hidden_size), (inter, hidden_size), (inter, out)):
            bound = (6.0 / i) ** 0.5     # uniform with fan_in = in: activations stay O(1) (the reference's kaiming_uniform_ on the
                                         # 3-d tensor uses fan_in = in * out; training overwrites either)
            ws.append((torch.rand(num_experts, i, o, generator=g) * 2 - 1) * bound)
            bs.append(torch.full((num_experts, o), 0.01))
        gate = []
        for i, o in ((inp, 64), (64, 64), (64, num_experts)):
            bound = 1.0 / i ** 0.5
            gate.append(((torch.rand(o, i, generator=g) * 2 - 1) * bound, (torch.rand(o, generator=g) * 2 - 1) * bound))
        return cls(ws, bs, gate, num_envs, device, latent_size)


def _cast_cols(src, dst, col0, cols, lo=-3.0e38, hi=3.0e38, row_mask=None):
    """dst[:rows, col0:col0+cols] = bf16(clamp(src[:, :cols])) through the strided view (col0 elements into each row of dst)"""
    assert src.dtype == torch.float32 and src.stride(-1) == 1
    view_ptr = dst.data_ptr() + col0 * 2
    if row_mask is not None:
        assert row_mask.dtype == torch.bool and row_mask.is_contiguous() and row_mask.shape[0] == src.shape[0]
        _check(lib().b200nn_cast_rows_masked(src.data_ptr(), src.stride(0), view_ptr, dst.shape[1], src.shape[0], cols, row_mask.data_ptr(),
                                             lo, hi, _stream()))
        return
    _check(lib().b200nn_cast_rows(src.data_ptr(), src.stride(0), view_ptr, dst.shape[1], src.shape[0], cols, None, None, lo, hi, _stream()))
