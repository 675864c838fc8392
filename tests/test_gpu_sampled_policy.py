"""GPU checks of the sampled action (a stochastic test-time player): the noise of the last wgmma layer against the float64 restatement
oracle/ref_port_sampled_policy.py, its statistics over many draws, sigma 0 against the deterministic layer, the dual policy's per-network
sigma, the imitation layer's order (residual, noise, clamp), and the players' run_test driven by a sampling policy (same seed, same
trajectory; graphed = eager).

eps is read back as (action - mu) / sigma in float64 where mu is the same policy built deterministic on the same operand: both launches
compute mu with the same instructions, so the only rounding is that of the fused mu + sigma * eps (<= ulp(|action|) / 2).  With
|mu| <= ~1 and sigma >= 0.13 that is below 1e-6 in eps.  The kernel's float32 logf / sqrtf / cosf against the restatement's float64
ones: 1e-5, plus 4 float32 ulps of log(u1) times 1 / sqrt(-2 ln u1) for the draws with u1 near 1 (|eps| ~ 1e-4), where an error in the
log is amplified (the bound tests/test_gpu_v2p_launch.py holds the pre-step's normals to)."""
import numpy as np
import pytest
import torch

from helpers import SIM_PARAMS, im_cfg
from oracle import ref_port_sampled_policy as S
from test_gpu_v2p_policy import ACT, OBS, make_env, networks

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL = 1e-5
SEED = 10 * 7 + 3


def tol(step, N, A, ldo=None):
    return TOL + 4 * 2.0 ** -23 * S.log_amplification(SEED, step, np.arange(N), np.arange(A), ldo or A)


def with_sigma(nets, seed, lo=-2.0, hi=-0.5, scale=(1.0, 3.0)):
    """the networks with a fixed sigma = exp(U(lo, hi)) each, network p's scaled by scale[p] (the two players' sigmas far apart)"""
    g = torch.Generator().manual_seed(seed)
    return [dict(n, sigma=torch.exp(torch.rand(ACT, generator=g) * (hi - lo) + lo) * scale[p]) for p, n in enumerate(nets)]


def pair(nets, N, seed=SEED, **kw):
    from vid2player3d_b200 import nn
    return nn.V2PPolicy(nets, N, DEV, **kw), nn.V2PPolicy(nets, N, DEV, deterministic=False, seed=seed, **kw)


def env_sigma(nets, N):
    """sigma of every output in env order: network p's for envs p, p + 2, ..."""
    s = torch.stack([n["sigma"] for n in nets]).double().to(DEV)
    return s[torch.arange(N, device=DEV) % len(nets)]


CASES = [("single", n) for n in (1, 63, 64, 65, 127, 8192)] + [("dual", 2 * 8192)]


@pytest.mark.parametrize("mode,N", CASES)
def test_eps_matches_the_restatement(mode, N):
    P = 2 if mode == "dual" else 1
    nets = with_sigma(networks(P, seed=N), seed=N)
    det, smp = pair(nets, N, clip_obs=6.0)
    obs = torch.randn(N, OBS, device=DEV, generator=torch.Generator(device=DEV).manual_seed(N)) * 3
    mu = det(obs).double()
    sig = env_sigma(nets, N)
    for step in range(3):
        a = smp(obs).double()
        torch.cuda.synchronize()
        eps = ((a - mu) / sig).cpu().numpy()
        want = S.counter_normal(SEED, step, np.arange(N), np.arange(ACT), ACT)
        err = np.abs(eps - want)
        assert (err <= tol(step, N, ACT)).all(), (step, err.max(), int((err > TOL).sum()))
        if P == 2:      # the other network's sigma on a player's rows would scale eps by 3 or 1/3
            other = ((a - mu) / env_sigma(nets[::-1], N)).cpu().numpy()
            assert np.abs(other - want).max() > 0.1
    assert [int(s) for s in smp.noise_steps] == [3] * P and det.noise_steps == []


def test_statistics_over_64_steps():
    N, steps = 8192, 64
    nets = with_sigma(networks(1, seed=2), seed=2)
    det, smp = pair(nets, N, clip_obs=6.0)
    obs = torch.randn(N, OBS, device=DEV, generator=torch.Generator(device=DEV).manual_seed(2)) * 3
    mu = det(obs).double()
    sig = env_sigma(nets, N)
    eps = torch.empty(steps, N, ACT, device=DEV, dtype=torch.float64)
    for t in range(steps):
        eps[t] = (smp(obs).double() - mu) / sig
    n = eps.numel()
    flat = eps.reshape(-1)
    assert bool(torch.isfinite(flat).all())
    assert abs(float(flat.mean())) < 5 / n ** 0.5
    assert abs(float(flat.var()) - 1) < 5 * (2 / n) ** 0.5
    srt = torch.sort(flat).values
    cdf = torch.special.ndtr(srt)
    i = torch.arange(1, n + 1, device=DEV, dtype=torch.float64)
    ks = float(torch.maximum(i / n - cdf, cdf - (i - 1) / n).max())
    assert ks < 1.63 / n ** 0.5, ks

    def corr(x, y):
        x, y = x.reshape(-1) - x.mean(), y.reshape(-1) - y.mean()
        return float((x * y).mean() / (x.std() * y.std()))
    for name, (x, y) in dict(rows=(eps[:, :-1], eps[:, 1:]), cols=(eps[:, :, :-1], eps[:, :, 1:]), steps=(eps[:-1], eps[1:])).items():
        m = x.numel()
        assert abs(corr(x, y)) < 5 / m ** 0.5, name


@pytest.mark.parametrize("mode,N", [("single", 65), ("single", 8192), ("dual", 16384)])
def test_sigma_zero_is_the_deterministic_action_bit_for_bit(mode, N):
    P = 2 if mode == "dual" else 1
    nets = [dict(n, sigma=torch.zeros(ACT)) for n in networks(P, seed=5)]
    det, smp = pair(nets, N, clip_actions=0.5)
    obs = torch.randn(N, OBS, device=DEV) * 3
    obs[0, :7] = float("nan")                   # a NaN row stays NaN in both
    want = det(obs).clone()
    for _ in range(2):
        got = smp(obs)
        assert torch.equal(got.view(torch.int32), want.view(torch.int32))


@pytest.mark.parametrize("N", [1, 129, 8192])
def test_imitation_layer_adds_residual_then_noise_then_clamps(N):
    from vid2player3d_b200 import nn
    g = torch.Generator().manual_seed(N)
    A, nd, clip = 75, 69, 0.4
    dims = (256, 512, 256, 256, A)
    layers = [((torch.rand(dims[i + 1], dims[i], generator=g) * 2 - 1) / dims[i] ** 0.5,
               (torch.rand(dims[i + 1], generator=g) * 2 - 1) / dims[i] ** 0.5 * 0.3) for i in range(4)]
    sigma = torch.exp(torch.rand(A, generator=g) * 1.5 - 2.0)
    resid = (torch.randn(N, nd, generator=g) * 0.3).to(DEV)
    obs = torch.randn(N, dims[0], device=DEV, generator=torch.Generator(device=DEV).manual_seed(N))
    det = nn.PolicyMLP(layers, N, DEV, residual=(resid, nd))
    smp = nn.PolicyMLP(layers, N, DEV, residual=(resid, nd), clamp_actions=clip, noise_sigma=sigma, seed=SEED)
    mu = det(obs).double().cpu().numpy()           # includes the residual
    a = smp(obs).double().cpu().numpy()
    assert int(smp.noise_step) == 1 and det.noise_step is None
    lim = float(np.float32(clip))
    want = mu + sigma.double().numpy()[None] * S.counter_normal(SEED, 0, np.arange(N), np.arange(A), A)
    inside = np.abs(a) < lim
    assert inside.any() and (~inside).any()
    err = np.abs((a - mu) / sigma.double().numpy()[None] - S.counter_normal(SEED, 0, np.arange(N), np.arange(A), A))
    assert (err <= tol(0, N, A))[inside].all(), err[inside].max()
    assert set(np.unique(a[~inside])) <= {-lim, lim}
    sure = np.abs(want) > lim + 1e-5                  # the restatement clamps these: the kernel must have clamped them to the sign
    np.testing.assert_array_equal(a[sure], np.sign(want[sure]) * lim)
    assert np.abs(want[inside]).max() <= lim + 1e-5


def _controller_run(mode, tmp, seed, graph, monkeypatch, run):
    N, frames = 256, 40
    d = tmp / f"{mode}_{run}"
    d.mkdir()
    monkeypatch.chdir(d)
    env = make_env(mode, N, record=True, num_rec_frames=frames, num_eg=3, episodeLength=25)
    nets = with_sigma(networks(2 if mode == "dual" else 1, seed=9), seed=9)
    from vid2player3d_b200 import nn
    pol = nn.V2PPolicy(nets, N, DEV, clip_obs=5.0, clip_actions=1.0, deterministic=False, seed=seed)
    torch.manual_seed(1)
    with pytest.raises(SystemExit):
        env.run_test(pol, frames + 5, graph=graph)
    steps = [int(s) for s in pol.noise_steps]
    return {k: v.cpu().numpy() for k, v in env._rec.items()}, steps


@pytest.mark.parametrize("mode", ["single", "dual"])
def test_controller_run_test_same_seed_same_episodes(mode, tmp_path, monkeypatch):
    """the recorded episodes of V2PPlayer.run with a sampling policy: bitwise equal for the same seed, graphed or eager; another seed
    records others; every replay of the step graph advanced the noise counter"""
    r0, s0 = _controller_run(mode, tmp_path, 11, True, monkeypatch, 0)
    r1, s1 = _controller_run(mode, tmp_path, 11, True, monkeypatch, 1)
    r2, s2 = _controller_run(mode, tmp_path, 11, False, monkeypatch, 2)
    r3, _ = _controller_run(mode, tmp_path, 12, True, monkeypatch, 3)
    for k in r0:
        np.testing.assert_array_equal(r0[k], r1[k], k)
        np.testing.assert_array_equal(r0[k], r2[k], k)
    assert any(not np.array_equal(r0[k], r3[k]) for k in r0 if r0[k].dtype.kind == "f")
    assert s0 == s1 == s2 and min(s0) >= 30          # one draw per step, graph replays included


def _im_network(seed):
    g = torch.Generator().manual_seed(seed)
    dims = (734, 1024, 1024, 512, 75)
    layers = [((torch.rand(dims[i + 1], dims[i], generator=g) * 2 - 1) / dims[i] ** 0.5,
               (torch.rand(dims[i + 1], generator=g) * 2 - 1) / dims[i] ** 0.5) for i in range(4)]
    return dict(layers=layers, mean=None, rstd=None, clip=float("inf"), sigma=torch.exp(torch.full((75,), -1.5)))


def _im_run(seed, graph, capsys):
    from vid2player3d_b200 import model_compiler, motion_lib
    from vid2player3d_b200.tasks import HumanoidSMPLIMVis
    torch.manual_seed(0)
    model = model_compiler.load_compiled("smpl_mesh_humanoid_amass_v1")
    flat = motion_lib.synthetic(model, num_motions=4, num_frames=60, seed=1)
    cfg = im_cfg(512, flat, stateInit="Start")
    cfg["seed"] = seed
    task = HumanoidSMPLIMVis(cfg, SIM_PARAMS, 1, "cuda", 0, True)
    capsys.readouterr()
    out = task.run_test(_im_network(4), games_num=700, max_steps=60, clip_obs=5.0, clip_actions=1.0, graph=graph)
    lines = capsys.readouterr().out.splitlines()
    return out, lines, int(task._im_policy.noise_step), task._im_policy.out.clone()


def test_imitation_run_test_same_seed_same_statistics(capsys):
    o0, l0, s0, a0 = _im_run(21, True, capsys)
    o1, l1, s1, a1 = _im_run(21, True, capsys)
    o2, l2, s2, a2 = _im_run(21, False, capsys)
    o3, l3, _, a3 = _im_run(22, True, capsys)
    assert len([l for l in l0 if l.startswith("reward:")]) > 0
    assert l0 == l1 == l2 and o0 == o1 == o2
    assert torch.equal(a0, a1) and torch.equal(a0, a2)
    assert l3 != l0 and not torch.equal(a3, a0)
    assert s0 == s1 == s2 and s0 >= 1
