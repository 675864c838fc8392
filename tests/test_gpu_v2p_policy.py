"""GPU checks of the tennis controller's high-level policy at test time: the operand row the post launch writes (b200v2p_ctrl_t.policy_*),
nn.V2PPolicy's wgmma layers against the float64 restatement oracle/ref_port_v2p_policy.py, and the test loop of MVAEControllerVis /
MVAEControllerVisDual graphed against the same loop run eagerly.

Tolerance of the actions.  As tests/test_gpu_nn.py states for a whole fp32 module: operands are bf16 (8 significant bits), accumulation
fp32; each product carries a relative error of 2^-8 twice, so after the three hidden layers the action is within ~1 % of max|mu|;
LOOSE = 2.5e-2 of max|mu| per output (the action clamp is 1-Lipschitz and does not widen it).  The operand row itself has no
tolerance: it is bit for bit the cast launch of libb200nn.so (nn.cast_rows) on the same observation."""
import numpy as np
import pytest
import torch

from helpers import SIM_PARAMS, v2p_cfg, v2p_dual_cfg
from oracle import ref_port_v2p_policy as R

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
LOOSE = 2.5e-2
OBS, ACT, UNITS = 257, 35, (1024, 1024, 512)
SENTINEL = -7.75


def networks(P, seed, identity_second=False):
    """random actors of the shipped shape with RunningNorm-like statistics (float32, CPU), as v2p_networks_from_checkpoint returns"""
    g = torch.Generator().manual_seed(seed)
    nets = []
    for p in range(P):
        dims = (OBS,) + UNITS + (ACT,)
        layers = [((torch.rand(dims[i + 1], dims[i], generator=g) * 2 - 1) / dims[i] ** 0.5,
                   (torch.rand(dims[i + 1], generator=g) * 2 - 1) / dims[i] ** 0.5) for i in range(4)]
        if identity_second and p == 1:
            nets.append(dict(layers=layers, mean=None, rstd=None, clip=float("inf")))
        else:
            std = torch.rand(OBS, generator=g) * 2 + 0.05
            nets.append(dict(layers=layers, mean=torch.randn(OBS, generator=g), rstd=1.0 / (std + 1e-8), clip=5.0))
    return nets


def oracle_nets(nets):
    """the same networks in the restatement's form (float64)"""
    out = []
    for n in nets:
        layers = [(w.double(), b.double()) for w, b in n["layers"]]
        if n["mean"] is None:
            out.append(dict(layers=layers, norm=None))
        else:   # rstd = 1 / (std + 1e-8) given: RunningNorm with std = 1 / rstd - 1e-8
            out.append(dict(layers=layers, norm="running", n=1, mean=n["mean"].double(), std=1.0 / n["rstd"].double() - 1e-8))
    return out


def on_device(nets):
    return [dict(n, layers=[(w.to(DEV), b.to(DEV)) for w, b in n["layers"]], **{k: n[k].to(DEV) for k in ("mean", "std") if k in n})
            for n in nets]


def policy(nets, N, **kw):
    from vid2player3d_b200 import nn
    return nn.V2PPolicy(nets, N, DEV, **kw)


SINGLE_N = (1, 2, 126, 127, 128, 129, 130, 256, 258, 8192)
DUAL_N = (2, 126, 128, 130, 256, 258, 8192)
CASES = [("single", n) for n in SINGLE_N] + [("dual", n) for n in DUAL_N]


@pytest.mark.parametrize("clip_actions", [None, 0.05])
@pytest.mark.parametrize("mode,N", CASES)
def test_actions_match_restatement(mode, N, clip_actions):
    P = 2 if mode == "dual" else 1
    nets = networks(P, seed=N, identity_second=(N % 4 == 2))
    pol = policy(nets, N, clip_obs=6.0, clip_actions=clip_actions)
    g = torch.Generator(device=DEV).manual_seed(N)
    obs = torch.randn(N, OBS, device=DEV, generator=g) * 4
    mu = pol(obs).clone()
    ref = on_device(oracle_nets(nets))
    want = R.act(obs.double(), ref, clip_obs=6.0, clip_actions=clip_actions)
    assert mu.shape == (N, ACT) and bool(torch.isfinite(mu).all())
    err = (mu.double() - want).abs().max()
    scale = R.act(obs.double(), ref, clip_obs=6.0).abs().max()        # max|mu| before the action clamp
    assert float(err) <= LOOSE * float(scale), (float(err), float(scale))
    if clip_actions:
        lim = torch.tensor(clip_actions, dtype=torch.float32)          # the clamp bound as the launch holds it
        assert float(mu.abs().max()) <= float(lim) and bool((mu.abs() == float(lim)).any())


@pytest.mark.parametrize("N", [2, 130, 258, 8192])
def test_dual_equals_two_single_runs(N):
    nets = networks(2, seed=7)
    dual = policy(nets, N, clip_actions=0.5)
    obs = torch.randn(N, OBS, device=DEV) * 3
    got = dual(obs).clone()
    for p in range(2):
        single = policy([nets[p]], N // 2, clip_actions=0.5)
        assert torch.equal(got[p::2], single(obs[p::2].contiguous()))


# ------------------------------------------------------------------------------------------------ the operand row of the post launch
def make_env(mode, N, tmp=None, **env_over):
    from vid2player3d_b200.tasks import MVAEControllerVis, MVAEControllerVisDual
    torch.manual_seed(0)
    np.random.seed(0)
    cfg = v2p_dual_cfg(N) if mode == "dual" else v2p_cfg(N)
    cfg["env"].update(env_over)
    cls = MVAEControllerVisDual if mode == "dual" else MVAEControllerVis
    return cls(cfg, SIM_PARAMS, 1, "cuda", 0, True)


def expected_operand(env, pol, rows=None):
    """nn.cast_rows on the same obs_buf, player block by player block"""
    from vid2player3d_b200 import nn
    N, P = env.num_envs, 2 if pol.dual else 1
    H = N // P
    want = torch.full_like(pol.x, SENTINEL)
    obs = torch.clamp(env.obs_buf, -pol.clip_obs, pol.clip_obs)
    for p in range(P):
        src = obs[p::P].contiguous()
        nn.cast_rows(src, want[p * H:], OBS, pol.mean[p] if pol.mean is not None else None, pol.rstd[p] if pol.rstd is not None else None,
                     -pol.clip[p], pol.clip[p])
    if rows is not None:      # the rows that were not refreshed keep the sentinel
        keep = torch.ones(pol.x.shape[0], dtype=torch.bool, device=DEV)
        env_rows = torch.arange(N, device=DEV)
        blk = (env_rows & 1) * H + (env_rows >> 1) if pol.dual else env_rows
        keep[blk[rows]] = False
        want[keep] = SENTINEL
    else:
        want[:, OBS:] = 0
        want[N:] = 0
    return want


@pytest.mark.parametrize("mode,N", [("single", 130), ("dual", 258)])
def test_operand_row_is_the_cast_of_obs_buf(mode, N):
    env = make_env(mode, N)
    pol = policy(networks(2 if mode == "dual" else 1, seed=3, identity_second=True), N, clip_obs=5.0, clip_actions=5.0)
    env.set_policy(pol)
    env.reset()
    for _ in range(3):                          # full steps: every row, every step
        env.test_step(graph=False)
        torch.cuda.synchronize()
        assert torch.equal(pol.x.view(torch.int16), expected_operand(env, pol).view(torch.int16))
    # the masked refresh of the reset path: the rows of the listed envs are rewritten, the others are left alone
    ids = torch.tensor([0, 1, 3, 6, N - 1], device=DEV)
    pol.x.fill_(SENTINEL)
    env._compute_observations(ids)
    torch.cuda.synchronize()
    mask = torch.zeros(N, dtype=torch.bool, device=DEV)
    mask[ids] = True
    assert torch.equal(pol.x.view(torch.int16), expected_operand(env, pol, rows=mask).view(torch.int16))


@pytest.mark.parametrize("mode", ["single", "dual"])
def test_post_without_policy_pointer_is_unchanged(mode):
    """the post launch with the operand fields writes exactly what it writes without them, everywhere else"""
    from vid2player3d_b200 import native_v2p
    N = 66
    env = make_env(mode, N)
    env.reset()
    for _ in range(2):
        env.step(torch.randn(N, env.num_actions, device=DEV))
    pol = policy(networks(2 if mode == "dual" else 1, seed=5), N, clip_actions=1.0)
    base = {k: v.clone() for k, v in env._tensors().items() if v is not None}
    outs = []
    for with_policy in (False, True):
        t = {k: v.clone() for k, v in base.items()}
        cfg = dict(env._post_cfg, advance=1)
        if with_policy:
            c, pt = pol.operand()
            cfg.update(c)
            t.update(pt)
        native_v2p.controller_post(cfg, t)
        outs.append(t)
    torch.cuda.synchronize()
    for k in base:
        assert torch.equal(outs[0][k].view(torch.uint8), outs[1][k].view(torch.uint8)), k
    assert not torch.equal(pol.x, torch.zeros_like(pol.x))


@pytest.mark.parametrize("mode", ["single", "dual"])
def test_graphed_loop_equals_eager_loop(mode, tmp_path, monkeypatch):
    """V2PPlayer.run driven by the policy: the graphed loop and the eager loop record the same episodes, meters and .npz files over a
    run that crosses resets and ends at the recording's end"""
    N, frames = 256, 60
    results = []
    for graph in (False, True):
        d = tmp_path / ("graph" if graph else "eager")
        d.mkdir()
        monkeypatch.chdir(d)
        env = make_env(mode, N, record=True, num_rec_frames=frames, num_eg=3, episodeLength=25)
        pol = policy(networks(2 if mode == "dual" else 1, seed=9), N, clip_obs=5.0, clip_actions=1.0)
        torch.manual_seed(1)
        with pytest.raises(SystemExit):
            env.run_test(pol, frames + 5, graph=graph)
        assert graph == (env._test_graphs is not None)
        rec = {k: v.cpu().numpy() for k, v in env._rec.items()}
        extra = {k: v.cpu().numpy() for k, v in (env._best.items() if mode == "dual" else
                                                  dict(sum=env._meter_sum, count=env._meter_count, avg=env._meter_avg, max=env._meter_max).items())}
        files = [dict(np.load(p)) for p in env.exported]
        resets = int(env._num_reset.sum())
        results.append((rec, extra, files, resets, [p.split("/")[-1] for p in env.exported]))
    (r0, e0, f0, n0, p0), (r1, e1, f1, n1, p1) = results
    assert n0 == n1 and ((n0 > N) if mode == "single" else len(f0) > 0)      # envs were reset during the run
    assert p0 == p1 and len(f0) > 0
    for k in r0:
        np.testing.assert_array_equal(r0[k], r1[k], k)
    for k in e0:
        np.testing.assert_array_equal(e0[k], e1[k], k)
    for a, b in zip(f0, f1):
        assert a.keys() == b.keys()
        for k in a:
            np.testing.assert_array_equal(a[k], b[k], k)
