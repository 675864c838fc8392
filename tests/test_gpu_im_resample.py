"""The training resample of HumanoidSMPLIM (cfg.env.b200_resample_motions, b200_hard_motion_share) on the GPU, against the restatement
oracle/ref_port_motion_resample.py:

1. b200env_resample_motions at N in {1, 33, 8197} x M in {1, 7, 3N, 100 000}, eagerly at several counters and in graph replays: the
   motion ids, bitwise body rows, assets and counts of the restatement; unmasked envs and envs that played no step untouched.
2. b200env_motion_weights: rates exact, the CDF within 1e-12 relative, the counts zeroed, the same bits on every call.
3. Resample + masked reset equals the same ids, bodies and assets written by hand and the masked reset of a task without the key, for the
   reset and 10 steps, on one body and on 3 and 64 bodies.
4. The id-list reset and the masked reset of the same envs draw the same motions.
5. A graphed rollout (step graph + reset_done graph, pre_epoch rebuilds between) equals the eager one bitwise, and repeats.
6. The motion draw and the motion-time draw are uncorrelated.
7. Without the key nothing new runs: the reset launches the parent's kernels and motion ids never change."""
import numpy as np
import pytest
import torch

import test_gpu_assets as TA
import test_gpu_im_motion_queue as GQ
from oracle import ref_port_motion_resample as R
from test_gpu_im_reset_masked import differing, reset_mask_of
from vid2player3d_b200 import native

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
N = 8 * 16 + 3
CONTACT = ["R_Ankle", "L_Ankle", "R_Toe", "L_Toe"]


def rtask(n, flat, S=1, key=True, h=0.5, **over):
    """an imitation task on `flat`; S > 1: motion m runs body m % S (scaled copies of the SMPL humanoid)"""
    from helpers import SIM_PARAMS, im_cfg
    from vid2player3d_b200.tasks import HumanoidSMPLIM
    if key:
        over = dict(over, b200_resample_motions=True, b200_hard_motion_share=h)
    if S > 1:
        base = TA._model(TA.AMASS)
        bodies = [TA.scaled(base, 0.9 + 0.2 * k / (S - 1)) for k in range(S)]
        over["motion_assets"] = [bodies[m % S] for m in range(flat.num_motions())]
    cfg = im_cfg(n, flat, episode_length=300, contactBodies=CONTACT, terminationBodyHeight=0.3, **over)
    cfg["seed"] = 10
    torch.manual_seed(0)
    return HumanoidSMPLIM(cfg, SIM_PARAMS, 1, "cuda", 0, True)


def start(tasks, steps, seed=3):
    """every task: the full reset at the same torch seed, then the same `steps` random steps"""
    for t in tasks:
        torch.manual_seed(1)
        t.reset()
    g = torch.Generator(device=DEV).manual_seed(seed)
    for _ in range(steps):
        a = (torch.rand(tasks[0].num_envs, tasks[0].num_actions, device=DEV, generator=g) * 2 - 1) * 0.6
        for t in tasks:
            t.step(a)
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------------------- 1. the sampler
def sampler_state(n, M, rng, sd=11, S=5):
    cdf_w = rng.random(M)
    cdf_w[rng.random(M) < 0.2] = 0.0
    cdf_w[rng.integers(0, M)] = 1.0
    f = lambda x, dt: torch.from_numpy(np.ascontiguousarray(x)).to(DEV, dt)  # noqa: E731
    s = dict(cdf=f(np.cumsum(cdf_w / cdf_w.sum()), torch.float64), lib_motion_bodies=f(rng.normal(size=(M, sd)), torch.float32),
             motion_asset=f(rng.integers(0, S, M), torch.int32), motion_ids=f(rng.integers(0, M, n), torch.int64),
             motion_bodies=f(rng.normal(size=(n, sd)), torch.float32), env_asset=f(rng.integers(0, S, n), torch.int32),
             mask=f(rng.random(n) < 0.6, torch.bool), progress_buf=f(rng.integers(0, 3, n), torch.int64),
             terminate_buf=f(rng.integers(0, 2, n), torch.int64), counter=f(np.array([rng.integers(0, 1 << 40)]), torch.int64),
             done=torch.zeros(1, device=DEV, dtype=torch.int32), tries=torch.zeros(M, device=DEV, dtype=torch.long),
             fails=torch.zeros(M, device=DEV, dtype=torch.long))
    s["mask"][0] = True
    s["progress_buf"][0] = 1
    return s


def host(s):
    return {k: v.cpu().numpy().copy() for k, v in s.items()}


def near_boundary(cdf, u, ids):
    """draws whose u * total lies within 2^-40 (relative) of the boundaries around the drawn motion"""
    x = u * cdf[-1]
    lo = np.where(ids > 0, cdf[np.maximum(ids - 1, 0)], 0.0)
    return int(((np.abs(x - cdf[ids]) < 2.0 ** -40 * cdf[-1]) | (np.abs(x - lo) < 2.0 ** -40 * cdf[-1])).sum())


def check_launch(s, plain, before, seed, launch):
    """one launch (launch()) against the restatement from the host copy `before`; `plain` (no counts, no assets) must draw the same"""
    M = len(before["cdf"])
    ora = R.Resampler(np.ones(M), 0.5, seed)
    ora.cdf, ora.counter = before["cdf"], int(before["counter"][0])
    want, drew = ora.resample(before["motion_ids"], before["mask"], before["progress_buf"], before["terminate_buf"])
    u = R.uniforms(seed, ora.counter, len(want))
    launch()
    torch.cuda.synchronize()
    got = host(s)
    assert np.array_equal(got["motion_ids"], want)
    assert got["motion_bodies"].tobytes() == np.where(drew[:, None], before["lib_motion_bodies"][want], before["motion_bodies"]).tobytes()
    assert np.array_equal(got["env_asset"], np.where(drew, before["motion_asset"][want], before["env_asset"]))
    assert np.array_equal(got["tries"] - before["tries"], ora.tries) and np.array_equal(got["fails"] - before["fails"], ora.fails)
    assert int(got["counter"][0]) == ora.counter and int(got["done"][0]) == 0
    assert np.array_equal(plain["motion_ids"].cpu().numpy(), want)
    assert plain["motion_bodies"].cpu().numpy().tobytes() == got["motion_bodies"].tobytes()
    return near_boundary(before["cdf"], u[drew], want[drew]), int(drew.sum())


@pytest.mark.parametrize("n", [1, 33, 8197])
@pytest.mark.parametrize("Mk", ["1", "7", "3N", "100000"])
def test_the_sampler_draws_the_restatements_motions(n, Mk):
    M = {"1": 1, "7": 7, "3N": 3 * n, "100000": 100000}[Mk]
    rng = np.random.default_rng(n * 7 + M)
    seed = 10
    s = sampler_state(n, M, rng)
    plain = {k: v.clone() for k, v in s.items() if k not in ("tries", "fails", "motion_asset", "env_asset")}
    sc = dict(n=n, num_motions=M, shape_dim=11, seed=seed)

    def launch():
        native.resample_motions(sc, s)
        native.resample_motions(sc, plain)

    near = drawn = 0
    for _ in range(3):                                        # eager, at three counters
        a, b = check_launch(s, plain, host(s), seed, launch)
        near, drawn = near + a, drawn + b
        s["progress_buf"].copy_(torch.from_numpy(rng.integers(0, 3, n)).to(DEV))
        plain["progress_buf"].copy_(s["progress_buf"])
    g = torch.cuda.CUDAGraph()
    torch.cuda.synchronize()
    with torch.cuda.graph(g):
        launch()
    for _ in range(2):                                        # replays draw at the next counters
        a, b = check_launch(s, plain, host(s), seed, g.replay)
        near, drawn = near + a, drawn + b
    print(f"\nN {n} M {M}: {drawn} draws, {near} within 2^-40 of a CDF boundary")
    assert near == 0


# ---------------------------------------------------------------------------------------------------------- 2. the rebuild
@pytest.mark.parametrize("M", [1, 7, 11000, 100000])
@pytest.mark.parametrize("h", [0.0, 0.3, 1.0])
@pytest.mark.parametrize("lengths", [False, True])
def test_the_rebuild_against_the_restatement(M, h, lengths):
    rng = np.random.default_rng(M + int(10 * h))
    L = rng.uniform(0.0, 5.0, M).astype(np.float32)
    L[rng.random(M) < 0.1] = 0.0
    L[0] = 1.5
    tries = rng.integers(0, 4, M) * (rng.random(M) < 0.7)
    fails = np.minimum(rng.integers(0, 3, M), tries)
    rate = rng.random(M)
    ora = R.Resampler(R.base_weights(L, lengths), h, 10)
    ora.tries[:], ora.fails[:], ora.rate[:] = tries, fails, rate
    ora.rebuild()
    f = lambda x, dt: torch.from_numpy(np.ascontiguousarray(x)).to(DEV, dt)  # noqa: E731
    t = dict(base=f(L, torch.float32) if lengths else None, tries=f(tries, torch.int64), fails=f(fails, torch.int64),
             rate=f(rate, torch.float64), cdf=torch.full((M,), float("nan"), device=DEV, dtype=torch.float64))
    native.motion_weights(dict(num_motions=M, h=h), t if h > 0 else dict(base=t["base"], cdf=t["cdf"]))
    got = {k: v.cpu().numpy() for k, v in t.items() if v is not None}
    if h > 0:
        assert got["rate"].tobytes() == ora.rate.tobytes()
        assert not got["tries"].any() and not got["fails"].any()
    np.testing.assert_allclose(got["cdf"], ora.cdf, rtol=1e-12, atol=0)
    again = t["cdf"].clone()
    t["cdf"].fill_(float("nan"))
    t["rate"].copy_(torch.from_numpy(got["rate"]))           # counts are zero: the same rates, the same distribution
    native.motion_weights(dict(num_motions=M, h=h), t if h > 0 else dict(base=t["base"], cdf=t["cdf"]))
    assert torch.equal(t["cdf"], again)


def test_the_rebuild_falls_back_to_the_base_without_failures():
    M = 1000
    rng = np.random.default_rng(1)
    L = rng.uniform(0.5, 2.0, M).astype(np.float32)
    f = lambda x, dt: torch.from_numpy(np.ascontiguousarray(x)).to(DEV, dt)  # noqa: E731
    t = dict(base=f(L, torch.float32), tries=f(np.ones(M), torch.int64), fails=f(np.zeros(M), torch.int64),
             rate=f(np.ones(M), torch.float64), cdf=torch.zeros(M, device=DEV, dtype=torch.float64))
    native.motion_weights(dict(num_motions=M, h=0.8), t)
    assert not t["rate"].any()
    np.testing.assert_allclose(t["cdf"].cpu().numpy(), np.cumsum(L.astype(np.float64) / L.astype(np.float64).sum()), rtol=1e-12, atol=0)


# ---------------------------------------------------------------------------------------------------------- 3. resample + reset
def rs_host(t):
    return {k: t._rs[k].cpu().numpy().copy() for k in ("cdf", "counter", "tries", "fails", "rate") if k in t._rs}


@pytest.mark.parametrize("S", [1, 3, 64])
def test_resample_then_reset_equals_a_hand_written_reset(S):
    flat = GQ.lib(96, 45, 6)
    over = dict(stateInit="Random", motion_weights_from_length=True)
    a, b = rtask(N, flat, S, **over), rtask(N, flat, S, key=False, **over)
    assert torch.equal(a._reset_ref_motion_ids, b._reset_ref_motion_ids)
    if S > 1:
        assert a._env.asset_plan_mixed and len(a._asset_models) == S
        b._env.fix_mixed_plan()
    ora_cdf = R.Resampler(R.base_weights(flat.motion_lengths, True), 0.5, 10).cdf
    np.testing.assert_allclose(a._rs["cdf"].cpu().numpy(), ora_cdf, rtol=1e-12, atol=0)
    start([a, b], 6)
    assert differing(a, b) == []
    mask = reset_mask_of(N)
    for t in (a, b):
        t.progress_buf[[0, 9]] = 0                           # masked, but played no step: keeps its motion
    before = {k: v.cpu().numpy().copy() for k, v in dict(ids=a._reset_ref_motion_ids, prog=a.progress_buf, term=a._terminate_buf).items()}
    st = rs_host(a)
    ora = R.Resampler(R.base_weights(flat.motion_lengths, True), 0.5, 10)
    ora.cdf, ora.counter = st["cdf"], int(st["counter"][0])
    want, drew = ora.resample(before["ids"], mask, before["prog"], before["term"])
    assert drew.sum() > 10 and not drew[[0, 9]].any() and (want[drew] != before["ids"][drew]).any()
    a.reset_masked(torch.from_numpy(mask).to(DEV))
    ids = torch.from_numpy(want).to(DEV)
    b._reset_ref_motion_ids.copy_(ids)
    b._reset_ref_motion_bodies.copy_(b._ml_t["motion_bodies"][ids])
    if S > 1:
        ea = torch.from_numpy(b._motion_asset[want]).to(DEV, torch.int32)
        err = torch.zeros(1, device=DEV, dtype=torch.int32)
        b._env.set_env_assets(ea, err)
        assert torch.equal(a._rs["env_asset"], ea)
    b.reset_masked(torch.from_numpy(mask).to(DEV))
    torch.cuda.synchronize()
    assert differing(a, b) == [], "resample + reset differs from the hand-written reset"
    got = rs_host(a)
    assert np.array_equal(got["tries"], ora.tries) and np.array_equal(got["fails"], ora.fails)
    g = torch.Generator(device=DEV).manual_seed(8)
    for k in range(10):
        act = (torch.rand(N, a.num_actions, device=DEV, generator=g) * 2 - 1) * 0.6
        a.step(act)
        b.step(act)
        torch.cuda.synchronize()
        assert differing(a, b) == [], f"step {k}"
    a.pre_epoch(1)
    torch.cuda.synchronize()
    ora.rebuild()
    assert a._rs["rate"].cpu().numpy().tobytes() == ora.rate.tobytes()
    print(f"\nS {S}: {int(drew.sum())} of {N} envs drew, {int((want[drew] != before['ids'][drew]).sum())} changed motion")


# ---------------------------------------------------------------------------------------------------------- 4. the two reset paths
def test_the_id_list_and_masked_resets_draw_the_same_motions():
    flat = GQ.lib(50, 45, 6)
    a, b = rtask(N, flat, stateInit="Random"), rtask(N, flat, stateInit="Random")
    start([a, b], 4)
    mask = reset_mask_of(N, seed=9)
    a.reset(torch.from_numpy(np.flatnonzero(mask)).to(DEV))
    b.reset_masked(torch.from_numpy(mask).to(DEV))
    torch.cuda.synchronize()
    assert torch.equal(a._reset_ref_motion_ids, b._reset_ref_motion_ids)
    assert torch.equal(a._reset_ref_motion_bodies.view(torch.int32), b._reset_ref_motion_bodies.view(torch.int32))
    for k in ("tries", "fails", "counter"):
        assert torch.equal(a._rs[k], b._rs[k]), k
    assert int(a._rs["tries"].sum()) == int(mask.sum())


# ---------------------------------------------------------------------------------------------------------- 5. the graphed rollout
def rollout(graph, steps=64, over=None):
    from vid2player3d_b200.tasks.vec_task import VecTaskPythonWrapper
    flat = GQ.lib(40, 45, 6)
    t = rtask(N, flat, **dict(dict(stateInit="Hybrid", hybridInitProb=0.5), **(over or {})))
    w = VecTaskPythonWrapper(t, t.device)
    if graph:
        w.enable_cuda_graph(reset_graph=True)
    else:
        for _ in range(3):                                     # what the capture's warm-up runs
            t.step(torch.zeros(N, t.num_actions, device=DEV))
        t.reset_masked(torch.zeros(N, dtype=torch.bool, device=DEV))
    g = torch.Generator(device=DEV).manual_seed(11)
    acts = [torch.rand(N, t.num_actions, device=DEV, generator=g) * 2 - 1 for _ in range(steps)]
    ids0 = t._reset_ref_motion_ids.clone()
    resets = torch.zeros((), dtype=torch.long, device=DEV)
    torch.cuda.synchronize()
    if graph:                                                  # the graphed rollout, rebuilds included, never waits for the device
        torch.cuda.set_sync_debug_mode("error")
    try:
        for i in range(steps):
            w.step(acts[i])
            resets += t.reset_buf.sum()
            w.reset_done()
            if i % 16 == 15:
                t.pre_epoch(i // 16)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    return t, int(resets), int((t._reset_ref_motion_ids != ids0).sum())


def test_the_graphed_rollout_equals_the_eager_one_and_repeats():
    a, resets, changed = rollout(True)
    b, _, _ = rollout(False)
    c, _, _ = rollout(True)
    assert resets > 0 and changed > 0, "no game ended or no motion changed: the rollout did not exercise the resample"
    for other in (b, c):
        assert differing(a, other) == []
        for k, v in a._rs.items():
            if v is not None:
                assert torch.equal(v, other._rs[k]), k
    print(f"\n64 steps of {N} envs: {resets} resets, {changed} envs on another motion at the end")


# ---------------------------------------------------------------------------------------------------------- 6. independence
def test_the_motion_draw_and_the_time_draw_are_uncorrelated():
    n, M, K = 8192, 16, 64
    t = rtask(n, GQ.lib(M, 45, 6), stateInit="Random", truncate_time=False, h=0.0)
    full = torch.ones(n, dtype=torch.bool, device=DEV)
    L = t._ml_t["motion_lengths"]
    um, ut = [], []
    for _ in range(K):
        c = int(t._rs["counter"])
        t.progress_buf.fill_(1)
        t.reset_masked(full)
        ids = t._reset_ref_motion_ids
        ut.append((t._reset_ref_motion_times.double() / L[ids].double()).cpu().numpy())
        u = R.uniforms(10, c, n)
        assert np.array_equal(ids.cpu().numpy(), R.draw(t._rs["cdf"].cpu().numpy(), u))
        um.append(u)
    um, ut = np.concatenate(um), np.concatenate(ut)
    rho = np.corrcoef(um, ut)[0, 1]
    print(f"\n{K} x {n} resets: correlation of the motion and time draws {rho:+.5f}")
    assert abs(rho) < 5.0 / np.sqrt(len(um))
    counts = np.bincount((um * M).astype(np.int64), minlength=M)
    assert counts.min() > 0.9 * len(um) / M


# ---------------------------------------------------------------------------------------------------------- 7. without the key
def test_without_the_key_nothing_new_runs(monkeypatch):
    from vid2player3d_b200.tasks.physics_mvae_controller import PhysicsMVAEController
    calls = []
    for name in ("resample_motions", "motion_weights"):
        real = getattr(native, name)
        monkeypatch.setattr(native, name, lambda *a, _r=real: calls.append(a) or _r(*a))
    flat = GQ.lib(40, 45, 6)
    kernels = {}
    for name, key, S in (("off", False, 1), ("on", True, 1), ("on, 3 bodies", True, 3)):
        t = rtask(N, flat, S, key=key)
        none = torch.zeros(N, dtype=torch.bool, device=DEV)
        t.reset_masked(none)                                   # the first call allocates the context window
        kernels[name] = PhysicsMVAEController._count_kernels(lambda: t.reset_masked(none))
        if not key:
            assert not calls and t._rs is None
            ids0 = t._reset_ref_motion_ids.clone()
            from vid2player3d_b200.tasks.vec_task import VecTaskPythonWrapper
            w = VecTaskPythonWrapper(t, t.device)
            w.enable_cuda_graph(reset_graph=True)
            resets = 0
            for i in range(32):
                w.step(torch.rand(N, t.num_actions, device=DEV) * 2 - 1)
                resets += int(t.reset_buf.sum())
                w.reset_done()
                t.pre_epoch(i)
            assert resets > 0 and torch.equal(t._reset_ref_motion_ids, ids0) and not calls
    print(f"\nkernels of one masked reset: {kernels}")
    assert kernels == {"off": 2, "on": 3, "on, 3 bodies": 4}
