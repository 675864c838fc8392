"""The mixed plan of a handle of several assets (b200env_create_assets; step_kernel_packed<true, false, true>), on the GPU.  A CTA batch
holds 32 consecutive envs whatever their assets; each env's lanes read its own asset's constants from global memory.

1. Exactness: after three steps every output row of a mixed handle is bit-identical to a single-asset handle of that env's body, at
   N = 1, B-1, B, B+1 with S = 2 and S = N distinct bodies, interleaved and at random; at N = B G + 5 and 2 B G + 5 (a second and a third
   round) with S = 2, 64 and N, against the grouped plan of the same assets (which tests/test_gpu_assets.py ties to single-asset
   handles) and against single-asset handles of a few of the bodies.
2. Parity with the float64 restatement, and the end-to-end task run against the numpy task oracle: the checks of
   tests/test_gpu_assets.py on a mixed handle.
3. A HumanoidSMPLIM rollout with motion_assets, graphed with reset_done on a mixed handle, equals the eager rollout with
   reset_masked on a grouped handle bit for bit.
4. The rule: 8192 envs over 256 bodies at random take the mixed plan, over one body the grouped one."""
import numpy as np
import pytest
import torch

import test_gpu_assets as TA
from test_gpu_launch import _pool

pytestmark = pytest.mark.gpu

AMASS = TA.AMASS


def _variants(S):
    base = TA._model(AMASS)
    return [base] + [TA.scaled(base, 0.88 + 0.24 * i / max(S - 1, 1)) for i in range(1, S)]


def _plan(monkeypatch, plan):
    monkeypatch.setenv("B200ENV_ASSET_PLAN", plan)


def _rows_of(monkeypatch, plan, assets, ea, envs, pool):
    _plan(monkeypatch, plan)
    t = TA._multi(AMASS, assets, ea)
    assert t._env.asset_plan_mixed == (plan == "mixed")
    B, G = TA._launch_shape(t)
    rows = TA._run(t, pool, envs)
    del t
    return rows, B, G


def _compare(got, ref, idx, label):
    for k in ref:
        a = ref[k].view(np.uint8).reshape(len(idx), -1)
        b = got[k][idx].view(np.uint8).reshape(len(idx), -1)
        bad = np.flatnonzero((a != b).any(1))
        assert not len(bad), f"{label}: {len(bad)} of {len(idx)} envs differ in {k}; first env {int(idx[bad[0]])} (batch {int(idx[bad[0]]) // 32})"


def _single_rows(assets, ea, a, envs, pool):
    mine = np.flatnonzero(ea == a)
    return mine, TA._run(TA._single(AMASS, assets, a, ea[mine]), pool, envs[mine])


@pytest.mark.parametrize("n", [1, 31, 32, 33])
@pytest.mark.parametrize("S,assign", [(2, "interleaved"), (2, "random"), ("N", "interleaved")])
def test_small_mixed_batches_match_single_asset_handles(monkeypatch, n, S, assign):
    S = n if S == "N" else S
    assets = _variants(S)
    rng = np.random.default_rng(n * 7 + S)
    ea = np.arange(n) % S if assign == "interleaved" else rng.integers(0, S, n)
    pool = _pool("humanoid")
    envs = np.arange(n) % len(pool["kind"])
    got, _, _ = _rows_of(monkeypatch, "mixed", assets, ea, envs, pool)
    monkeypatch.delenv("B200ENV_ASSET_PLAN")
    for a in range(S):
        if (ea == a).any():
            mine, ref = _single_rows(assets, ea, a, envs, pool)
            _compare(got, ref, mine, f"N = {n}, S = {S} {assign}, asset {a}")


@pytest.mark.parametrize("rounds,S", [(2, 2), (2, 64), (2, "N"), (3, 2), (3, 64)])
def test_mixed_rounds_match_grouped_plan_and_single_asset_handles(monkeypatch, rounds, S):
    t0 = TA._memo("probe", lambda: TA._multi(AMASS, [TA._model(AMASS)], [0]))
    B, G = TA._launch_shape(t0)
    n = (rounds - 1) * B * G + 5
    S = n if S == "N" else S
    assets = _variants(S)
    ea = np.arange(n) if S == n else np.random.default_rng(S).integers(0, S, n)
    pool = _pool("humanoid")
    envs = np.arange(n) % len(pool["kind"])
    got, B, G = _rows_of(monkeypatch, "mixed", assets, ea, envs, pool)
    assert -(-n // B) > (rounds - 1) * G
    grouped, _, _ = _rows_of(monkeypatch, "grouped", assets, ea, envs, pool)
    _compare(got, grouped, np.arange(n), f"N = {n}, S = {S}: mixed against grouped")
    monkeypatch.delenv("B200ENV_ASSET_PLAN")
    for a in (0, 1, S - 1):
        mine, ref = _single_rows(assets, ea, a, envs, pool)
        _compare(got, ref, mine, f"N = {n}, S = {S}, asset {a}: mixed against a single-asset handle")
    print(f"\nN = {n}, S = {S}: {-(-n // B)} mixed batches, G = {G}, {-(-n // (B * G))} rounds; bit-identical")


def test_mixed_launch_matches_float64_restatement_per_asset(monkeypatch):
    _plan(monkeypatch, "mixed")
    TA.test_launch_matches_float64_restatement_per_asset()


def test_mixed_task_end_to_end_against_the_task_oracle(monkeypatch):
    _plan(monkeypatch, "mixed")
    TA.test_motion_assets_task_end_to_end()


def test_graphed_reset_done_on_mixed_handle_equals_eager_grouped(monkeypatch):
    """U(-1, 1) actions for 48 steps over 2 bodies: a mixed handle behind the step and reset_done graphs against a grouped handle
    stepped and reset_masked eagerly"""
    import test_gpu_im_reset_masked as RM
    from vid2player3d_b200.tasks.vec_task import VecTaskPythonWrapper
    over = dict(stateInit="Hybrid", hybridInitProb=0.5, motion_assets=RM._assets_cfg())
    n, steps = RM.N, 48
    _plan(monkeypatch, "mixed")
    a = RM.make_task(n, 0.3, **over)
    _plan(monkeypatch, "grouped")
    b = RM.make_task(n, 0.3, **over)
    assert a._env.asset_plan_mixed and not b._env.asset_plan_mixed and a._env.asset_plan[0] == 2
    w = VecTaskPythonWrapper(a, a.device)
    w.enable_cuda_graph(reset_graph=True)
    for _ in range(3):
        b.step(torch.clamp(torch.zeros(n, b.num_actions, device=b.device), -1.0, 1.0))
    b.reset_masked(torch.zeros(n, dtype=torch.bool, device=b.device))
    torch.cuda.synchronize()
    assert RM.differing(a, b) == []
    g = torch.Generator(device=a.device).manual_seed(11)
    acts = [torch.rand(n, a.num_actions, device=a.device, generator=g) * 2 - 1 for _ in range(steps)]
    mask_b = torch.zeros(n, dtype=torch.bool, device=b.device)
    resets = torch.zeros((), dtype=torch.long, device=a.device)
    for i in range(steps):
        w.step(acts[i])
        resets += a.reset_buf.sum()
        obs = w.reset_done()
    for i in range(steps):
        b.step(torch.clamp(acts[i], -1.0, 1.0))
        torch.ne(b.reset_buf, 0, out=mask_b)
        b.reset_masked(mask_b)
    torch.cuda.synchronize()
    assert int(resets) > 0, "no env finished: the rollout did not exercise the reset"
    assert RM.differing(a, b) == [], "graphed mixed rollout differs from the eager grouped one"
    assert torch.equal(obs, torch.clamp(b.obs_buf, -5.0, 5.0))


def test_rule_on_a_real_handle():
    from vid2player3d_b200 import native
    t0 = TA._memo("probe", lambda: TA._multi(AMASS, [TA._model(AMASS)], [0]))
    models, verts = zip(*[t0._pack(m) for m in _variants(4)])
    cfg = t0._cfg_struct
    n = 8192
    _, G = TA._launch_shape(t0)
    for S, want in ((1, False), (256, True)):
        ea = np.random.default_rng(S).integers(0, S, n)
        e = native.Env([models[i % 4] for i in range(S)], [verts[i % 4] for i in range(S)], cfg, n, 0, env_asset=ea)
        assert e.asset_plan_mixed == want == native.choose_asset_plan(ea, S, G)
        na, rows, batches = e.asset_plan
        assert na == S
        r2, b2 = native.plan_assets(ea, S, 32, mixed=want)
        assert np.array_equal(rows, r2) and np.array_equal(batches, b2)
        e.close()
