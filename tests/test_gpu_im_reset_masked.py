"""The mask-driven reset of the imitation task (HumanoidSMPLIM.reset_masked / reset_done, include/b200env.h: b200env_reset_masked)
against the id-list path, on the GPU.

1. Masked equals the id list: a mask with the first, last and isolated envs over a ragged n (8 x 16 + 3); the drawn times and the
   Hybrid choice restated in numpy from the counter-based generator (uint64, bit for bit); a twin task in the same pre-state given
   exactly those ids and times through b200env_reset + b200env_motion_context (ref-state rows) and `_reset_default` (default rows):
   every buffer bit-identical, unmasked rows untouched.  Start, Random, Hybrid at p in {0, 0.3, 1}, Default, with and without
   truncate_time, and a task of several assets (cfg.env.motion_assets).
2. The draw at the edges of t = u * max(length - truncate, 0): lengths below, at and one ulp above the truncation (t exactly 0 up to
   there), zero length (a one-frame motion), the largest and a subnormal float32.
3. The launch counter: every call advances it by one and draws anew; the same seed and counter draw the same times.
4. An empty mask changes no byte; a full mask equals reset(None) given the same times.
5. A random-policy rollout with the step graph and the reset_done graph is bit-identical to the same rollout run eagerly with
   reset_masked, and the graphed reset_done makes no host synchronisation.
6. With cfg.env.transform_specs, reset_done is the id-list reset."""
import numpy as np
import pytest
import torch

from test_gpu_task import _ml, make_task

pytestmark = pytest.mark.gpu

N = 8 * 16 + 3
F = np.float32


def buffers(t):
    t._context_buffers()
    return dict(root=t._root_states, dof=t._dof_state, rb=t._rigid_body_state, cf=t._contact_force_tensor, obs=t.obs_buf, rew=t.rew_buf,
                sub=t._sub_rewards, prog=t.progress_buf, reset=t.reset_buf, term=t._terminate_buf, times=t._cur_ref_motion_times,
                reset_times=t._reset_ref_motion_times, acts=t.actions, pd=t._pd_target_dof_pos, p_dof=t._prev_target_dof_pos,
                p_dofv=t._prev_target_dof_vel, p_rbp=t._prev_target_rb_pos, p_rbr=t._prev_target_rb_rot, t_rootp=t._target_root_pos,
                t_rootr=t._target_root_rot, t_dof=t._target_dof_pos, t_rootv=t._target_root_vel, t_rootav=t._target_root_ang_vel,
                t_dofv=t._target_dof_vel, t_key=t._target_key_pos, t_rbp=t._target_rb_pos, t_rbr=t._target_rb_rot,
                init_root=t._initial_humanoid_root_states, init_dof=t._initial_dof_pos, init_dofv=t._initial_dof_vel, ctx=t.context_feat,
                ctx_mask=t.context_mask, motion_ids=t._reset_ref_motion_ids, motion_bodies=t._reset_ref_motion_bodies)


def prefill(tasks, seed=3):
    """the same seeded values in every buffer of every task (motion ids and bodies as the tasks sampled them)"""
    rng = np.random.default_rng(seed)
    for k, b in buffers(tasks[0]).items():
        if k in ("motion_ids", "motion_bodies"):
            continue
        if b.dtype == torch.bool:
            v = torch.from_numpy(rng.integers(0, 2, tuple(b.shape)).astype(bool))
        elif b.dtype.is_floating_point:
            v = torch.from_numpy(rng.normal(0, 1, tuple(b.shape)).astype(F))
        else:
            v = torch.from_numpy(rng.integers(0, 3, tuple(b.shape)))
        for t in tasks:
            buffers(t)[k].copy_(v.to(b.dtype))
    torch.cuda.synchronize()


def _bits(b):
    return b.view(torch.int32) if b.dtype == torch.float32 else b


def snapshot(t):
    return {k: _bits(b).clone() for k, b in buffers(t).items()}


def differing(a, b):
    """names of the buffers of two snapshots / tasks that differ in any bit"""
    a = a if isinstance(a, dict) else snapshot(a)
    b = b if isinstance(b, dict) else snapshot(b)
    return [k for k in a if not torch.equal(a[k], b[k])]


def draws(seed, counter, n):
    """numpy restatement of the kernel's draws: u_k = (splitmix hash of (seed, counter, 2e + k)) >> 40, times 2^-24"""
    from oracle.ref_port_v2p import counter_hash
    e = np.arange(n, dtype=np.uint64)
    u = lambda k: (counter_hash(seed, counter, e * np.uint64(2) + np.uint64(k)) >> np.uint64(40)).astype(F) * F(2.0 ** -24)  # noqa: E731
    return u(0), u(1)


def expected(t, counter, lengths=None):
    """(motion times, ref-state init?) of every env for the task's state init, in float32 like the kernel"""
    sample = t._state_init in ("Random", "Hybrid")
    p = {"Start": 1.0, "Random": 1.0, "Hybrid": min(float(t._hybrid_init_prob), 1.0), "Default": 0.0}[t._state_init]
    u0, u1 = draws(t.cfg.get("seed", 10), counter, t.num_envs)
    L = (t._ml_t["motion_lengths"] if lengths is None else lengths).cpu().numpy()[t._reset_ref_motion_ids.cpu().numpy()].astype(F)
    trunc = F(t.context_length * t.dt) if t.truncate_time else F(0)
    times = (u0 * np.maximum((L - trunc).astype(F), F(0))).astype(F) if sample else np.zeros(t.num_envs, F)
    return times, u1 < F(p)


def id_list_reset(t, mask, times, ref):
    """the same reset through the id-list launches: b200env_reset + the reset times + b200env_motion_context for the ref-state rows,
    `_reset_default` for the others"""
    dev = t.device
    ids = torch.from_numpy(np.flatnonzero(mask & ref)).to(dev)
    dids = torch.from_numpy(np.flatnonzero(mask & ~ref)).to(dev)
    if len(dids):
        t._reset_default(dids)
    if len(ids):
        tt = torch.from_numpy(times).to(dev)[ids].contiguous()
        t._env.reset(ids, tt)
        t._reset_ref_motion_times[ids] = tt
        t._init_context(ids, t._reset_ref_motion_ids[ids], tt)
    torch.cuda.synchronize()


def reset_mask_of(n, seed=5):
    rng = np.random.default_rng(seed)
    m = rng.random(n) < 0.3
    m[[0, n - 1, 64, 9]] = True
    m[[1, 8, 10, 63, 65, n - 2]] = False          # 9 and 64 isolated
    return m


def _assets_cfg():
    from test_gpu_assets import scaled
    from vid2player3d_b200 import model_compiler
    big = scaled(model_compiler.load_compiled("smpl_mesh_humanoid_amass_v1"), 1.1)
    return ["mjcf/smpl_mesh_humanoid_amass_v1.xml" if m % 2 == 0 else big for m in range(len(_ml()["num_frames"]))]


CASES = [("Start", 1.0, True, False), ("Random", 1.0, True, False), ("Random", 1.0, False, False), ("Hybrid", 1.0, True, False),
         ("Hybrid", 1.0, False, False), ("Hybrid", 0.3, True, False), ("Hybrid", 0.0, True, False), ("Default", 1.0, True, False),
         ("Hybrid", 0.3, True, True)]


@pytest.mark.parametrize("state_init,p,truncate,multi", CASES,
                         ids=[f"{s}-p{p}-{'trunc' if tr else 'notrunc'}{'-assets' if mu else ''}" for s, p, tr, mu in CASES])
def test_masked_reset_equals_id_list(state_init, p, truncate, multi):
    over = dict(stateInit=state_init, hybridInitProb=p, truncate_time=truncate)
    if multi:
        over["motion_assets"] = _assets_cfg()
    a, b = make_task(N, 0.3, **over), make_task(N, 0.3, **over)
    assert torch.equal(a._reset_ref_motion_ids, b._reset_ref_motion_ids)
    if multi:
        assert a._env.asset_plan[0] == 2
    prefill([a, b])
    mask = reset_mask_of(N)
    c0 = int(a._reset_rng.item())
    times, ref = expected(a, c0)
    before = snapshot(a)
    a.reset_masked(torch.from_numpy(mask).to(a.device))
    torch.cuda.synchronize()
    assert int(a._reset_rng.item()) == c0 + 1 and not a._reset_work[:2].any()
    got = a._reset_ref_motion_times.cpu().numpy()
    rows = np.flatnonzero(mask & ref)
    assert np.array_equal(got[rows].view(np.uint32), times[rows].view(np.uint32)), "drawn times differ from the numpy restatement"
    id_list_reset(b, mask, times, ref)
    assert differing(a, b) == [], f"{state_init}: the masked reset differs from the id-list reset"
    after = snapshot(a)
    for k in before:
        if after[k].dim() and after[k].shape[0] == N:
            assert torch.equal(after[k][~torch.from_numpy(mask).to(a.device)], before[k][~torch.from_numpy(mask).to(a.device)]), k
    if state_init == "Hybrid" and 0 < p < 1:
        assert 0 < ref[mask].sum() < mask.sum()
    print(f"\n{state_init} p {p}: {int(mask.sum())} of {N} envs reset, {int((mask & ref).sum())} from the MoCap")


def test_draw_at_the_edges_of_the_product():
    """motion lengths around the truncation and at the float32 extremes: the kernel's times equal the numpy restatement bit for bit,
    and t is exactly 0 for every length up to the truncation"""
    a = make_task(N, 0.3, stateInit="Random")
    M = len(_ml()["num_frames"])
    a._reset_ref_motion_ids.copy_(torch.arange(N, device=a.device) % M)
    trunc = F(a.context_length * a.dt)
    edges = np.array([np.nextafter(trunc, F(0)), trunc, np.nextafter(trunc, F(np.inf)), F(0), np.finfo(F).max, F(1e-40), F(0.05),
                      trunc * F(3)], F)
    assert len(edges) == M
    lengths = a._ml_t["motion_lengths"].clone()
    a._ml_t["motion_lengths"].copy_(torch.from_numpy(edges).to(a.device))
    try:
        for _ in range(3):
            c = int(a._reset_rng.item())
            times, _ = expected(a, c)
            a.reset_masked(torch.ones(N, dtype=torch.bool, device=a.device))
            got = a._reset_ref_motion_times.cpu().numpy()
            assert np.array_equal(got.view(np.uint32), times.view(np.uint32)), c
            mid = np.arange(N) % M
            assert (got[edges[mid] <= trunc] == 0).all() and (got[edges[mid] > trunc] > 0).any()
            assert (got[mid == 4] > F(1e38)).any() and np.isfinite(got).all()
    finally:
        a._ml_t["motion_lengths"].copy_(lengths)


def test_counter_draws_anew_and_replays():
    """without truncate_time every env has a positive range of times, so a new draw moves every time"""
    a = make_task(N, 0.3, stateInit="Random", truncate_time=False)
    full = torch.ones(N, dtype=torch.bool, device=a.device)
    a.reset_masked(full)
    t1 = a._reset_ref_motion_times.clone()
    a.reset_masked(full)
    t2 = a._reset_ref_motion_times.clone()
    assert int(a._reset_rng.item()) == 2
    assert (t1 != t2).float().mean() > 0.9, "two launches drew the same times"
    a._reset_rng.fill_(0)
    a.reset_masked(full)
    assert torch.equal(a._reset_ref_motion_times, t1)
    b = make_task(N, 0.3, stateInit="Random", truncate_time=False)
    b.reset_masked(full)
    assert torch.equal(b._reset_ref_motion_times, t1)


def test_empty_mask_and_full_mask():
    a, b = make_task(N, 0.3, stateInit="Random"), make_task(N, 0.3, stateInit="Random")
    prefill([a, b])
    before = snapshot(a)
    a.reset_masked(torch.zeros(N, dtype=torch.bool, device=a.device))
    torch.cuda.synchronize()
    assert differing(before, a) == [] and int(a._reset_rng.item()) == 1
    times, _ = expected(a, 1)
    a.reset_masked(torch.ones(N, dtype=torch.bool, device=a.device))
    tt = torch.from_numpy(times).to(b.device)
    b.sample_time = lambda motion_ids, truncate_time=None: tt.clone()
    b.reset(None)
    torch.cuda.synchronize()
    assert differing(a, b) == [], "reset_masked(all) differs from reset(None) at the same times"


def _graphed_and_eager(n, over):
    """two tasks in the same state: `a` behind a VecTaskPythonWrapper with the step and reset graphs, `b` eager after the same warm-up
    (3 steps and an empty reset); then every env of both reset through reset_done / reset_masked"""
    from vid2player3d_b200.tasks.vec_task import VecTaskPythonWrapper
    a, b = make_task(n, 0.3, **over), make_task(n, 0.3, **over)
    w = VecTaskPythonWrapper(a, a.device)
    w.enable_cuda_graph(reset_graph=True)
    for _ in range(3):
        b.step(torch.clamp(torch.zeros(n, b.num_actions, device=b.device), -1.0, 1.0))
    b.reset_masked(torch.zeros(n, dtype=torch.bool, device=b.device))
    torch.cuda.synchronize()
    assert differing(a, b) == []
    a.reset_buf.fill_(1)
    w.reset_done()
    b.reset_masked(torch.ones(n, dtype=torch.bool, device=b.device))
    torch.cuda.synchronize()
    assert differing(a, b) == []
    return w, a, b


def test_graphed_rollout_equals_eager_reset_masked():
    """U(-1, 1) actions for 48 steps: step graph + reset_done graph against step + reset_masked(reset_buf != 0) eagerly"""
    n, steps = N, 48
    w, a, b = _graphed_and_eager(n, dict(stateInit="Hybrid", hybridInitProb=0.5))
    g = torch.Generator(device=a.device).manual_seed(11)
    acts = [torch.rand(n, a.num_actions, device=a.device, generator=g) * 2 - 1 for _ in range(steps)]
    mask_b = torch.zeros(n, dtype=torch.bool, device=b.device)
    resets = torch.zeros((), dtype=torch.long, device=a.device)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for i in range(steps):
            w.step(acts[i])
            resets += a.reset_buf.sum()
            obs = w.reset_done()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    for i in range(steps):
        b.step(torch.clamp(acts[i], -1.0, 1.0))
        torch.ne(b.reset_buf, 0, out=mask_b)
        b.reset_masked(mask_b)
    torch.cuda.synchronize()
    assert int(resets) > 0, "no env finished: the rollout did not exercise the reset"
    assert differing(a, b) == [], "graphed step + reset_done differs from the eager rollout"
    assert torch.equal(obs, torch.clamp(b.obs_buf, -5.0, 5.0))
    assert int(a._reset_rng.item()) == int(b._reset_rng.item()) == steps + 2
    print(f"\n{steps} steps of {n} envs: {int(resets)} resets")


def test_transform_specs_fall_back_to_the_id_list():
    """with cfg.env.transform_specs no reset graph is captured, reset_masked refuses, and reset_done is reset(reset_buf.nonzero())"""
    from vid2player3d_b200.tasks.vec_task import VecTaskPythonWrapper
    over = dict(stateInit="Random", transform_specs={"mask_joints": {"joints": ["L_Hand", "R_Toe"]}})
    a, b = make_task(N, 0.3, **over), make_task(N, 0.3, **over)
    with pytest.raises(ValueError):
        a.reset_masked(torch.ones(N, dtype=torch.bool, device=a.device))
    wa, wb = VecTaskPythonWrapper(a, a.device), VecTaskPythonWrapper(b, b.device)
    for w in (wa, wb):
        w.enable_cuda_graph(reset_graph=True)
    assert a._reset_graph is None
    torch.cuda.synchronize()
    assert differing(a, b) == []
    for t in (a, b):
        t.reset_buf.copy_(torch.from_numpy(reset_mask_of(N).astype(np.int64)).to(t.device))
    torch.manual_seed(4)
    obs = wa.reset_done()
    torch.manual_seed(4)
    b.reset(b.reset_buf.nonzero(as_tuple=False).flatten())
    torch.cuda.synchronize()
    assert differing(a, b) == [], "reset_done with transform_specs differs from the id-list reset"
    assert torch.equal(obs, torch.clamp(b.obs_buf, -5.0, 5.0))
