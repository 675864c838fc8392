"""The edge catalogue of tests/test_physics_edges.py on the GPU.

1. b200env_physics_only in float64 with the DOF force sensor on every finite case, against the float64 restatement within 1e-9 of
   each env's scale.
2. The real step (HumanoidSMPLIM on amass, HumanoidSMPLIMMVAE on federer) at N = 2 B G + 5 with the edge envs placed at every env
   slot g of a full batch in both rounds and in the ragged last batch.  Every placement of a case gives the same rows bit for bit;
   against the restatement fed the PD targets the launch consumed, each case is held to the float32 bound of its kind
   (test_physics_edges.f32_failures: the free / settled bounds of tests/test_gpu_parity.py scaled by the state's angular speed,
   q compared as a geodesic angle within 1e-2 of pi, a vector flip accepted only there); the sensor rows of the limit cases lie within
   tests/test_gpu_dof_force.float_bound.
3. Exact invariants: negating the root quaternion negates every rigid-body quaternion row, and with them the quaternion columns
   of the imitation task's raw-state observation, and leaves the root position and velocities, the dof rows, the contact forces,
   every other observation column, the reset flags and the sensor rows bit-identical.  The reward is held to round-off only: it
   takes the angle of each body's rotation difference as 2 acos(w) (ref_quat_to_angle_axis, as the reference's
   quat_to_angle_axis), and w changes sign with -Q, so the same angle may come out of a different float path.
4. Non-finite envs: NaN and +Inf in each of the root position, root quaternion, one joint q, one joint qd, one PD action, the
   residual wrench and (federer) the ball position and velocity, each alone in its warp - at every slot g of full batches in the
   first and second round, and in the ragged last batch - so that the three finite envs sharing the warp are compared too: every
   other env's rows are bit-identical to the run where they are finite; an env whose restatement fails or goes non-finite keeps a
   non-finite row; a NaN action or joint angle gives a NaN PD target, as torch.maximum / torch.minimum do.
5. DOF force sensor rows bit-identical across launch sizes, a seeded permuted layout and the sorted hand-out (B200ENV_SORT=1)."""
import numpy as np
import pytest
import torch

import test_physics_edges as E
from test_dof_force import model_arrays, sensor_from_state, start_of_last_substep
from test_gpu_dof_force import float_bound
from test_gpu_launch import EPW, RES, _by_env, _form, _load, _pool, _read, assert_identical, Layout, layout_problems, permuted_layout

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------ 1. float64 test launch
def test_physics_only_float64_matches_restatement():
    from vid2player3d_b200 import native
    cases = E.catalogue()
    fails, seen = [], 0
    for grp in E._groups(cases):
        W = grp[0].W
        n = len(grp)
        env = native.Env(W.ms, W.verts, W.cfg, n, 0)
        if W.faces is not None:
            env.set_hull_faces(*W.faces)
        S = lambda k: torch.tensor(np.stack([c.st[k] for c in grp]), dtype=torch.float64, device="cuda:0").contiguous()  # noqa: E731
        r, q, qd, tar, ext = S("root"), S("q"), S("qd"), S("tar"), S("ext")
        ball = S("ball") if W.has_ball else None
        hits = torch.zeros(n, dtype=torch.int32, device="cuda:0") if W.has_ball else None
        rb = torch.zeros(n, W.nb, 13, dtype=torch.float64, device="cuda:0")
        cf = torch.zeros(n, W.nb, 3, dtype=torch.float64, device="cuda:0")
        tau = torch.full((n, W.nd), float("nan"), dtype=torch.float64, device="cuda:0")
        env.physics_only(r, q, qd, tar, ext, rb, cf, n_steps=1, ball=ball, ball_hits=hits, dof_force=tau)
        torch.cuda.synchronize()
        g = lambda x: x.cpu().numpy() if x is not None else None  # noqa: E731
        got = dict(root=g(r), q=g(q), qd=g(qd), rb=g(rb), cf=g(cf), ball=g(ball), hits=g(hits), tau=g(tau))
        ref = E.restate(W, [c.st for c in grp])
        names = [c.name for c in grp]
        fails += E.f64_failures(names, got, ref, keys=("root", "q", "qd", "rb", "cf", "ball"))
        free = [i for i in range(n) if np.linalg.norm(ref["qd"][i].reshape(-1, 3), axis=-1).max() < E.WMAX * (1 - 1e-9)]
        sen = E.restate_sensor(W, [grp[i].st for i in free])
        fails += E.f64_failures([names[i] for i in free], dict(tau=got["tau"][free]), sen, keys=("tau",))
        if W.has_ball and not np.array_equal(got["hits"], ref["hits"]):
            fails.append(f"{W.name}: racket hits {got['hits'].tolist()} != {ref['hits'].tolist()}")
        seen += n
    print(f"\n{seen} edge cases, b200env_physics_only float64 against the restatement")
    assert not fails, "\n".join(fails)


# ------------------------------------------------------------------------------------------------ tasks with the sensor
_tasks = {}


def _task(wl, n, form="default"):
    from test_gpu_dof_force import _amass_task, _ball_task
    with _form(form):
        t = _amass_task(n) if wl == "humanoid" else _ball_task(n)
    return t


def _shape(wl):
    if wl not in _tasks:
        _tasks[wl] = _task(wl, 1)._env.physics_launch_shape
    return _tasks[wl]


def _rows(t, wl, n):
    rows = _read(t, wl, n)
    g = lambda x: x.detach().cpu().numpy().reshape(n, -1).copy()  # noqa: E731
    rows.update(obs=g(t.obs_buf), rew=g(t.rew_buf), reset=g(t.reset_buf), term=g(t._terminate_buf), pd=g(t._pd_target_dof_pos),
                tau=g(t.dof_force_tensor))
    return rows


def _phys(rows):
    """the rows that depend on the env's state and actions only (the observation, reward and reset flags also depend on the
    reference motion each env index is given when the task is made)"""
    return {k: v for k, v in rows.items() if k not in ("obs", "rew", "reset", "term")}


class _TaskWorkload:
    """the restatement's inputs from a task (test_physics_edges.restate takes a Workload)"""

    def __init__(self, t, wl):
        from vid2player3d_b200 import abi
        self.ms, self.verts, self.cfg = t._model_struct, t._verts, t._cfg_struct
        self.faces = abi.pack_faces(t._model, t._verts) if wl == "ball" else None
        self.has_ball = wl == "ball"


def _step(wl, pool, perm, form="default"):
    n = len(perm)
    t = _task(wl, n, form)
    a = _load(t, wl, pool, perm)
    t.step(a)
    torch.cuda.synchronize()
    return t, _rows(t, wl, n)


def _case_pool(wl, cases, P):
    """the launch pool of test_gpu_launch with the cases' states: actions that give the cases' PD targets (pd_mode 0: the target;
    pd_mode 1: target dof = the target, action 0), no residual wrench"""
    pool = {k: v[:P].copy() for k, v in _pool(wl).items()}
    for j, c in enumerate(cases):
        st = c.st
        pool["root"][j] = st["root"]
        pool["q"][j], pool["qd"][j] = st["q"], st["qd"]
        if wl == "humanoid":
            pool["act"][j] = np.concatenate([st["tar"], st["ext"][:6] / RES])
        else:
            pool["act"][j] = 0.0
            pool["t_dof"][j] = st["tar"]
            pool["ball"][j] = st["ball"]
        pool["kind"][j] = -1
    return pool


def _placements(ncases, B, G, n):
    """positions of case j: slot g of a full batch in round 0 and in round 1, for every g, and (the first EPW + 1 cases) the
    ragged last batch"""
    pos = {}
    for j in range(ncases):
        p = []
        for rnd in (0, 1):
            base = rnd * B * G + (1 + j) * B     # batch 1 + j of the round: full batches
            p += [base + 4 * (j % (B // 4)) + g for g in range(EPW)]
        pos[j] = p
    tail = (n - 1) // B * B
    for j in range(min(ncases, n - tail)):
        pos[j].append(tail + j)
    return pos


# ------------------------------------------------------------------------------------------------ 2. + 3. float32 step launch
@pytest.mark.parametrize("wl", ["humanoid", "ball"])
def test_step_launch_on_the_edge_cases(wl):
    B, G = _shape(wl)
    n = 2 * B * G + 5
    W = E.workload("amass", "sub2") if wl == "humanoid" else E.workload("federer", "ball")
    cases = [c for c in E.catalogue() if c.W is W]
    assert len(cases) >= 10
    P = len(_pool(wl)["kind"])
    pool = _case_pool(wl, cases, P)
    pos = _placements(len(cases), B, G, n)
    taken = [p for ps in pos.values() for p in ps]
    assert len(set(taken)) == len(taken)
    perm = np.empty(n, np.int64)
    for j, ps in pos.items():
        perm[ps] = j
    free_pos = np.setdiff1d(np.arange(n), taken)
    perm[free_pos] = np.arange(len(cases), len(cases) + len(free_pos))       # the other pool envs fill the rest
    t, rows = _step(wl, pool, perm)
    # every placement of a case: bit-identical rows
    fails = []
    for j, ps in pos.items():
        for p in ps[1:]:
            for key, v in _phys(rows).items():
                if not E._bits_equal(v[ps[0]], v[p]):
                    fails.append(f"{cases[j].name}: {key} at position {p} differs from position {ps[0]}")
    # against the restatement, fed the PD targets of the launch
    first = [ps[0] for ps in pos.values()]
    f64 = lambda x: np.ascontiguousarray(x, np.float64)  # noqa: E731
    pd = rows["pd"][first]
    lim = np.float32(t._cfg_struct.pd_tar_lim)
    sts = []
    for j, c in enumerate(cases):
        st = dict(c.st, tar=f64(pd[j]), ext=np.zeros(6))
        for key in ("root", "q", "qd", "ball"):
            if st.get(key) is not None:
                st[key] = f64(np.float32(st[key]))
        sts.append(st)
    ref = E.restate(_TaskWorkload(t, wl), sts)
    got = dict(root=rows["root"][first, :13], q=rows["dof"][first].reshape(-1, 69, 2)[..., 0], qd=rows["dof"][first].reshape(-1, 69, 2)[..., 1])
    fails += E.f32_failures(cases, got, ref)
    if wl == "ball":
        hit = rows["racket_hit_now"][first, 0] != 0
        if not np.array_equal(hit, ref["hits"] > 0):
            fails.append(f"racket hits {hit.astype(int).tolist()} != restatement {(ref['hits'] > 0).astype(int).tolist()}")
    # the PD targets: the clamp of step_prologue
    base = pool["act"][:len(cases), :69] if wl == "humanoid" else pool["t_dof"][:len(cases)] + pool["act"][:len(cases), :69]
    want = np.maximum(np.minimum(base, pool["q"][:len(cases)] + lim), pool["q"][:len(cases)] - lim)
    if not np.array_equal(pd, want):
        fails.append("PD targets differ from the clamp")
    # sensor rows of the limit cases within the float32 bound, on the step's own end state
    lim_j = [j for j, c in enumerate(cases) if c.branch.startswith("limit")]
    if lim_j:
        ms, cfg = t._model_struct, t._cfg_struct
        q64, qd64 = got["q"][lim_j].astype(np.float64), got["qd"][lim_j].astype(np.float64)
        qs, qdp = start_of_last_substep(ms, cfg, q64, qd64)
        tar = pd[lim_j].astype(np.float64)
        ref_tau, bound = sensor_from_state(ms, cfg, qs, qdp, tar), float_bound(ms, cfg, qs, qdp, tar)
        a = model_arrays(ms)
        edge = (np.abs(qs - a["lim_lo"]) < 1e-4) | (np.abs(qs - a["lim_hi"]) < 1e-4)
        ratio = np.where(edge, 0.0, np.abs(rows["tau"][first][lim_j] - ref_tau) / bound)
        print(f"\nlimit cases: worst sensor error / float32 bound {ratio.max():.3f}")
        if not ratio.max() <= 1.0:
            fails.append(f"limit cases: sensor error / bound {ratio.max():.3f} > 1")
    # -Q: the case "root w < 0" run again with -Q in its places (same positions, so the same reference motion): rigid-body
    # quaternions negated, every other row bit-identical; the reward to round-off
    names = [c.name for c in cases]
    if "root w < 0" in names:
        ja = names.index("root w < 0")
        pool2 = {k: v.copy() for k, v in pool.items()}
        pool2["root"][ja, 3:7] *= -1
        _, rows2 = _step(wl, pool2, perm)
        a_ = pos[ja][0]
        nb = t.num_bodies
        ra, rb_ = rows["rb"][a_].reshape(-1, 13), rows2["rb"][a_].reshape(-1, 13)
        if not E._bits_equal(ra[:nb, 3:7], -rb_[:nb, 3:7]):
            fails.append("-Q: rigid-body quaternions are not negated")
        if not (E._bits_equal(ra[:nb, :3], rb_[:nb, :3]) and E._bits_equal(ra[:nb, 7:], rb_[:nb, 7:])):
            fails.append("-Q: rigid-body positions / velocities differ")
        r1, r2 = rows["root"][a_], rows2["root"][a_]
        if not (E._bits_equal(r1[3:7], -r2[3:7]) and E._bits_equal(r1[:3], r2[:3]) and E._bits_equal(r1[7:], r2[7:])):
            fails.append("-Q: root rows")
        for key in [k for k in rows if k not in ("root", "rb", "rew", "obs")]:
            if not E._bits_equal(rows[key][a_], rows2[key][a_]):
                fails.append(f"-Q: {key} differs")
        # the raw-state observation of HumanoidSMPLIM (humanoid_smpl_im.py:653-668) holds the rigid-body quaternions at [3 nb, 7 nb)
        o1, o2 = rows["obs"][a_], rows2["obs"][a_]
        qc = np.zeros(len(o1), bool)
        qc[3 * nb:7 * nb] = True
        if not (E._bits_equal(o1[qc], -o2[qc]) and E._bits_equal(o1[~qc], o2[~qc])):
            fails.append(f"-Q: observation columns {np.flatnonzero((o1 != o2) & ~qc)[:20].tolist()} differ, or the quaternion columns "
                         f"{np.flatnonzero((o1 != -o2) & qc)[:20].tolist()} are not negated")
        if not np.allclose(rows["rew"][a_], rows2["rew"][a_], rtol=1e-5, atol=1e-6):
            fails.append(f"-Q: reward {rows['rew'][a_]} vs {rows2['rew'][a_]}")
    print(f"\n{wl}: {len(cases)} edge cases at {sum(len(p) for p in pos.values())} positions of N = {n} (B = {B}, G = {G})")
    assert not fails, "\n".join(fails)


# ------------------------------------------------------------------------------------------------ 4. non-finite envs
NONFINITE_FIELDS = (("root position", "root", 0), ("root quaternion", "root", 3), ("joint q", "q", E.KNEE), ("joint qd", "qd", E.KNEE + 1),
                    ("PD action", "act", E.KNEE), ("residual wrench", "act", 69), ("ball position", "ball", 0), ("ball velocity", "ball", 8))


def nonfinite_spots(nmut, B, G, n):
    """launch positions of the non-finite envs: mutation i in a warp of its own of a full batch in the first round (slot i % 4) and
    in the second round (slot (i + 1) % 4), and mutation 0 at slot 3 of the ragged last batch's first warp.  Every other env of
    those warps is finite, so a leak inside a warp reaches a compared env."""
    wpb = B // EPW
    spots = []
    for i in range(nmut):
        off = (1 + i // wpb) * B + EPW * (i % wpb)
        spots += [(off + i % EPW, i), (B * G + off + (i + 1) % EPW, i)]
    spots.append(((n - 1) // B * B + 3, 0))
    return spots


@pytest.mark.parametrize("wl", ["humanoid", "ball"])
def test_nonfinite_envs(wl):
    from oracle import physics_ref, ref_port as R
    from test_gpu_launch import position
    from vid2player3d_b200 import abi
    B, G = _shape(wl)
    n = 2 * B * G + 5
    muts = [(f"{'NaN' if np.isnan(v) else '+Inf'} {name}", key, idx, v) for name, key, idx in NONFINITE_FIELDS for v in (np.nan, np.inf)
            if key != "ball" or wl == "ball"]
    spots = nonfinite_spots(len(muts), B, G, n)
    where = [position(p, B, G) for p, _ in spots]
    warps = [(w[1], w[2]) for w in where]
    assert len(set(warps)) == len(warps), "one non-finite env per warp"
    assert {w[3] for w in where if w[0] == 0} == {w[3] for w in where if w[0] == 1} == set(range(EPW))
    assert where[-1][0] == 2 and (n - 1) // B * B + 3 < n
    pool = {k: v.copy() for k, v in _pool(wl).items()}
    perm = np.arange(n)
    _, ref_rows = _step(wl, pool, perm)
    bad = {}
    for p, i in spots:
        name, key, idx, val = muts[i]
        pool[key][p, idx] = val
        bad[p] = name
    t, rows = _step(wl, pool, perm)
    others = np.setdiff1d(np.arange(n), [p for p, _ in spots])
    Lay = Layout("natural order", B, G, np.arange(len(pool["kind"])))
    assert_identical({k: v for k, v in ref_rows.items()}, rows, others, Lay, Lay)
    fails = []
    lim = np.float32(t._cfg_struct.pd_tar_lim)
    cfg = t._cfg_struct
    for p, name in bad.items():
        a = pool["act"][p, :69]
        base = a if wl == "humanoid" else pool["t_dof"][p] + a
        want = np.maximum(np.minimum(base, pool["q"][p] + lim), pool["q"][p] - lim)
        pd = rows["pd"][p]
        if not (np.array_equal(np.isnan(pd), np.isnan(want)) and np.array_equal(pd[~np.isnan(want)], want[~np.isnan(want)])):
            fails.append(f"{name} at {p}: PD target {pd[np.isnan(want) != np.isnan(pd)]} where the clamp of torch.maximum / torch.minimum "
                         f"gives {want[np.isnan(want) != np.isnan(pd)]}")
        f64 = lambda x: np.ascontiguousarray(x, np.float64)  # noqa: E731
        _, _, force, torque = R.pre_physics(f64(pool["act"][p:p + 1]), np.zeros(1), f64(pool["q"][p:p + 1]), f64(pool["root"][p:p + 1, 3:7]),
                                            69, float(lim), float(cfg.res_force_scale), float(cfg.res_torque_scale))
        o = dict(root=f64(pool["root"][p:p + 1]), q=f64(pool["q"][p:p + 1]), qd=f64(pool["qd"][p:p + 1]))
        ball = f64(pool["ball"][p:p + 1]) if wl == "ball" else None
        if wl == "ball":
            physics_ref.set_hull_faces(*abi.pack_faces(t._model, t._verts))
        try:
            physics_ref.control_step(t._model_struct, t._verts, cfg, o["root"], o["q"], o["qd"], f64(pd[None]), f64(np.concatenate([force, torque], 1)),
                                     ball=ball, hits=np.zeros(1, np.int32) if ball is not None else None)
            ref_bad = not (np.isfinite(o["root"]).all() and np.isfinite(o["q"]).all() and np.isfinite(o["qd"]).all()
                           and (ball is None or np.isfinite(ball).all()))
        except RuntimeError:
            ref_bad = True
        finally:
            physics_ref.clear_hull_faces()
        mine_bad = not (np.isfinite(rows["root"][p]).all() and np.isfinite(rows["dof"][p]).all())
        if ref_bad and not mine_bad:
            fails.append(f"{name} at {p}: the restatement goes non-finite, the launch repaired the env to a finite state")
        print(f"  {name:24s} at {p:5d} (round {(p // B) // G}, g {p % EPW}): restatement non-finite {ref_bad}, launch non-finite {mine_bad}")
    print(f"{len(spots)} non-finite envs, each alone in its warp; the other {len(others)} envs bit-identical")
    nan_pd = [p for p, nm in bad.items() if nm in ("NaN PD action", "NaN joint q")]
    assert nan_pd and all(np.isnan(rows["pd"][p]).any() for p in nan_pd), "a NaN action or joint angle must give a NaN PD target"
    assert not fails, "\n".join(fails)


# ------------------------------------------------------------------------------------------------ 5. sensor rows by position and form
@pytest.mark.parametrize("wl", ["humanoid", "ball"])
def test_sensor_rows_do_not_depend_on_the_launch_position_or_form(wl):
    B, G = _shape(wl)
    BG = B * G
    pool = _pool(wl)
    P = len(pool["kind"])
    n_ref = 2 * BG + 5
    _, ref = _step(wl, pool, np.arange(n_ref))
    ref = _by_env(_phys(ref), np.arange(n_ref), P)
    lay = Layout(f"natural order at N={n_ref}", B, G, np.arange(P))
    for n in (1, 5, B + 1, BG + 1):
        _, r = _step(wl, pool, np.arange(n))
        assert_identical(ref, _by_env(_phys(r), np.arange(n), P), np.arange(n), lay, Layout(f"natural order at N={n}", B, G, np.arange(P)))
    perm = permuted_layout(n_ref, B, G, pool["kind"][:n_ref], seed=11)
    assert layout_problems(perm, pool["kind"][:n_ref], B, G) == []
    _, r = _step(wl, pool, perm)
    assert_identical(ref, _by_env(_phys(r), perm, P), np.arange(n_ref), lay, Layout.of_perm(f"permuted layout at N={n_ref}", B, G, perm, P))
    for n in (5, n_ref):
        t, r = _step(wl, pool, np.arange(n), form="sort")
        assert t._env.kernel_form == "packed"
        assert_identical(ref, _by_env(_phys(r), np.arange(n), P), np.arange(n), lay, Layout(f"sorted hand-out at N={n}", B, G, np.arange(P)))
    assert np.isfinite(ref["tau"][:n_ref]).all() and np.abs(ref["tau"][:n_ref]).max() > 0
    print(f"\n{wl}: sensor and state rows bit-identical across sizes, a permuted layout and the sorted hand-out")
