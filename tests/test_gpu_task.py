"""The imitation task's own launches against the numpy task oracle (oracle/ref_port.py, pinned to the reference by
test_oracle_golden.py): MoCap sampling (sample_motion through b200env_motion_state), the reset (reset_kernel), the context window
(motion_context_kernel) and the two task launches of a step (pre_kernel and post_kernel; the fused form runs the same prologue and
epilogue inside its physics launch).  The physics itself is covered by test_gpu_launch.py / test_gpu_parity.py: here the oracle is
resynchronised from the post-physics state the GPU wrote, and only the task logic is under test.

1. An edge motion library: 30, 60 and 24 fps (1/24 is not exact in float32), a 2-frame and a 3-frame motion, a run of bit-identical
   frames (slerp's c >= 1 / sin < 1e-3 branches), quaternions negated from frame to frame (c < 0), near-identity joint rotations,
   nonzero min_verts_h and motion_bodies, and frame velocities that differ from frame to frame (so f0 is visible in them).
2. Sampling at -2dt, -dt, -1 ulp, 0, every frame time and midpoint, length -1 ulp, length, length +1 ulp, length + dt and
   length + 2dt: blend < 0 and > 1 extrapolate, as in the reference (motion_lib.py:427-436 clamps the phase, not the blend).
3. Reset and context: every row the launch writes against the oracle, every other row bit-identical to the sentinel it held.
4. One step from chosen per-env cases that land exactly on every threshold of compute_humanoid_reset and its caller, in float32:
   the updated ref time at the motion length and one ulp either side, progress at max_len - 2 / max_len - 1, a body's z at its
   termination height and one ulp below, a contact body below its height, a fall at progress 1 and 2, sticky resets with both
   terminate values.  The z cases come from the launch itself: a probe step of one copy of an upright pose gives the post-physics z of
   its lowest non-contact body, and the termination height is set to that value (z == height: no fall) or to the next float above
   (z one ulp below: fall).  Copies of the pose give the same rows at every position (test_gpu_launch.py).
5. The task outputs of the default, B200ENV_SORT=1, fused and tmem forms are bit-identical; with two env slices, pre_kernel writes
   actions_used and the PD targets of its own rows only.
6. CPU negative controls: every comparator rejects a mutated oracle and names the env (or sample) and the field.

Quirks of the reference kept by the oracle and so required of the kernels: a time before 0 or past the end extrapolates from the first
or the last frame pair (blend = t / dt - i0 is not clamped); an env already flagged for reset gets reward 0 and keeps its terminate
flag; a fall only terminates from progress 2 on (progress > 1 after the increment)."""
import numpy as np
import pytest
import torch

from helpers import lib_dict

SENT = np.float32(12345.0)     # float rows are filled with it before a launch; integer rows with ISENT
ISENT = 7777
MAX_LEN = 300
DT = np.float32(2) * np.float32(1.0 / 60.0)     # control dt: controlFrequencyInv 2 x sim dt, in float32 as the kernels form it
CONTACT = ["R_Ankle", "L_Ankle", "R_Toe", "L_Toe"]
HEAD = 13
INF = np.float32(np.inf)

EXACT = "exact"
EXPMAP = "expmap"
SAMPLE_SPEC = dict(root_vel=EXACT, root_ang_vel=EXACT, dof_vel=EXACT, root_pos=1e-5, root_rot=1e-5, key_pos=1e-5, rb_pos=1e-5,
                   rb_rot=1e-5, dof_pos=EXPMAP)
TARGETS = dict(t_rootp="root_pos", t_rootr="root_rot", t_dof="dof_pos", t_rootv="root_vel", t_rootav="root_ang_vel",
               t_dofv="dof_vel", t_key="key_pos", t_rbp="rb_pos", t_rbr="rb_rot")
STEP_SPEC = dict(acts=EXACT, pd=EXACT, p_dof=EXACT, p_dofv=EXACT, p_rbp=EXACT, p_rbr=EXACT, prog=EXACT, reset=EXACT, term=EXACT,
                 times=EXACT, obs=EXACT, rew=1e-5, sub=1e-5,
                 **{k: SAMPLE_SPEC[v] for k, v in TARGETS.items()})
KINDS = ("bulk", "t = length", "t = length - ulp", "t = length + ulp", "progress max-2", "progress max-1", "z = height",
         "fall at progress 1", "fall at progress 2", "sticky reset, term 0", "sticky reset, term 1", "bulk")


# ------------------------------------------------------------------------------------------------ edge library and times (CPU)
def nxt(x, d):
    return np.nextafter(np.float32(x), np.float32(d)).astype(np.float32)


def edge_lib(model, seed=0):
    """the seeded FlatMotionLib of the module docstring (8 motions on amass_v1)"""
    from vid2player3d_b200 import motion_lib
    spec = ((30.0, 2, 40, True), (60.0, 2, 50, True), (24.0, 2, 30, True), (30.0, 1, 2, False), (24.0, 1, 3, False))
    flat = motion_lib.FlatMotionLib.merge([motion_lib.synthetic(model, num_motions=m, num_frames=nf, fps=fps, seed=seed + 10 * i,
                                                                sigma=0.06, ragged=rag) for i, (fps, m, nf, rag) in enumerate(spec)])
    rng = np.random.default_rng(seed)
    kw = {k: np.array(getattr(flat, k)) for k in flat.FIELDS}
    M, s = len(kw["num_frames"]), kw["length_starts"]
    for k in ("grvs", "gravs", "dvs"):           # the synthetic copies the second-last frame into the last: make every frame differ
        kw[k] += rng.normal(0, 0.3, kw[k].shape).astype(np.float32)
    run = np.arange(s[0] + 5, s[0] + 9)          # motion 0: four bit-identical frames
    for k in ("gts", "grs", "lrs"):
        kw[k][run] = kw[k][run[0]]
    odd = np.arange(s[1] + 1, s[1] + kw["num_frames"][1], 2)   # motion 1: root and some joints negated on every other frame
    kw["grs"][odd[:, None], [0, 3, 12]] *= -1
    kw["lrs"][odd[:, None], [0, 3, 7, 12]] *= -1
    fr = np.arange(s[2], s[2] + kw["num_frames"][2])           # motion 2: near-identity rotations of three joints
    v = rng.normal(0, 1e-4, (len(fr), 3, 3))
    ang = np.linalg.norm(v, axis=-1, keepdims=True)
    kw["lrs"][fr[:, None], [2, 6, 16]] = np.concatenate([v / ang * np.sin(ang / 2), np.cos(ang / 2)], -1).astype(np.float32)
    kw["grs"][s[6] + 1, 0] *= -1                 # the 2-frame motion: the root flips sign
    kw["min_verts_h"] = rng.uniform(-0.03, 0.05, M).astype(np.float32)
    kw["motion_bodies"] = rng.normal(size=(M, 11)).astype(np.float32)
    return motion_lib.FlatMotionLib(**kw)


def edge_times(ml):
    """every (motion, time, edge class) of the sampling test"""
    ids, ts, cls = [], [], []
    for m in range(len(ml["num_frames"])):
        L, dt, nf = ml["motion_lengths"][m], ml["motion_dt"][m], int(ml["num_frames"][m])
        fi = np.arange(nf, dtype=np.float32)
        groups = (("t < 0", [-2 * dt, -dt, nxt(0, -1)]), ("t = 0", [np.float32(0)]), ("frame", fi * dt),
                  ("midpoint", (fi[:-1] + np.float32(0.5)) * dt), ("length - ulp", [nxt(L, -INF)]), ("length", [L]),
                  ("length + ulp", [nxt(L, INF)]), ("past the end", [L + dt, L + 2 * dt]))
        for c, t in groups:
            t = np.asarray(t, np.float32)
            ids += [m] * len(t)
            ts.append(t)
            cls += [c] * len(t)
    return np.array(ids, np.int64), np.concatenate(ts).astype(np.float32), np.array(cls)


def solve_time(f, target, x0):
    """a float32 x near x0 with f(x) == target, for f monotone non-decreasing in x (stepping one ulp at a time)"""
    x = np.float32(x0)
    for _ in range(4096):
        y = f(x)
        if y == target:
            return x
        x = nxt(x, INF if y < target else -INF)
    raise AssertionError(f"no float32 time reaches {target!r}")


def time_before(target, dt=DT):
    """ref_t with fl(ref_t + dt) == target: the updated ref time of the step lands exactly on target"""
    return solve_time(lambda x: np.float32(x + dt), np.float32(target), np.float32(target) - dt)


# ------------------------------------------------------------------------------------------------ comparators (CPU)
def _flat(a):
    a = np.ascontiguousarray(a)
    return a.reshape(a.shape[0], int(np.prod(a.shape[1:])))


def compare(got, ref, spec, label="env", names=None):
    """got, ref: field -> array [rows, ...]; spec: field -> EXACT (bit for bit), a float tolerance, or EXPMAP (the close_expmap rule of
    test_gpu_parity.py: entries below 2e-3 on both sides within 2e-3, the rest within 1e-5 and at most 1 % of the entries beyond 1e-5;
    and a joint that one side gives as exactly (0, 0, 0) within 1e-2: quat_to_exp_map masks sin_theta = sqrt(1 - w w) <= 1e-5,
    NaN included, and the float32 slerp of a near-identity pair can leave w one ulp at or above 1 on one side only, with |xyz| up to
    ~3e-3 left by the norm error of the blend, so the other side's 2 |xyz| survives).
    Returns (failure lines naming the field and the row, worst |error| per field)."""
    fails, worst = [], {}
    for k, how in spec.items():
        g, r = _flat(got[k]), _flat(ref[k])
        n = g.shape[0]
        rows = names if names is not None else np.arange(n)
        if how == EXACT:
            r = np.ascontiguousarray(r.astype(g.dtype))
            u = f"u{g.dtype.itemsize}"
            bad_e = g.view(u) != r.view(u)
            bad = bad_e.any(1)
            err = np.abs(g.astype(np.float64) - r.astype(np.float64))
            worst[k] = float(np.nanmax(err)) if err.size else 0.0
        else:
            err = np.abs(g.astype(np.float64) - r.astype(np.float64))
            tol = float(how) if how != EXPMAP else 1e-5
            allow = tol
            if how == EXPMAP:
                allow = np.where((np.abs(g) < 2e-3) & (np.abs(r) < 2e-3), 2e-3, tol)
                g3, r3 = g.reshape(n, -1, 3).astype(np.float64), r.reshape(n, -1, 3).astype(np.float64)
                masked = ((g3 == 0).all(-1) | (r3 == 0).all(-1)) & (np.linalg.norm(g3, axis=-1) < 1e-2) & (np.linalg.norm(r3, axis=-1) < 1e-2)
                allow = np.maximum(allow, np.repeat(np.where(masked, 1e-2, 0.0), 3, axis=1))
            bad = (~(err <= allow)).any(1)
            worst[k] = float(np.nanmax(err)) if err.size else 0.0
            if how == EXPMAP and err.size and (err > tol).mean() >= 0.01:
                fails.append(f"{k}: {(err > tol).mean():.3%} of the entries beyond {tol:g} (at most 1 %)")
        for i in np.flatnonzero(bad)[:3]:
            j = int(np.flatnonzero(bad_e[i])[0]) if how == EXACT else int(np.nanargmax(np.where(np.isnan(err[i]), np.inf, err[i])))
            fails.append(f"{k}: {int(bad.sum())} of {n} rows differ; {label} {rows[i]}: column {j} got {g[i, j]!r} ref {r[i, j]!r}"
                         f" (|diff| {np.abs(float(g[i, j]) - float(r[i, j])):.3e}, bound {how})")
    return fails, worst


def assert_match(got, ref, spec, label="env", names=None, what=""):
    fails, worst = compare(got, ref, spec, label, names)
    assert not fails, f"{what}\n" + "\n".join(fails)
    return worst


def sample_rows(ml, ids, times):
    """R.get_motion_state as a field dict"""
    from oracle import ref_port as R
    names = ("root_pos", "root_rot", "dof_pos", "root_vel", "root_ang_vel", "dof_vel", "key_pos", "rb_pos", "rb_rot")
    return dict(zip(names, R.get_motion_state(ml, np.asarray(ids), np.asarray(times, np.float32))))


def oracle_step(ml, inp, rbs, dofs, cfg):
    """ImTaskOracle from the pre-step rows `inp`, stepped on the post-physics state rbs [n,B,13], dofs [n,D,2]; field dict of every
    task output.  The previous targets come from the target rows the step started from."""
    from oracle import ref_port as R
    n = len(inp["mids"])
    orc = R.ImTaskOracle(ml, inp["mids"], inp["times"], inp["prog"], inp["reset"], inp["term"], DT, MAX_LEN, cfg["th"],
                         cfg["contact_ids"], np.ones(rbs.shape[1], np.float32), ml["motion_bodies"][inp["mids"]],
                         enable_early_termination=cfg["early"], pd_tar_lim=cfg["lim"], res_scale=cfg["res"])
    orc.t_dof_pos, orc.t_dof_vel, orc.t_rb_pos, orc.t_rb_rot = inp["t_dof"], inp["t_dofv"], inp["t_rbp"], inp["t_rbr"]
    nd = dofs.shape[1]
    acts = inp["acts"] if inp["acts"].shape[1] == nd + 6 else np.concatenate([inp["acts"], np.zeros((n, 6), np.float32)], 1)
    a, pd, _, _ = orc.pre_physics(acts, inp["q"], inp["rb0_rot"])
    obs, rew, sub = orc.post_physics(rbs, dofs)
    return dict(acts=a[:, :inp["acts"].shape[1]], pd=pd, p_dof=orc.p_dof_pos, p_dofv=orc.p_dof_vel, p_rbp=orc.p_rb_pos,
                p_rbr=orc.p_rb_rot, obs=obs, rew=rew, sub=sub, reset=orc.reset_buf, term=orc.terminate_buf, prog=orc.progress,
                times=orc.ref_times, t_rootp=orc.t_root_pos, t_rootr=orc.t_root_rot, t_dof=orc.t_dof_pos, t_rootv=orc.t_root_vel,
                t_rootav=orc.t_root_ang_vel, t_dofv=orc.t_dof_vel, t_key=orc.t_key_pos, t_rbp=orc.t_rb_pos, t_rbr=orc.t_rb_rot)


def case_counts(ml, inp, out, rbs, cfg):
    """envs of each threshold case that the step reached with the case deciding the outcome (no other reset or fall in play)"""
    z, th = rbs[..., 2], cfg["th"]
    nc = np.ones(len(th), bool)
    nc[cfg["contact_ids"]] = False
    alive = inp["reset"] == 0
    fallen = (z[:, nc] < th[nc]).any(1) & cfg["early"]
    L = ml["motion_lengths"][inp["mids"]]
    quiet = alive & ~fallen & (out["prog"] < MAX_LEN - 2)
    t, p = out["times"], out["prog"]
    below = nxt(th, -INF)
    return {"t = length": quiet & (t == L), "t = length - ulp": quiet & (t == nxt(L, -INF)), "t = length + ulp": quiet & (t == nxt(L, INF)),
            "progress max-2": alive & ~fallen & (t < L) & (p == MAX_LEN - 2),
            "progress max-1": alive & ~fallen & (t < L) & (p == MAX_LEN - 1),
            "z = height": quiet & cfg["early"] & (z[:, nc] == th[nc]).any(1),
            "z = height - ulp": alive & (t < L) & (p > 1) & (p < MAX_LEN - 1) & cfg["early"] & (z[:, nc] == below[nc]).any(1)
            & ~(z[:, nc] < below[nc]).any(1),
            "contact body below height": quiet & cfg["early"] & (z[:, ~nc] < th[~nc]).any(1),
            "fall at progress 1": alive & fallen & (p == 1) & (t < L),
            "fall at progress 2": alive & fallen & (p == 2) & (t < L),
            "sticky reset, term 0": ~alive & (inp["term"] == 0), "sticky reset, term 1": ~alive & (inp["term"] == 1)}


# ------------------------------------------------------------------------------------------------ negative controls (CPU)
_cpu = {}


def _model():
    from vid2player3d_b200 import model_compiler
    if "model" not in _cpu:
        _cpu["model"] = model_compiler.load_compiled("smpl_mesh_humanoid_amass_v1")
    return _cpu["model"]


def _ml():
    if "ml" not in _cpu:
        _cpu["flat"] = edge_lib(_model())
        _cpu["ml"] = lib_dict(_cpu["flat"], _model())
    return _cpu["ml"]


def _cpu_scenario(n=24, seed=4):
    """pre-step rows and a made-up post-physics state (the oracle takes it as given) with one env per threshold case"""
    from vid2player3d_b200 import abi
    ml, model = _ml(), _model()
    rng = np.random.default_rng(seed)
    c = abi.make_cfg(model, contact_bodies=tuple(CONTACT), termination_body_height=0.3)
    cfg = dict(th=np.array(list(c.termination_height)[:24], np.float32), contact_ids=np.array([3, 4, 7, 8]), early=True,
               lim=np.float32(c.pd_tar_lim), res=np.float32(31.85))
    M = len(ml["num_frames"])
    mids = rng.integers(0, M, n)
    mids[:9] = 0                            # the case envs play a long motion: their step ends well before its length
    L = ml["motion_lengths"][mids]
    times = (rng.uniform(0, 0.5, n) * L).astype(np.float32)
    prog = rng.integers(2, 100, n)
    reset, term = np.zeros(n, np.int64), rng.integers(0, 2, n)
    rbs = rng.normal(0, 0.2, (n, 24, 13)).astype(np.float32)
    rbs[..., 2] = rng.uniform(0.6, 1.5, (n, 24)).astype(np.float32)
    rbs[..., 3:7] /= np.linalg.norm(rbs[..., 3:7], axis=-1, keepdims=True)
    rbs[:, HEAD, 2] = 1.6                   # above the head's termination height: only the fall cases fall
    case = {}
    case["t = length"], case["t = length - ulp"], case["t = length + ulp"] = 0, 1, 2
    for e, tgt in ((0, L[0]), (1, nxt(L[1], -INF)), (2, nxt(L[2], INF))):
        times[e] = time_before(tgt)
    case["progress max-1"] = 3
    prog[3] = MAX_LEN - 2
    case["z = height"] = 4
    rbs[4, 10, 2] = cfg["th"][10]
    case["fall at progress 1"] = 5
    prog[5], rbs[5, 16, 2] = 0, np.float32(0.1)
    case["sticky reset"] = 6
    reset[6] = 1
    case["late frame"] = 7                  # the targets of env 7 sample the middle of the last frame pair
    times[7] = solve_time(lambda x: np.float32(np.float32(x + DT) + DT), np.float32(L[7] - np.float32(0.5) * ml["motion_dt"][0]),
                          L[7] - np.float32(2.5) * DT)
    case["extrapolated"] = 8                # ... and env 8 a time before 0
    times[8] = np.float32(-3) * DT
    inp = dict(mids=mids, times=times, prog=prog, reset=reset, term=term, acts=rng.normal(0, 1, (n, 75)).astype(np.float32),
               q=rng.normal(0, 0.3, (n, 69)).astype(np.float32), rb0_rot=rbs[:, 0, 3:7].copy())
    st = sample_rows(ml, mids, times + DT)
    inp.update(t_dof=st["dof_pos"], t_dofv=st["dof_vel"], t_rbp=st["rb_pos"], t_rbr=st["rb_rot"])
    dofs = rng.normal(0, 0.3, (n, 69, 2)).astype(np.float32)
    return ml, inp, rbs, dofs, cfg, case


def test_edge_library_has_every_edge():
    ml, flat = _ml(), _cpu["flat"]
    assert set(np.round(1.0 / ml["motion_dt"]).astype(int)) == {24, 30, 60} and float(np.float32(1 / 24)) != 1 / 24
    assert {2, 3} <= set(ml["num_frames"].tolist())
    s = ml["length_starts"]
    assert np.array_equal(flat.grs[s[0] + 5], flat.grs[s[0] + 8])
    assert (np.sum(flat.grs[s[1]:s[1] + 10, 0] * flat.grs[s[1] + 1:s[1] + 11, 0], -1) < 0).all()
    v = np.linalg.norm(flat.lrs[s[2]:s[2] + 5, 2, :3], axis=-1)
    assert ((v > 0) & (v < 1e-3)).all()
    assert (ml["min_verts_h"] != 0).all() and (ml["motion_bodies"] != 0).all()
    last = s + ml["num_frames"] - 1
    assert (ml["grvs"][last] != ml["grvs"][last - 1]).all() and (ml["dvs"][last] != ml["dvs"][last - 1]).any(1).all()


def test_sampling_comparator_rejects_mutated_oracles(monkeypatch):
    """f0 one frame late at the last frame, and the blend clamped to [0, 1]: the comparator names the sample and the field"""
    from oracle import ref_port as R
    ml = _ml()
    ids, ts, cls = edge_times(ml)
    ref = sample_rows(ml, ids, ts)
    assert compare(ref, ref, SAMPLE_SPEC, "sample")[0] == []
    orig = R.calc_frame_blend

    def late(time, length, num_frames, dt):
        i0, i1, b = orig(time, length, num_frames, dt)
        i0 = np.where(i0 == num_frames - 2, num_frames - 1, i0)
        return i0, i1, b

    def clamped(time, length, num_frames, dt):
        i0, i1, b = orig(time, length, num_frames, dt)
        return i0, i1, np.clip(b, 0, 1).astype(b.dtype)

    i0 = orig(ts, ml["motion_lengths"][ids], ml["num_frames"][ids], ml["motion_dt"][ids])[0]
    for mut, field, where in ((late, "dof_vel", i0 == ml["num_frames"][ids] - 2), (clamped, "rb_pos", cls == "t < 0")):
        monkeypatch.setattr(R, "calc_frame_blend", mut)
        bad = sample_rows(ml, ids, ts)
        monkeypatch.setattr(R, "calc_frame_blend", orig)
        fails = compare(ref, bad, SAMPLE_SPEC, "sample")[0]
        first = int(np.flatnonzero(where)[0])
        assert any(f.startswith(field) and f"sample {first}:" in f for f in fails), (mut.__name__, fails)


def test_step_comparator_rejects_mutated_oracles(monkeypatch):
    """each mutation of the task oracle is a plausible kernel bug; the step comparator names the env it shows on and the field"""
    from oracle import ref_port as R
    ml, inp, rbs, dofs, cfg, case = _cpu_scenario()
    ref = oracle_step(ml, inp, rbs, dofs, cfg)
    assert compare(ref, ref, STEP_SPEC)[0] == []
    counts = {k: int(v.sum()) for k, v in case_counts(ml, inp, ref, rbs, cfg).items()}
    for k in ("t = length", "t = length - ulp", "t = length + ulp", "progress max-1", "z = height", "fall at progress 1"):
        assert counts[k] >= 1, (k, counts)
    reset_, caller = R.compute_humanoid_reset, R.compute_reward_caller

    def gt_not_ge(reset_buf, progress, cids, pos, max_len, early, th, t, lens):        # `>` for `>=` in the reset condition
        return reset_(reset_buf, progress, cids, pos, max_len + 1, early, th, t, nxt(lens, INF))

    def le_fall(reset_buf, progress, cids, pos, max_len, early, th, t, lens):          # `<=` in the fall test
        return reset_(reset_buf, progress, cids, pos, max_len, early, nxt(th, INF), t, lens)

    def term_at_1(reset_buf, progress, cids, pos, max_len, early, th, t, lens):        # termination from progress 1
        return reset_(reset_buf, progress + 1, cids, pos, max_len + 1, early, th, t, lens)

    muts = ((gt_not_ge, "reset", case["t = length"]), (gt_not_ge, "reset", case["progress max-1"]),
            (le_fall, "term", case["z = height"]), (term_at_1, "term", case["fall at progress 1"]))
    for mut, field, env in muts:
        monkeypatch.setattr(R, "compute_humanoid_reset", mut)
        bad = oracle_step(ml, inp, rbs, dofs, cfg)
        monkeypatch.setattr(R, "compute_humanoid_reset", reset_)
        fails = compare(ref, bad, STEP_SPEC)[0]
        assert any(f.startswith(field + ":") and f"env {env}:" in f for f in fails), (mut.__name__, fails)
    monkeypatch.setattr(R, "compute_reward_caller", lambda rew, sub, reset_buf: (rew, sub))   # a sticky-reset env keeps its reward
    bad = oracle_step(ml, inp, rbs, dofs, cfg)
    monkeypatch.setattr(R, "compute_reward_caller", caller)
    assert any(f.startswith("rew:") and f"env {case['sticky reset']}:" in f for f in compare(ref, bad, STEP_SPEC)[0])
    # blend clamped to [0, 1] / f0 one frame late, seen in the targets of the step
    orig = R.calc_frame_blend
    for mut, field, env in ((lambda *a: (lambda i0, i1, b: (i0, i1, np.clip(b, 0, 1).astype(b.dtype)))(*orig(*a)), "t_rbp", case["extrapolated"]),
                            (lambda t_, l_, nf, d: (lambda i0, i1, b: (np.where(i0 == nf - 2, nf - 1, i0), i1, b))(*orig(t_, l_, nf, d)),
                             "t_dofv", case["late frame"])):
        monkeypatch.setattr(R, "calc_frame_blend", mut)
        bad = oracle_step(ml, inp, rbs, dofs, cfg)
        monkeypatch.setattr(R, "calc_frame_blend", orig)
        assert any(f.startswith(field + ":") and f"env {env}:" in f for f in compare(ref, bad, STEP_SPEC)[0]), field
    # a neighbour's row written into an env; p_* not refreshed; one target 1 ulp off where the bound is exact
    for field, env, mutate in (("obs", 9, lambda b: b["obs"].__setitem__(9, b["obs"][10])),
                               ("p_rbp", 11, lambda b: b["p_rbp"].__setitem__(11, SENT)),
                               ("t_rootv", 12, lambda b: b["t_rootv"].__setitem__((12, 1), nxt(b["t_rootv"][12, 1], INF))),
                               ("times", 13, lambda b: b["times"].__setitem__(13, nxt(b["times"][13], -INF)))):
        bad = {k: v.copy() for k, v in ref.items()}
        mutate(bad)
        fails = compare(ref, bad, STEP_SPEC)[0]
        assert any(f.startswith(field + ":") and f"env {env}:" in f for f in fails), (field, fails)


def test_time_solvers_land_on_the_threshold():
    ml = _ml()
    for L in ml["motion_lengths"]:
        for tgt in (nxt(L, -INF), L, nxt(L, INF)):
            x = time_before(tgt)
            assert np.float32(x + DT) == tgt


# ------------------------------------------------------------------------------------------------ GPU: tasks and pools
_cache = {}


def _memo(key, fn):
    if key not in _cache:
        _cache[key] = fn()
    return _cache[key]


def make_task(n, H, form="default", **over):
    from helpers import SIM_PARAMS, im_cfg
    from test_gpu_launch import _form
    from vid2player3d_b200.tasks import HumanoidSMPLIM
    _ml()
    cfg = im_cfg(n, _cpu["flat"], episode_length=MAX_LEN, contactBodies=CONTACT, terminationBodyHeight=float(H), **over)
    with _form(form):
        torch.manual_seed(0)
        t = HumanoidSMPLIM(cfg, SIM_PARAMS, 1, "cuda", 0, True)
    assert t._env.kernel_form == ("tmem" if form == "tmem" else "packed")
    return t


def task_cfg(t):
    c = t._cfg_struct
    return dict(th=np.array(list(c.termination_height)[:t.num_bodies], np.float32), contact_ids=t._contact_body_ids.cpu().numpy(),
                early=bool(c.enable_early_termination), lim=np.float32(c.pd_tar_lim), res=np.float32(c.res_force_scale))


def _upright(z, lying=False):
    from oracle import ref_port as R
    root = np.zeros(13)
    root[2] = z
    base = np.array([0.5, 0.5, 0.5, 0.5])
    root[3:7] = R.quat_mul(R.quat_from_angle_axis(np.array(np.pi / 2), np.array([1.0, 0, 0])), base) if lying else base
    return root


def launch_shape():
    return _memo("shape", lambda: make_task(1, 0.3)._env.physics_launch_shape)


def sizes():
    B, G = launch_shape()
    return [1, 7, 8, 9, 8 * 128 + 3, 2 * B * G + 5, 8195]


def pool():
    """seeded pre-step rows of P envs, kind KINDS[e % len(KINDS)]"""
    def make():
        ml = _ml()
        P = max(sizes())
        rng = np.random.default_rng(77)
        kind = np.array([KINDS.index(KINDS[e % len(KINDS)]) for e in range(P)])
        M = len(ml["num_frames"])
        mids = rng.integers(0, M, P)
        L, mdt = ml["motion_lengths"][mids], ml["motion_dt"][mids]
        times = (rng.uniform(0, 1, P) * L).astype(np.float32)
        bulk = kind == 0
        times[bulk] = rng.uniform(-2 * mdt[bulk], L[bulk] + 2 * mdt[bulk]).astype(np.float32)
        for k, f in ((1, lambda l: l), (2, lambda l: nxt(l, -INF)), (3, lambda l: nxt(l, INF))):
            for e in np.flatnonzero(kind == k):
                times[e] = time_before(f(L[e]))
        prog = rng.integers(2, MAX_LEN - 4, P)
        prog[kind == 4], prog[kind == 5] = MAX_LEN - 3, MAX_LEN - 2
        prog[kind == 7], prog[kind == 8] = 0, 1
        reset = np.isin(kind, (9, 10)).astype(np.int64)
        term = rng.integers(0, 2, P)
        term[kind == 9], term[kind == 10] = 0, 1
        ms = sample_rows(ml, mids, times)
        root = np.concatenate([ms["root_pos"], ms["root_rot"], ms["root_vel"], ms["root_ang_vel"]], 1).astype(np.float64)
        root[:, 7:13] += rng.normal(0, 0.1, (P, 6))
        q = ms["dof_pos"] + rng.normal(0, 0.05, (P, 69))
        qd = ms["dof_vel"] * 0.2 + rng.normal(0, 0.3, (P, 69))
        acts = rng.normal(0, 0.5, (P, 75))
        safe = np.isin(kind, (1, 2, 3, 4, 5))
        root[safe] = _upright(2.0)                           # high in the air: no body near its termination height
        q[safe], qd[safe] = 0, 0
        za = kind == 6
        root[za], q[za], qd[za], acts[za] = _upright(1.0), 0, 0, 0   # identical copies: the probe's pose
        low = np.isin(kind, (7, 8))
        root[low], q[low], qd[low] = _upright(0.35, lying=True), 0, 0
        st = sample_rows(ml, mids, times + DT)
        p = dict(kind=kind, mids=mids, times=times, prog=prog, reset=reset, term=term, root=root, q=q, qd=qd, acts=acts,
                 t_dof=st["dof_pos"], t_dofv=st["dof_vel"], t_rbp=st["rb_pos"], t_rbr=st["rb_rot"])
        return {k: (v.astype(np.float32) if v.dtype == np.float64 else v) for k, v in p.items()}
    return _memo("pool", make)


def heights():
    """(height with z == height for the probe pose, next float above): the post-physics z of the lowest non-contact, non-head body
    of one upright copy stepped alone"""
    def probe():
        pl = pool()
        e = int(np.flatnonzero(pl["kind"] == 6)[0])
        t = make_task(1, 0.3)
        rows = step_rows(t, pl, np.array([e]))
        z = rows["rbs"][0, :, 2]
        nc = np.ones(len(z), bool)
        nc[CONTACT_IDS()] = False
        nc[HEAD] = False
        H = np.float32(z[nc].min())
        assert z[HEAD] > 1.0 and (z[~nc & (np.arange(len(z)) != HEAD)] < H).all(), "the probe pose must have its feet lowest"
        return H, nxt(H, INF)
    return _memo("heights", probe)


def CONTACT_IDS():
    names = [str(x) for x in _model()["body_names"]]
    return np.array([names.index(c) for c in CONTACT])


def _fill(t):
    """sentinel in every task row a step writes"""
    for x in (t.obs_buf, t.rew_buf, t._sub_rewards, t._target_root_pos, t._target_root_rot, t._target_root_vel, t._target_root_ang_vel,
              t._target_key_pos, t._prev_target_dof_pos, t._prev_target_dof_vel, t._prev_target_rb_pos, t._prev_target_rb_rot,
              t.actions, t._pd_target_dof_pos, t._rigid_body_state, t._contact_force_tensor):
        x.fill_(float(SENT))


def load(t, pl, idx):
    """pool envs idx[p] into the task's rows p; returns the action rows"""
    n = len(idx)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a[idx])).to(t.device)  # noqa: E731
    _fill(t)
    t._root_states.copy_(T(pl["root"]))
    dof = t._dof_state.view(n, -1, 2)
    dof[..., 0] = T(pl["q"])
    dof[..., 1] = T(pl["qd"])
    t._rigid_body_state.view(n, -1, 13)[:, 0, 3:7] = T(pl["root"][:, 3:7])    # the residual wrench turns with rigid body 0
    t._reset_ref_motion_ids.copy_(T(pl["mids"]))
    t._reset_ref_motion_bodies.copy_(torch.from_numpy(_ml()["motion_bodies"][pl["mids"][idx]]).to(t.device))
    t._cur_ref_motion_times.copy_(T(pl["times"]))
    t.progress_buf.copy_(T(pl["prog"]))
    t.reset_buf.copy_(T(pl["reset"]))
    t._terminate_buf.copy_(T(pl["term"]))
    for name, k in (("_target_dof_pos", "t_dof"), ("_target_dof_vel", "t_dofv"), ("_target_rb_pos", "t_rbp"), ("_target_rb_rot", "t_rbr")):
        getattr(t, name).copy_(T(pl[k]))
    return T(pl["acts"])[:, :t.num_actions].contiguous()


def read(t):
    g = lambda x: x.detach().cpu().numpy().copy()  # noqa: E731
    n = t.num_envs
    return dict(acts=g(t.actions), pd=g(t._pd_target_dof_pos), p_dof=g(t._prev_target_dof_pos), p_dofv=g(t._prev_target_dof_vel),
                p_rbp=g(t._prev_target_rb_pos), p_rbr=g(t._prev_target_rb_rot), obs=g(t.obs_buf), rew=g(t.rew_buf), sub=g(t._sub_rewards),
                reset=g(t.reset_buf), term=g(t._terminate_buf), prog=g(t.progress_buf), times=g(t._cur_ref_motion_times),
                t_rootp=g(t._target_root_pos), t_rootr=g(t._target_root_rot), t_dof=g(t._target_dof_pos), t_rootv=g(t._target_root_vel),
                t_rootav=g(t._target_root_ang_vel), t_dofv=g(t._target_dof_vel), t_key=g(t._target_key_pos), t_rbp=g(t._target_rb_pos),
                t_rbr=g(t._target_rb_rot), rbs=g(t._rigid_body_state).reshape(n, -1, 13), dofs=g(t._dof_state).reshape(n, -1, 2))


def step_rows(t, pl, idx):
    a = load(t, pl, idx)
    t.step(a)
    torch.cuda.synchronize()
    return read(t)


def motion_state(t, ids, times, extra=0):
    """b200env_motion_state into sentinel-filled outputs with `extra` rows past n: returns (rows 0..n-1, the extra rows)"""
    n, nb, nd = len(ids), t._num_lib_bodies, t.num_dof
    shapes = dict(root_pos=(3,), root_rot=(4,), dof_pos=(nd,), root_vel=(3,), root_ang_vel=(3,), dof_vel=(nd,), key_pos=(4, 3),
                  rb_pos=(nb, 3), rb_rot=(nb, 4))
    out = {k: torch.full((n + extra,) + s, float(SENT), device=t.device) for k, s in shapes.items()}
    t._env.motion_state(torch.from_numpy(np.asarray(ids, np.int64)).to(t.device), torch.from_numpy(np.asarray(times, np.float32)).to(t.device), out)
    torch.cuda.synchronize()
    o = {k: v.cpu().numpy() for k, v in out.items()}
    return {k: v[:n] for k, v in o.items()}, {k: v[n:] for k, v in o.items()}


def order(n, seed):
    """pool envs of a launch of n envs: the first n in order for small n, a seeded shuffle of the pool beyond"""
    return np.arange(n) if n < 64 else np.random.default_rng(seed).permutation(len(pool()["kind"]))[:n]


def check_step(t, pl, idx, rows, label):
    """rows of one step of the task against the oracle and against b200env_motion_state; returns (worst errors, case masks)"""
    n = len(idx)
    inp = {k: v[idx] for k, v in pl.items()}
    inp["acts"] = inp["acts"][:, :t.num_actions]
    inp["rb0_rot"] = inp["root"][:, 3:7]
    cfg = task_cfg(t)
    ml = _ml()
    ref = oracle_step(ml, inp, rows["rbs"], rows["dofs"], cfg)
    worst = assert_match(rows, ref, STEP_SPEC, what=f"{label}: step against the task oracle")
    ms, _ = motion_state(t, inp["mids"], rows["times"] + DT)
    assert_match(rows, {k: ms[v] for k, v in TARGETS.items()}, {k: EXACT for k in TARGETS}, what=f"{label}: targets against b200env_motion_state")
    assert n == t.num_envs
    return worst, case_counts(ml, inp, ref, rows["rbs"], cfg)


# ------------------------------------------------------------------------------------------------ GPU tests
@pytest.mark.gpu
def test_motion_state_at_every_edge():
    """b200env_motion_state vs R.get_motion_state at every edge time of every motion, at ragged n in shuffled order; rows past n
    keep their sentinel"""
    ml = _ml()
    t = make_task(8, 0.3)
    ids, ts, cls = edge_times(ml)
    N = len(ids)
    print(f"\n{N} samples over {len(ml['num_frames'])} motions (frames {ml['num_frames'].tolist()}, dt {ml['motion_dt'].tolist()})")
    for seed, n in enumerate((1, 7, 8, 9, 8 * 40 + 3, N)):
        sel = np.random.default_rng(seed).permutation(N)[:n]
        got, past = motion_state(t, ids[sel], ts[sel], extra=5)
        assert all((v == SENT).all() for v in past.values()), f"n = {n}: a row past n was written"
        ref = sample_rows(ml, ids[sel], ts[sel])
        worst = assert_match(got, ref, SAMPLE_SPEC, "sample", names=sel, what=f"n = {n}")
        if n == N:
            print("  worst |error| per edge class:")
            for c in np.unique(cls):
                m = cls[sel] == c
                w = compare({k: v[m] for k, v in got.items()}, {k: v[m] for k, v in ref.items()}, SAMPLE_SPEC)[1]
                print(f"    {c:14s} ({m.sum():4d}): " + " ".join(f"{k} {v:.1e}" for k, v in w.items()))
        else:
            print(f"  n = {n:4d}: worst " + " ".join(f"{k} {v:.1e}" for k, v in worst.items()))


@pytest.mark.gpu
def test_reset_rows_and_context_window():
    """b200env_reset on an unsorted id list (first, last and isolated envs) at edge times: every written row against the oracle and
    the targets bit-identical to b200env_motion_state at (id, t + dt); every other row keeps its sentinel.  Then b200env_motion_context
    with windows that start before 0 and end past length + 2 dt, the mask exact, including frames at length + 2 dt exactly."""
    from oracle import ref_port as R
    ml = _ml()
    n = 8 * 16 + 3
    t = make_task(n, 0.3)
    rng = np.random.default_rng(5)
    M = len(ml["num_frames"])
    mids = rng.integers(0, M, n)
    t._reset_ref_motion_ids.copy_(torch.from_numpy(mids).to(t.device))
    t._reset_ref_motion_bodies.copy_(torch.from_numpy(ml["motion_bodies"][mids]).to(t.device))
    ids = np.concatenate([[n - 1, 0, 64, 9], rng.choice(np.setdiff1d(np.arange(12, n - 2), [64]), 40, replace=False)])
    ids = ids[rng.permutation(len(ids))]
    L, mdt = ml["motion_lengths"][mids[ids]], ml["motion_dt"][mids[ids]]
    edge = [lambda l, d: -2 * d, lambda l, d: -d, lambda l, d: nxt(0, -1), lambda l, d: np.float32(0), lambda l, d: d,
            lambda l, d: nxt(l, -INF), lambda l, d: l, lambda l, d: nxt(l, INF), lambda l, d: l + d, lambda l, d: l + 2 * d,
            lambda l, d: np.float32(0.5) * l]
    times = np.array([edge[i % len(edge)](L[i], mdt[i]) for i in range(len(ids))], np.float32)
    bufs = dict(root=t._root_states, dof=t._dof_state, rb=t._rigid_body_state, cf=t._contact_force_tensor, obs=t.obs_buf, rew=t.rew_buf,
                sub=t._sub_rewards, prog=t.progress_buf, reset=t.reset_buf, term=t._terminate_buf, times=t._cur_ref_motion_times,
                acts=t.actions, pd=t._pd_target_dof_pos, p_dof=t._prev_target_dof_pos, p_dofv=t._prev_target_dof_vel,
                p_rbp=t._prev_target_rb_pos, p_rbr=t._prev_target_rb_rot, t_rootp=t._target_root_pos, t_rootr=t._target_root_rot,
                t_dof=t._target_dof_pos, t_rootv=t._target_root_vel, t_rootav=t._target_root_ang_vel, t_dofv=t._target_dof_vel,
                t_key=t._target_key_pos, t_rbp=t._target_rb_pos, t_rbr=t._target_rb_rot)
    for k, b in bufs.items():
        b.fill_(ISENT if not b.dtype.is_floating_point else float(SENT))
    torch.cuda.synchronize()
    g = lambda b: b.detach().cpu().numpy().reshape(n, -1).copy()  # noqa: E731
    before = {k: g(b) for k, b in bufs.items()}
    t._env.reset(torch.from_numpy(ids).to(t.device), torch.from_numpy(times).to(t.device))
    torch.cuda.synchronize()
    after = {k: g(b) for k, b in bufs.items()}
    other = np.setdiff1d(np.arange(n), ids)
    assert_match({k: v[other] for k, v in after.items()}, {k: v[other] for k, v in before.items()}, {k: EXACT for k in bufs}, names=other,
                 what="rows the reset does not list must keep their sentinel")
    unwritten = ("cf", "rew", "sub", "acts", "pd", "p_dof", "p_dofv", "p_rbp", "p_rbr")
    assert_match({k: after[k][ids] for k in unwritten}, {k: before[k][ids] for k in unwritten}, {k: EXACT for k in unwritten}, names=ids,
                 what="rows of a listed env the reset does not own")
    a = {k: v[ids] for k, v in after.items()}
    s = sample_rows(ml, mids[ids], times)
    nl = len(ids)
    rb, dof = a["rb"].reshape(nl, 24, 13), a["dof"].reshape(nl, 69, 2)
    got = dict(root_pos=a["root"][:, 0:3], root_rot=a["root"][:, 3:7], root_vel=a["root"][:, 7:10], root_ang_vel=a["root"][:, 10:13],
               dof_pos=dof[..., 0], dof_vel=dof[..., 1], rb_pos=rb[..., 0:3], rb_rot=rb[..., 3:7])
    assert_match(got, s, {k: SAMPLE_SPEC[k] for k in got}, names=ids, what="reset state against R.get_motion_state(t)")
    z = np.zeros((nl, 1), np.float32)
    assert_match(dict(rbv=rb[..., 7:13], prog=a["prog"], reset=a["reset"], term=a["term"], times=a["times"],
                      obs=a["obs"]),
                 dict(rbv=np.zeros_like(rb[..., 7:13]), prog=z.astype(np.int64), reset=z.astype(np.int64), term=z.astype(np.int64),
                      times=times[:, None], obs=R.compute_humanoid_obs_raw(rb[..., 0:3], rb[..., 3:7], dof[..., 0], dof[..., 1], rb[..., 7:10],
                                                                           rb[..., 10:13], ml["motion_bodies"][mids[ids]])),
                 dict(rbv=EXACT, prog=EXACT, reset=EXACT, term=EXACT, times=EXACT, obs=EXACT), names=ids, what="reset flags and obs")
    tt = (times + DT).astype(np.float32)
    ms, _ = motion_state(t, mids[ids], tt)
    assert_match(a, {k: ms[v].reshape(nl, -1) for k, v in TARGETS.items()}, {k: EXACT for k in TARGETS}, names=ids,
                 what="reset targets against b200env_motion_state(t + dt)")
    ref = sample_rows(ml, mids[ids], tt)
    worst = assert_match({k: a[k] for k in TARGETS}, {k: ref[v].reshape(nl, -1) for k, v in TARGETS.items()},
                         {k: SAMPLE_SPEC[v] for k, v in TARGETS.items()}, names=ids, what="reset targets against R.get_motion_state(t + dt)")
    print(f"\nreset of {nl} of {n} envs: targets worst " + " ".join(f"{k} {v:.1e}" for k, v in worst.items()))

    # ---- the context window: 48 frames from t + dt - 8 dt
    P, first = 48, -8
    cm = rng.integers(0, M, 60)
    cl, cd = ml["motion_lengths"][cm], ml["motion_dt"][cm]
    ct = np.empty(60, np.float32)
    for i in range(60):
        kind = i % 4
        if kind == 0:
            ct[i] = -DT                                                      # starts 8 frames before 0
        elif kind == 1:
            ct[i] = cl[i] - np.float32(20) * DT                              # runs past length + 2 dt
        else:                                                                # a window frame lands on length + 2 dt exactly
            edge_t = np.float32(cl[i] + np.float32(2) * DT)
            # frame offset j' >= 0 with j' dt <= half the edge time: no cancellation, so every float near the edge is reachable
            step = np.float32(min(12 + 7 * (i % 3) + (kind - 2), int(0.5 * edge_t / DT))) * DT
            ct[i] = solve_time(lambda x: np.float32(np.float32(x + DT) + step), edge_t, edge_t - step - DT)
    rows = rng.permutation(n)[:60]
    feat = torch.full((n, P, 378), float(SENT), device=t.device)
    mask = torch.zeros(n, P, dtype=torch.bool, device=t.device)
    t._env.motion_context(torch.from_numpy(rows).to(t.device), torch.from_numpy(cm).to(t.device), torch.from_numpy(ct).to(t.device),
                          P, first, float(DT), feat, mask)
    torch.cuda.synchronize()
    f, mk = feat.cpu().numpy(), mask.cpu().numpy()
    rf, rmask = R.init_context(ml, cm, ct, DT, context_length=32, context_padding=8)
    others = np.setdiff1d(np.arange(n), rows)
    assert (f[others] == SENT).all() and not mk[others].any(), "the context launch wrote a row it was not given"
    f, mk = f[rows], mk[rows]
    cols = dict(body_pos=(0, 72, 1e-5), body_rot=(72, 168, 1e-5), dof_pos=(168, 237, EXPMAP), body_pos_gt=(237, 309, 1e-5),
                dof_pos_gt=(309, 378, EXPMAP))
    worst = assert_match({k: f[..., a:b].reshape(60 * P, -1) for k, (a, b, _) in cols.items()},
                         {k: rf[..., a:b].reshape(60 * P, -1) for k, (a, b, _) in cols.items()}, {k: c for k, (_, _, c) in cols.items()},
                         "window frame", what="context features against R.init_context")
    assert_match(dict(mask=mk), dict(mask=rmask), dict(mask=EXACT), names=rows, what="context mask")
    tj = np.float32(ct + DT)[:, None] + (DT * np.arange(first, first + P).astype(np.float32))[None]
    at_edge = tj.astype(np.float32) == np.float32(cl + np.float32(2) * DT)[:, None]
    print(f"context of 60 envs: worst " + " ".join(f"{k} {v:.1e}" for k, v in worst.items()) +
          f"; {int(at_edge.sum())} frames at length + 2 dt exactly (masked in), {int((~rmask).sum())} past it, "
          f"{int((tj < 0).sum())} before 0")
    assert at_edge.sum() >= 30 and mk[at_edge].all() and (~rmask).any() and (tj < 0).any()


@pytest.mark.gpu
def test_step_task_logic_at_every_threshold():
    """one step at every size of sizes() with the per-env cases of KINDS, against ImTaskOracle resynchronised from the GPU's post-physics
    state (exact: actions_used, PD targets, previous targets, progress, flags, ref times, the raw obs; targets exact against
    b200env_motion_state and within 1e-5 of the oracle; reward and sub-rewards 1e-5).  Termination height H: the probe pose's z (no
    fall) and the next float above (fall)."""
    H_eq, H_below = heights()
    pl = pool()
    B, G = launch_shape()
    total = {}
    print(f"\nB = {B}, G = {G}; termination height {H_eq!r} (the probe pose's lowest non-contact body) and {H_below!r}")
    for n in sizes():
        idx = order(n, n)
        for var, H in (("z = height", H_eq), ("z one ulp below", H_below)):
            t = make_task(n, H)
            rows = step_rows(t, pl, idx)
            worst, cases = check_step(t, pl, idx, rows, f"N = {n}, {var}")
            if var == "z = height":
                _cache[("rows", n)] = rows
            for k, m in cases.items():
                total[k] = total.get(k, 0) + int(m.sum())
            print(f"  N = {n:5d} ({var:16s}): worst rew {worst['rew']:.1e} sub {worst['sub']:.1e} t_rbp {worst['t_rbp']:.1e} "
                  f"t_rbr {worst['t_rbr']:.1e} t_dof {worst['t_dof']:.1e}; resets {int(rows['reset'].sum())}, terminated "
                  f"{int(rows['term'].sum())}")
            del t
    print("  envs that reached each case: " + ", ".join(f"{k} {v}" for k, v in total.items()))
    missing = [k for k, v in total.items() if v == 0]
    assert not missing, f"cases never reached: {missing}"


@pytest.mark.gpu
def test_step_without_early_termination_or_residual_wrench():
    """the same cases with enableEarlyTermination off (no env terminates, z cases reset only by time / progress) and with
    residual_force_scale 0 (69-wide action rows)"""
    H_eq, _ = heights()
    pl = pool()
    n = 8 * 128 + 3
    idx = order(n, 3)
    for over in (dict(enableEarlyTermination=False), dict(residual_force_scale=0.0)):
        t = make_task(n, H_eq, **over)
        rows = step_rows(t, pl, idx)
        worst, cases = check_step(t, pl, idx, rows, str(over))
        if "enableEarlyTermination" in over:
            assert not rows["term"][pl["reset"][idx] == 0].any()
        else:
            assert rows["acts"].shape[1] == 69
        print(f"\n{over}: worst rew {worst['rew']:.1e}; resets {int(rows['reset'].sum())}, terminated {int(rows['term'].sum())}")


PHYSICS_FREE = ("acts", "pd", "p_dof", "p_dofv", "p_rbp", "p_rbr", "prog", "times") + tuple(TARGETS)


@pytest.mark.gpu
@pytest.mark.parametrize("form", ["sort", "fused", "tmem"])
def test_task_outputs_identical_across_kernel_forms(form):
    """the form's task rows at every size against the default form's.  B200ENV_SORT=1 runs the same physics in another hand-out order:
    every row, state rows included, bit-identical.  The fused and tmem forms' physics rows differ from the default form's in the last
    bits (test_gpu_launch.py compares each with itself), so there the rows the physics does not feed (actions_used, PD and previous
    targets, progress, ref times, targets) are bit-identical, and obs, reward and flags are bit-identical on every env whose post-physics
    rows are, and held to the oracle from the form's own post-physics rows on the others.  The fused form runs the epilogue inside its
    physics launch, so its ragged tail is its own code path."""
    H_eq, _ = heights()
    pl = pool()
    for n in sizes():
        idx = order(n, n)
        ref = _cache.get(("rows", n))
        if ref is None:
            ref = step_rows(make_task(n, H_eq), pl, idx)
            _cache[("rows", n)] = ref
        t = make_task(n, H_eq, form)
        rows = step_rows(t, pl, idx)
        what = f"{form} form against the default form at N = {n}"
        if form == "sort":
            assert_match(rows, ref, {k: EXACT for k in ref}, what=what)
            continue
        assert_match(rows, ref, {k: EXACT for k in PHYSICS_FREE}, what=what)
        same = np.flatnonzero([np.array_equal(rows["rbs"][e], ref["rbs"][e]) and np.array_equal(rows["dofs"][e], ref["dofs"][e])
                               for e in range(n)])
        assert_match({k: rows[k][same] for k in ref}, {k: ref[k][same] for k in ref}, {k: EXACT for k in ref}, names=same,
                     what=what + " (envs with bit-identical physics rows)")
        check_step(t, pl, idx, rows, f"{form} form at N = {n}")
        print(f"\n{form}, N = {n}: {len(same)} of {n} envs with bit-identical physics rows")


@pytest.mark.gpu
@pytest.mark.parametrize("per_slice", [13, 8 * 4 + 3])
def test_pre_kernel_writes_only_its_env_slice(per_slice):
    """two handles over the even / odd rows (federer, task_mode 1, PD target = clamp(target dof + action, q -+ lim)): stepping one
    handle writes actions_used and the PD targets of its rows, bit for bit, and leaves every bit of the other slice's"""
    from test_gpu_launch import _load, _make_pool, _task
    n = 2 * per_slice
    t = _task("ball", n, "default", handles=2)
    assert len(t._envs) == 2
    pl = _make_pool("ball", n)
    a = _load(t, "ball", pl, np.arange(n))
    t.actions.fill_(float(SENT))
    t._pd_target_dof_pos.fill_(float(SENT))
    torch.cuda.synchronize()
    lim = np.float32(t._cfg_struct.pd_tar_lim)
    for k, h in enumerate(t._envs):
        mine, other = np.arange(k, n, 2), np.arange(1 - k, n, 2)
        before = dict(acts=t.actions.cpu().numpy().copy(), pd=t._pd_target_dof_pos.cpu().numpy().copy())
        q = t._dof_state.view(n, -1, 2)[..., 0].cpu().numpy()[mine]
        tdof = t._target_dof_pos.cpu().numpy()[mine]
        h.step(a)
        torch.cuda.synchronize()
        after = dict(acts=t.actions.cpu().numpy(), pd=t._pd_target_dof_pos.cpu().numpy())
        assert_match({x: v[other] for x, v in after.items()}, {x: v[other] for x, v in before.items()}, dict(acts=EXACT, pd=EXACT),
                     names=other, what=f"slice {k}'s step wrote a row of the other slice")
        an = a.cpu().numpy()[mine]
        pd = np.maximum(np.minimum(tdof + an[:, :69], q + lim), q - lim)
        assert_match({x: v[mine] for x, v in after.items()}, dict(acts=an, pd=pd), dict(acts=EXACT, pd=EXACT), names=mine,
                     what=f"slice {k}'s own rows")
    print(f"\nenv slices of {per_slice} envs: each pre_kernel wrote exactly its own rows")
