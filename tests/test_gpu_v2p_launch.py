"""The vid2player task launches (include/b200env_v2p.h) against the numpy oracle (oracle/ref_port_v2p.py, whose pieces are pinned to
the reference by test_oracle_golden_v2p.py), at ragged sizes and on every threshold, with every row the launch must not write checked.

1. Sizes 1 ... 8195 (ragged last block of the warp-per-env kernels and of the 128 / 256-thread ones).  Outputs start as a sentinel and
   have slack rows past n; rows past n and rows whose mask is clear must stay bit-identical.
2. controller_post: a per-env case table where each case lands exactly on a threshold or one float32 ulp to either side of it:
   in_court for the true and the estimated bounce, the out-of-court box, "behind", progress at max_len - 2 / max_len - 1 (with and
   without the advance increment), tar_time reaching tar_time_total, the flag combinations of tar_action / contact / bounce, one NaN in
   each observation block, the estimator's validity tests (x_net = +-4 included), its half-even cell edges and clamps, and the net test
   tx + z = 1.07.  Flags, counters, observations (except the rot6d block), the trajectory / history windows and the estimator outputs
   are exact; rewards, distance and rot6d have stated bounds.
3. The estimator cases run on a coarse table and on the reference's 0.1 / 0.1 / 0.2 grid with a table whose rows encode their index.
4. task_reset, ctrl_reset, pre_step and stream_gather against their restatements.
5. CPU negative controls: each comparator rejects a mutated oracle and names the env and the field.

Quirks of the reference kept by the oracle and so required of the kernels: the rot6d observation feeds the xyzw body quaternion to the
wxyz converter; the reset FSM terminates on a NaN anywhere in the observation row; the estimator only writes the rows with a valid
contact and leaves the z of est_bounce_pos alone; recovery envs roll their ball history in an observation refresh only outside dual mode.

Bounds that are not exact, and why: the kernels contract products into fma in the reward (squared distances), in distance (|v_xy|) and
in the quaternion -> matrix conversion of the rot6d observation; each is held to a few float32 ulps of its value.  The welded racket row of
actor_reset has no reference formula (the reference reads it from the simulator) and is held to 4e-7."""
import ctypes as C

import numpy as np
import pytest

from oracle import ref_port_v2p as V

f32 = np.float32
SENT = f32(12345.0)      # float rows start as it, integer rows as ISENT, bool rows as True (the flags the kernels clear)
ISENT = 7777
INF = f32(np.inf)
SIZES = (1, 2, 3, 4, 5, 7, 9, 127, 129, 257, 4097, 8191, 8195)
SLACK = 3
MAX_LEN = 300
COURT_MIN, COURT_MAX = (f32(-5), f32(-16)), (f32(5), f32(-10))
COARSE = np.array([[10, 65, 1], [-5, 10, 1], [-10, 10, 2], [0, 30, 0.5], [0, 3, 0.1]], np.float64)
FINE = np.array([[10, 15, 0.1], [-5, 10, 0.1], [-10, 10, 0.2], [0, 30, 0.5], [0, 3, 0.1]], np.float64)   # truncated VX: ~360 MB
NX, NY = 60, 30
SCALES = {"pos": 50.0, "phase": 10.0, "bounce_pos": 1.0, "bounce_time": 0.5}
WEIGHTS = {"pos": 0.5, "ball_pos": 0.5}

INT_FIELDS = ("swing_type", "swing_type_cycle", "tar_action", "tar_time", "tar_time_total", "progress", "reset", "terminate")
BOOL_FIELDS = ("has_contact", "has_contact_now", "has_bounce", "has_bounce_now", "bounce_in", "est_bounce_in", "reset_reaction",
               "reset_recovery")
GPU_NAME = dict(rbs="rigid_body_state", obs="obs_buf", rew="rew_buf", sub="sub_rewards", reset="reset_buf", terminate="terminate_buf",
                progress="progress_buf")
ROT6D = slice(78, 222)
# comparison spec: "exact", or an absolute bound scaled by max(1, |value|)
POST_SPEC = dict(obs="obs", rew=2e-6, sub=2e-6, distance=2e-6, **{k: "exact" for k in INT_FIELDS + BOOL_FIELDS},
                 est_bounce_pos="exact", est_bounce_time="exact", est_max_height="exact", ball_traj="exact", ball_obs="exact")


def nxt(x, d, k=1):
    x = f32(x)
    for _ in range(k):
        x = np.nextafter(x, f32(d)).astype(f32)
    return x


# ------------------------------------------------------------------------------------------------ comparator (CPU)
def compare(ref, got, spec, rows=None, limit=8):
    """-> list of "field: env i: ..." failures (the first `limit` differing envs per field), over `rows` (default all)"""
    fails = []
    for k, how in spec.items():
        if k not in ref or ref[k] is None:
            continue
        a, b = np.asarray(ref[k]), np.asarray(got[k])
        if rows is not None:
            a, b = a[rows], b[rows]
        a2, b2 = a.reshape(len(a), -1), b.reshape(len(b), -1)
        if how == "obs":
            bad = ~((a2 == b2) | (np.isnan(a2) & np.isnan(b2)))
            bad[:, ROT6D] = ~((np.abs(a2[:, ROT6D] - b2[:, ROT6D]) <= 1e-6) | (np.isnan(a2[:, ROT6D]) & np.isnan(b2[:, ROT6D])))
        elif how == "exact":
            bad = ~((a2 == b2) | (np.isnan(a2) & np.isnan(b2))) if a2.dtype.kind == "f" else a2 != b2
        else:
            bad = ~((np.abs(a2.astype(np.float64) - b2) <= how * np.maximum(1, np.abs(a2.astype(np.float64)))) | (np.isnan(a2) & np.isnan(b2)))
        for r in np.flatnonzero(bad.any(1))[:limit]:
            c = int(np.flatnonzero(bad[r])[0])
            env = int(rows[r]) if rows is not None else int(r)
            fails.append(f"{k}: env {env}: column {c} got {b2[r, c]!r} ref {a2[r, c]!r} ({int(bad.any(1).sum())} envs differ)")
    return fails


# ------------------------------------------------------------------------------------------------ tables and states (CPU)
def coarse_tables(seed=3):
    """random out-estimator tables on the COARSE grid; the distance at the last height index is 0 (then the estimated bounce is the
    contact point itself, which puts the est_bounce_in cases exactly on the court lines)"""
    rows = 55 * 15 * 10
    rng = np.random.default_rng(seed)
    tx = rng.uniform(0, 1, (rows, NX)).astype(f32)
    ty = np.stack([rng.uniform(5, 25, (rows, NY)), rng.uniform(0.3, 1.5, (rows, NY))], -1).astype(f32)
    ty[:, NY - 1, 0] = 0
    return tx, ty


class IndexTable:
    """the FINE-grid tables as a function of the row: tx[r] = (r, 0, ...), ty[r, h] = (h + 1, r); est_max_height = z + r and
    est_bounce_time = r name the row, the bounce distance names the height index"""
    rows = 50 * 150 * 100

    def __init__(self, which):
        self.which = which

    def __getitem__(self, r):
        r = np.asarray(r)
        if self.which == "x":
            out = np.zeros(r.shape + (NX,), f32)
            out[..., 0] = r
            return out
        out = np.zeros(r.shape + (NY, 2), f32)
        out[..., 0] = np.arange(1, NY + 1, dtype=f32)
        out[..., 1] = r[..., None]
        return out


def base_state(n, rng, L=10, history=False):
    """a plausible controller state: the player on its court box, the ball incoming, nobody on a threshold"""
    u = lambda lo, hi, *s: rng.uniform(lo, hi, s).astype(f32)  # noqa: E731
    q = rng.normal(size=(n, 26, 4))
    q /= np.linalg.norm(q, axis=-1, keepdims=True)
    rbs = np.concatenate([u(-1, 1, n, 26, 3), q.astype(f32), u(-2, 2, n, 26, 6)], -1).astype(f32)
    root = np.stack([u(-3, 3, n), u(-14.5, -11.5, n), u(0.8, 1.0, n)], -1)
    rbs[:, 0, 0:3] = root
    bs = np.concatenate([u(-2, 2, n, 1), u(-11, -8, n, 1), u(0.5, 2.5, n, 1), u(-1, 1, n, 4), u(-3, 3, n, 1), u(12, 40, n, 1),
                         u(-4, 9, n, 1), u(-40, 40, n, 3)], 1)
    s = dict(rbs=rbs, ball_states=bs, root_pos=root, root_vel=u(-3, 3, n, 3), racket_pos=rbs[:, 24, 0:3].copy(),
             racket_normal=u(-1, 1, n, 3), ball_pos=np.stack([u(-3, 3, n), u(-9, 11, n), u(0.1, 3, n)], -1),
             bounce_pos=u(-5, 5, n, 3), ball_traj=u(-10, 10, n, 100, 3), target_bounce_pos=u(-3, 3, n, 3), phase=u(0, 6, n),
             est_bounce_pos=u(-5, 5, n, 3), est_bounce_time=u(0, 1, n), est_max_height=u(0, 3, n), distance=u(0, 50, n),
             obs=np.full((n, 225 + 3 * L + 2), SENT, f32), rew=np.full(n, SENT, f32), sub=np.full((n, 2), SENT, f32),
             ball_obs=u(-10, 10, n, L, 3) if history or L else None)
    s.update(swing_type=rng.integers(-1, 4, n), swing_type_cycle=rng.integers(-1, 4, n), tar_action=rng.integers(0, 2, n),
             tar_time_total=rng.integers(65, 75, n), progress=rng.integers(0, MAX_LEN - 4, n), reset=np.full(n, ISENT, np.int64),
             terminate=np.full(n, ISENT, np.int64))
    s["tar_time"] = s["tar_time_total"] - rng.integers(3, 60, n)
    for k in BOOL_FIELDS:
        s[k] = rng.random(n) < 0.3
    s["has_contact_now"] &= s["has_contact"]
    return s


def ball_case(s, i, b0=0.0, b1=-10.0, b2=2.0, b7=0.0, b8=20.0, b9=2.0, w=(0.0, 0.0, 0.0)):
    s["ball_states"][i, [0, 1, 2, 7, 8, 9, 10, 11, 12]] = np.array([b0, b1, b2, b7, b8, b9, *w], f32)
    s["has_contact_now"][i] = s["has_contact"][i] = True


def fma_cases(rng, kind, count, grid):
    """ball states where an fma-contracted x_net / vel_x / vspin differs from the separately rounded one in its outcome: validity at
    x_net = +-4, or the table row at a cell edge (fma emulated in float64: exact products, one rounding of the sum)"""
    out = []
    VX, VS = grid[0], grid[2]
    while len(out) < count:
        if kind == "x_net":
            b8, b1, b7 = f32(rng.uniform(12, 30)), f32(rng.uniform(-14, -8)), f32(rng.uniform(-8, 8))
            qq = np.abs(b1 / b8)
            tgt = f32(4) if rng.random() < 0.5 else f32(-4)
            b0 = f32(tgt - b7 * qq)
            for k in range(-3, 4):
                c = nxt(b0, INF if k > 0 else -INF, abs(k))
                sep, fm = f32(c + f32(b7 * qq)), f32(np.float64(b7) * np.float64(qq) + np.float64(c))
                if (abs(sep) < 4) != (abs(fm) < 4):
                    out.append(dict(b0=c, b1=b1, b7=b7, b8=b8))
                    break
        elif kind == "vel_x":
            k = rng.integers(1, int((VX[1] - VX[0]) / VX[2]) - 1)
            edge = f32(VX[0] + (k + 0.5) * VX[2])
            b7 = f32(rng.uniform(0.5, 3))
            b8 = f32(np.sqrt(np.float64(edge) ** 2 - np.float64(b7) ** 2))
            for j in range(-40, 41):
                c = nxt(b8, INF if j > 0 else -INF, abs(j))
                sq7, sq8 = f32(b7 * b7), f32(c * c)
                sep = np.sqrt(f32(sq7 + sq8))
                fms = [np.sqrt(f32(np.float64(c) * np.float64(c) + np.float64(sq7))), np.sqrt(f32(np.float64(b7) * np.float64(b7) + np.float64(sq8)))]
                ix = lambda v: np.rint((np.clip(v, f32(VX[0]), f32(VX[1] - VX[2])) - f32(VX[0])) / f32(VX[2]))  # noqa: E731
                if any(ix(fm) != ix(sep) for fm in fms):
                    out.append(dict(b7=b7, b8=c))
                    break
        else:   # vspin: |w| / 2pi at a cell edge
            k = rng.integers(1, int((VS[1] - VS[0]) / VS[2]) - 1)
            edge = (VS[0] + (k + 0.5) * VS[2]) * 2 * np.pi
            w0, w1 = f32(rng.uniform(1, 10)), f32(rng.uniform(1, 10))
            w2 = f32(np.sqrt(max(edge ** 2 - float(w0) ** 2 - float(w1) ** 2, 1.0)))
            for j in range(-60, 61):
                c = nxt(w2, INF if j > 0 else -INF, abs(j))
                a, b, d = f32(w0 * w0), f32(w1 * w1), f32(c * c)
                sep = np.sqrt(f32(f32(a + b) + d)) / f32(2 * np.pi)
                fm = np.sqrt(f32(np.float64(c) * np.float64(c) + np.float64(f32(np.float64(w1) * np.float64(w1) + np.float64(a))))) / f32(2 * np.pi)
                ix = lambda v: np.rint((np.clip(v, f32(VS[0]), f32(VS[1] - VS[2])) - f32(VS[0])) / f32(VS[2]))  # noqa: E731
                if ix(fm) != ix(sep):
                    out.append(dict(w=(w0, w1, c)))
                    break
    return out


def case_table(rng, grid, est_x):
    """[(kind, fn(s, i))]: each fn puts env i exactly on (or one ulp beside) a threshold"""
    cases = []

    def add(kind, fn):
        cases.append((kind, fn))
    for x in (f32(-4.11), f32(4.11)):
        for d in (0, -INF, INF):
            xv = nxt(x, d) if d else x
            add(f"bounce_in x {xv!r}", lambda s, i, xv=xv: (s["bounce_pos"].__setitem__((i, slice(0, 2)), (xv, 5)),
                                                             s["tar_action"].__setitem__(i, 0), s["has_bounce_now"].__setitem__(i, True)))
    for y in (f32(0), f32(11.89)):
        for d in (0, -INF, INF):
            yv = nxt(y, d) if d else y
            add(f"bounce_in y {yv!r}", lambda s, i, yv=yv: (s["bounce_pos"].__setitem__((i, slice(0, 2)), (0, yv)),
                                                             s["tar_action"].__setitem__(i, 0), s["has_bounce_now"].__setitem__(i, True)))
    for ax, val in ((0, COURT_MIN[0]), (1, COURT_MIN[1]), (0, COURT_MAX[0]), (1, COURT_MAX[1])):
        for d in (0, -INF, INF):
            v = nxt(val, d) if d else val
            add(f"court axis {ax} {v!r}", lambda s, i, ax=ax, v=v: s["root_pos"].__setitem__((i, ax), v))
    for k in (0, -INF, INF):
        def behind(s, i, k=k):
            by = f32(s["root_pos"][i, 1] - f32(1))
            s["ball_pos"][i, 1] = nxt(by, k) if k else by
            s["tar_action"][i] = 1
        add(f"behind {k}", behind)
    def quiet(s, i):    # no other reason to reset: the counters alone decide
        s["tar_action"][i] = 0
        for k in ("has_contact", "has_contact_now", "has_bounce", "has_bounce_now"):
            s[k][i] = False
    for p in (MAX_LEN - 3, MAX_LEN - 2, MAX_LEN - 1):
        add(f"progress {p}", lambda s, i, p=p: (quiet(s, i), s["progress"].__setitem__(i, p)))
    for dt in (-2, -1, 0, 1):
        add(f"tar_time total{dt:+d}", lambda s, i, dt=dt: (quiet(s, i), s["tar_time"].__setitem__(i, s["tar_time_total"][i] + dt)))
    for bits in range(32):
        def flags(s, i, bits=bits):
            s["tar_action"][i] = bits & 1
            s["has_contact"][i], s["has_contact_now"][i] = bool(bits & 2), bool(bits & 2) and bool(bits & 4)
            s["has_bounce"][i], s["has_bounce_now"][i] = bool(bits & 8), bool(bits & 16)
        add(f"flags {bits}", flags)
    nan_at = (("root_pos", (0,)), ("root_vel", (1,)), ("rbs", (5, 1)), ("rbs", (3, 4)), ("racket_normal", (2,)), ("ball_traj", (2, 1)),
              ("ball_obs", (4, 2)), ("target_bounce_pos", (0,)), ("rbs", (24, 0)))
    for k, idx in nan_at:
        add(f"nan {k}{idx}", lambda s, i, k=k, idx=idx: s[k].__setitem__((i,) + idx, np.nan))
    VX, VY, TY = grid[0], grid[1], grid[4]
    for kind, kw in (("b8 = VX lo", dict(b8=f32(VX[0]))), ("b8 = VX lo + ulp", dict(b8=nxt(VX[0], INF))),
                     ("b9 = VY lo", dict(b9=f32(VY[0]))), ("b9 = VY lo + ulp", dict(b9=nxt(VY[0], INF))),
                     ("b9 = VY hi", dict(b9=f32(VY[1]))), ("b9 = VY hi - ulp", dict(b9=nxt(VY[1], -INF))),
                     ("b2 = TY hi", dict(b2=f32(TY[1]))), ("b2 = TY hi - ulp", dict(b2=nxt(TY[1], -INF)))):
        add("valid " + kind, lambda s, i, kw=kw: ball_case(s, i, **kw))
    for kw in fma_cases(rng, "x_net", 6, grid) + fma_cases(rng, "vel_x", 6, grid) + fma_cases(rng, "vspin", 6, grid):
        add(f"fma {sorted(kw)}", lambda s, i, kw=kw: ball_case(s, i, **kw))
    for k in range(int((VX[1] - VX[0]) / VX[2]) + 2):   # vel_x = |b8| at every half cell and past both clamps
        add(f"vel_x half {k}", lambda s, i, k=k: ball_case(s, i, b8=f32(VX[0] + (k - 0.5) * VX[2]) if k else nxt(VX[0], INF)))
    for b9 in list(np.arange(VY[0] + VY[2] / 2, VY[1], VY[2] * 7)) + [VY[1] - VY[2] / 2, nxt(VY[1], -INF)]:
        add(f"vy {b9}", lambda s, i, b9=f32(b9): ball_case(s, i, b9=b9))
    for wz in (0.0, 1e3, 3.0):
        add(f"vspin w {wz}", lambda s, i, wz=wz: ball_case(s, i, w=(0, 0, wz)))
    for b2 in (0.0, 0.05, 0.15, 1.45, 2.85, 2.9, 2.95, float(nxt(3.0, -INF))):
        add(f"height {b2}", lambda s, i, b2=f32(b2): ball_case(s, i, b2=b2))
    for b1 in (0.0, -1e-30, -5.0, -14.75, -40.0, -300.0):
        add(f"net dist b1 {b1}", lambda s, i, b1=f32(b1): ball_case(s, i, b1=b1, b8=f32(20), b7=f32(0.0)))
    for d in (0, -INF, INF):     # tx + z = 1.07: z solved for the row / net index the case selects
        def net(s, i, d=d):
            ball_case(s, i, b1=f32(-10), b2=f32(0.5), b7=f32(0.0), b8=f32(20), b9=f32(2))
            b = s["ball_states"][i:i + 1, :13]
            ti, ni = est_row(b, grid)
            tx = est_x[ti][0, ni[0]]
            z = f32(f32(1.07) - tx)
            for _ in range(64):
                y = f32(tx + z)
                if y == f32(1.07):
                    break
                z = nxt(z, INF if y < f32(1.07) else -INF)
            s["ball_states"][i, 2] = nxt(z, d) if d else z
        add(f"net height {d}", net)
    for x in (f32(-4.11), f32(4.11)):   # est_bounce_in on the court lines: zero distance at the last height index -> bounce = contact
        for d in (0, -INF, INF):
            xv = nxt(x, d) if d else x
            add(f"est_bounce_in x {xv!r}", lambda s, i, xv=xv: ball_case(s, i, b0=xv, b1=f32(5), b2=f32(2.95),
                                                                         b7=f32(-2 if xv > 0 else 2), b8=f32(20)))
    for y in (f32(0), f32(11.89)):
        for d in (0, -INF, INF):
            yv = nxt(y, d) if d else y
            add(f"est_bounce_in y {yv!r}", lambda s, i, yv=yv: ball_case(s, i, b1=yv, b2=f32(2.95)))
    return cases


def est_row(b, grid):
    """(table row, net index) the estimator reads for ball rows b (the oracle's float32 index math)"""
    VX, VY, VS, TX = [tuple(float(v) for v in r) for r in grid[:4]]
    idx = lambda v, r: V.est_round((np.clip(v, f32(r[0]), f32(r[1] - r[2])) - f32(r[0])) / f32(r[2]))  # noqa: E731
    vel = np.linalg.norm(b[:, 7:9], axis=-1)
    vs = np.linalg.norm(b[:, 10:13], axis=1) / f32(2 * np.pi)
    d1, d2 = f32((VY[1] - VY[0]) / VY[2]), f32((VS[1] - VS[0]) / VS[2])
    ti = (idx(vel, VX) * d1 * d2 + idx(b[:, 9], VY) * d2 + idx(vs, VS)).astype(np.int64)
    return ti, idx(-b[:, 1] / b[:, 8] * vel, TX).astype(np.int64)


def apply_cases(s, cases, rng):
    """case k on env perm[k] (all of them if n allows); -> {env: kind}"""
    n = len(s["root_pos"])
    perm = rng.permutation(n)
    where = {}
    for k, (kind, fn) in enumerate(cases[:n]):
        fn(s, perm[k])
        where[int(perm[k])] = kind
    return where


def post_cfg(L=10, use_target=1, rtype="return_w_estimate", et=1, est=None, grid=COARSE, **flags):
    return dict(obs_traj_len=L, use_target=use_target, reward_type=rtype, early_termination=et, max_len=MAX_LEN, court_min=COURT_MIN,
                court_max=COURT_MAX, scales=SCALES, weights=WEIGHTS, est=None if est is None else (est[0], est[1], grid), **flags)


# ------------------------------------------------------------------------------------------------ GPU runners
def _dev(a, dtype=None):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to("cuda:0")


def _pad(a, fill):
    pad = np.full((SLACK,) + a.shape[1:], fill, a.dtype)
    return np.concatenate([a, pad])


def run_post(s, cfg, est_dev=None, touch_mask=None):
    """one b200v2p_controller_post launch over a copy of s with SLACK sentinel rows; -> (state after, slack rows untouched?)"""
    import torch
    from vid2player3d_b200 import native_v2p as NV
    n = len(s["root_pos"])
    L = cfg["obs_traj_len"]
    width = 225 + 3 * L + (2 if cfg["use_target"] else 0)
    t = {}
    for k, v in s.items():
        if v is None or k == "touch_mask":
            continue
        if k == "obs":
            v = v[:, :width]
        fill = {"b": True, "i": ISENT}.get(v.dtype.kind, SENT)
        t[GPU_NAME.get(k, k)] = _dev(_pad(v, fill))
    if touch_mask is not None:
        t["touch_mask"] = _dev(_pad(touch_mask, True))
    t["est_x"], t["est_y"] = est_dev if est_dev is not None else (None, None)
    if not cfg.get("use_history") and s.get("ball_obs") is None:
        t["ball_obs"] = None
    grid = cfg["est"][2] if cfg.get("est") else np.zeros((5, 3))
    c = dict(n=n, bodies_per_env=26, ball_stride=13, racket_body=24, num_obs=width, obs_traj_len=L, use_target=cfg["use_target"],
             reward_type=NV.REWARD_TYPES[cfg["reward_type"]], early_termination=cfg["early_termination"], max_episode_length=MAX_LEN,
             est_nx=NX if est_dev is not None else 0, est_ny=NY if est_dev is not None else 0, scale_pos=SCALES["pos"],
             scale_phase=SCALES["phase"], scale_bounce_pos=SCALES["bounce_pos"], scale_bounce_time=SCALES["bounce_time"],
             w_pos=WEIGHTS["pos"], w_ball_pos=WEIGHTS["ball_pos"], court_min=COURT_MIN, court_max=COURT_MAX,
             est_params=np.asarray(grid, np.float32).reshape(-1), obs_only=cfg.get("obs_only", 0), dual=cfg.get("dual", 0),
             use_history=cfg.get("use_history", 0), advance=cfg.get("advance", 0))
    NV.controller_post(c, t)
    torch.cuda.synchronize()
    out, clean = {}, True
    for k, v in s.items():
        if v is None or k == "touch_mask":
            out[k] = v
            continue
        g = t[GPU_NAME.get(k, k)].cpu().numpy()
        fill = {"b": True, "i": ISENT}.get(g.dtype.kind, SENT)
        clean &= bool((g[n:] == fill).all())
        out[k] = g[:n]
    out["obs"] = np.concatenate([out["obs"], s["obs"][:, width:]], 1) if width < s["obs"].shape[1] else out["obs"]
    return out, clean


def check_post(s, cfg, est_np=None, est_dev=None, touch_mask=None, label=""):
    if touch_mask is not None:
        s = dict(s, touch_mask=touch_mask)
    L = cfg["obs_traj_len"]
    width = 225 + 3 * L + (2 if cfg["use_target"] else 0)
    s = dict(s, obs=s["obs"][:, :width].copy())
    got, clean = run_post(s, cfg, est_dev, touch_mask)
    assert clean, f"{label}: a row past n was written"
    ref = V.controller_post(s, cfg)
    fails = compare(ref, got, POST_SPEC)
    assert not fails, f"{label}: " + "; ".join(fails[:6])
    return ref, got


# ------------------------------------------------------------------------------------------------ CPU: validation and controls
def test_controller_post_rejects_odd_dual_and_wrong_obs_width():
    """b200v2p_controller_post checks its descriptor before any launch, so fake (never dereferenced) pointers reach every rule on a
    machine without a GPU: dual mode with an odd n, and an observation row wider or narrower than the columns the launch writes"""
    from vid2player3d_b200 import abi
    from vid2player3d_b200 import native_v2p as NV
    from vid2player3d_b200.native import lib
    L = lib()
    L.b200v2p_last_error.restype = C.c_char_p

    def run(**kw):
        c = abi.V2PCtrl()
        base = dict(n=8, bodies_per_env=26, ball_stride=13, racket_body=24, num_obs=257, obs_traj_len=10, use_target=1, reward_type=2,
                    max_episode_length=300)
        base.update(kw)
        for k, v in base.items():
            setattr(c, k, v)
        return L.b200v2p_controller_post(C.byref(c), None), L.b200v2p_last_error().decode()
    for kw, msg in ((dict(dual=1, n=7), "even number of envs"), (dict(dual=1, n=1), "even number of envs"),
                    (dict(num_obs=258), "observation width"), (dict(num_obs=256), "observation width"),
                    (dict(use_target=0), "observation width"), (dict(obs_traj_len=101, num_obs=530), "observation width")):
        rc, err = run(**kw)
        assert rc == -2 and msg in err, (kw, rc, err)
    assert NV.REWARD_TYPES["return_w_estimate"] == 2


def _cpu_scenario(n=300, seed=0):
    rng = np.random.default_rng(seed)
    tx, ty = coarse_tables()
    s = base_state(n, rng)
    cases = case_table(rng, COARSE, tx)
    where = apply_cases(s, cases, rng)
    return s, (tx, ty), where


def test_post_comparator_rejects_mutated_oracles(monkeypatch):
    """each mutation of the oracle is a plausible kernel bug; the comparator names the env it shows on and the field"""
    s, est, where = _cpu_scenario()
    env_of = {v: k for k, v in where.items()}
    cfg = post_cfg(est=est, advance=1)
    ref = V.controller_post(s, cfg)

    def rejects(field, env, **patch):
        orig = {k: getattr(V, k) for k in patch}
        for k, fn in patch.items():
            monkeypatch.setattr(V, k, fn)
        bad = V.controller_post(s, cfg)
        for k, fn in orig.items():
            monkeypatch.setattr(V, k, fn)
        fails = compare(ref, bad, POST_SPEC, limit=None)
        assert any(x.startswith(field + ":") and f"env {env}:" in x for x in fails), (field, env, fails[:8])

    in_court = lambda p: (p[:, 0] >= f32(-4.11)) & (p[:, 0] < f32(4.11)) & (p[:, 1] > 0) & (p[:, 1] < f32(11.89))  # noqa: E731
    rejects("bounce_in", env_of[f"bounce_in x {f32(-4.11)!r}"], in_court=in_court)
    rejects("est_bounce_in", env_of[f"est_bounce_in x {f32(-4.11)!r}"], in_court=in_court)
    x_net_env = min(e for e, k in where.items() if k.startswith("fma ['b0'"))
    rejects("est_max_height", x_net_env, net_crossing_x=lambda b: b[:, 0] + b[:, 7] * (b[:, 1] / b[:, 8]))   # x_net without abs
    half_away = lambda v: np.sign(v) * np.floor(np.abs(v) + f32(0.5))  # noqa: E731
    rejects("est_max_height", env_of["vel_x half 1"], est_round=half_away)
    adv = V.advance_counters

    def late(s_):       # the reaction test done before the increment: tar_time counts after the reset FSM
        adv(s_)
        s_["tar_time"] = s_["tar_time"] - 1
    rejects("reset_reaction", env_of["tar_time total-1"], advance_counters=late)
    reset = V.controller_reset

    def keeps_recovery(*a, **k):
        r, t, rea, rec = reset(*a, **k)
        tar_action, has_contact, ball_pos, root_pos = a[8], a[9], a[10], a[0]
        return r, t, rea, (tar_action == 1) & (has_contact | (ball_pos[:, 1] < root_pos[:, 1] - 1))
    rejects("reset_recovery", env_of["behind -inf"], controller_reset=keeps_recovery)

    def at_max_len(*a, **k):
        a = list(a)
        a[5] = a[5] + 1
        return reset(*a, **k)
    rejects("reset", env_of[f"progress {MAX_LEN - 2}"], controller_reset=at_max_len)
    # a neighbour's row, one value 1 ulp off
    for field, env, mutate in (("obs", 9, lambda b: b["obs"].__setitem__(9, b["obs"][10])),
                               ("est_max_height", env_of["height 0.0"],
                                lambda b: b["est_max_height"].__setitem__(env_of["height 0.0"], nxt(b["est_max_height"][env_of["height 0.0"]], INF))),
                               ("ball_traj", 11, lambda b: b["ball_traj"].__setitem__((11, 0, 0), nxt(b["ball_traj"][11, 0, 0], INF)))):
        bad = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in ref.items()}
        mutate(bad)
        assert any(x.startswith(field + ":") and f"env {env}:" in x for x in compare(ref, bad, POST_SPEC, limit=None)), field


def test_post_comparator_rejects_history_roll_and_dual_partner(monkeypatch):
    """ball_obs rolled on rows an observation refresh must not touch; the dual partner taken as e + 1"""
    rng = np.random.default_rng(4)
    s = base_state(64, rng, history=True)
    s["reset_reaction"][:], s["reset_recovery"][:] = False, False
    s["reset_reaction"][[3, 40]] = True
    s["reset_recovery"][[7]] = True
    touch = np.zeros(64, bool)
    touch[[7, 12]] = True
    cfg = post_cfg(obs_only=1, use_history=1)
    st = dict(s, touch_mask=touch)
    ref = V.controller_post(st, cfg)
    hr = V.history_rows
    monkeypatch.setattr(V, "history_rows", lambda s_, c_: np.ones(len(s_["root_pos"]), bool))
    bad = V.controller_post(st, cfg)
    monkeypatch.setattr(V, "history_rows", hr)
    fails = compare(ref, bad, POST_SPEC, limit=None)
    assert any(x.startswith("ball_obs:") and "env 12:" in x for x in fails), fails
    # dual: partner e + 1 (wrong for odd e)
    s = base_state(64, rng)
    s["tar_action"][:] = 1
    s["has_contact"][:] = False
    s["ball_pos"][5, 1] = s["root_pos"][5, 1] - 3       # env 5 misses: its partner 4 must be flagged for reaction
    cfg = post_cfg(dual=1, est=None)
    ref = V.controller_post(s, cfg)
    dr = V.dual_controller_reset

    def wrong_partner(tar_action, has_contact, has_bounce, ball_pos, root_pos, root_vel, bounce_in, distance, reset_buf):
        reset, rea, rec, dist = dr(tar_action, has_contact, has_bounce, ball_pos, root_pos, root_vel, bounce_in, distance, reset_buf)
        miss = (tar_action == 1) & (has_contact | (ball_pos[:, 1] < root_pos[:, 1] - f32(1)))
        rea = np.zeros_like(rea)
        rea[:-1] = miss[1:]
        return reset, rea, rec, dist
    monkeypatch.setattr(V, "dual_controller_reset", wrong_partner)
    bad = V.controller_post(s, cfg)
    monkeypatch.setattr(V, "dual_controller_reset", dr)
    assert any(x.startswith("reset_reaction:") and "env 4:" in x for x in compare(ref, bad, POST_SPEC, limit=None))


def test_counter_normal_matches_box_muller():
    """the uint64 restatement against Python integers for a few draws; the normals are finite with unit scale"""
    seed, step = 10 * 7919 + 13, 5

    def sm(x):
        x = (x + 0x9E3779B97F4A7C15) & V.M64
        x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & V.M64
        x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & V.M64
        return x ^ (x >> 31)
    idx = np.arange(0, 5000, 7)
    want = [sm((sm(seed ^ ((step * 0xD1B54A32D192ED03) & V.M64)) + int(i)) & V.M64) for i in idx]
    assert [int(h) for h in V.counter_hash(seed, step, idx)] == want
    z = V.counter_normal(seed, step, np.arange(200000))
    assert np.isfinite(z).all() and abs(float(z.mean())) < 0.02 and abs(float(z.std()) - 1) < 0.02


# ------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
def test_controller_post_sizes_and_cases():
    """every size, the case table on the coarse estimator table, advance on at odd sizes; rows past n untouched"""
    tx, ty = coarse_tables()
    est_dev = (_dev(tx), _dev(ty))
    full = []
    for j, n in enumerate(SIZES):
        rng = np.random.default_rng(100 + n)
        s = base_state(n, rng)
        cases = case_table(rng, COARSE, tx)
        where = apply_cases(s, cases, rng)
        if len(where) == len(cases):
            full.append((n, j % 2))
        check_post(s, post_cfg(est=(tx, ty), advance=j % 2), est_dev=est_dev, label=f"n = {n}")
    assert {a for _, a in full} == {0, 1} and len(full) >= 3, f"the whole case table ran only at {full}: it must run with and without advance"


@pytest.mark.gpu
@pytest.mark.parametrize("rtype", V.REWARD_NAMES)
def test_controller_post_mode_matrix(rtype):
    """reward type x early_termination x use_target x use_history x advance at n = 129, the case table in every one"""
    tx, ty = coarse_tables()
    est_dev = (_dev(tx), _dev(ty))
    for et in (0, 1):
        for use_target in (0, 1):
            for hist in (0, 1):
                for adv in (0, 1):
                    rng = np.random.default_rng(et * 8 + use_target * 4 + hist * 2 + adv)
                    s = base_state(129, rng, history=True)
                    apply_cases(s, case_table(rng, COARSE, tx), rng)
                    check_post(s, post_cfg(rtype=rtype, et=et, use_target=use_target, est=(tx, ty), use_history=hist, advance=adv),
                               est_dev=est_dev, label=f"{rtype} et {et} target {use_target} history {hist} advance {adv}")


@pytest.mark.gpu
def test_controller_post_traj_lengths_obs_only_and_dual():
    """obs_traj_len 0 / 1 / 10 / 100 (300-float shift buffers), the observation refresh with and without a touch mask (history mode,
    rows outside the masks untouched), and the dual FSM at even sizes"""
    tx, ty = coarse_tables()
    est_dev = (_dev(tx), _dev(ty))
    for L in (0, 1, 10, 100):
        for hist in ((0, 1) if L else (0,)):
            rng = np.random.default_rng(L + hist)
            s = base_state(257, rng, L=L, history=True)
            apply_cases(s, [c for c in case_table(rng, COARSE, tx) if not c[0].startswith("nan ball_obs") or L > 4], rng)
            check_post(s, post_cfg(L=L, est=(tx, ty), use_history=hist, advance=1), est_dev=est_dev, label=f"L = {L} history {hist}")
    for n in (1, 2, 9, 4097):
        for touch in (False, True):
            rng = np.random.default_rng(n)
            s = base_state(n, rng, history=True)
            tm = rng.random(n) < 0.2 if touch else None
            ref, got = check_post(s, post_cfg(est=(tx, ty), obs_only=1, use_history=1), est_dev=est_dev, touch_mask=tm,
                                  label=f"obs_only n = {n} touch {touch}")
            if touch:
                skip = ~(tm | s["reset_reaction"] | s["reset_recovery"])
                assert (got["obs"][skip] == SENT).all(), "an observation row outside the masks was written"
    for n in (2, 4, 8, 128, 130, 258, 4098, 8194):
        rng = np.random.default_rng(n)
        s = base_state(n, rng)
        apply_cases(s, [c for c in case_table(rng, COARSE, tx) if not c[0].startswith(("valid", "fma", "vel_x", "vy", "vspin", "height",
                                                                                        "net", "est_"))], rng)
        s["has_contact_now"][:] = False
        check_post(s, post_cfg(dual=1, advance=n % 4 == 0), label=f"dual n = {n}")


@pytest.mark.gpu
def test_estimator_on_the_reference_grid():
    """the estimator cases on the 0.1 / 0.1 / 0.2 grid (VX truncated to 10..15) with a table whose rows encode their index"""
    import torch
    rows = IndexTable.rows
    ex = torch.zeros(rows, NX, device="cuda:0")
    ex[:, 0] = torch.arange(rows, device="cuda:0", dtype=torch.float32)
    ey = torch.zeros(rows, NY, 2, device="cuda:0")
    ey[:, :, 0] = torch.arange(1, NY + 1, device="cuda:0", dtype=torch.float32)
    ey[:, :, 1] = torch.arange(rows, device="cuda:0", dtype=torch.float32)[:, None]
    est = (IndexTable("x"), IndexTable("y"))
    for n in (257, 1031):
        rng = np.random.default_rng(n)
        s = base_state(n, rng)
        cases = [c for c in case_table(rng, FINE, est[0]) if c[0].startswith(("valid", "fma", "vel_x", "vy", "vspin", "height", "net"))]
        where = apply_cases(s, cases, rng)
        assert len(where) == len(cases)
        check_post(s, post_cfg(est=est, grid=FINE), est_dev=(ex, ey), label=f"fine grid n = {n}")


@pytest.mark.gpu
def test_task_reset_sizes_and_edges():
    """b200v2p_task_reset against the restatement: pool index edges (x whose index lands at -1, 0, P-1, P; side_rand at its ends;
    ball_y at 0 and +-1 ulp), a pool of one row, reaction / recovery / both, both target modes (seeds at 0.33 / 0.67 +-1 ulp), history
    rows, the ball's rigid-body row; rows without a flag untouched"""
    import torch
    from vid2player3d_b200 import native_v2p as NV
    for n in SIZES:
        for P, mode, hist in ((257, "discrete", False), (1, "continuous", True), (1000, None, False)):
            rng = np.random.default_rng(n * 7 + P)
            pool = rng.uniform(-20, 20, (P, 307)).astype(f32)
            pool[:, 6] = rng.uniform(-10, 10, P)
            bp = np.stack([rng.uniform(-3, 3, n), rng.uniform(-5, 11, n), rng.uniform(0, 3, n)], -1).astype(f32)
            # x edges (index -1, 0, P - 1, P and the truncation at 8 / P) with side_rand 0, so no clamp hides the truncation, at
            # ball_y 0 / +-1 ulp; then the side_rand ends on the near path (y > 0) at both ends of the pool
            edges = [f32(-4), nxt(-4, INF), nxt(-4, -INF), f32(-4 - 8 / P), f32(4), nxt(4, -INF), f32(-4 + 8 / P), nxt(f32(-4 + 8 / P), -INF),
                     f32(-5), f32(5)]
            ys = [nxt(0, INF), f32(0), nxt(0, -INF)]
            side = rng.integers(-1000, 1000, n)
            for k in range(min(n, len(edges) * len(ys))):
                bp[k, 0], bp[k, 1], side[k] = edges[k % len(edges)], ys[k // len(edges)], 0
            for j, (x, sd) in enumerate(((-3.9, -1000), (3.9, 999), (0.0, -1000), (0.0, 999), (-3.9, 999), (3.9, -1000))):
                k = len(edges) * len(ys) + j
                if k < n:
                    bp[k, 0], bp[k, 1], side[k] = x, 5, sd
            seeds = np.concatenate([[f32(0.33), nxt(0.33, INF), nxt(0.33, -INF), f32(0.67), nxt(0.67, INF), nxt(0.67, -INF)],
                                    rng.random(max(n - 6, 0)).astype(f32)])[:n] if mode == "discrete" else rng.random(3).astype(f32)
            L = 10
            s = dict(ball_pos=bp, ball_vel=rng.normal(size=(n, 3)).astype(f32), bounce_pos=rng.normal(size=(n, 3)).astype(f32),
                     ball_traj=rng.normal(size=(n, 100, 3)).astype(f32), est_bounce_pos=rng.normal(size=(n, 3)).astype(f32),
                     est_bounce_time=rng.random(n).astype(f32), est_max_height=rng.random(n).astype(f32),
                     target_bounce_pos=rng.normal(size=(n, 3)).astype(f32), ball_states=rng.normal(size=(n, 13)).astype(f32),
                     rbs_ball=rng.normal(size=(n, 13)).astype(f32), has_bounce=rng.random(n) < 0.5, has_contact=rng.random(n) < 0.5,
                     bounce_in=rng.random(n) < 0.5, est_bounce_in=rng.random(n) < 0.5, tar_time=rng.integers(0, 80, n),
                     tar_time_total=rng.integers(60, 80, n), tar_action=rng.integers(0, 2, n), num_reset_reaction=rng.integers(0, 5, n),
                     swing_type_cycle=rng.integers(-1, 4, n), reset_reaction=rng.random(n) < 0.5, reset_recovery=rng.random(n) < 0.4,
                     ball_obs=rng.normal(size=(n, L, 3)).astype(f32) if hist else None)
            s["reset_reaction"][: min(n, 36)] = True
            draws = dict(pool_rand=rng.integers(0, P, n), side_rand=side, frame_rand=rng.integers(-5, 5, n), target_seed=seeds)
            cfg = dict(pool=pool, reaction_nframes=70, target_mode=mode, target_min=(-3, 9, 0), target_max=(3, 11, 0))
            ref = V.task_reset(s, cfg, draws)
            rbs = np.full((n + SLACK, 26, 13), SENT, f32)
            rbs[:n, 25] = s["rbs_ball"]
            t = {k: _dev(_pad(v, {"b": True, "i": ISENT}.get(v.dtype.kind, SENT))) for k, v in s.items()
                 if v is not None and k not in ("rbs_ball", "reset_reaction", "reset_recovery")}
            t.update(reset_reaction=_dev(_pad(s["reset_reaction"], True)), reset_recovery=_dev(_pad(s["reset_recovery"], True)),
                     rigid_body_state=_dev(rbs), pool=_dev(pool), ball_obs=t.get("ball_obs"),
                     **{k: _dev(v) for k, v in draws.items() if k != "target_seed"}, target_seed=_dev(seeds))
            NV.task_reset(dict(n=n, pool_size=P, ball_stride=13, bodies_per_env=26, reaction_nframes=70,
                               target_mode={None: 0, "continuous": 1, "discrete": 2}[mode], target_min=(-3, 9, 0), target_max=(3, 11, 0),
                               obs_traj_len=L), t)
            torch.cuda.synchronize()
            got = {k: t[k].cpu().numpy() for k in t if s.get(k) is not None}
            rb = t["rigid_body_state"].cpu().numpy()
            got["rbs_ball"] = rb[:, 25]
            for k, v in got.items():
                fill = {"b": True, "i": ISENT}.get(v.dtype.kind, SENT)
                assert (v[n:] == fill).all(), f"n = {n}: {k} written past n"
                got[k] = v[:n]
            assert (rb[:, :25] == SENT).all(), "a humanoid body row was written"
            spec = {k: "exact" for k in ref if ref[k] is not None and k not in ("pool",)}
            fails = compare(ref, got, spec)
            assert not fails, f"n = {n} P = {P} mode {mode}: " + "; ".join(fails[:6])


def check_normals(got, ref, rows, seed, step):
    """counter normals within 4 float32 ulps of the value plus 4 ulps of 1 in logf(u1), which 1 / sqrt(-2 ln u1) amplifies for u1 near 1"""
    n, nl = got.shape
    h = V.counter_hash(seed, step, np.arange(n)[:, None] * 35 + np.arange(nl))
    u1 = ((h >> np.uint64(40)).astype(np.float64) + 1) / 16777217.0
    bound = 4 * 2.0 ** -23 * (np.abs(ref) + 1 / np.sqrt(-2 * np.log(u1)))
    err = np.abs(got.astype(np.float64) - ref)
    bad = rows[:, None] & ~(err <= bound)
    assert not bad.any(), f"{int(bad.sum())} normals off; worst at {np.unravel_index(np.argmax(np.where(rows[:, None], err / bound, 0)), err.shape)}"


@pytest.mark.gpu
def test_ctrl_reset_pre_step_and_stream_gather():
    """ctrl_reset on a mask; pre_step's counter normals (logf / cosf within 4 ulp), its step counter advancing once per launch from
    one block to many with done_counter back at 0, a graph replay drawing fresh numbers; stream_gather with frames = 1, negative
    offsets and a reseed mask that leaves the other envs alone"""
    import torch
    from vid2player3d_b200 import native_v2p as NV
    dev = "cuda:0"
    for n in SIZES:
        rng = np.random.default_rng(n)
        mask = rng.random(n) < 0.4
        s = dict(progress=rng.integers(0, 300, n), reset=rng.integers(0, 2, n), terminate=rng.integers(0, 2, n),
                 num_reset_reaction=rng.integers(0, 9, n), distance=rng.random(n).astype(f32), num_reset=rng.integers(0, 9, n))
        ref = V.ctrl_reset(s, mask)
        t = {k: _dev(_pad(v, {"i": ISENT}.get(v.dtype.kind, SENT))) for k, v in s.items()}
        NV.ctrl_reset(_dev(mask), t["progress"], t["reset"], t["terminate"], t["num_reset_reaction"], t["distance"], t["num_reset"])
        got = {k: v.cpu().numpy() for k, v in t.items()}
        assert all((got[k][n:] == _pad(s[k], {"i": ISENT}.get(s[k].dtype.kind, SENT))[n:]).all() for k in got)
        assert not compare(ref, {k: v[:n] for k, v in got.items()}, {k: "exact" for k in s})
        # pre_step
        na, nl, nr = 35, 32, 3
        acts = rng.normal(size=(n, na)).astype(f32)
        tar = rng.integers(0, 2, n)
        cfg = dict(n=n, num_actions=na, num_latent=nl, num_res_dof=nr, random_walk_in_recovery=1, vae_action_scale=1.5,
                   residual_dof_scale=0.4, seed=79203)
        step = torch.tensor([int(rng.integers(0, 1 << 40))], device=dev)
        done = torch.zeros(1, dtype=torch.int32, device=dev)
        mv, rd = torch.full((n + SLACK, nl), float(SENT), device=dev), torch.full((n + SLACK, nr), float(SENT), device=dev)
        for rep in range(2):
            s0 = int(step.item())
            NV.pre_step(cfg, dict(actions=_dev(acts), tar_action=_dev(tar), step_counter=step, done_counter=done, mvae_actions=mv,
                                  res_dof_actions=rd))
            torch.cuda.synchronize()
            assert int(step.item()) == s0 + 1 and int(done.item()) == 0
            lat, res = V.pre_step(acts, tar, s0, cfg)
            g = mv.cpu().numpy()
            assert (g[n:] == SENT).all() and (rd.cpu().numpy()[n:] == SENT).all()
            assert np.array_equal(rd.cpu().numpy()[:n], res)
            walk = tar == 0
            assert np.array_equal(g[:n][~walk], lat[~walk])
            check_normals(g[:n], lat, walk, cfg["seed"], s0)
        # stream_gather
        K = 1 if n % 2 else 5
        ring = dict(ring_rotmat=rng.normal(size=(K * n, 24, 9)).astype(f32), ring_root_pos=rng.normal(size=(K * n, 3)).astype(f32),
                    ring_racket_pos=rng.normal(size=(K * n, 3)).astype(f32), ring_phase=rng.normal(size=K * n).astype(f32),
                    ring_swing_type=rng.integers(-1, 4, K * n), ring_swing_type_cycle=rng.integers(-1, 4, K * n))
        live = dict(rotmat=np.full((n + SLACK, 24, 9), SENT, f32), root_pos=np.full((n + SLACK, 3), SENT, f32),
                    racket_pos=np.full((n + SLACK, 3), SENT, f32), phase=np.full(n + SLACK, SENT, f32),
                    swing_type=np.full(n + SLACK, ISENT, np.int64), swing_type_cycle=np.full(n + SLACK, ISENT, np.int64))
        off = rng.integers(-3 * K, 3 * K, n)
        clock0 = int(rng.integers(0, 100))
        t = {k: _dev(v) for k, v in {**ring, **live}.items()}
        t.update(clock=torch.tensor([clock0], device=dev), done_counter=torch.zeros(1, dtype=torch.int32, device=dev), offset=_dev(_pad(off, ISENT)))
        reseed = rng.random(n) < 0.3
        for adv, rm in ((1, None), (0, reseed)):
            before = {k: t[k].cpu().numpy().copy() for k in live}
            frame, new_off = V.stream_frames(int(t["clock"].item()), adv, t["offset"].cpu().numpy()[:n], K, n, seed=99, reseed_mask=rm)
            NV.stream_gather(n, K, adv, t, reseed_mask=None if rm is None else _dev(rm), seed=99)
            torch.cuda.synchronize()
            assert int(t["clock"].item()) == clock0 + 1 and int(t["done_counter"].item()) == 0
            assert np.array_equal(t["offset"].cpu().numpy()[:n], new_off)
            sel = np.ones(n, bool) if rm is None else rm
            row = frame * n + np.arange(n)
            for k, rk in (("rotmat", "ring_rotmat"), ("root_pos", "ring_root_pos"), ("racket_pos", "ring_racket_pos"), ("phase", "ring_phase"),
                          ("swing_type", "ring_swing_type"), ("swing_type_cycle", "ring_swing_type_cycle")):
                g = t[k].cpu().numpy()
                assert np.array_equal(g[:n][sel], ring[rk][row][sel]), (n, k)
                assert np.array_equal(g[:n][~sel], before[k][:n][~sel]) and np.array_equal(g[n:], before[k][n:]), (n, k)


@pytest.mark.gpu
def test_pre_step_graph_replay_draws_fresh_numbers():
    import torch
    from vid2player3d_b200 import native_v2p as NV
    n, dev = 8195, "cuda:0"
    cfg = dict(n=n, num_actions=35, num_latent=32, num_res_dof=3, random_walk_in_recovery=1, vae_action_scale=1.5, residual_dof_scale=0.4,
               seed=5)
    t = dict(actions=torch.zeros(n, 35, device=dev), tar_action=torch.zeros(n, dtype=torch.long, device=dev),
             step_counter=torch.zeros(1, dtype=torch.long, device=dev), done_counter=torch.zeros(1, dtype=torch.int32, device=dev),
             mvae_actions=torch.zeros(n, 32, device=dev), res_dof_actions=torch.zeros(n, 3, device=dev))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        NV.pre_step(cfg, t)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        NV.pre_step(cfg, t)
    outs = []
    for _ in range(3):
        st = int(t["step_counter"].item())
        g.replay()
        torch.cuda.synchronize()
        outs.append(t["mvae_actions"].cpu().numpy().copy())
        lat, _ = V.pre_step(np.zeros((n, 35), f32), np.zeros(n, np.int64), st, cfg)
        check_normals(outs[-1], lat, np.ones(n, bool), cfg["seed"], st)
    assert not np.array_equal(outs[0], outs[1]) and not np.array_equal(outs[1], outs[2])


@pytest.mark.gpu
def test_actor_reset_id_lists_masks_and_racket_weld():
    """b200v2p_actor_reset against the restatement at every size: a shuffled, unsorted id list, and the mask form (ids 0..N-1 with a
    mask); one and two players (dual: odd envs weld the racket to the second player's parent with its offset).  Every row the launch
    writes must match (the racket row within 2 ulps: the kernel rotates the offset by the algebraically equal 2 q x (q x o) form); rows
    outside the list or the mask, rows past N, the ball body and the other columns of the root rows stay bit-identical."""
    import torch
    from vid2player3d_b200 import native_v2p as NV
    nd, B, RS = 69, 26, 16
    for N in SIZES:
        for form, dual in (("list", False), ("mask", True), ("list", True)):
            if dual and N % 2:
                continue
            rng = np.random.default_rng(N * 3 + dual)
            q = rng.normal(size=(N, 24, 4))
            q /= np.linalg.norm(q, axis=-1, keepdims=True)
            r = rng.normal(size=(N, 4))
            r /= np.linalg.norm(r, axis=-1, keepdims=True)
            src = dict(root_pos=rng.normal(size=(N, 3)).astype(f32), root_rot=r.astype(f32), dof_pos=rng.normal(size=(N, nd)).astype(f32),
                       rb_pos=rng.normal(size=(N, 24, 3)).astype(f32), rb_rot=q.astype(f32))
            g = lambda *sh: rng.normal(size=sh).astype(f32)  # noqa: E731
            s = dict(root_states=g(N, RS), dof_state=g(N, nd, 2), rbs=g(N, B, 13), prev_target_root_pos=g(N, 3), prev_target_rb_rot=g(N, 24, 4),
                     root_pos=g(N, 3), root_vel=g(N, 3), pd_target_dof_pos=g(N, nd), target_root_pos=g(N, 3),
                     progress=rng.integers(1, 300, N), reset=rng.integers(0, 2, N) + 1, terminate=rng.integers(0, 2, N) + 1)
            cfg = dict(racket_body=24, racket_parent=22, racket_offset=(0.5, -0.02, 0.01))
            if dual:
                cfg.update(dual=1, racket_parent2=17, racket_offset2=(-0.5, 0.03, -0.01))
            if form == "list":
                ids = rng.permutation(N)[: max(1, N // 3)]
                mask = None
            else:
                mask = rng.random(N) < 0.3
                ids = np.flatnonzero(mask)
            ref = V.actor_reset(s, src, ids, cfg)
            t = {k: _dev(_pad(v, {"i": ISENT}.get(v.dtype.kind, SENT))) for k, v in s.items()}
            srcd = {k: _dev(v) for k, v in src.items()}
            lid = np.arange(N) if form == "mask" else ids
            NV.actor_reset(dict(n=len(lid), num_dof=nd, bodies_per_env=B, root_stride=RS, **cfg),
                           dict(env_ids=_dev(lid.astype(np.int64)), src_root_pos=srcd["root_pos"], src_root_rot=srcd["root_rot"],
                                src_dof_pos=srcd["dof_pos"], src_rb_pos=srcd["rb_pos"], src_rb_rot=srcd["rb_rot"], root_states=t["root_states"],
                                dof_state=t["dof_state"], rigid_body_state=t["rbs"], prev_target_root_pos=t["prev_target_root_pos"],
                                prev_target_rb_rot=t["prev_target_rb_rot"], root_pos=t["root_pos"], root_vel=t["root_vel"],
                                pd_target_dof_pos=t["pd_target_dof_pos"], target_root_pos=t["target_root_pos"], progress_buf=t["progress"],
                                reset_buf=t["reset"], terminate_buf=t["terminate"], mask=None if mask is None else _dev(mask)))
            torch.cuda.synchronize()
            got = {k: v.cpu().numpy() for k, v in t.items()}
            for k, v in got.items():
                assert (v[N:] == {"i": ISENT}.get(v.dtype.kind, SENT)).all(), f"N = {N}: {k} written past N"
                got[k] = v[:N]
            racket = (slice(None), 24, slice(0, 3))
            spec = {k: "exact" for k in s}
            a, b = ref["rbs"].copy(), got["rbs"].copy()
            fails = compare({"racket": a[racket]}, {"racket": b[racket]}, {"racket": 4e-7})
            a[racket], b[racket] = 0, 0
            fails += compare({**ref, "rbs": a}, {**got, "rbs": b}, spec)
            assert not fails, f"N = {N} {form} dual {dual}: " + "; ".join(fails[:6])


@pytest.mark.gpu
def test_idlist_reset_refreshes_only_the_reset_rows_in_history_mode():
    """PhysicsMVAEController._reset_envs_idlist, the reference-shaped reset (:173-201), in use_history_ball_obs mode: its observation
    refresh (_compute_observations(reset_all_env_ids), :197-198) writes the obs rows of the reset envs and rolls their ball history
    (:345-346), like V.controller_post(obs_only) on those rows; the history, obs, bounce_in and est_* of every other env stay as they were"""
    import torch
    from helpers import SIM_PARAMS, v2p_cfg
    from vid2player3d_b200.tasks import PhysicsMVAEController
    N = 64
    torch.manual_seed(7)
    env = PhysicsMVAEController(v2p_cfg(N, use_history_ball_obs=True), SIM_PARAMS, 1, "cuda", 0, True)
    env.reset()
    for _ in range(3):
        env.step(torch.clamp(torch.randn(N, env.num_actions, device="cuda:0"), -5, 5))
        env.reset(env.reset_buf.nonzero(as_tuple=False).flatten())
    task = env._physics_player.task
    rea, rec = torch.zeros(N, dtype=torch.bool, device="cuda:0"), torch.zeros(N, dtype=torch.bool, device="cuda:0")
    rea[[2, 9, 30]], rec[[5, 9, 41, 60]] = True, True
    env._reset_reaction_buf.copy_(rea)
    env._reset_recovery_buf.copy_(rec)
    # a bounce this step on envs in recovery: a full post step would rewrite their bounce_in (set to the opposite of in_court here)
    env._tar_action[:] = torch.where(rea | rec, env._tar_action, torch.zeros_like(env._tar_action))
    task._has_bounce_now[:] = True
    task._bounce_pos[:, 0:2] = torch.tensor([0.0, 5.0], device="cuda:0")
    env._bounce_in[:] = False
    g = lambda x: x.detach().cpu().numpy().copy()  # noqa: E731
    names = ("_ball_obs", "obs_buf", "_bounce_in", "_est_bounce_pos", "_est_bounce_time", "_est_max_height", "_est_bounce_in", "_distance")
    before = {k: g(getattr(env, k)) for k in names}
    env._reset_envs_idlist(torch.zeros(0, dtype=torch.long, device="cuda:0"))
    torch.cuda.synchronize()
    after = {k: g(getattr(env, k)) for k in names}
    rows = g(rea | rec)
    pre = before["_ball_obs"].copy()              # the history the refresh starts from: reaction rows were reset to the launch position
    pre[g(rea)] = g(task._ball_pos)[g(rea)][:, None, :]
    s = dict(rbs=g(task._rigid_body_state.view(N, 26, 13)), root_pos=g(task._root_pos), root_vel=g(task._root_vel),
             racket_normal=g(task._racket_normal), ball_pos=g(task._ball_pos), ball_traj=g(env._ball_traj),
             target_bounce_pos=g(env._target_bounce_pos), ball_obs=pre, obs=before["obs_buf"], reset_reaction=rows,
             reset_recovery=np.zeros(N, bool), touch_mask=np.zeros(N, bool))
    ref = V.controller_post(s, post_cfg(obs_only=1, use_history=1))
    fails = compare(ref, {"obs": after["obs_buf"], "ball_obs": after["_ball_obs"]}, {"obs": "obs", "ball_obs": "exact"})
    keep = ~rows
    fails += compare({k: before[k] for k in names}, after, {k: "exact" for k in names if k not in ("_ball_obs", "obs_buf")}, rows=np.flatnonzero(keep))
    assert not fails, "; ".join(fails[:6])
