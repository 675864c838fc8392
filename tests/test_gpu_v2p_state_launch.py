"""The FK target, head look-at, state refresh, ball reset, incoming-ball estimator and ball aerodynamics launches
(include/b200env_v2p.h) against the numpy oracle (oracle/ref_port_v2p.py, pinned to the reference by test_oracle_golden_v2p.py), at
ragged sizes, on every branch and threshold, with every row the launch must not write checked.

1. Sizes 1 ... 8195: the ragged last block of the warp-per-env kernels (4 warps per block) and of the 128-thread ones.  Every output
   starts as a sentinel and has SLACK rows past n; rows past n, rows whose mask is clear and envs missing from an id list stay
   bit-identical.  Row r of an 8195-env launch is bitwise equal to the same row of an (r + 1)-env launch of the same inputs, and two
   launches are bitwise equal.
2. Exact (==, NaN equal to NaN) against the float32 oracle: every field written by copies, subtractions, divisions or explicitly
   rounded intrinsics in the oracle's order - ball_reset and ball_in_estimate entirely (the selected table row included), the copies,
   contact flags and velocity-jump detector of update_state, the flags and bounce_pos of ball_aero, and root_vel, prev_root_pos_update
   and target_root_pos_out of smpl_to_sim.
3. Bounded against a float64 oracle run on the same float32 inputs, where nvcc contracts products into fma or libm differs.  u = 2^-24;
   each bound is absolute and already scaled as stated:
   - smpl_to_sim FK.  A level of the chain G = G_parent R adds at most 9u in the spectral norm (nine entries, each a 3-term dot of unit
     rows and columns rounded twice), so depth 8 carries <= 72u.  rb_pos sums G rel + P_parent along the chain (sum |rel| < 1.2 m,
     |P| < 1.5 m): 72u * 1.2 + 3u * 8 * 1.5 + 2u * |root| < 160u * max(1, |v|).  rb_rot / root_rot: the branch taken has sq >= 2, so a
     component moves by <= 2 * 72u + 6u < 160u.  dof_pos converts an exact input matrix: <= 12u in the quaternion, |d aa / d q| <= pi + 2
     over four components, plus 3 ulp of atan2f: < 128u * max(1, |v|).
   - smpl_to_sim velocities: the condition of 2 acos(w).  With Q = 160u the error of the current quaternion, the normalised difference
     carries <= 4.1Q in w and in its vector part; st = sqrt(1 - w^2) moves by (4.1Q + u) / st, the angle by 8.2Q / st + 10u pi, the axis
     by 4.1Q / st + (4.1Q + u) / st^2, and angle / st <= pi for w >= 0.  So |d dof_vel| <= (24Q / st + 16Q) / dt, st taken from the
     float64 run; root_ang_vel is divided by dt once more (the reference quirk).
   - fix_head: the yaw error d moves by 64u / |look_xy| (the look vector of a normalised quaternion, entries <= 45u off) plus
     2u (|ball_xy| + |head_xy|) / |ball_xy - head_xy| plus 16u of atan2f; a term is 0 where its vector is exactly 0 (both sides take
     the 1e-12 clamp).  The corrected matrix moves by 2 * (128u * 4 + d_err / 2) + 16u = 1040u + d_err.  Random envs are kept 1e-3
     away from d = +-pi, where one rounding flips the wrap by 2 pi; the wrap cases are built 0.5 rad past it.
   - update_state: racket_normal < 64u * max(1, |v|) (normalisation 3u, each matrix entry <= 34u, a 3-term dot with a unit grip);
     ball_vspin < 8u * max(1, |v|) (three squares, sqrt, and 6.283185307179586f against 2 pi).
   - ball_aero force: <= 32u * KF * (CD + 0.5) * |v|^2 per component (drag and lift each within 32u of their magnitudes; |cl| <= 1/2).
4. Quaternion sign: where the float64 FK rotation lies within 1e-4 of a branch switch of rotmat_to_quat_wxyz (trace 0 or a tie on the
   diagonal) both signs are valid and float32 rounding picks one, so rb_rot is compared up to sign there, below the root only (the root's
   matrix is the input itself, so both sides take the same branch).
5. CPU negative controls: each comparator rejects a mutated oracle and names the env and the field.

Out of scope: duplicate ids in ball_reset are undefined, as in the reference's indexed assignment (callers pass unique ids); an
out-of-range pool_index is not checked (the ABI does not carry the pool's row count, and the caller clamps)."""
import ctypes as C
import math

import numpy as np
import pytest

from conftest import golden
from oracle import ref_port as R
from oracle import ref_port_v2p as V
from test_gpu_v2p_launch import INF, SENT, SIZES, SLACK, _dev, _pad, fma_cases, nxt

f32, f64 = np.float32, np.float64
U = 2.0 ** -24
DT = float(f32(1 / 30))
DEV = "cuda:0"
BIG = SIZES[-1]
WORST = {}
SM_OUT = dict(root_rot=(4,), dof_pos=(69,), root_vel=(3,), root_ang_vel=(3,), dof_vel=(69,), rb_pos=(24, 3), rb_rot=(24, 4))
IN_COARSE = golden("v2p_dual.npz")["in_params"]          # HEIGHT, VEL_X, VEL_Y, VSPIN: 5 x 4 x 2 x 4 rows
IN_SHIPPED = golden("v2p_dual.npz")["in_params_full"]    # 15 x 50 x 30 x 50 rows
PLAYERS = (dict(grip="eastern", wrist=22, racket=24), dict(grip="semi_western", wrist=17, racket=23))


@pytest.fixture(scope="module", autouse=True)
def report_worst_ratio():
    yield
    if WORST:
        print("\nworst |got - ref| / bound per field: " + ", ".join(f"{k}: {r:.3g}" for k, r in sorted(WORST.items())))


# ------------------------------------------------------------------------------------------------ comparator (CPU)
def compare(ref, got, spec, rows=None, limit=8, tag=""):
    """-> list of "field: env i: ..." failures.  spec[field] = "exact", or an absolute bound (scalar or array of the field's shape);
    NaN equals NaN.  The worst error / bound ratio of each bounded field goes to WORST."""
    fails = []
    for k, how in spec.items():
        a, b = np.asarray(ref[k]), np.asarray(got[k])
        bd = None if isinstance(how, str) else np.broadcast_to(np.asarray(how, f64), a.shape)
        if rows is not None:
            a, b = a[rows], b[rows]
            bd = None if bd is None else bd[rows]
        if len(a) == 0:
            continue
        a2, b2 = a.reshape(len(a), -1), b.reshape(len(b), -1)
        both_nan = (np.isnan(a2) & np.isnan(b2)) if a2.dtype.kind == "f" else np.zeros(a2.shape, bool)
        if bd is None:
            bad = ~((a2 == b2) | both_nan)
        else:
            bd2 = bd.reshape(len(a), -1)
            with np.errstate(invalid="ignore"):
                err = np.abs(a2.astype(f64) - b2.astype(f64))
                bad = ~((a2 == b2) | (err <= bd2) | both_nan)
                fin = np.isfinite(err) & (bd2 > 0) & np.isfinite(bd2)
            if tag and fin.any():
                WORST[tag + k] = max(WORST.get(tag + k, 0.0), float((err[fin] / bd2[fin]).max()))
        for r in np.flatnonzero(bad.any(1))[:limit]:
            c = int(np.flatnonzero(bad[r])[0])
            env = int(rows[r]) if rows is not None else int(r)
            fails.append(f"{k}: env {env}: column {c} got {b2[r, c]!r} ref {a2[r, c]!r} ({int(bad.any(1).sum())} envs differ)")
    return fails


def place(n, cases, rng):
    """case k on env perm[k] (as many as n allows); -> {env: name}"""
    perm = rng.permutation(n)
    out = {}
    for k, (name, fn) in enumerate(cases[:n]):
        fn(int(perm[k]))
        out[int(perm[k])] = name
    return out


# ------------------------------------------------------------------------------------------------ smpl_to_sim (CPU side)
def skeleton():
    g = golden("v2p_smpl_to_sim.npz")
    return g["rest"].astype(f32), g["parents"].astype(np.int32), g["smpl_2_mujoco"].astype(np.int32)


def rand_rot(rng, *shape):
    q = rng.normal(size=shape + (4,))
    return V.quaternion_to_rotation_matrix_wxyz(q / np.linalg.norm(q, axis=-1, keepdims=True))


def rot_x(deg):
    c, s = math.cos(math.radians(deg)), math.sin(math.radians(deg))
    return np.array([[1, 0, 0], [0, c, -s], [0, s, c]], f32)


# exact matrices on every branch of rotmat_to_quat_wxyz (trace > 0 / m00 largest / m11 > m22 / else) and both signs of w
SPECIAL_ROTS = (("identity matrix", np.eye(3, dtype=f32)), ("180 about x", np.diag([1, -1, -1]).astype(f32)),
                ("180 about y", np.diag([-1, 1, -1]).astype(f32)), ("180 about z", np.diag([-1, -1, 1]).astype(f32)),
                ("tie m00 == m11 > m22", np.array([[0, 1, 0], [1, 0, 0], [0, 0, -1]], f32)),
                ("tie m11 == m22", np.array([[-1, 0, 0], [0, 0, 1], [0, 1, 0]], f32)),
                ("trace 0, w > 0", np.array([[0, 0, 1], [1, 0, 0], [0, 1, 0]], f32)),
                ("trace 0, w < 0", np.array([[0, 1, 0], [0, 0, 1], [1, 0, 0]], f32)), ("-150 about x, w < 0", rot_x(-150)))


def quat_branch(m):
    """(branch of rotmat_to_quat_wxyz, w) in float64"""
    m = m.astype(f64)
    tr = m[0, 0] + m[1, 1] + m[2, 2]
    b = 0 if tr > 0 else (1 if m[0, 0] > m[1, 1] and m[0, 0] > m[2, 2] else (2 if m[1, 1] > m[2, 2] else 3))
    return b, float(V.rotation_matrix_to_quaternion_wxyz(m)[0])


def fk_quat64(inp, e):
    """float64 FK body quaternions (MuJoCo order, xyzw) of env e"""
    _, par, s2m = skeleton()
    K = len(inp["rest"])
    return V.smpl_to_sim(inp["root"][e:e + 1].astype(f64), inp["rot"][e:e + 1].astype(f64), inp["rest"][e % K][None].astype(f64),
                         par, s2m, DT)[7][0]


def make_smpl(n, K, seed):
    rest0, _, _ = skeleton()
    rng = np.random.default_rng(seed)
    rest = np.stack([rest0 * f32(1 + 0.1 * k) + rng.normal(0, 0.01, (24, 3)) for k in range(K)]).astype(f32)
    q = rng.normal(size=(n, 24, 4))
    inp = dict(rest=rest, rot=rand_rot(rng, n, 24).astype(f32), root=rng.uniform(-3, 3, (n, 3)).astype(f32),
               prev_rot=(q / np.linalg.norm(q, axis=-1, keepdims=True)).astype(f32))
    inp["prev_root"] = (inp["root"] + rng.normal(0, 0.05, (n, 3))).astype(f32)
    cases = []

    def identity(e):   # prev == cur == identity: d = (0, 0, 0, 1) exactly, st = 0 <= 1e-5: angle 0, axis (0, 0, 1)
        inp["rot"][e] = np.eye(3, dtype=f32)
        inp["prev_rot"][e] = (0, 0, 0, 1)
    cases.append(("identity env", identity))
    for i, (name, m) in enumerate(SPECIAL_ROTS):
        cases.append((name, lambda e, m=m, i=i: (inp["rot"].__setitem__((e, 0), m), inp["rot"].__setitem__((e, 1 + i % 23), m))))
    place_later = [("near pi", 1.0), ("near pi, sign flip", -1.0), ("prev = cur", 0.0)]
    for name, _ in place_later:
        cases.append((name, lambda e: None))
    where = place(n, cases, rng)
    for e, name in where.items():       # previous frames defined against the float64 FK of the final rotations
        for pname, sgn in place_later:
            if name != pname:
                continue
            cur = fk_quat64(inp, e)
            if sgn == 0.0:
                inp["prev_rot"][e] = cur.astype(f32)
                continue
            ax = rng.normal(size=(24, 3))
            ax /= np.linalg.norm(ax, axis=-1, keepdims=True)
            ang = np.pi - 1e-3       # frame-to-frame rotation just under pi
            delta = np.concatenate([ax * np.sin(ang / 2), np.full((24, 1), np.cos(ang / 2))], -1)
            prev = R.quat_mul(cur, R.quat_conjugate(delta))        # conj(prev) cur = delta
            inp["prev_rot"][e] = (sgn * prev / np.linalg.norm(prev, axis=-1, keepdims=True)).astype(f32)
    inp["where"] = where
    return inp


def smpl_expected(inp, n, mode, rest_of=lambda e, K: e % K, ang_div_dt=2):
    """(reference outputs, spec).  float64 run for the bounded fields, float32 run for root_vel"""
    _, par, s2m = skeleton()
    K = len(inp["rest"])
    rest_env = inp["rest"][rest_of(np.arange(n), K)]
    prev = mode != "fresh"
    p64 = (inp["prev_root"][:n].astype(f64), inp["prev_rot"][:n].astype(f64)) if prev else (None, None)
    p32 = (inp["prev_root"][:n], inp["prev_rot"][:n]) if prev else (None, None)
    with np.errstate(invalid="ignore", divide="ignore"):
        o64 = V.smpl_to_sim(inp["root"][:n].astype(f64), inp["rot"][:n].astype(f64), rest_env.astype(f64), par, s2m, DT, *p64)
        o32 = V.smpl_to_sim(inp["root"][:n], inp["rot"][:n], rest_env, par, s2m, DT, *p32)
    ref = dict(root_rot=o64[1], dof_pos=o64[2], root_vel=o32[3], root_ang_vel=o64[4] * DT ** (2 - ang_div_dt), dof_vel=o64[5],
               rb_pos=o64[6], rb_rot=o64[7])
    Q = 160 * U
    spec = dict(root_rot=Q, dof_pos=128 * U * np.maximum(1, np.abs(o64[2])), root_vel="exact", rb_pos=160 * U * np.maximum(1, np.abs(o64[6])),
                rb_rot=Q)
    if prev:
        w = V.quat_mul_norm(R.quat_conjugate(p64[1]), o64[7])[..., 3]
        with np.errstate(divide="ignore"):
            bd = (24 * Q / np.sqrt(np.maximum(0, 1 - w * w)) + 16 * Q) / DT
        spec.update(dof_vel=np.repeat(bd[:, 1:], 3, 1), root_ang_vel=np.repeat(bd[:, :1] / DT, 3, 1))
        ref["prev_root_pos_update"] = ref["target_root_pos_out"] = inp["root"][:n]
    else:
        spec.update(dof_vel="exact", root_ang_vel="exact")
    G = V.batch_rigid_transform(inp["rot"][:n].astype(f64), rest_env.astype(f64), par)[1][:, s2m]
    d = np.stack([G[..., 0, 0], G[..., 1, 1], G[..., 2, 2]], -1)
    near = ((np.abs(d.sum(-1)) <= 1e-4) | (np.abs(d[..., 0] - d[..., 1]) <= 1e-4) | (np.abs(d[..., 0] - d[..., 2]) <= 1e-4) |
            (np.abs(d[..., 1] - d[..., 2]) <= 1e-4))
    near[:, 0] = False
    ref["_near_branch"] = near
    return ref, spec


def align_sign(got_rot, ref):
    """flip got's quaternion where the float64 rotation sits on a branch switch and -got is the closer one"""
    g = got_rot.copy()
    flip = ref["_near_branch"] & (np.abs(g + ref["rb_rot"]).sum(-1) < np.abs(g - ref["rb_rot"]).sum(-1))
    g[flip] *= -1
    return g


# ------------------------------------------------------------------------------------------------ fix_head (CPU side)
def yaw_error(head_rot, head_pos, ball):
    """float64 restatement of the correction's inputs: (raw d before the wrap, |look_xy|, |ball_xy - head_xy|)"""
    m = V.quaternion_to_rotation_matrix_wxyz(head_rot.astype(f64)[:, [3, 0, 1, 2]])
    look = m[:, :2, 2]
    hb = ball[:, :2].astype(f64) - head_pos[:, :2].astype(f64)
    ln, bn = np.linalg.norm(look, axis=-1), np.linalg.norm(hb, axis=-1)
    lk = look / np.maximum(ln, 1e-12)[:, None]
    bb = hb / np.maximum(bn, 1e-12)[:, None]
    return np.arctan2(bb[:, 1], bb[:, 0]) - np.arctan2(lk[:, 1], lk[:, 0]), ln, bn


def quat_xyzw(axis, ang):
    axis = np.asarray(axis, f64) / np.linalg.norm(axis)
    return np.concatenate([axis * np.sin(ang / 2), [np.cos(ang / 2)]])


def head_tilted(alpha):
    """head quaternion whose z axis points along yaw alpha in the xy plane: R_z(alpha) R_y(90 deg)"""
    return R.quat_mul(quat_xyzw((0, 0, 1), alpha), quat_xyzw((0, 1, 0), np.pi / 2))


def make_head(n, seed):
    rng = np.random.default_rng(seed)
    q = rng.normal(size=(n, 24, 4))
    inp = dict(rb_rot=(q / np.linalg.norm(q, axis=-1, keepdims=True)).astype(f32), rb_pos=rng.uniform(-1, 1, (n, 24, 3)).astype(f32),
               root=np.stack([rng.uniform(-3, 3, n), rng.uniform(-14, -9, n), rng.uniform(0.8, 1, n)], -1).astype(f32),
               rot=rand_rot(rng, n, 24).astype(f32))
    inp["rb_pos"][:, 13] = inp["root"] + np.array([0, 0, 0.6], f32)
    inp["ball"] = np.stack([rng.uniform(-3.9, 3.9, n), rng.uniform(-10, 12, n), rng.uniform(0.1, 3, n)], -1).astype(f32)
    cases = []

    def miss_y(k):
        def fn(e):
            y = f32(inp["root"][e, 1] - f32(0.5))       # exact: root y and root y - 0.5 share a binade
            inp["ball"][e, 1] = nxt(y, INF if k > 0 else -INF) if k else y
        return fn
    for k in (0, -1, 1):
        cases.append((f"ball_y = root_y - 0.5 {k:+d} ulp", miss_y(k)))
    for x in (f32(4), f32(-4)):
        for k in (0, -1, 1):
            cases.append((f"ball_x {x} {k:+d} ulp", lambda e, x=x, k=k: inp["ball"].__setitem__((e, 0), nxt(x, INF if k > 0 else -INF) if k else x)))

    def wrap(alpha, beta):
        def fn(e):
            inp["rb_rot"][e, 13] = head_tilted(alpha).astype(f32)
            inp["rb_pos"][e, 13, :2] = (0, inp["root"][e, 1])         # ball 1 m away: |sin beta| < 0.5 keeps it clear of the miss test
            inp["ball"][e, :2] = (np.cos(beta), inp["root"][e, 1] + np.sin(beta))
        return fn
    cases.append(("wrap -2 pi", wrap(2.8, 0.4 - np.pi)))       # raw d = 0.4 - pi - 2.8 < -pi
    cases.append(("wrap +2 pi", wrap(-2.8, np.pi - 0.4)))      # raw d = pi - 0.4 + 2.8 > pi
    cases.append(("head up (identity)", lambda e: inp["rb_rot"].__setitem__((e, 13), (0, 0, 0, 1))))
    cases.append(("head up (yaw only)", lambda e: inp["rb_rot"].__setitem__((e, 13), quat_xyzw((0, 0, 1), 1.1).astype(f32))))
    cases.append(("ball above head", lambda e: inp["ball"].__setitem__((e, slice(0, 2)), inp["rb_pos"][e, 13, :2])))

    def taylor(corrected):
        def fn(e):
            if corrected:       # head up: d = atan2(ball direction) exactly known; joints yawed by -d/2 + 3e-4 -> theta^2 ~ 9e-8
                inp["rb_rot"][e, 13] = (0, 0, 0, 1)
                inp["ball"][e, :2] = inp["rb_pos"][e, 13, :2] + np.array([0.6, 1.7], f32)
                d = float(yaw_error(inp["rb_rot"][e:e + 1, 13], inp["rb_pos"][e:e + 1, 13], inp["ball"][e:e + 1])[0][0])
                a = -d / 2 + 3e-4
            else:               # miss: no correction, theta^2 = 2.5e-7
                inp["ball"][e, 0] = 4.5
                a = 5e-4
            for j in (15, 12):
                inp["rot"][e, j] = V.angle_axis_to_rotation_matrix(np.array([0, a, 0], f64)).astype(f32)
        return fn
    cases.append(("taylor, miss", taylor(False)))
    cases.append(("taylor, corrected", taylor(True)))
    where = place(n, cases, rng)
    d, _, _ = yaw_error(inp["rb_rot"][:, 13], inp["rb_pos"][:, 13], inp["ball"])
    for e in range(n):   # random envs: 1e-3 away from the wrap at +-pi
        if e not in where:
            while abs(abs(d[e]) - np.pi) < 1e-3 or abs(abs(d[e]) - 3 * np.pi) < 1e-3:
                inp["ball"][e, 0] = f32(inp["ball"][e, 0] * 0.9)
                d[e] = yaw_error(inp["rb_rot"][e:e + 1, 13], inp["rb_pos"][e:e + 1, 13], inp["ball"][e:e + 1])[0][0]
    inp["where"] = where
    return inp


def head_expected(inp, n):
    s = slice(0, n)
    ref = V.fix_head_orientation(inp["rot"][s].astype(f64), inp["rb_rot"][s, 13].astype(f64), inp["rb_pos"][s, 13].astype(f64),
                                 inp["ball"][s].astype(f64), inp["root"][s].astype(f64))
    _, ln, bn = yaw_error(inp["rb_rot"][s, 13], inp["rb_pos"][s, 13], inp["ball"][s])
    mag = np.linalg.norm(inp["ball"][s, :2].astype(f64), axis=-1) + np.linalg.norm(inp["rb_pos"][s, 13, :2].astype(f64), axis=-1)
    with np.errstate(divide="ignore", invalid="ignore"):
        derr = np.where(ln > 0, 64 * U / ln, 0) + np.where(bn > 0, 2 * U * mag / bn, 0) + 16 * U
    bound = np.zeros((n, 24, 3, 3))
    bound[:, [12, 15]] = (1040 * U + derr)[:, None, None, None]
    return ref, bound


# ------------------------------------------------------------------------------------------------ update_state (CPU side)
def body_of(e, dual, key):
    return PLAYERS[1][key] if dual and e % 2 else PLAYERS[0][key]


def make_state(n, seed, ball_stride=13, root_stride=13, dual=False):
    rng = np.random.default_rng(seed)
    rbs = rng.uniform(-2, 2, (n, 26, 13)).astype(f32)
    rbs[..., 3:7] = rng.normal(size=(n, 26, 4))
    ball = rng.normal(size=(n, ball_stride)).astype(f32)
    ball[:, 8] = rng.uniform(-30, 30, n)
    inp = dict(rbs=rbs, root=rng.normal(size=(n, root_stride)).astype(f32), ball=ball, dual=dual,
               prev_vel=rng.uniform(-20, 20, (n, 3)).astype(f32), contact=rng.random(n) < 0.3, now=rng.random(n) < 0.5)

    def det(b8, prev, contact=False):
        def fn(e):
            inp["ball"][e, 8], inp["prev_vel"][e, 1], inp["contact"][e] = b8, prev, contact
        return fn
    wq = lambda q: lambda e: inp["rbs"].__setitem__((e, body_of(e, dual, "wrist"), slice(3, 7)), q)  # noqa: E731
    cases = [("ball[8] = 0", det(f32(0), f32(-20))), ("ball[8] = +1 ulp", det(nxt(0, INF), f32(-20))),
             ("jump = 10", det(f32(25), f32(15))), ("jump = 10 + ulp", det(nxt(25, INF), f32(15))),
             ("jump = 10 - ulp", det(nxt(25, -INF), f32(15))), ("contact already set", det(f32(30), f32(0), True)),
             ("zero wrist quaternion", wq((0, 0, 0, 0))), ("nan wrist quaternion", wq((np.nan, 0.5, 0.5, 0.5)))]
    inp["where"] = place(n, cases, rng)
    return inp


def state_before(inp, n):
    sent3 = np.full((n, 3), SENT, f32)
    return dict(has_contact=inp["contact"][:n], has_contact_now=inp["now"][:n], root_pos=sent3, root_vel=sent3, racket_pos=sent3,
                racket_vel=sent3, racket_normal=sent3, ball_pos=sent3, ball_vel=inp["prev_vel"][:n], ball_vspin=np.full(n, SENT, f32))


def state_expected(inp, n, mask=None, odd_player=1):
    """(ref, spec): float32 oracle for the exact fields, float64 for racket_normal / ball_vspin; rows whose mask is clear keep their
    values.  odd_player: the player whose grip / bodies the odd envs use in dual mode"""
    ref = {k: v.copy() for k, v in state_before(inp, n).items()}
    ref64 = {}
    for p in ((0, 1) if inp["dual"] else (0,)):
        rows = np.arange(p, n, 2) if inp["dual"] else np.arange(n)
        pl = PLAYERS[odd_player if p else 0]
        args = (inp["rbs"][rows], inp["root"][rows], inp["ball"][rows], inp["prev_vel"][rows], inp["contact"][rows], pl["grip"], pl["racket"],
                pl["wrist"])
        with np.errstate(invalid="ignore"):
            o = V.update_state_from_sim(*args)
            o64 = V.update_state_from_sim(*[a.astype(f64) if a.dtype == f32 else a for a in args[:5]], *args[5:])
        if mask is not None:
            rows = rows[mask[rows]]
            o = {k: v[mask[np.arange(p, n, 2) if inp["dual"] else np.arange(n)]] for k, v in o.items()}
            o64 = {k: v[mask[np.arange(p, n, 2) if inp["dual"] else np.arange(n)]] for k, v in o64.items()}
        for k in ("root_pos", "root_vel", "racket_pos", "racket_vel", "ball_pos", "ball_vel", "ball_vspin"):
            ref[k][rows] = o[k]
        ref["racket_normal"][rows] = o64["racket_normal"]
        ref["ball_vspin"] = ref["ball_vspin"].astype(f64)
        ref["ball_vspin"][rows] = o64["ball_vspin"]
        ref["has_contact"][rows], ref["has_contact_now"][rows] = o["contact"], o["contact_now"]
    ref["has_contact"], ref["has_contact_now"] = ref["has_contact"].copy(), ref["has_contact_now"].copy()
    spec = {k: "exact" for k in ref}
    with np.errstate(invalid="ignore"):
        spec.update(racket_normal=64 * U * np.maximum(1, np.abs(ref["racket_normal"].astype(f64))),
                    ball_vspin=8 * U * np.maximum(1, np.abs(ref["ball_vspin"])))
    return ref, spec


# ------------------------------------------------------------------------------------------------ ball_reset (CPU side)
def make_ball_reset(n, seed, order, stride):
    rng = np.random.default_rng(seed)
    N = 2 * n + 1 if order == "strided" else n + n // 2 + 1
    ids = {"ascending": lambda: np.sort(rng.choice(N, n, replace=False)), "descending": lambda: np.sort(rng.choice(N, n, replace=False))[::-1],
           "strided": lambda: np.arange(n) * 2 + 1, "permuted": lambda: rng.permutation(N)[:n]}[order]()
    P = 257
    pool = rng.uniform(-20, 20, (P, 307)).astype(f32)
    pool[:, 6] = rng.uniform(-10, 10, P)
    pool[[0, 100], 3:5] = 0                                     # vertical launches: v x (0, 0, -1) = 0, normalise clamps at 1e-12
    pidx = rng.integers(0, P, n)
    pidx[: min(n, 3)] = (0, P - 1, 100)[: min(n, 3)]
    g = lambda *s: rng.normal(size=s).astype(f32)  # noqa: E731
    before = dict(ball=np.full((N, stride), SENT, f32), ball_pos=g(N, 3), ball_vel=g(N, 3), has_bounce=rng.random(N) < 0.5,
                  bounce_pos=g(N, 3), has_contact=rng.random(N) < 0.5, traj=g(N, 100, 3))
    before["ball"][:, stride - 13:] = g(N, 13)
    return dict(ids=ids.astype(np.int64), pidx=pidx.astype(np.int64), pool=pool, stride=stride, before=before)


def ball_reset_expected(inp):
    ref = {k: v.copy() for k, v in inp["before"].items()}
    ids, o = inp["ids"], inp["stride"] - 13
    traj, pos, vel, w = V.ball_reset(inp["pool"], inp["pidx"])
    ref["ball"][ids, o:o + 3], ref["ball"][ids, o + 7:o + 10], ref["ball"][ids, o + 10:o + 13] = pos, vel, w
    ref["ball_pos"][ids], ref["ball_vel"][ids], ref["bounce_pos"][ids], ref["traj"][ids] = pos, vel, 0, traj
    ref["has_bounce"][ids], ref["has_contact"][ids] = False, False
    return ref


# ------------------------------------------------------------------------------------------------ ball_in_estimate (CPU side)
class RowTable:
    """incoming-ball table whose row r holds distances 1..50 and heights r: the selected row is traj[:, k, 2]"""
    def __init__(self, rows, shift=0):
        self.rows, self.shift = rows, shift      # shift: the negative control reads the row next to the selected one

    def __getitem__(self, r):
        r = np.asarray(r) + self.shift
        out = np.empty(r.shape + (50, 2), f32)
        out[..., 0] = np.arange(1, 51, dtype=f32)
        out[..., 1] = r[..., None]
        return out


def in_rows(params):
    return int(np.prod([round((hi - lo) / st) for lo, hi, st in params]))


def axis_value(axis, x):
    """float32 value the estimator rounds on `axis` when the ball carries x in the field the case sets (vel_x: b8 with b7 = 0; vspin:
    w = (0, 0, x))"""
    x = f32(x)
    if axis == 1:
        return np.sqrt(f32(x * x))
    if axis == 3:
        return f32(np.sqrt(f32(x * x)) / f32(2 * np.pi))
    return x


def in_index(v, lo, hi, st):
    """in_round with CUDA's fminf / fmaxf (a NaN clamps to lo), float32"""
    with np.errstate(invalid="ignore"):
        c = np.fmin(np.fmax(np.asarray(v, f32), f32(lo)), f32(hi - st))
        return np.rint(f32(c - f32(lo)) / f32(st)).astype(f32)


def tie_cases(params, axis, count=2):
    """inputs x whose float32 (axis_value(x) - lo) / step is exactly k + 0.5 (half-even ties), searched over +-200 ulps of the edge"""
    lo, hi, st = (float(v) for v in params[axis])
    out = []
    for k in range(int(round((hi - lo) / st)) - 1):
        x0 = (lo + (k + 0.5) * st) * (2 * np.pi if axis == 3 else 1)
        for j in range(401):
            x = nxt(x0, INF if j % 2 else -INF, (j + 1) // 2)
            if f32(f32(axis_value(axis, x) - f32(lo)) / f32(st)) == f32(k + 0.5):
                out.append((k, x))
                break
        if len(out) >= count:
            break
    return out


def set_axis(b, axis, x):
    if axis == 0:
        b[2] = x
    elif axis == 1:
        b[7], b[8] = 0, x
    elif axis == 2:
        b[9] = x
    else:
        b[10:13] = (0, 0, x)


def make_in(n, seed, params, stride):
    rng = np.random.default_rng(seed)
    N = n + 5
    (h0, h1, _), (x0, x1, _), (y0, y1, _), (s0, s1, _) = params
    b = np.zeros((N, stride), f32)
    b[:, :13] = rng.normal(size=(N, 13))
    vx = rng.uniform(x0 - 0.3, x1 + 0.3, N)
    ang = rng.uniform(0, 2 * np.pi, N)
    b[:, 2], b[:, 7], b[:, 8], b[:, 9] = rng.uniform(h0 - 0.2, h1 + 0.2, N), vx * np.cos(ang), vx * np.sin(ang), rng.uniform(y0 - 0.3, y1 + 0.3, N)
    w = rng.normal(size=(N, 3))
    b[:, 10:13] = w / np.linalg.norm(w, axis=-1, keepdims=True) * rng.uniform(s0 - 0.3, s1 + 0.3, (N, 1)) * 2 * np.pi
    ids = rng.permutation(N)[:n]
    cases, bad = [], set()
    for axis in range(4):
        lo, hi, st = (float(v) for v in params[axis])
        for k, x in tie_cases(params, axis):
            for dx in (0, -1, 1):
                cases.append((f"axis {axis} tie {k} {dx:+d} ulp", lambda e, a=axis, x=nxt(x, INF if dx > 0 else -INF) if dx else x: set_axis(b[e], a, x)))
        scale = 2 * np.pi if axis == 3 else 1
        for name, x in (("lo - 1", (lo - 1) * scale), ("lo", lo * scale), ("hi - step", (hi - st) * scale), ("hi", hi * scale), ("hi + 1", (hi + 1) * scale)):
            cases.append((f"axis {axis} {name}", lambda e, a=axis, x=f32(x): set_axis(b[e], a, x)))
    grid = np.asarray(params[1:], f64)
    for kw in fma_cases(rng, "vel_x", 3, grid) + fma_cases(rng, "vspin", 3, grid):
        def fma(e, kw=kw):
            if "w" in kw:
                b[e, 10:13] = kw["w"]
            else:
                b[e, 7], b[e, 8] = kw["b7"], kw["b8"]
        cases.append((f"fma {sorted(kw)}", fma))
    cases.append(("v_xy = 0", lambda e: b[e, 7:9].__setitem__(slice(None), 0)))
    for col in (2, 7, 8, 9, 10, 12):
        for v in (np.nan, np.inf, -np.inf):
            cases.append((f"non-finite b[{col}] = {v}", lambda e, col=col, v=v: b[e].__setitem__(col, v)))
    perm = rng.permutation(n)
    where = {}
    for k, (name, fn) in enumerate(cases[:n]):
        fn(int(ids[perm[k]]))
        where[int(perm[k])] = name
        if name.startswith("non-finite"):
            bad.add(int(perm[k]))
    if n > len(cases) + 4:     # repeated contact ids, after the case rows
        free = perm[len(cases):]
        ids[free[:3]] = ids[free[3]]
    return dict(b=b, ids=ids.astype(np.int64), params=params, stride=stride, where=where, nonfinite=np.array(sorted(bad), np.int64))


def in_expected_row(b, params):
    """the row the kernel selects, with CUDA's NaN-dropping clamps, clamped into the table"""
    with np.errstate(invalid="ignore", over="ignore"):
        vel_x = np.sqrt(f32(f32(b[:, 7] * b[:, 7]) + f32(b[:, 8] * b[:, 8])))
        vs = f32(np.sqrt(f32(f32(f32(b[:, 10] * b[:, 10]) + f32(b[:, 11] * b[:, 11])) + f32(b[:, 12] * b[:, 12]))) / f32(2 * np.pi))
    r = [in_index(v, *(float(x) for x in params[k])) for k, v in enumerate((b[:, 2], vel_x, b[:, 9], vs))]
    dim = [f32((float(hi) - float(lo)) / float(st)) for lo, hi, st in params]
    fi = f32(f32(f32(f32(f32(f32(r[0] * dim[1]) * dim[2]) * dim[3]) + f32(f32(r[1] * dim[2]) * dim[3])) + f32(r[2] * dim[3])) + r[3])
    return np.clip(fi.astype(np.int64), 0, in_rows(params) - 1)


def in_expected(inp, n, row_shift=0):
    bs = inp["b"][inp["ids"][:n], :13]
    table = RowTable(in_rows(inp["params"]), row_shift)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        tt, s_in, s_out = V.in_estimator_estimate(bs, table, inp["params"])
    return dict(traj=tt, s_in=s_in, s_out=s_out)


# ------------------------------------------------------------------------------------------------ ball_aero (CPU side)
THR = {s: f32(V.BALL_R * (6 if s > 2 else 4)) for s in (1, 2, 3, 6)}


def make_aero(n, seed, stride):
    rng = np.random.default_rng(seed)
    b = np.full((n, stride), SENT, f32)
    b[:, :13] = rng.normal(size=(n, 13))
    b[:, 2], b[:, 7:10], b[:, 10:13] = rng.uniform(0, 1, n), rng.normal(0, 10, (n, 3)), rng.normal(0, 30, (n, 3))
    inp = dict(b=b, has_bounce=rng.random(n) < 0.3, now=rng.random(n) < 0.3, bounce_pos=rng.normal(size=(n, 3)).astype(f32))
    cases = []
    for s in (4, 6):
        for k in (0, -1, 1):
            def z(e, s=s, k=k):
                t = f32(V.BALL_R * s)
                b[e, 2] = nxt(t, INF if k > 0 else -INF) if k else t
                inp["has_bounce"][e] = False
            cases.append((f"z = {s}R {k:+d} ulp", z))
    cases.append(("has_bounce set, z = 0", lambda e: (b[e].__setitem__(2, 0), inp["has_bounce"].__setitem__(e, True))))
    cases.append(("at rest", lambda e: b[e, 7:10].__setitem__(slice(None), 0)))
    cases.append(("zero spin", lambda e: b[e, 10:13].__setitem__(slice(None), 0)))
    cases.append(("at rest, zero spin", lambda e: b[e, 7:13].__setitem__(slice(None), 0)))
    inp["where"] = place(n, cases, rng)
    return inp


def aero_expected(inp, n, substeps, spin):
    b = inp["b"][:n, :13]
    _, hb, now = V.ball_aero(b, inp["has_bounce"][:n], substeps, spin)
    with np.errstate(invalid="ignore", divide="ignore"):
        force = V.ball_aero(b.astype(f64), inp["has_bounce"][:n], substeps, spin)[0]
    ref = dict(force=force, has_bounce=hb, has_bounce_now=inp["now"][:n] | now,
               bounce_pos=np.where(now[:, None], b[:, :3], inp["bounce_pos"][:n]))
    vs2 = (b[:, 7:10].astype(f64) ** 2).sum(-1)
    spec = dict(force=np.repeat((32 * U * V.KF * (V.BASE_CD + 0.5) * vs2)[:, None], 3, 1), has_bounce="exact", has_bounce_now="exact",
                bounce_pos="exact")
    return ref, spec


# ------------------------------------------------------------------------------------------------ CPU: constructors, controls, refusals
def test_case_constructors_lie_on_their_branches_and_thresholds():
    """every constructed case is where its name says, checked in float64"""
    branches = {quat_branch(m)[0] for _, m in SPECIAL_ROTS}
    assert branches == {0, 1, 2, 3}, branches
    assert any(quat_branch(m)[1] < 0 and quat_branch(m)[0] > 0 for _, m in SPECIAL_ROTS)       # the c < 0 branch of the angle-axis
    for name, m in SPECIAL_ROTS:
        assert abs(np.linalg.det(m.astype(f64)) - 1) < 1e-6 and np.abs(m.astype(f64) @ m.T.astype(f64) - np.eye(3)).max() < 1e-6, name
    assert quat_branch(SPECIAL_ROTS[6][1])[0] == 3 and np.trace(SPECIAL_ROTS[6][1]) == 0
    inp = make_smpl(300, 3, 5)
    env = {v: k for k, v in inp["where"].items()}
    for name in ("near pi", "near pi, sign flip"):
        e = env[name]
        cur = fk_quat64(inp, e)
        d = V.quat_mul_norm(R.quat_conjugate(inp["prev_rot"][e].astype(f64)), cur)
        ang = 2 * np.arccos(np.clip(d[:, 3], -1, 1))
        assert np.all((ang > np.pi - 2e-3) & (ang < np.pi)), (name, ang)
        if "flip" in name:
            assert np.all(R.quat_mul(R.quat_conjugate(inp["prev_rot"][e].astype(f64)), cur)[:, 3] < 0)   # quat_pos has to flip it
    # fix_head
    h = make_head(300, 6)
    env = {v: k for k, v in h["where"].items()}
    for k, want in ((0, False), (-1, True), (1, False)):
        e = env[f"ball_y = root_y - 0.5 {k:+d} ulp"]
        assert f32(h["root"][e, 1] - f32(0.5)) == f64(h["root"][e, 1]) - 0.5
        assert (f64(h["ball"][e, 1]) < f64(h["root"][e, 1]) - 0.5) == want
    for x in (4, -4):
        for k, want in ((0, False), (-1, x < 0), (1, x > 0)):
            assert (abs(f64(h["ball"][env[f"ball_x {f32(x)} {k:+d} ulp"], 0])) > 4) == want
    d, ln, bn = yaw_error(h["rb_rot"][:, 13], h["rb_pos"][:, 13], h["ball"])
    assert d[env["wrap -2 pi"]] < -np.pi - 0.1 and d[env["wrap +2 pi"]] > np.pi + 0.1
    assert ln[env["head up (identity)"]] == 0 and ln[env["head up (yaw only)"]] < 1e-7 and bn[env["ball above head"]] == 0
    for name, corrected in (("taylor, miss", False), ("taylor, corrected", True)):
        e = env[name]
        dd = 0.0 if not corrected else np.arctan2(*(h["ball"][e, 1::-1] - h["rb_pos"][e, 13, 1::-1]).astype(f64))
        aa = V.rotation_matrix_to_angle_axis(h["rot"][e, [15, 12]].astype(f64))
        aa[:, 1] += dd / 2
        th2 = (aa ** 2).sum(-1)
        assert np.all(th2 < 0.5e-6), (name, th2)
    far = np.array([e for e in range(300) if e not in h["where"]])
    assert np.all(np.abs(np.abs(d[far]) - np.pi) >= 1e-3)
    # update_state detector
    s = make_state(300, 7)
    env = {v: k for k, v in s["where"].items()}
    for name, jump in (("jump = 10", 0), ("jump = 10 + ulp", 1), ("jump = 10 - ulp", -1)):
        e = env[name]
        diff = f64(s["ball"][e, 8]) - f64(s["prev_vel"][e, 1])
        assert np.sign(diff - 10) == jump and f32(s["ball"][e, 8] - s["prev_vel"][e, 1]) == f32(diff)
    # estimator ties and the aero thresholds
    for params in (IN_COARSE, IN_SHIPPED):
        for axis in range(4):
            ties = tie_cases(params, axis)
            assert ties, (axis, params[axis])
            for k, x in ties:
                assert in_index(axis_value(axis, x), *(float(v) for v in params[axis])) == (k if k % 2 == 0 else k + 1)
    assert THR[2] == f32(f32(0.032) * f32(4)) and THR[3] == f32(f32(0.032) * f32(6))


def test_comparators_reject_mutated_oracles():
    """a plausible kernel bug in each comparator's oracle is caught and named by env and field"""
    def rejects(fails, field, env=None):
        assert any(x.startswith(field + ":") and (env is None or f"env {env}:" in x) for x in fails), (field, env, fails[:6])
    # per-shape rest from e % 1 instead of e % K
    inp = make_smpl(40, 3, 1)
    ref, spec = smpl_expected(inp, 40, "fused")
    bad, _ = smpl_expected(inp, 40, "fused", rest_of=lambda e, K: e % 1)
    rejects(compare(ref, bad, {k: spec[k] for k in ("rb_pos",)}, limit=None), "rb_pos", 1)
    # root_ang_vel divided by dt once
    bad, _ = smpl_expected(inp, 40, "fused", ang_div_dt=1)
    rejects(compare(ref, bad, {"root_ang_vel": spec["root_ang_vel"]}), "root_ang_vel", 0)
    # odd envs given the even player's grip
    s = make_state(40, 2, dual=True)
    ref, spec = state_expected(s, 40)
    bad, _ = state_expected(s, 40, odd_player=0)
    rejects(compare(ref, bad, spec, limit=None), "racket_normal", 1)
    # a masked-out row written
    mask = np.arange(40) % 3 == 0
    ref, spec = state_expected(s, 40, mask=mask)
    bad, _ = state_expected(s, 40)
    rejects(compare(ref, bad, spec, limit=None), "root_pos", 1)
    # a table row off by one
    inp = make_in(64, 3, IN_COARSE, 13)
    fin = np.setdiff1d(np.arange(64), inp["nonfinite"])
    ref = in_expected(inp, 64)
    bad = in_expected(inp, 64, row_shift=1)
    rejects(compare(ref, bad, {"traj": "exact"}, rows=fin, limit=None), "traj", int(fin[0]))


def test_descriptor_entry_points_refuse_bad_arguments():
    """update_state (n < 0, strides below 13, racket / wrist bodies of either player outside [0, bodies_per_env)), ball_reset (stride
    below 13) and ball_in_estimate (stride below 13, a grid step <= 0 or NaN) refuse before any launch: fake, never dereferenced
    pointers reach every rule on a machine without a GPU"""
    from vid2player3d_b200 import abi
    from vid2player3d_b200.native import lib
    L = lib()
    L.b200v2p_last_error.restype = C.c_char_p

    def state(**kw):
        s = abi.V2PState()
        base = dict(n=8, bodies_per_env=26, ball_stride=26, root_stride=26, racket_body=24, wrist_body=22, dual=0, racket_body2=23, wrist_body2=17)
        base.update(kw)
        for k, v in base.items():
            setattr(s, k, v)
        for k in ("rigid_body_state", "root_states", "ball_states", "has_contact", "has_contact_now", "root_pos", "root_vel", "racket_pos",
                  "racket_vel", "racket_normal", "ball_pos", "ball_vel", "ball_vspin"):
            setattr(s, k, 256)
        return L.b200v2p_update_state(C.byref(s), None), L.b200v2p_last_error().decode()
    for kw, rc_want, msg in ((dict(n=-1), -1, "bad arguments"), (dict(ball_stride=12), -1, "bad arguments"), (dict(root_stride=12), -1, "bad arguments"),
                             (dict(racket_body=26), -2, "racket and wrist"), (dict(racket_body=-1), -2, "racket and wrist"),
                             (dict(wrist_body=26), -2, "racket and wrist"), (dict(dual=1, racket_body2=26), -2, "racket and wrist"),
                             (dict(dual=1, wrist_body2=-1), -2, "racket and wrist"), (dict(bodies_per_env=24), -2, "racket and wrist")):
        rc, err = state(**kw)
        assert rc == rc_want and msg in err and "update_state" in err, (kw, rc, err)
    fake = lambda S, **kw: S(**kw, **{f: 256 for f, ct in S._fields_ if issubclass(ct, C.c_void_p)})  # noqa: E731
    rc = L.b200v2p_ball_reset(C.byref(fake(abi.V2PBallReset, n=4, stride=12)), None)
    assert rc == -1 and "ball_reset" in L.b200v2p_last_error().decode()
    good = [float(v) for v in IN_COARSE.reshape(-1)]

    def est(stride, params):
        rc = L.b200v2p_ball_in_estimate(C.byref(fake(abi.V2PInEst, n=4, stride=stride, table_rows=160, params=(C.c_double * 12)(*params))), None)
        return rc, L.b200v2p_last_error().decode()
    rc, err = est(12, good)
    assert rc == -1 and "ball_in_estimate" in err
    for axis in range(4):
        for step in (0.0, -0.1, float("nan")):
            bad = list(good)
            bad[axis * 3 + 2] = step
            rc, err = est(13, bad)
            assert rc == -2 and "grid steps must be positive" in err, (axis, step, rc, err)


# ------------------------------------------------------------------------------------------------ GPU runners
def _full(shape, fill=SENT, dtype=None):
    import torch
    if dtype is torch.bool:
        return torch.full(shape, bool(fill), dtype=torch.bool, device=DEV)
    return torch.full(shape, float(fill), device=DEV)


def run_smpl(inp, n, mode, mask=None):
    """one b200v2p_smpl_to_sim launch; mode 'fresh' (no prev_*), 'fused' (prev_root_pos_update aliases prev_root_pos, target set) or
    'separate' (its own update buffer, no target); -> every buffer (n + SLACK rows) as numpy"""
    import torch
    from vid2player3d_b200 import native_v2p as NV
    _, par, s2m = skeleton()
    out = {k: _full((n + SLACK,) + s) for k, s in SM_OUT.items()}
    kw = {}
    if mode != "fresh":
        prev = _dev(_pad(inp["prev_root"][:n], SENT))
        kw = dict(prev_root_pos=prev, prev_rb_rot=_dev(inp["prev_rot"][:n]),
                  prev_root_pos_update=prev if mode == "fused" else _full((n + SLACK, 3)),
                  target_root_pos_out=_full((n + SLACK, 3)) if mode == "fused" else None)
    NV.smpl_to_sim(_dev(inp["root"][:n]), _dev(inp["rot"][:n]), _dev(inp["rest"]), _dev(par), _dev(s2m), DT, out,
                   only_mask=None if mask is None else _dev(mask[:n]), **kw)
    torch.cuda.synchronize()
    got = {k: v.cpu().numpy() for k, v in out.items()}
    for k in ("prev_root_pos", "prev_root_pos_update", "target_root_pos_out"):
        if kw.get(k) is not None:
            got[k] = kw[k].cpu().numpy()
    return got


def check_smpl(inp, n, mode, label):
    got = run_smpl(inp, n, mode)
    for k, v in got.items():
        want = _pad(inp["prev_root"][:n], SENT) if (k == "prev_root_pos" and mode == "separate") else None
        if want is not None:
            assert np.array_equal(v, want), f"{label}: prev_root_pos written in separate mode"
        else:
            assert (v[n:] == SENT).all(), f"{label}: {k} written past n"
    ref, spec = smpl_expected(inp, n, mode)
    g = {k: v[:n] for k, v in got.items()}
    g["rb_rot"] = align_sign(g["rb_rot"], ref)
    if mode != "fresh":
        spec.update(prev_root_pos_update="exact", **({"target_root_pos_out": "exact"} if mode == "fused" else {}))
    fails = compare(ref, g, spec, tag="smpl_to_sim.")
    assert not fails, f"{label}: " + "; ".join(fails[:6])
    env = {v: k for k, v in inp["where"].items()}
    if "identity env" in env and mode != "fresh":
        e = env["identity env"]
        assert (g["dof_vel"][e] == 0).all() and (g["root_ang_vel"][e] == 0).all(), f"{label}: prev == cur did not take the st <= 1e-5 branch"
    return got


# ------------------------------------------------------------------------------------------------ GPU: smpl_to_sim
@pytest.mark.gpu
def test_smpl_to_sim_sizes_modes_and_rotation_edges():
    """every size x (fresh, fused, separate) with 1, 2 or 3 rest skeletons (K = 3 leaves n % K != 0 at the tail), the branch cases of
    rotmat_to_quat_wxyz at the root and at a child joint, prev == cur, a frame-to-frame rotation just under pi with and without a sign
    flip (quat_pos)"""
    for j, n in enumerate(SIZES):
        for i, mode in enumerate(("fresh", "fused", "separate")):
            K = 1 + (j + i) % 3
            check_smpl(make_smpl(n, K, 10 * n + i), n, mode, f"n = {n} {mode} K = {K}")
    for K in (1, 2, 3):
        check_smpl(make_smpl(BIG, K, K), BIG, "fused", f"n = {BIG} K = {K}")


@pytest.mark.gpu
def test_smpl_to_sim_mask_nan_batch_independence_and_determinism():
    """only_mask: masked rows bitwise equal to the unmasked launch, every other row of all nine outputs untouched; a NaN in one env's
    rotations stays in that env; row r of an 8195-env launch equals an (r + 1)-env launch; two launches are equal"""
    inp = make_smpl(BIG, 3, 77)
    for mode in ("fused", "separate", "fresh"):
        full = run_smpl(inp, BIG, mode)
        again = run_smpl(inp, BIG, mode)
        for k in full:
            assert np.array_equal(full[k], again[k], equal_nan=True), f"{mode}: {k} differs between two launches"
        for n in SIZES[:-1]:
            part = run_smpl(inp, n, mode)
            for k in part:
                assert np.array_equal(part[k][:n], full[k][:n], equal_nan=True), f"{mode}: {k} of a {n}-env launch differs from rows of {BIG}"
        rng = np.random.default_rng(5)
        for n in (1, 5, 129, BIG):
            mask = rng.random(n) < 0.4
            mask[n - 1] = True
            masked = run_smpl(inp, n, mode, mask=mask)
            for k in masked:
                keep = ~mask
                assert np.array_equal(masked[k][:n][mask], full[k][:n][mask], equal_nan=True), f"{mode} n = {n}: masked row of {k} differs"
                aliased = k == "prev_root_pos" or (k == "prev_root_pos_update" and mode == "fused")
                before = _pad(inp["prev_root"][:n], SENT) if aliased else np.full_like(masked[k], SENT)
                assert np.array_equal(masked[k][:n][keep], before[:n][keep]), f"{mode} n = {n}: {k} written on a row whose mask is clear"
                assert np.array_equal(masked[k][n:], before[n:]), f"{mode} n = {n}: {k} written past n"
    e = 4097
    bad = dict(inp, rot=inp["rot"].copy())
    bad["rot"][e, 5, 1, 1] = np.nan
    full, nan = run_smpl(inp, BIG, "fused"), run_smpl(bad, BIG, "fused")
    assert np.isnan(nan["rb_pos"][e]).any(), "a NaN rotation did not reach the FK of its descendants"
    for k in full:
        other = np.arange(BIG + SLACK) != e
        assert np.array_equal(full[k][other], nan[k][other], equal_nan=True), f"the NaN of env {e} leaked into another env's {k}"


# ------------------------------------------------------------------------------------------------ GPU: fix_head
def run_head(inp, n):
    import torch
    from vid2player3d_b200 import native_v2p as NV
    rot = _dev(_pad(inp["rot"][:n], SENT))
    NV.fix_head(_dev(inp["rb_pos"][:n]), _dev(inp["rb_rot"][:n]), _dev(inp["ball"][:n]), _dev(inp["root"][:n]), rot, head_body=13)
    torch.cuda.synchronize()
    return rot.cpu().numpy()


@pytest.mark.gpu
def test_fix_head_sizes_thresholds_wrap_and_clamps():
    """the miss tests exactly on ball_y = root_y - 0.5 and |ball_x| = 4 and one ulp to either side, the +-2 pi wrap both ways, a head
    looking straight up and a ball directly above it (the 1e-12 clamps), the Taylor branch of aa_to_rotmat with and without a correction;
    joints other than Head and Neck, and rows past n, bit-identical; batch independence and determinism at 8195"""
    for n in SIZES:
        inp = make_head(n, 3 * n)
        got = run_head(inp, n)
        assert (got[n:] == SENT).all(), f"n = {n}: written past n"
        ref, bound = head_expected(inp, n)
        other = np.ones(24, bool)
        other[[12, 15]] = False
        assert np.array_equal(got[:n, other], inp["rot"][:n, other]), f"n = {n}: a joint other than Head / Neck was written"
        fails = compare({"joint_rotmat": ref}, {"joint_rotmat": got[:n]}, {"joint_rotmat": bound}, tag="fix_head.")
        assert not fails, f"n = {n}: " + "; ".join(fails[:6])
        env = {v: k for k, v in inp["where"].items()}
        for name in ("ball_y = root_y - 0.5 -1 ulp", f"ball_x {f32(4)} +1 ulp", f"ball_x {f32(-4)} -1 ulp", "taylor, miss"):
            if name in env:     # a miss leaves the rotation as the round trip matrix -> angle-axis -> matrix gives it
                e = env[name]
                want = V.angle_axis_to_rotation_matrix(V.rotation_matrix_to_angle_axis(inp["rot"][e, [15, 12]].astype(f64)))
                assert np.abs(got[e, [15, 12]] - want).max() <= 1040 * U, name
    inp = make_head(BIG, 1)
    full, again = run_head(inp, BIG), run_head(inp, BIG)
    assert np.array_equal(full, again)
    for n in SIZES[:-1]:
        assert np.array_equal(run_head(inp, n)[:n], full[:n]), f"a {n}-env launch differs from the rows of {BIG}"


# ------------------------------------------------------------------------------------------------ GPU: update_state
def run_state(inp, n, mask=None):
    import torch
    from vid2player3d_b200 import native_v2p as NV
    before = state_before(inp, n)
    t = {k: _dev(_pad(v, True if v.dtype == bool else SENT)) for k, v in before.items()}
    dual = inp["dual"]
    pick = lambda key: [PLAYERS[0][key], PLAYERS[1][key]] if dual else PLAYERS[0][key]  # noqa: E731
    NV.update_state(n, 26, _dev(inp["rbs"][:n]), _dev(_pad(inp["root"][:n], SENT)), inp["root"].shape[1], _dev(_pad(inp["ball"][:n], SENT)),
                    inp["ball"].shape[1], t, grip=pick("grip"), racket_body=pick("racket"), wrist_body=pick("wrist"),
                    only_mask=None if mask is None else _dev(mask[:n]))
    torch.cuda.synchronize()
    got = {k: v.cpu().numpy() for k, v in t.items()}
    for k, v in got.items():
        assert (v[n:] == (True if v.dtype == bool else SENT)).all(), f"n = {n}: {k} written past n"
    return {k: v[:n] for k, v in got.items()}


@pytest.mark.gpu
def test_update_state_sizes_strides_dual_and_mask():
    """ball / root strides 13 and 26; dual mode with another grip, wrist and racket for odd envs (odd n: the last env is an even one);
    the detector at ball[8] = 0 and at a jump of exactly 10 and one ulp to either side, has_contact already set; a zero wrist
    quaternion (identity matrix: the normal is the grip) and a NaN one (a NaN normal); only_mask; batch independence and determinism"""
    for j, n in enumerate(SIZES):
        for bs, rs in ((13, 13), (26, 26), (26, 13)):
            for dual in (False, True):
                inp = make_state(n, n + bs + 2 * rs + dual, bs, rs, dual)
                got = run_state(inp, n)
                ref, spec = state_expected(inp, n)
                fails = compare(ref, got, spec, tag="update_state.")
                assert not fails, f"n = {n} strides {bs}/{rs} dual {dual}: " + "; ".join(fails[:6])
                env = {v: k for k, v in inp["where"].items()}
                if "zero wrist quaternion" in env:
                    e = env["zero wrist quaternion"]
                    grip = V.GRIP_NORMAL[PLAYERS[int(dual and e % 2)]["grip"]]
                    assert np.array_equal(got["racket_normal"][e], np.asarray(grip, f32)), "zero quaternion: normal != grip"
                if "nan wrist quaternion" in env:
                    assert np.isnan(got["racket_normal"][env["nan wrist quaternion"]]).all()
                if j % 4 == 0 or n == BIG:
                    mask = np.random.default_rng(n).random(n) < 0.5
                    gm = run_state(inp, n, mask)
                    ref_m, spec_m = state_expected(inp, n, mask=mask)
                    fails = compare(ref_m, gm, {k: "exact" for k in spec_m}, rows=np.flatnonzero(~mask))
                    fails += compare(got, gm, {k: "exact" for k in spec_m}, rows=np.flatnonzero(mask))
                    assert not fails, f"n = {n} masked: " + "; ".join(fails[:6])
    for dual in (False, True):
        inp = make_state(BIG, 9, 26, 26, dual)
        full, again = run_state(inp, BIG), run_state(inp, BIG)
        assert not compare(full, again, {k: "exact" for k in full})
        for n in SIZES[:-1]:
            part = run_state(inp, n)
            assert not compare({k: v[:n] for k, v in full.items()}, part, {k: "exact" for k in full}), f"dual {dual}: {n}-env launch"


# ------------------------------------------------------------------------------------------------ GPU: ball_reset
def run_ball_reset(inp, n=None):
    import torch
    from vid2player3d_b200 import native_v2p as NV
    n = len(inp["ids"]) if n is None else n
    t = {k: _dev(_pad(v, True if v.dtype == bool else SENT)) for k, v in inp["before"].items()}
    o = inp["stride"] - 13
    NV.ball_reset(_dev(inp["ids"][:n]), _dev(inp["pidx"][:n]), _dev(inp["pool"]), t["ball"].view(-1)[o:], t["ball_pos"], t["ball_vel"],
                  t["has_bounce"], t["bounce_pos"], t["has_contact"], t["traj"], stride=inp["stride"])
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in t.items()}


@pytest.mark.gpu
def test_ball_reset_id_orders_pool_edges_and_stride():
    """ascending, descending, strided and permuted id lists; pool_index at the first and last pool row; stride 13 and 26 (the ball is
    actor 1 of 2); vertical launches (zero spin through the normalise clamp).  All seven outputs are exact, and every env missing from the
    list, the humanoid half of a 26-float row and the slack rows stay bit-identical"""
    for j, n in enumerate(SIZES):
        for order in ("ascending", "descending", "strided", "permuted"):
            inp = make_ball_reset(n, n * 5 + j, order, (13, 26)[(j + len(order)) % 2])
            got = run_ball_reset(inp)
            ref = ball_reset_expected(inp)
            fails = compare({k: _pad(v, True if v.dtype == bool else SENT) for k, v in ref.items()}, got, {k: "exact" for k in ref})
            assert not fails, f"n = {n} {order} stride {inp['stride']}: " + "; ".join(fails[:6])
            vert = inp["ids"][inp["pidx"] == 0]
            o = inp["stride"] - 13
            assert (got["ball"][vert, o + 10:o + 13] == 0).all()
    inp = make_ball_reset(BIG, 1, "permuted", 26)
    full, again = run_ball_reset(inp), run_ball_reset(inp)
    assert all(np.array_equal(full[k], again[k]) for k in full)
    for n in SIZES[:-1]:      # the first n ids: their rows equal the full launch, the rest untouched
        part = run_ball_reset(inp, n)
        ids = inp["ids"][:n]
        for k in full:
            assert np.array_equal(part[k][ids], full[k][ids]), (n, k)


# ------------------------------------------------------------------------------------------------ GPU: ball_in_estimate
def in_table_dev(params):
    import torch
    rows = in_rows(params)
    t = torch.empty(rows, 50, 2, device=DEV)
    t[:, :, 0] = torch.arange(1, 51, device=DEV, dtype=torch.float32)
    t[:, :, 1] = torch.arange(rows, device=DEV, dtype=torch.float32)[:, None]
    return t


def run_in(inp, n, table):
    import torch
    from vid2player3d_b200 import native_v2p as NV
    traj, s_in, s_out = _full((n + SLACK, 50, 3)), _full((n + SLACK, 13)), _full((n + SLACK, 13))
    NV.ball_in_estimate(_dev(inp["ids"][:n]), _dev(inp["b"]), inp["stride"], table, inp["params"], traj[:n], s_in[:n], s_out[:n])
    torch.cuda.synchronize()
    got = dict(traj=traj.cpu().numpy(), s_in=s_in.cpu().numpy(), s_out=s_out.cpu().numpy())
    for k, v in got.items():
        assert (v[n:] == SENT).all(), f"n = {n}: {k} written past n"
    return {k: v[:n] for k, v in got.items()}


@pytest.mark.gpu
def test_ball_in_estimate_rows_ties_and_non_finite_states():
    """a table whose row r encodes r, on the golden coarse grid and the shipped 15 x 50 x 30 x 50 grid: half-even ties on all four
    axes and one ulp beside them, values below lo and at / above hi - step, fma-sensitive vel_x and vspin, unsorted and repeated contact
    ids, stride 13 and 26, v_xy = 0 (a NaN direction on both sides) - all exact against the float32 oracle, the selected row included.
    Non-finite ball states (the masked dual reset passes them for unused rows): the oracle would index the table with a garbage row
    (numpy's cast of a NaN) and the reference would raise; the kernel's defined behaviour is pinned instead - fminf / fmaxf drop a NaN
    to lo, +-Inf clamps to an end, and the row computed here from those clamps lies inside the table and is the one selected.
    The v_xy = 0 case caught the kernel writing the z of omega as a literal 0 in both snapped states, where the reference's normalize
    of a NaN direction gives NaN; the kernel now keeps the NaN through its 1e-12 clamp."""
    for params in (IN_COARSE, IN_SHIPPED):
        table = in_table_dev(params)
        rows = in_rows(params)
        for j, n in enumerate(SIZES):
            inp = make_in(n, n + rows % 97, params, (13, 26)[j % 2])
            got = run_in(inp, n, table)
            ref = in_expected(inp, n)
            fin = np.setdiff1d(np.arange(n), inp["nonfinite"])
            fails = compare(ref, got, {k: "exact" for k in ref}, rows=fin)
            assert not fails, f"n = {n} rows {rows}: " + "; ".join(fails[:6])
            want = in_expected_row(inp["b"][inp["ids"][:n], :13], params)
            assert np.array_equal(got["traj"][:, 0, 2].astype(np.int64), want), f"n = {n}: selected row differs from the defined clamps"
            assert ((want >= 0) & (want < rows)).all()
            assert np.array_equal(got["traj"][:, :, 2], np.repeat(want[:, None], 50, 1).astype(f32))
        inp = make_in(BIG, 2, params, 26)
        full, again = run_in(inp, BIG, table), run_in(inp, BIG, table)
        assert all(np.array_equal(full[k], again[k], equal_nan=True) for k in full)
        for n in SIZES[:-1]:
            part = run_in(inp, n, table)
            assert all(np.array_equal(part[k], full[k][:n], equal_nan=True) for k in full), f"a {n}-env launch differs"
        del table


# ------------------------------------------------------------------------------------------------ GPU: ball_aero
def run_aero(inp, n, substeps, spin):
    import torch
    from vid2player3d_b200 import native_v2p as NV
    hb, now = _dev(_pad(inp["has_bounce"][:n], True)), _dev(_pad(inp["now"][:n], True))
    bp, force = _dev(_pad(inp["bounce_pos"][:n], SENT)), _full((n + SLACK, 3))
    NV.ball_aero(_dev(inp["b"][:n]).view(-1), hb[:n], now[:n], bp[:n], force[:n], substeps, spin, stride=inp["b"].shape[1])
    torch.cuda.synchronize()
    got = dict(has_bounce=hb.cpu().numpy(), has_bounce_now=now.cpu().numpy(), bounce_pos=bp.cpu().numpy(), force=force.cpu().numpy())
    for k, v in got.items():
        assert (v[n:] == (True if v.dtype == bool else SENT)).all(), f"n = {n}: {k} written past n"
    return {k: v[:n] for k, v in got.items()}


@pytest.mark.gpu
def test_ball_aero_thresholds_substeps_and_stride():
    """z exactly at the 4R and 6R thresholds and one ulp beside, substeps 1, 2, 3 and 6; has_bounce already set; a ball at rest and zero
    spin; stride 13 and 26.  Flags and bounce_pos exact (has_bounce_now and has_bounce are |=, as in the reference), force bounded"""
    for j, n in enumerate(SIZES):
        for substeps in (1, 2, 3, 6):
            inp = make_aero(n, n * 7 + substeps, (13, 26)[(j + substeps) % 2])
            got = run_aero(inp, n, substeps, (1.0, 5.0)[j % 2])
            ref, spec = aero_expected(inp, n, substeps, (1.0, 5.0)[j % 2])
            fails = compare(ref, got, spec, tag="ball_aero.")
            assert not fails, f"n = {n} substeps {substeps}: " + "; ".join(fails[:6])
            env = {v: k for k, v in inp["where"].items()}
            R_ = 6 if substeps > 2 else 4
            for k, hit in ((0, True), (-1, True), (1, False)):
                if f"z = {R_}R {k:+d} ulp" in env:
                    assert bool(got["has_bounce"][env[f"z = {R_}R {k:+d} ulp"]]) == hit
    inp = make_aero(BIG, 3, 26)
    full, again = run_aero(inp, BIG, 6, 1.0), run_aero(inp, BIG, 6, 1.0)
    assert all(np.array_equal(full[k], again[k]) for k in full)
    for n in SIZES[:-1]:
        part = run_aero(inp, n, 6, 1.0)
        assert all(np.array_equal(part[k], full[k][:n]) for k in full), n


# ------------------------------------------------------------------------------------------------ GPU: refusals and the fused target path
@pytest.mark.gpu
def test_refusals_through_native_v2p():
    import torch
    from vid2player3d_b200 import native_v2p as NV
    n = 4
    t = {k: torch.zeros(n, 3, device=DEV) for k in ("root_pos", "root_vel", "racket_pos", "racket_vel", "racket_normal", "ball_pos", "ball_vel")}
    t.update(has_contact=torch.zeros(n, dtype=torch.bool, device=DEV), has_contact_now=torch.zeros(n, dtype=torch.bool, device=DEV),
             ball_vspin=torch.zeros(n, device=DEV))
    rbs, rows = torch.zeros(n, 26, 13, device=DEV), torch.zeros(n, 26, device=DEV)
    for kw, msg in ((dict(racket_body=26), "racket and wrist"), (dict(wrist_body=[22, 26]), "racket and wrist"),
                    (dict(racket_body=[24, -1]), "racket and wrist")):
        with pytest.raises(RuntimeError, match=msg):
            NV.update_state(n, 26, rbs, rows, 26, rows, 26, t, **kw)
    with pytest.raises(RuntimeError, match="bad arguments"):
        NV.update_state(n, 26, rbs, rows, 12, rows, 26, t)
    ids = torch.arange(n, device=DEV)
    with pytest.raises(RuntimeError, match="ball_reset: bad arguments"):
        NV.ball_reset(ids, ids, torch.zeros(3, 307, device=DEV), rows, t["ball_pos"], t["ball_vel"], t["has_contact"], t["ball_pos"],
                      t["has_contact_now"], torch.zeros(n, 100, 3, device=DEV), stride=12)
    tab, traj, si, so = torch.zeros(160, 50, 2, device=DEV), torch.zeros(n, 50, 3, device=DEV), torch.zeros(n, 13, device=DEV), torch.zeros(n, 13, device=DEV)
    with pytest.raises(RuntimeError, match="ball_in_estimate: bad arguments"):
        NV.ball_in_estimate(ids, rows, 12, tab, IN_COARSE, traj, si, so)
    bad = IN_COARSE.copy()
    bad[3, 2] = 0
    with pytest.raises(RuntimeError, match="grid steps must be positive"):
        NV.ball_in_estimate(ids, rows, 13, tab, bad, traj, si, so)
    torch.cuda.synchronize()
    assert (traj == 0).all() and (t["root_pos"] == 0).all()


@pytest.mark.gpu
def test_fused_target_path_matches_three_step_path():
    """PhysicsMVAEController's targets from the one fused smpl_to_sim launch (prev_root_pos_update aliasing prev_root_pos, the target
    root stored by the kernel) equal the three-step path (FK with a cloned previous rotation, then two copies) bitwise, over ten steps
    and a masked reset"""
    import torch
    from helpers import SIM_PARAMS, v2p_cfg
    from vid2player3d_b200.tasks import PhysicsMVAEController
    N = 64
    names = ("_target_root_pos", "_target_root_rot", "_target_dof_pos", "_target_root_vel", "_target_root_ang_vel", "_target_dof_vel",
             "_target_rb_pos", "_target_rb_rot", "_prev_target_root_pos")
    mask = torch.zeros(N, dtype=torch.bool)
    mask[[1, 7, 30, 63]] = True
    runs = []
    for fast in (True, False):
        torch.manual_seed(3)
        env = PhysicsMVAEController(v2p_cfg(N), SIM_PARAMS, 1, "cuda", 0, True)
        task = env._physics_player.task
        assert task._fast_targets, "the single-player config builds the fused path"
        task._fast_targets = fast
        env.reset()
        gen = torch.Generator().manual_seed(11)
        rec = []
        for i in range(10):
            env.step(torch.clamp(torch.randn(N, env.num_actions, generator=gen), -5, 5).to(DEV))
            if i == 5:
                env._reset_envs_masked(mask.to(DEV))
            torch.cuda.synchronize()
            rec.append({k: getattr(task, k).detach().cpu().numpy().copy() for k in names})
        runs.append(rec)
        del env
    for i, (a, b) in enumerate(zip(*runs)):
        for k in names:
            assert np.array_equal(a[k], b[k], equal_nan=True), f"step {i}: {k} differs between the fused and the three-step path"
