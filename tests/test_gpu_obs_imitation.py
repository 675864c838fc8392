"""The imitation observation launch (obs_imitation_kernel, DESIGN.md row a6) through both entry points - b200env_obs_imitation on
contiguous gathers and b200env_obs_imitation_rows on the Isaac-layout state rows, with the policy's bf16 operand row - against the
numpy oracle (oracle/ref_port.py: compute_humanoid_observations_imitation and _jpos, pinned to the reference by
test_oracle_golden.py), on two handles: HumanoidSMPLIM on amass_v1 (24 bodies) and HumanoidSMPLIMMVAE on federer (25 bodies, welded
racket last, 26 state rows per env).

1. Sizes 1 ... 8195: the ragged last CTA (8 warps, one env each).  The float obs starts as SENT = 12345.0 and the bf16 operand as
   SENT_BF16 = -7.75 (exact in bf16), each with SLACK rows past n; rows past n and operand columns past the row width W stay
   bit-identical.  Row r of an 8195-env launch equals the same row of an (r + 1)-env launch bit for bit, and two launches are equal.
2. Both variants (full, 734 wide; _jpos, 513 wide) under all four (local_root_obs, root_height_obs).  The rows entry equals the
   gathered entry bitwise at bodies_per_env 24, 25 and 26; every state row the launch must not read (past the 24 humanoid bodies:
   racket, ball, padding) holds NaN, so a stride bug shows as NaN.  A float obs one float off 8-byte alignment takes the scalar store
   path and must equal the aligned float2 path bitwise.
3. Exact (==, NaN equal to NaN) against the float32 oracle, fields written by a copy or one subtraction: root_h (+0 when off),
   dof_vel, target_rel_root_h, target_rel_dof_pos, motion_bodies.
4. Exact invariances: negating any body or target quaternion leaves the row unchanged (every use is quadratic in q or a product whose
   sign cancels, and round-to-nearest is symmetric) - bitwise, except that an exact zero may change sign; root_height_obs changes
   column 0 only; local_root_obs changes the root tan-norm slot only; the _jpos row's columns up to the end of dof_vel, its
   target_rel_root_h / target_rel_2d_pos and its target_rel_body_pos block equal the full row's.
5. Bounded against float64 on the same float32 inputs, u = 2^-24, bounds absolute per component:
   - The heading.  The de-based root r = q (x) conj(base) is a 4-term sum of exact halves per component (<= 3u); its x axis
     d = rotate(r, e_x) has d_x = 2w^2 - 1 + 2x^2 and d_y = 2wz + 2xy, so |dd_xy| <= 2 * 2 * 2 * 3u + 4 roundings < 64u.  With
     rho = |d_xy| from the float64 run the heading moves by dh <= 64u / rho + 16u (3 ulp of atan2f at |h| <= pi is 12u); the same
     for the target heading (dh_t, rho_t).  sinf / cosf of h / 2 add 2u to the heading quaternion, inside the terms below.
   - A rotated vector l = rotate(hq, v), v = a float32 difference (<= u|v|) or an input: the rotation formula on a heading quaternion
     of norm 1 +- 2u is within 16u|v| of the exact rotation by the kernel's heading, which is |v_xy| dh away from the float64 one:
     bound 16u|v| + |v_xy| dh per component (local_body_pos, local_body_vel / ang_vel, target_rel_2d_pos, target_rel_body_pos).
   - Tan-norm blocks: the product quaternion carries <= 4u per component and the two quadratic forms add a few u more, so 24u; the
     de-headed body rotations (local_body_rot) add |t_xy| dh per 3-vector; target_rel_root_rot chains two de-based rotations: 32u;
     target_rel_body_rot: 24u; the root slot with local_root_obs: 24u, heading-free.
   - Heading vector (cos, sin)(h_t - h): dh + dh_t + 16u (the subtraction at |h_t - h| <= 2 pi, cosf / sinf).
   Where rho < RHO_MIN the heading is ill-conditioned: the kernel's and the oracle's headings may differ by anything, and both are
   valid.  There only what a rotation about z cannot change is compared: every heading-rotated 3-vector becomes (|xy|, 0, z), the 2-d
   target position its length, within twice the bound without the dh term (|xy| carries at most sqrt 2 of a component's error); the
   heading vector becomes its length, held to 1 within 16u; every heading-free field keeps its bound or stays exact.  Where only
   rho_t < RHO_MIN, only the heading vector is reduced to its length.
   Constructed cases at seeded positions of the random bulk: heading at +pi and -pi with d_y = +-0 and d_y = +-1 ulp; the x axis
   vertical, and 1e-3 and 1e-6 rad off vertical; target heading minus root heading just either side of +-pi; identity root, its
   negation and the upright base rotation; zero velocities and dofs; court-scale positions (|x|, |y| <= 30 m); near-unit quaternions
   (|q|^2 - 1 of a few u, as physics writes them).
6. The bf16 operand row, ld_bf16 in {768, 736, 1024}, mean / rstd given or NULL, clamp in {5, 0.25, inf}: equal to
   torch.clamp((obs - mean) * rstd, -c, c).to(bfloat16) of the launch's own float row as int16 bit patterns (so -0 != +0), NaN
   positions equal, and to the unfused nn.cast_rows of that row.  One env with a NaN input, one with +inf, one with -inf: NaN stays
   NaN, +-inf becomes +-clamp, every other row is bit-identical to a run without them.
7. Live wiring: a PhysicsMVAEController with the fused PolicyMLP at n = 1029, a few steps of random actions; then
   task._compute_observations() on the live rows holds the bounds above and policy.x holds the operand formula, with the config's
   localRootObs / rootHeightObs on and off.
8. The host refusals (include/b200env.h): ld_bf16 < W, odd ld_bf16, obs_bf16 not 4-byte aligned, shape_dim outside [0, 32] at create.
9. CPU negative controls: each comparator rejects a mutated oracle and names the env and the field."""
import ctypes as C
import math

import numpy as np
import pytest

from oracle import ref_port as R

f32, f64 = np.float32, np.float64
U = 2.0 ** -24
DEV = "cuda:0"
SENT = f32(12345.0)
SENT_BF16 = -7.75
SLACK = 3
SIZES = (1, 7, 8, 9, 63, 64, 65, 127, 129, 4095, 8191, 8192, 8195)
BIG = SIZES[-1]
MID = 1029
RHO_MIN = 1e-4
NB, ND, SD = 24, 69, 11
NAMES = ("body_pos", "body_rot", "target_pos", "target_rot", "dof_pos", "dof_vel", "target_dof_pos", "body_vel", "body_ang_vel",
         "motion_bodies")
WORST = {}


@pytest.fixture(scope="module", autouse=True)
def report_worst_ratio():
    yield
    if WORST:
        print("\nworst |got - ref| / bound per field: " + ", ".join(f"{k}: {r:.3g}" for k, r in sorted(WORST.items())))


# ------------------------------------------------------------------------------------------------ row layout (CPU)
def layout(jpos, local_root_obs=True, nb=NB, nd=ND, sd=SD):
    """[(field, width, kind)] of the row in column order.  kind: exact | vec3 (heading-rotated 3-vectors) | vec2 (their xy) |
    tn_h (heading-rotated tan-norm pairs) | tn (heading-free tan-norm pairs) | hvec (the heading vector)"""
    f = [("root_h", 1, "exact"), ("local_body_pos", (nb - 1) * 3, "vec3"), ("local_root_rot", 6, "tn" if local_root_obs else "tn_h"),
         ("local_body_rot", (nb - 1) * 6, "tn_h"), ("local_body_vel", nb * 3, "vec3"), ("local_body_ang_vel", nb * 3, "vec3"),
         ("dof_vel", nd, "exact"), ("target_rel_root_h", 1, "exact")]
    if jpos:
        f += [("target_rel_2d_pos", 2, "vec2")]
    else:
        f += [("target_rel_root_rot", 6, "tn"), ("target_rel_2d_pos", 2, "vec2"), ("target_rel_heading_vec", 2, "hvec"),
              ("target_rel_dof_pos", nd, "exact")]
    f += [("target_rel_body_pos", nb * 3, "vec3")]
    if not jpos:
        f += [("target_rel_body_rot", nb * 6, "tn")]
    return f + [("motion_bodies", sd, "exact")]


def width(jpos):
    return sum(w for _, w, _ in layout(jpos))


def split(row, jpos, local_root_obs=True):
    out, c = {}, 0
    for k, w, _ in layout(jpos, local_root_obs):
        out[k] = np.asarray(row)[:, c:c + w]
        c += w
    assert c == row.shape[1], (c, row.shape)
    return out


def field_cols(jpos, name):
    c = 0
    for k, w, _ in layout(jpos):
        if k == name:
            return c, c + w
        c += w
    raise KeyError(name)


# ------------------------------------------------------------------------------------------------ inputs (CPU)
def quat_z(h):
    return np.array([0.0, 0.0, math.sin(h / 2), math.cos(h / 2)])


def quat_axis(axis, ang):
    a = np.asarray(axis, f64) / np.linalg.norm(axis)
    return np.concatenate([a * math.sin(ang / 2), [math.cos(ang / 2)]])


BASE = np.array([0.5, 0.5, 0.5, 0.5])


def from_debased(r):
    """the body quaternion whose de-based rotation is r: r (x) base"""
    return R.quat_mul(np.asarray(r, f64), BASE)


def x_axis_tilted(off, yaw):
    """de-based root whose x axis is `off` rad from vertical (up), at heading yaw"""
    return R.quat_mul(quat_z(yaw), quat_axis((0, 1, 0), -(math.pi / 2 - off)))


def make_inputs(n, seed):
    """float32 inputs of n envs, the constructed cases at seeded positions; -> (inputs, {env: case})"""
    rng = np.random.default_rng(seed)
    q = rng.normal(size=(n, NB, 4))
    tq = rng.normal(size=(n, NB, 4))
    root = np.stack([rng.uniform(-3, 3, n), rng.uniform(-3, 3, n), rng.uniform(0.5, 1.2, n)], -1)
    bp = root[:, None] + rng.normal(0, 0.4, (n, NB, 3))
    bp[:, 0] = root
    inp = dict(body_pos=bp, body_rot=q / np.linalg.norm(q, axis=-1, keepdims=True), target_pos=bp + rng.normal(0, 0.1, (n, NB, 3)),
               target_rot=tq / np.linalg.norm(tq, axis=-1, keepdims=True), dof_pos=rng.normal(0, 0.5, (n, ND)),
               dof_vel=rng.normal(0, 3, (n, ND)), body_vel=rng.normal(0, 2, (n, NB, 3)), body_ang_vel=rng.normal(0, 4, (n, NB, 3)),
               motion_bodies=rng.normal(size=(n, SD)))
    inp["target_dof_pos"] = inp["dof_pos"] + rng.normal(0, 0.2, (n, ND))
    inp = {k: v.astype(f32) for k, v in inp.items()}
    ulp = 2.0 ** -23

    def root_rot(r):
        return lambda e: inp["body_rot"].__setitem__((e, 0), from_debased(r).astype(f32))

    def target_root(r):
        return lambda e: inp["target_rot"].__setitem__((e, 0), from_debased(r).astype(f32))

    def both(a, b):
        return lambda e: (a(e), b(e))

    def zero_motion(e):
        for k in ("body_vel", "body_ang_vel", "dof_pos", "dof_vel", "target_dof_pos"):
            inp[k][e] = 0

    def court(e):
        shift = np.array([rng.uniform(-30, 30), rng.uniform(-30, 30), 0])
        shift[rng.integers(2)] = rng.choice([-30.0, 30.0])
        for k in ("body_pos", "target_pos"):
            inp[k][e] = (inp[k][e].astype(f64) + shift).astype(f32)

    def near_unit(e):
        for k in ("body_rot", "target_rot"):
            s = 1 + rng.integers(-4, 5, NB)[:, None] * U
            inp[k][e] = (inp[k][e].astype(f64) * s).astype(f32)

    def negate_root(e):
        inp["body_rot"][e, 0] = -inp["body_rot"][e, 0]

    cases = [("heading +pi, d_y +0", root_rot(quat_z(math.pi))), ("heading -pi, d_y -0", root_rot(-quat_z(math.pi))),
             ("heading pi, d_y +1 ulp", root_rot(quat_z(math.pi - ulp))), ("heading -pi, d_y -1 ulp", root_rot(quat_z(-math.pi + ulp))),
             ("heading pi, d_y +1/2 ulp", root_rot(quat_z(math.pi - ulp / 2))),
             ("x axis vertical", root_rot(quat_axis((0, 1, 0), -math.pi / 2))), ("x axis vertical down", root_rot(quat_axis((0, 1, 0), math.pi / 2))),
             ("x axis 1e-3 off vertical", root_rot(x_axis_tilted(1e-3, 0.7))), ("x axis 1e-6 off vertical", root_rot(x_axis_tilted(1e-6, -2.0))),
             ("target x axis vertical", target_root(quat_axis((0, 1, 0), -math.pi / 2))),
             ("target - root heading just under pi", both(root_rot(quat_z(0.4)), target_root(quat_z(0.4 + math.pi - 1e-4)))),
             ("target - root heading just over pi", both(root_rot(quat_z(0.4)), target_root(quat_z(0.4 + math.pi + 1e-4)))),
             ("target - root heading just over -pi", both(root_rot(quat_z(2.9)), target_root(quat_z(2.9 - math.pi + 1e-4)))),
             ("target - root heading just under -pi", both(root_rot(quat_z(2.9)), target_root(quat_z(2.9 - math.pi - 1e-4)))),
             ("identity root", lambda e: inp["body_rot"].__setitem__((e, 0), (0, 0, 0, 1))),
             ("negated identity root", lambda e: inp["body_rot"].__setitem__((e, 0), (-0.0, -0.0, -0.0, -1))),
             ("upright base rotation", lambda e: inp["body_rot"].__setitem__((e, 0), (0.5, 0.5, 0.5, 0.5))),
             ("upright, all bodies identity", lambda e: (inp["body_rot"].__setitem__((e, slice(None)), (0, 0, 0, 1)),
                                                         inp["target_rot"].__setitem__((e, slice(None)), (0, 0, 0, 1)))),
             ("zero velocities and dofs", zero_motion), ("zero motion, upright", both(zero_motion, root_rot(np.array([0, 0, 0, 1.0])))),
             ("negated root quaternion", negate_root), ("near-unit quaternions", near_unit), ("near-unit, heading pi",
                                                                                             both(root_rot(quat_z(math.pi)), near_unit))]
    cases += [(f"court scale {k}", court) for k in range(4)]
    perm = rng.permutation(n)
    where = {}
    for k, (name, fn) in enumerate(cases[:n]):
        fn(int(perm[k]))
        where[int(perm[k])] = name
    return inp, where


# ------------------------------------------------------------------------------------------------ oracle and bounds (CPU)
def oracle(inp, n, jpos, lr, rh, dtype):
    fn = R.compute_humanoid_observations_imitation_jpos if jpos else R.compute_humanoid_observations_imitation
    with np.errstate(all="ignore"):
        return fn(*[inp[k][:n].astype(dtype) for k in NAMES], local_root_obs=bool(lr), root_height_obs=bool(rh))


def heading_rho(q):
    """|d_xy| of the de-based x axis, float64"""
    d = R.my_quat_rotate(R.remove_base_rot(q.astype(f64)), np.broadcast_to(np.array([1.0, 0, 0]), q.shape[:-1] + (3,)))
    return np.hypot(d[..., 0], d[..., 1])


def project(x, kind):
    """what a rotation about z leaves: 3-vectors -> (|xy|, 0, z), 2-vectors -> (|v|, 0)"""
    x = np.asarray(x, f64)
    if kind in ("vec3", "tn_h"):
        v = x.reshape(len(x), -1, 3)
        return np.stack([np.hypot(v[..., 0], v[..., 1]), np.zeros(v.shape[:-1]), v[..., 2]], -1).reshape(x.shape)
    return np.stack([np.hypot(x[:, 0], x[:, 1]), np.zeros(len(x))], -1)


def expected(inp, n, jpos, lr, rh):
    """(ref fields, spec, ill rows, target-ill rows): float64 oracle for the bounded fields, float32 for the exact ones"""
    o64 = split(oracle(inp, n, jpos, lr, rh, f64), jpos, lr)
    o32 = split(oracle(inp, n, jpos, lr, rh, f32), jpos, lr)
    rho, rho_t = heading_rho(inp["body_rot"][:n, 0]), heading_rho(inp["target_rot"][:n, 0])
    ill, ill_t = rho < RHO_MIN, rho_t < RHO_MIN
    with np.errstate(divide="ignore"):
        dh = np.where(ill, 0.0, 64 * U / rho + 16 * U)
        dh_t = np.where(ill_t, 0.0, 64 * U / rho_t + 16 * U)
    d2 = inp["target_pos"][:n, 0].astype(f64) - inp["body_pos"][:n, 0].astype(f64)
    ref, spec = {}, {}
    for k, w, kind in layout(jpos, lr):
        a = o64[k]
        if kind == "exact":
            ref[k], spec[k] = o32[k], "exact"
            continue
        ref[k] = a
        if kind in ("vec3", "tn_h"):
            v = a.reshape(n, -1, 3)
            mag = np.linalg.norm(v, axis=-1) if kind == "vec3" else np.ones(v.shape[:-1])
            c = 16 * U if kind == "vec3" else 24 * U
            bd = c * mag + np.hypot(v[..., 0], v[..., 1]) * dh[:, None]
            bd = np.where(ill[:, None], 2 * c * mag, bd)
            spec[k] = np.repeat(bd, 3, 1)
        elif kind == "vec2":
            bd = 16 * U * np.linalg.norm(d2, axis=-1) + np.hypot(d2[:, 0], d2[:, 1]) * dh
            bd = np.where(ill, 32 * U * np.linalg.norm(d2, axis=-1), bd)
            spec[k] = np.repeat(bd[:, None], 2, 1)
        elif kind == "tn":
            spec[k] = np.full(a.shape, (32 if k == "target_rel_root_rot" else 24) * U)
        elif kind == "hvec":
            spec[k] = np.where((ill | ill_t)[:, None], 16 * U, (dh + dh_t + 16 * U)[:, None] * np.ones((1, 2)))
    return ref, spec, ill, ill_t


def reduce_ill(fields, jpos, lr, ill, ill_t):
    """rows with an ill-conditioned heading compared on their rotation-invariant parts only"""
    out = {k: np.array(v, f64) if kind != "exact" else v for (k, _, kind) in layout(jpos, lr) for v in [fields[k]]}
    for k, _, kind in layout(jpos, lr):
        if kind in ("vec3", "tn_h", "vec2") and ill.any():
            out[k][ill] = project(out[k][ill], kind)
        if kind == "hvec" and (ill | ill_t).any():
            out[k][ill | ill_t] = project(out[k][ill | ill_t], kind)
    return out


def compare(ref, got, spec, limit=8, tag="", where=None):
    """-> list of "field: env i: column c ..." failures.  spec[field] = "exact" or an absolute bound array of the field's shape;
    NaN equals NaN.  The worst error / bound ratio of each bounded field goes to WORST under tag + field."""
    fails = []
    for k, how in spec.items():
        a, b = np.asarray(ref[k]), np.asarray(got[k])
        both_nan = np.isnan(a.astype(f64)) & np.isnan(b.astype(f64))
        if isinstance(how, str):
            bad = ~((a == b) | both_nan)
        else:
            with np.errstate(invalid="ignore"):
                err = np.abs(a.astype(f64) - b.astype(f64))
                bad = ~((a == b) | (err <= how) | both_nan)
                fin = np.isfinite(err) & (how > 0)
            if tag and fin.any():
                WORST[tag + k] = max(WORST.get(tag + k, 0.0), float((err[fin] / how[fin]).max()))
        for r in np.flatnonzero(bad.any(1))[:limit]:
            c = int(np.flatnonzero(bad[r])[0])
            case = f" ({where[int(r)]})" if where and int(r) in where else ""
            fails.append(f"{k}: env {int(r)}{case}: column {c} got {b[r, c]!r} ref {a[r, c]!r} ({int(bad.any(1).sum())} envs differ)")
    return fails


def check_row(inp, got_row, n, jpos, lr, rh, tag="", where=None):
    """failures of a launch's float rows [n, W] against the oracle"""
    ref, spec, ill, ill_t = expected(inp, n, jpos, lr, rh)
    got = split(np.asarray(got_row), jpos, lr)
    return compare(reduce_ill(ref, jpos, lr, ill, ill_t), reduce_ill(got, jpos, lr, ill, ill_t), spec, tag=tag, where=where)


def operand_want(obs, mean, rstd, clamp):
    """int16 bit patterns and NaN mask of torch.clamp((obs - mean) * rstd, -c, c).to(bfloat16), from the float rows"""
    import torch
    x = obs if mean is None else (obs - mean) * rstd
    b = torch.clamp(x, -clamp, clamp).to(torch.bfloat16)
    return b.view(torch.int16), torch.isnan(b)


def operand_fails(op, n, W, want_bits, want_nan, label):
    """failures of the bf16 operand buffer: the first n rows' W columns against the formula (bit patterns; NaN positions), rows past n
    and columns past W still the sentinel"""
    import torch
    fails = []
    got = op[:n, :W]
    gnan = torch.isnan(got.float())
    if not torch.equal(gnan, want_nan):
        r, c = (gnan != want_nan).nonzero()[0].tolist()
        fails.append(f"{label}: operand NaN at env {r} column {c}: got {float(got[r, c])}")
    bad = (got.view(torch.int16) != want_bits) & ~want_nan
    if bool(bad.any()):
        r, c = bad.nonzero()[0].tolist()
        fails.append(f"{label}: operand env {r} column {c}: got {float(got[r, c])!r} want {float(want_bits.view(torch.bfloat16)[r, c])!r} "
                     f"({int(bad.any(1).sum())} envs differ)")
    s = torch.tensor(SENT_BF16, dtype=torch.bfloat16, device=op.device).view(torch.int16)
    if not bool((op[n:].view(torch.int16) == s).all()):
        fails.append(f"{label}: operand row past n = {n} written (row {n + int((op[n:].view(torch.int16) != s).any(1).nonzero()[0])})")
    if not bool((op[:, W:].view(torch.int16) == s).all()):
        fails.append(f"{label}: operand padding column past W = {W} written (column {W + int((op[:, W:].view(torch.int16) != s).any(0).nonzero()[0])})")
    return fails


# ------------------------------------------------------------------------------------------------ GPU runners
@pytest.fixture(scope="module")
def handles():
    from helpers import SIM_PARAMS, im_cfg, v2p_cfg
    from vid2player3d_b200 import model_compiler, motion_lib
    from vid2player3d_b200.tasks import HumanoidSMPLIM, PhysicsMVAEController
    model = model_compiler.load_compiled("smpl_mesh_humanoid_amass_v1")
    flat = motion_lib.synthetic(model, num_motions=4, num_frames=30, seed=3)
    im = HumanoidSMPLIM(im_cfg(8, flat), SIM_PARAMS, 1, "cuda", 0, True)
    ctl = PhysicsMVAEController(v2p_cfg(8), SIM_PARAMS, 1, "cuda", 0, True)
    h = dict(amass=(im._env, 24), federer=(ctl._physics_player.task._env, 26))
    for env, _ in h.values():
        assert env.lib_bodies == NB and env.obs_row_width() == 734 and env.obs_row_width(True) == 513
    yield h
    del im, ctl


@pytest.fixture(scope="module")
def big_inputs():
    return make_inputs(BIG, 11)


def dev_inputs(inp, bpe):
    """device tensors: the gathers of the legacy entry and the Isaac-layout rows (every row past the 24 humanoid bodies NaN)"""
    import torch
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)  # noqa: E731
    n = len(inp["body_pos"])
    rbs = np.full((n, bpe, 13), np.nan, f32)
    for k, c in (("body_pos", 0), ("body_rot", 3), ("body_vel", 7), ("body_ang_vel", 10)):
        rbs[:, :NB, c:c + inp[k].shape[-1]] = inp[k]
    d = {k: t(v) for k, v in inp.items()}
    d["rbs"] = t(rbs)
    d["dofs"] = t(np.stack([inp["dof_pos"], inp["dof_vel"]], -1))
    d["bpe"] = bpe
    return d


def sent_obs(n, jpos):
    import torch
    return torch.full((n + SLACK, width(jpos)), float(SENT), device=DEV)


def sent_op(n, ld):
    import torch
    return torch.full((n + SLACK, ld), SENT_BF16, device=DEV, dtype=torch.bfloat16)


def run_rows(env, d, n, lr, rh, jpos, obs=None, op=None, mean=None, rstd=None, clamp=5.0):
    import torch
    obs = sent_obs(n, jpos) if obs is None else obs
    env.obs_imitation_rows(n, d["rbs"], d["bpe"], d["dofs"], d["target_pos"], d["target_rot"], d["target_dof_pos"], d["motion_bodies"],
                           lr, rh, obs, obs_bf16=op, mean=mean, rstd=rstd, clamp=clamp, jpos=jpos)
    torch.cuda.synchronize()
    return obs


def run_gathered(env, d, n, lr, rh, jpos):
    import torch
    obs = sent_obs(n, jpos)
    env.obs_imitation(*[d[k][:n] for k in ("body_pos", "body_rot", "target_pos", "target_rot", "dof_pos", "dof_vel", "target_dof_pos",
                                           "body_vel", "body_ang_vel", "motion_bodies")], lr, rh, obs, jpos=jpos)
    torch.cuda.synchronize()
    return obs


def bits(t):
    import torch
    return t.view(torch.int32) if t.dtype == torch.float32 else t.view(torch.int16)


def clean_slack(obs, n):
    return bool((obs[n:].cpu().numpy() == SENT).all())


# ------------------------------------------------------------------------------------------------ 1. sizes, sentinels, position
@pytest.mark.gpu
@pytest.mark.parametrize("asset", ["amass", "federer"])
def test_sizes_sentinels_and_position(handles, big_inputs, asset):
    import torch
    env, bpe = handles[asset]
    inp, where = big_inputs
    d = dev_inputs(inp, bpe)
    mean, rstd = torch.randn(734, device=DEV) * 0.1, torch.rand(734, device=DEV) + 0.5
    op_big = sent_op(BIG, 768)
    big = run_rows(env, d, BIG, 1, 1, False, op=op_big, mean=mean, rstd=rstd)
    again = run_rows(env, d, BIG, 1, 1, False, op=sent_op(BIG, 768), mean=mean, rstd=rstd)
    assert torch.equal(bits(big), bits(again)), "two launches of the same inputs differ"
    want_bits, want_nan = operand_want(big[:BIG], mean, rstd, 5.0)
    fails = operand_fails(op_big, BIG, 734, want_bits, want_nan, f"{asset} n={BIG}")
    for n in SIZES:
        op = sent_op(n, 768)
        obs = run_rows(env, d, n, 1, 1, False, op=op, mean=mean, rstd=rstd)
        if not clean_slack(obs, n):
            fails.append(f"n={n}: a float row past n was written")
        if not torch.equal(bits(obs[:n]), bits(big[:n])):
            r = int((bits(obs[:n]) != bits(big[:n])).any(1).nonzero()[0])
            fails.append(f"n={n}: row {r} differs from the {BIG}-env launch")
        fails += operand_fails(op, n, 734, want_bits[:n], want_nan[:n], f"{asset} n={n}")
    assert not fails, "; ".join(fails[:8])
    fails = check_row(inp, big[:BIG].cpu().numpy(), BIG, False, 1, 1, tag="full ", where=where)
    assert not fails, "; ".join(fails[:8])


# ------------------------------------------------------------------------------------------------ 2./3. entry points and layouts
@pytest.mark.gpu
@pytest.mark.parametrize("asset", ["amass", "federer"])
@pytest.mark.parametrize("jpos", [False, True], ids=["full", "jpos"])
@pytest.mark.parametrize("lr,rh", [(1, 1), (1, 0), (0, 1), (0, 0)])
def test_entry_points_and_layouts(handles, big_inputs, asset, jpos, lr, rh):
    import torch
    env, _ = handles[asset]
    inp = {k: v[:MID] for k, v in big_inputs[0].items()}
    where = {e: c for e, c in big_inputs[1].items() if e < MID}
    ref = run_gathered(env, dev_inputs(inp, NB), MID, lr, rh, jpos)
    assert clean_slack(ref, MID), "the gathered entry wrote a row past n"
    for bpe in (24, 25, 26):
        got = run_rows(env, dev_inputs(inp, bpe), MID, lr, rh, jpos)
        assert clean_slack(got, MID), f"bodies_per_env {bpe}: a row past n was written"
        diff = (bits(got) != bits(ref)).any(1)
        assert not bool(diff.any()), f"bodies_per_env {bpe}: rows entry differs from the gathered entry at env {int(diff.nonzero()[0])}"
    W = width(jpos)
    raw = torch.full((MID * W + 1,), float(SENT), device=DEV)       # one float off 8-byte alignment: the scalar store path
    mis = raw[1:].view(MID, W)
    assert mis.data_ptr() % 8 == 4
    run_rows(env, dev_inputs(inp, 26), MID, lr, rh, jpos, obs=mis)
    assert float(raw[0]) == SENT and torch.equal(bits(mis), bits(ref[:MID])), "scalar store path differs from the float2 path"
    fails = check_row(inp, ref[:MID].cpu().numpy(), MID, jpos, lr, rh, tag=("jpos " if jpos else "full ") + f"lr{lr} rh{rh} ", where=where)
    assert not fails, "; ".join(fails[:8])


@pytest.mark.gpu
def test_jpos_field_through_the_c_abi(handles, big_inputs):
    """the jpos field selects the 513-wide row on b200env_obs_imitation_rows, called through ctypes"""
    import torch
    from vid2player3d_b200 import abi
    from vid2player3d_b200.native import lib
    env, bpe = handles["federer"]
    inp = {k: v[:MID] for k, v in big_inputs[0].items()}
    d = dev_inputs(inp, bpe)
    want = run_rows(env, d, MID, 1, 1, True)
    obs, op = sent_obs(MID, True), sent_op(MID, 768)
    desc = abi.ObsRows(n=MID, bodies_per_env=bpe, local_root_obs=1, root_height_obs=1, jpos=1, ld_bf16=768, clamp=5.0,
                       rigid_body_state=d["rbs"].data_ptr(), dof_state=d["dofs"].data_ptr(), target_pos=d["target_pos"].data_ptr(),
                       target_rot=d["target_rot"].data_ptr(), target_dof_pos=d["target_dof_pos"].data_ptr(),
                       motion_bodies=d["motion_bodies"].data_ptr(), obs=obs.data_ptr(), obs_bf16=op.data_ptr())
    rc = lib().b200env_obs_imitation_rows(env._h, C.byref(desc), C.c_void_p(torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    assert rc == 0, lib().b200env_last_error()
    assert torch.equal(bits(obs), bits(want))
    wb, wn = operand_want(obs[:MID], None, None, 5.0)
    fails = operand_fails(op, MID, 513, wb, wn, "jpos via the C ABI")
    assert not fails, "; ".join(fails)


# ------------------------------------------------------------------------------------------------ 4. exact invariances
def same_bits_up_to_zero_sign(a, b):
    """bitwise equal, except that an exact zero may carry either sign; -> first differing (env, column) or None"""
    import torch
    bad = (bits(a) != bits(b)) & ~((a == 0) & (b == 0))
    return None if not bool(bad.any()) else tuple(bad.nonzero()[0].tolist())


@pytest.mark.gpu
def test_exact_invariances(handles, big_inputs):
    import torch
    env, bpe = handles["federer"]
    inp = {k: v[:MID].copy() for k, v in big_inputs[0].items()}
    base = run_rows(env, dev_inputs(inp, bpe), MID, 1, 1, False)[:MID]
    rng = np.random.default_rng(4)
    for k, what in (("body_rot", "body rotations"), ("target_rot", "target rotations")):
        neg = {kk: v.copy() for kk, v in inp.items()}
        m = rng.random((MID, NB)) < 0.5
        m[:, 0] |= rng.random(MID) < 0.5
        neg[k][m] = -neg[k][m]
        got = run_rows(env, dev_inputs(neg, bpe), MID, 1, 1, False)[:MID]
        bad = same_bits_up_to_zero_sign(got, base)
        assert bad is None, f"negated {what}: env {bad[0]} column {bad[1]} changed"
    for jpos in (False, True):
        rows = {(lr, rh): run_rows(env, dev_inputs(inp, bpe), MID, lr, rh, jpos)[:MID] for lr in (0, 1) for rh in (0, 1)}
        for lr in (0, 1):
            a, b = rows[(lr, 1)], rows[(lr, 0)]
            assert torch.equal(bits(a[:, 1:]), bits(b[:, 1:])), "root_height_obs changed a column other than 0"
            assert bool((b[:, 0] == 0).all()) and not bool(torch.signbit(b[:, 0]).any()) and torch.equal(a[:, 0], d0(inp))
        c0, c1 = field_cols(jpos, "local_root_rot")
        for rh in (0, 1):
            a, b = rows[(1, rh)], rows[(0, rh)]
            assert torch.equal(bits(a[:, :c0]), bits(b[:, :c0])) and torch.equal(bits(a[:, c1:]), bits(b[:, c1:])), \
                "local_root_obs changed a column outside the root tan-norm slot"
            assert bool((a[:, c0:c1] != b[:, c0:c1]).any(1).float().mean() > 0.99)
    full = run_rows(env, dev_inputs(inp, bpe), MID, 1, 1, False)[:MID]
    jp = run_rows(env, dev_inputs(inp, bpe), MID, 1, 1, True)[:MID]
    for name in ("root_h", "local_body_pos", "local_root_rot", "local_body_rot", "local_body_vel", "local_body_ang_vel", "dof_vel",
                 "target_rel_root_h", "target_rel_2d_pos", "target_rel_body_pos", "motion_bodies"):
        (a0, a1), (b0, b1) = field_cols(False, name), field_cols(True, name)
        assert torch.equal(bits(full[:, a0:a1]), bits(jp[:, b0:b1])), f"_jpos {name} differs from the full row's"


def d0(inp):
    import torch
    return torch.from_numpy(inp["body_pos"][:, 0, 2].copy()).to(DEV)


# ------------------------------------------------------------------------------------------------ 6. the bf16 operand row
@pytest.mark.gpu
@pytest.mark.parametrize("ld", [768, 736, 1024])
@pytest.mark.parametrize("norm", [True, False], ids=["mean_rstd", "raw"])
@pytest.mark.parametrize("clamp", [5.0, 0.25, math.inf], ids=["c5", "c0.25", "cinf"])
@pytest.mark.parametrize("jpos", [False, True], ids=["full", "jpos"])
def test_operand_row(handles, big_inputs, ld, norm, clamp, jpos):
    import torch
    from vid2player3d_b200 import nn
    env, bpe = handles["federer"]
    inp = {k: v[:MID] for k, v in big_inputs[0].items()}
    W = width(jpos)
    g = torch.Generator(device=DEV).manual_seed(ld)
    mean = torch.randn(W, device=DEV, generator=g) * 0.5 if norm else None
    rstd = torch.rand(W, device=DEV, generator=g) * 4 + 0.25 if norm else None
    op = sent_op(MID, ld)
    obs = run_rows(env, dev_inputs(inp, bpe), MID, 1, 1, jpos, op=op, mean=mean, rstd=rstd, clamp=clamp)
    wb, wn = operand_want(obs[:MID], mean, rstd, clamp)
    fails = operand_fails(op, MID, W, wb, wn, f"ld {ld}")
    assert not fails, "; ".join(fails)
    cast = sent_op(MID, ld)
    nn.cast_rows(obs[:MID], cast, W, mean, rstd, -clamp, clamp)
    torch.cuda.synchronize()
    assert torch.equal(bits(cast[:MID, :W]), bits(op[:MID, :W])), "fused operand row differs from nn.cast_rows of the float row"


@pytest.mark.gpu
@pytest.mark.parametrize("jpos", [False, True], ids=["full", "jpos"])
def test_operand_row_nonfinite_inputs(handles, big_inputs, jpos):
    """NaN stays NaN, +-inf becomes +-clamp, every other env is untouched by its neighbours' non-finite inputs"""
    import torch
    env, bpe = handles["federer"]
    inp = {k: v[:MID].copy() for k, v in big_inputs[0].items()}
    W = width(jpos)
    mean, rstd = torch.randn(W, device=DEV) * 0.5, torch.rand(W, device=DEV) * 4 + 0.25
    op0 = sent_op(MID, 768)
    clean = run_rows(env, dev_inputs(inp, bpe), MID, 1, 1, jpos, op=op0, mean=mean, rstd=rstd)
    bad = {5: np.nan, 600: np.inf, 1028: -np.inf}
    for e, v in bad.items():
        inp["dof_vel"][e, 7] = v
        inp["body_vel"][e, 3, 1] = v
    op = sent_op(MID, 768)
    obs = run_rows(env, dev_inputs(inp, bpe), MID, 1, 1, jpos, op=op, mean=mean, rstd=rstd)
    others = torch.ones(MID + SLACK, dtype=torch.bool, device=DEV)
    others[list(bad)] = False
    assert torch.equal(bits(obs[others]), bits(clean[others])) and torch.equal(bits(op[others]), bits(op0[others]))
    c = field_cols(jpos, "dof_vel")[0] + 7
    assert math.isnan(float(op[5, c])) and float(op[600, c]) == 5.0 and float(op[1028, c]) == -5.0
    wb, wn = operand_want(obs[:MID], mean, rstd, 5.0)
    fails = operand_fails(op, MID, W, wb, wn, "non-finite inputs")
    assert not fails, "; ".join(fails)


# ------------------------------------------------------------------------------------------------ 7. live wiring
@pytest.mark.gpu
@pytest.mark.parametrize("flags", [(True, True), (False, False)], ids=["local_height", "nolocal_noheight"])
def test_live_rows_and_policy_operand(flags):
    import torch
    from helpers import SIM_PARAMS, v2p_cfg
    from vid2player3d_b200 import nn
    from vid2player3d_b200.tasks import PhysicsMVAEController
    lr, rh = flags
    g = torch.Generator().manual_seed(8)
    mean, var = torch.randn(734, generator=g) * 0.5, torch.rand(734, generator=g) * 4 + 0.25
    policy = nn.PolicyMLP.random(MID, DEV, seed=3, out_gain=1.0, obs_mean=mean, obs_var=var, clamp_obs=5.0, clamp_actions=1.0)
    torch.manual_seed(4)
    cfg = v2p_cfg(MID)
    cfg["env"]["low_level_policy"] = policy
    cfg["env"]["physics"].update(localRootObs=lr, rootHeightObs=rh)
    env = PhysicsMVAEController(cfg, SIM_PARAMS, 1, "cuda", 0, True)
    task = env._physics_player.task
    assert task._obs_operand is not None and task._obs_operand[0] is policy.x
    env.reset()
    gen = torch.Generator(device=DEV).manual_seed(9)
    for _ in range(3):
        env.step(torch.clamp(torch.randn(MID, env.num_actions, device=DEV, generator=gen), -5, 5))
    task._compute_observations()
    torch.cuda.synchronize()
    rbs = task._rigid_body_state.view(MID, 26, 13).cpu().numpy()
    dofs = task._dof_state.view(MID, -1, 2).cpu().numpy()
    inp = dict(body_pos=rbs[:, :NB, 0:3], body_rot=rbs[:, :NB, 3:7], body_vel=rbs[:, :NB, 7:10], body_ang_vel=rbs[:, :NB, 10:13],
               dof_pos=dofs[..., 0], dof_vel=dofs[..., 1], target_pos=task._target_rb_pos.view(MID, NB, 3).cpu().numpy(),
               target_rot=task._target_rb_rot.view(MID, NB, 4).cpu().numpy(), target_dof_pos=task._target_dof_pos.cpu().numpy(),
               motion_bodies=task._reset_ref_motion_bodies.cpu().numpy())
    inp = {k: np.ascontiguousarray(v, f32) for k, v in inp.items()}
    fails = check_row(inp, task.obs_buf.cpu().numpy(), MID, False, lr, rh, tag=f"live lr{int(lr)} rh{int(rh)} ")
    assert not fails, "; ".join(fails[:8])
    if not rh:
        assert bool((task.obs_buf[:, 0] == 0).all())
    wb, wn = operand_want(task.obs_buf, policy.mean, policy.rstd, 5.0)
    got = policy.x[:MID, :734]
    assert torch.equal(torch.isnan(got.float()), wn) and torch.equal(got.view(torch.int16)[~wn], wb[~wn]), "policy.x differs from the formula"


# ------------------------------------------------------------------------------------------------ 8. refusals
@pytest.mark.gpu
def test_operand_argument_refusals(handles, big_inputs):
    """checked on the host before any launch: ld_bf16 below the row width, odd, or an operand address off 4-byte alignment"""
    import torch
    env, bpe = handles["federer"]
    inp = {k: v[:64] for k, v in big_inputs[0].items()}
    d = dev_inputs(inp, bpe)
    for jpos, ld, off, msg in ((False, 732, 0, "ld_bf16 is smaller"), (True, 512, 0, "ld_bf16 is smaller"), (False, 767, 0, "even"),
                               (False, 768, 1, "4-byte aligned")):
        buf = sent_op(64, ld + 2)
        op = buf.view(-1)[off:off + (64 + SLACK) * ld].view(64 + SLACK, ld)
        obs = sent_obs(64, jpos)
        with pytest.raises(RuntimeError, match=msg):
            run_rows(env, d, 64, 1, 1, jpos, obs=obs, op=op)
        assert clean_slack(obs, 0) and bool((buf.float() == SENT_BF16).all()), "a refused call wrote"
    with pytest.raises(AssertionError):
        run_rows(env, d, 64, 1, 1, False, obs=sent_obs(64, True))
    with pytest.raises(AssertionError):
        run_rows(env, d, 64, 1, 1, False, op=torch.zeros(63, 768, device=DEV, dtype=torch.bfloat16))


def test_create_refuses_shape_dim_outside_0_32():
    """b200env_create / b200env_create_assets refuse cfg.shape_dim outside [0, 32] before touching a device (the observation launches
    give one lane to each motion-body column)"""
    from vid2player3d_b200 import abi, model_compiler
    from vid2player3d_b200.native import lib
    model = model_compiler.load_compiled("smpl_mesh_humanoid_amass_v1")
    m, verts = abi.pack_model(model)
    L = lib()
    for sd in (33, -1, 1000):
        cfg = abi.make_cfg(model, shape_dim=sd)
        h = C.c_void_p()
        rc = L.b200env_create(C.byref(m), verts.ctypes.data_as(C.c_void_p), C.byref(cfg), C.c_int32(8), C.c_int32(0), C.byref(h))
        assert rc == -2 and b"shape_dim" in L.b200env_last_error(), (sd, rc, L.b200env_last_error())
        marr = (abi.Model * 1)(m)
        varr = (C.c_void_p * 1)(verts.ctypes.data)
        ea = np.zeros(8, np.int32)
        rc = L.b200env_create_assets(marr, varr, C.c_int32(1), ea.ctypes.data_as(C.c_void_p), C.byref(cfg), C.c_int32(8), C.c_int32(0),
                                     C.byref(h))
        assert rc == -2 and b"shape_dim" in L.b200env_last_error(), (sd, rc, L.b200env_last_error())


# ------------------------------------------------------------------------------------------------ 9. CPU negative controls
@pytest.fixture(scope="module")
def cpu_case():
    inp, where = make_inputs(300, 2)
    return inp, where


def _mutated(inp, jpos, lr, rh, mutate):
    """the float32 oracle's row (a stand-in for a correct kernel) with one field mutated"""
    row = oracle(inp, len(inp["body_pos"]), jpos, lr, rh, f32)
    f = split(row.copy(), jpos, lr)
    mutate(f, inp)
    return np.concatenate([f[k] for k, _, _ in layout(jpos, lr)], 1).astype(f32)


def test_oracle_row_passes_its_own_comparator(cpu_case):
    inp, where = cpu_case
    for jpos in (False, True):
        for lr, rh in ((1, 1), (0, 0)):
            fails = check_row(inp, oracle(inp, 300, jpos, lr, rh, f32), 300, jpos, lr, rh, where=where)
            assert not fails, fails[:4]
    ill = {where.get(int(e), "random") for e in np.flatnonzero(heading_rho(inp["body_rot"][:, 0]) < RHO_MIN)}
    # the body's identity quaternion de-bases to an x axis along z: the identity-root cases are ill-conditioned too
    assert ill == {"x axis vertical", "x axis vertical down", "x axis 1e-6 off vertical", "identity root", "negated identity root",
                   "upright, all bodies identity"}, ill


def _heading_flip(f, inp):
    """heading sign flipped: the de-heading rotation is the inverse one"""
    n = len(inp["body_pos"])
    rr = R.remove_base_rot(inp["body_rot"][:, 0])
    hq, _ = R.calc_heading_quat_inv_with_heading(rr)
    hq = R.quat_conjugate(hq)
    hr = np.broadcast_to(hq[:, None], (n, NB, 4))
    f["local_body_pos"][:] = R.my_quat_rotate(hr, inp["body_pos"] - inp["body_pos"][:, :1]).reshape(n, -1)[:, 3:]


def _shift_body(f, inp):
    v = f["local_body_pos"].reshape(len(inp["body_pos"]), -1, 3)
    f["local_body_pos"][:] = np.concatenate([v[:, 1:], v[:, :1]], 1).reshape(len(v), -1)


def _swap_tan_norm(f, inp):
    v = f["target_rel_body_rot"].reshape(len(inp["body_pos"]), -1, 2, 3)
    f["target_rel_body_rot"][:] = v[:, :, ::-1].reshape(len(v), -1)


def _negate_rel_dof(f, inp):
    f["target_rel_dof_pos"][:] = -f["target_rel_dof_pos"]


@pytest.mark.parametrize("mutate,field", [(_heading_flip, "local_body_pos"), (_shift_body, "local_body_pos"),
                                          (_swap_tan_norm, "target_rel_body_rot"), (_negate_rel_dof, "target_rel_dof_pos")],
                         ids=["heading_sign", "body_shift", "tan_norm_swap", "rel_dof_negated"])
def test_comparator_rejects_mutated_oracle(cpu_case, mutate, field):
    inp, where = cpu_case
    got = _mutated(inp, False, 1, 1, mutate)
    fails = check_row(inp, got, 300, False, 1, 1, where=where)
    assert fails and all(x.startswith(field + ": env ") for x in fails), fails[:4]
    assert "column" in fails[0]


def test_operand_comparator_rejects_one_ulp_and_slack_writes():
    """a 1-ulp change of one bf16 entry, a write into a slack row and one into the padding columns are each named"""
    import torch
    rng = np.random.default_rng(1)
    n, W, ld = 37, 513, 768
    obs = torch.from_numpy(rng.normal(0, 3, (n, W)).astype(f32))
    mean, rstd = torch.from_numpy(rng.normal(0, 0.5, W).astype(f32)), torch.from_numpy(rng.uniform(0.25, 4, W).astype(f32))
    wb, wn = operand_want(obs, mean, rstd, 5.0)
    op = torch.full((n + SLACK, ld), SENT_BF16, dtype=torch.bfloat16)
    op[:n, :W] = wb.view(torch.bfloat16)
    assert operand_fails(op, n, W, wb, wn, "clean") == []
    one = op.clone()
    one.view(torch.int16)[12, 100] += 1
    f = operand_fails(one, n, W, wb, wn, "ulp")
    assert len(f) == 1 and "env 12 column 100" in f[0]
    slack = op.clone()
    slack[n + 1, 3] = 0
    f = operand_fails(slack, n, W, wb, wn, "slack")
    assert len(f) == 1 and f"row {n + 1}" in f[0]
    pad = op.clone()
    pad[4, W] = 0
    f = operand_fails(pad, n, W, wb, wn, "pad")
    assert len(f) == 1 and f"column {W}" in f[0]


def test_float_slack_check_rejects_a_write():
    import torch
    obs = torch.full((10 + SLACK, 734), float(SENT))
    assert clean_slack(obs, 10)
    obs[11, 700] = 0.0
    assert not clean_slack(obs, 10)


def test_layout_matches_the_kernel_width():
    assert width(False) == 734 and width(True) == 513
    assert field_cols(False, "target_rel_body_pos") == (507, 579) and field_cols(True, "target_rel_body_pos") == (430, 502)
