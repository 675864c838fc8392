"""Edge catalogue of the physics step: named states of the amass and federer workloads that land on the branches the random states
of the other physics tests never reach, each proved on the float64 restatement (oracle/physics_ref.c) to lie on its branch with a
stated margin from the threshold; then the lane emulator of the device code (tests/emu, csrc/packed.cuh compiled as host C++) on them.

Branches (csrc/dyn_common.cuh, csrc/packed.cuh; the restatement has the same thresholds):
- rotation: the 1e-6 series switch of qexp (on |q|) and qlog (on sin(|q| / 2)) at |q| = 0, 5e-7, 1.5e-6, 2e-6, 4e-6; |q| near pi at rest; a joint carried across pi
  within the control step, which qlog wraps to the opposite vector of angle 2 pi - |q| (dof_pos stays in [0, pi]); a root quaternion
  with w < 0, paired with the same state at -Q;
- the angular-velocity clamp (|w| > max_ang_vel = 100 in pk_root_integrate / pk_forward) of the root and of one joint, at 150 (taken)
  and 99.9 (never taken), with 1, 2 and 6 substeps (one substep: h |w| = 1.67 rad, the float qexp_small series, not sin / cos);
- joint limits: federer's live wrist limits and amass with tight limits, one DOF below lo, above hi and inside, on its side at the
  start of every substep of the control step;
- contact load: 0, 1, 8, 9, 16, 17 and >= 20 bodies with penetrating vertices (rounds 0 to 3 of the 8-lane hand-out of
  pk_contact_phase), a body whose penetrating vertices all have index >= 32 (the high word of the mask only), a body with every
  vertex in the ground, a bounding sphere across z = 0 with no vertex below it;
- ball (federer, ball-body contact with the hull faces): z = R (1 +- 1e-3) moving down and up, the racket head rim at Rad +- 1e-3,
  a 70 m/s ball through the head, a ball centre inside a body hull, a ball at each end cap of the handle capsule;
- non-finite: NaN and +Inf in the root position, root quaternion, one joint q, one joint qd, one PD target, the residual wrench and
  the ball position and velocity.

Bounds.  The float64 emulator runs the restatement's algorithm, so every finite case is held to 1e-9 of its env's scale (the largest
magnitude of the row, at least 1; contact forces and DOF forces likewise).  The float32 emulator (the arithmetic the product kernel
runs, host libm for the MUFU approximations) is held per kind to the bounds of tests/test_gpu_parity.py, scaled by the state's size:
a float32 step carries a relative error of a few units of 2^-24 in every term, so the error of q after a control step grows with
the rotation h |w| it integrates.  With S = max(1, max(|w_root|, max_j |qd_j|) / 10):
- free flight: q and root 1e-5 S, qd 1e-3 S;
- contact (every contact-load case): q and root 1e-4 S, qd 2e-3 S;
- within delta = 1e-2 of pi, q is compared as the geodesic angle between exp(q) rotations, and a vector flip between the two sides
  is accepted there only.
Non-finite input must leave the other three envs of its warp bit-identical to the run where that env holds a finite state, and
must not be repaired to an all-finite state where the restatement fails or goes non-finite.  The comparators reject a joint vector
flipped outside the wrap band, a restatement without the clamp, an inverted limit branch and a NaN leaked into a neighbour.
Negating the root quaternion negates the rigid-body quaternions and leaves every other row of the step bit-identical."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "emu"))

from oracle import physics_ref  # noqa: E402
from test_dof_force import emu_lib, restatement_dof_force, with_tight_limits  # noqa: E402
from vid2player3d_b200 import abi, model_compiler  # noqa: E402

UPRIGHT = np.array([0.5, 0.5, 0.5, 0.5])
AXIS = np.array([0.6, 0.0, 0.8])             # the rotation axis of the joint cases
ROOT_AXIS = np.array([0.0, 0.0, 1.0])        # root spin of the clamp cases: about z the humanoid stays below 100 rad/s from 99.9
KNEE = 3                                     # first DOF of L_Knee (body 2): the joint of the rotation and joint-clamp cases
WMAX = 100.0
PI_BAND = 1e-2
EPW = 4


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


# ------------------------------------------------------------------------------------------------ workloads
_W = {}


class Workload:
    def __init__(self, name, variant):
        self.name, self.variant = name, variant
        asset = "smpl_mesh_humanoid_amass_v1" if name == "amass" else "smpl_mesh_humanoid_federer"
        self.mod = model_compiler.canonical_racket_last(model_compiler.load_compiled(asset))
        self.ms, self.verts = abi.pack_model(self.mod, float(self.mod["mass"].sum()) / 90.0)
        self.faces = None
        if name == "amass":
            sub = {"sub1": 1, "sub2": 2, "sub6": 6, "tight": 2}[variant]
            self.cfg = abi.make_cfg(self.mod, substeps=sub)
            if variant == "tight":
                self.ms = with_tight_limits(self.ms)
        else:
            self.cfg = abi.make_cfg(self.mod, substeps=6, ball={"ball_body_contact": 1}, task_mode=1, pd_mode=1)
            self.faces = abi.pack_faces(self.mod, self.verts)
        self.nb, self.nd = self.ms.nb, self.ms.nd
        self.names = [str(x) for x in self.mod["body_names"]]
        self.h = float(self.cfg.sim_dt) / self.cfg.substeps
        self.nsub = self.cfg.substeps * self.cfg.control_freq_inv

    @property
    def has_ball(self):
        return self.faces is not None

    def cfg_with(self, **kw):
        c = abi.Cfg.from_buffer_copy(self.cfg)
        for k, v in kw.items():
            setattr(c, k, v)
        return c


def workload(name, variant):
    if (name, variant) not in _W:
        _W[(name, variant)] = Workload(name, variant)
    return _W[(name, variant)]


def base_state(W, seed):
    """a humanoid at rest in free flight (root at z = 2, upright, small joint angles held by their PD targets), the ball far away"""
    rng = np.random.default_rng(seed)
    root = np.zeros(13)
    root[0:2], root[2], root[3:7] = rng.uniform(-1, 1, 2), 2.0, UPRIGHT
    q = rng.normal(0, 0.1, W.nd)
    st = dict(root=root, q=q, qd=np.zeros(W.nd), tar=q.copy(), ext=np.zeros(6), ball=None)
    if W.has_ball:
        ball = np.zeros(13)
        ball[0:3] = [root[0] + 3.0, root[1] + 6.0, 1.5]
        ball[7:10] = [0.0, -1.0, 0.0]
        st["ball"] = ball
    return st


def restate(W, sts, cfg=None, ms=None, n_steps=1):
    """the restatement on a list of states (copies); returns (root, q, qd, rb, cf, ball, hits) or raises on a failed solve"""
    n = len(sts)
    S = lambda k: np.ascontiguousarray(np.stack([s[k] for s in sts]), np.float64)  # noqa: E731
    root, q, qd, tar, ext = S("root"), S("q"), S("qd"), S("tar"), S("ext")
    ball = S("ball") if W.has_ball else None
    hits = np.zeros(n, np.int32) if W.has_ball else None
    if W.faces is not None:
        physics_ref.set_hull_faces(*W.faces)
    try:
        rb, cf = physics_ref.control_step(ms or W.ms, W.verts, cfg or W.cfg, root, q, qd, tar, ext, n_steps=n_steps, ball=ball, hits=hits)
    finally:
        physics_ref.clear_hull_faces()
    return dict(root=root, q=q, qd=qd, rb=rb, cf=cf, ball=ball, hits=hits)


def poses(W, root, q):
    """rigid-body rows [n, nb, 13] of the restatement at sim_dt = 1e-12 (forward kinematics) and its contact rows"""
    tiny = W.cfg_with(sim_dt=1e-12)
    n = len(root)
    rb, cf = physics_ref.control_step(W.ms, W.verts, tiny, np.ascontiguousarray(root, np.float64).copy(), np.ascontiguousarray(q, np.float64).copy(),
                                      np.zeros((n, W.nd)), np.ascontiguousarray(q, np.float64).copy(), None)
    return rb, cf


def _rot(quat):
    from scipy.spatial.transform import Rotation
    return Rotation.from_quat(quat).as_matrix()


def vertex_z(W, rb):
    """world z of every hull vertex [n, nb, vmax] (+inf past a body's vertex count)"""
    nv = list(W.ms.nverts)[:W.nb]
    out = np.full(rb.shape[:2] + (W.verts.shape[1],), np.inf)
    for b in range(W.nb):
        if nv[b] == 0:
            continue
        R = _rot(rb[:, b, 3:7])
        out[:, b, :nv[b]] = rb[:, b, None, 2] + np.einsum("nj,vj->nv", R[:, 2, :], W.verts[b, :nv[b]].astype(np.float64))
    return out


def substep_trace(W, st):
    """(root, q, qd) at the start of every substep of the control step and at its end: the restatement one substep at a time (a
    control step of one substep of length h), the residual wrench on the substeps of the first sim step.  Humanoid only."""
    one = W.cfg_with(sim_dt=W.h, substeps=1, control_freq_inv=1, has_ball=0)
    cur = {k: (v.copy() if v is not None else None) for k, v in st.items()}
    out = [(cur["root"].copy(), cur["q"].copy(), cur["qd"].copy())]
    for k in range(W.nsub):
        s = dict(cur, ext=cur["ext"] if k < W.cfg.substeps else np.zeros(6))
        root, q, qd = (np.ascontiguousarray(s[x][None], np.float64).copy() for x in ("root", "q", "qd"))
        physics_ref.control_step(W.ms, W.verts, one, root, q, qd, np.ascontiguousarray(s["tar"][None]), np.ascontiguousarray(s["ext"][None]))
        cur.update(root=root[0], q=q[0], qd=qd[0])
        out.append((root[0].copy(), q[0].copy(), qd[0].copy()))
    return out


# ------------------------------------------------------------------------------------------------ the catalogue
class Case:
    """a named state of one workload, the branch it lands on, and the restatement's proof: `value` against `threshold`, with
    `margin` = the distance to it on the side the branch needs (> 0 when the case lands on its branch)"""

    def __init__(self, name, W, st, kind, branch, value, threshold, margin):
        self.name, self.W, self.st, self.kind = name, W, st, kind
        self.branch, self.value, self.threshold, self.margin = branch, float(value), float(threshold), float(margin)

    @property
    def key(self):
        return (self.W.name, self.W.variant)


def _with_joint(st, d0, vec, vel=None):
    s = {k: (v.copy() if v is not None else None) for k, v in st.items()}
    s["q"][d0:d0 + 3] = vec
    s["tar"][d0:d0 + 3] = vec
    s["qd"][d0:d0 + 3] = 0.0 if vel is None else vel
    return s


def _drive_lead(W, d):
    """a PD target this far ahead of q along qd cancels the drive's damping at the start of the step (kp (tar - q - h qd) = kd qd):
    without it the implicit drive takes a joint from 150 rad/s to below 100 in one substep and its clamp is never reached"""
    return W.h + float(W.ms.kd[d]) / float(W.ms.kp[d])


def _qexp(v):
    """the restatement's q_exp (oracle/physics_ref.c): rotation vector -> quaternion (x, y, z, w)"""
    a = float(np.linalg.norm(v))
    f = 0.5 - a * a / 48.0 if a < 1e-6 else np.sin(0.5 * a) / a
    return np.array([f * v[0], f * v[1], f * v[2], np.cos(0.5 * a)])


def rotation_cases():
    W = workload("amass", "sub2")
    b = base_state(W, 1)
    out = []
    # the switches are evaluated on the restatement's own input: qexp on |q| when the step loads the joint, qlog on |xyz| of that
    # exp(q) = sin(|q| / 2) in the first substep's drive.  |q| = 2e-6 puts sin(|q| / 2) = 1e-6 - 1.7e-19 on qlog's switch (round-off
    # decides it, so it claims only its qexp branch); 1.5e-6 is the case strictly between the two switches.
    for a, name in ((0.0, "q = 0"), (5e-7, "|q| = 5e-7"), (1.5e-6, "|q| = 1.5e-6"), (2e-6, "|q| = 2e-6"), (4e-6, "|q| = 4e-6")):
        st = _with_joint(b, KNEE, a * AXIS)
        s = np.linalg.norm(_qexp(a * AXIS)[:3])
        branch = f"qexp {'series' if a < 1e-6 else 'sin/cos'}, "
        if name == "|q| = 2e-6":
            out.append(Case(name, W, st, "free", branch + "qlog at its switch", a, 1e-6, abs(a - 1e-6)))
        else:
            out.append(Case(name, W, st, "free", branch + f"qlog {'series' if s < 1e-6 else 'atan2'}", a, 1e-6,
                            min(abs(a - 1e-6), abs(s - 1e-6))))
    # |q| = pi - 1e-3 at rest: stays below pi (no flip) at every substep
    st = _with_joint(b, KNEE, (np.pi - 1e-3) * AXIS)
    tr = substep_trace(W, st)
    ang = np.array([np.linalg.norm(x[1][KNEE:KNEE + 3]) for x in tr])
    flip = min(float(np.dot(x[1][KNEE:KNEE + 3], AXIS)) for x in tr)
    out.append(Case("|q| = pi - 1e-3 at rest", W, st, "free", "qlog w > 0, no wrap", ang.max(), np.pi, min(np.pi - ang.max(), flip)))
    # carried across pi: the vector flips to the opposite side and ends outside the band around pi
    st = _with_joint(b, KNEE, (np.pi - 0.05) * AXIS, 20.0 * AXIS)
    st["tar"][KNEE:KNEE + 3] += _drive_lead(W, KNEE) * 20.0 * AXIS
    tr = substep_trace(W, st)
    dots = np.array([float(np.dot(x[1][KNEE:KNEE + 3], AXIS)) for x in tr])
    end = np.linalg.norm(tr[-1][1][KNEE:KNEE + 3])
    out.append(Case("|q| carried across pi (wrap)", W, st, "free", "qlog wrap at pi", end, np.pi - PI_BAND,
                    min(np.pi - PI_BAND - end, -dots[-1])))
    # root quaternion with w < 0, and the same state at -Q
    st = {k: (v.copy() if v is not None else None) for k, v in b.items()}
    Q = np.array([0.3, -0.5, 0.4, -0.7])
    st["root"][3:7] = Q / np.linalg.norm(Q)
    st["root"][10:13] = [0.4, -0.3, 0.2]
    neg = {k: (v.copy() if v is not None else None) for k, v in st.items()}
    neg["root"][3:7] *= -1
    out.append(Case("root w < 0", W, st, "free", "root Q, w < 0", st["root"][6], 0.0, -st["root"][6]))
    out.append(Case("root w < 0 at -Q", W, neg, "free", "root -Q, w > 0", neg["root"][6], 0.0, neg["root"][6]))
    return out


def clamp_cases():
    """the clamp is taken somewhere in the control step iff removing it changes the restatement's result"""
    out = []
    for variant in ("sub1", "sub2", "sub6"):
        W = workload("amass", variant)
        b = base_state(W, 2)
        for where in ("root", "joint"):
            for w in (150.0, 99.9):
                st = {k: (v.copy() if v is not None else None) for k, v in b.items()}
                if where == "root":
                    st["root"][10:13] = w * ROOT_AXIS
                else:
                    st["qd"][KNEE:KNEE + 3] = w * AXIS
                    st["tar"][KNEE:KNEE + 3] += _drive_lead(W, KNEE) * w * AXIS
                on = restate(W, [st])
                off = restate(W, [st], cfg=W.cfg_with(max_ang_vel=1e6))
                diff = max(float(np.abs(on[k] - off[k]).max()) for k in ("root", "q", "qd"))
                taken = w > WMAX
                if taken:
                    value, margin = diff, diff
                else:                                # below the clamp at the end of every substep, and removing it changes nothing
                    tr = substep_trace(W, st)
                    value = max(np.linalg.norm(x[0][10:13] if where == "root" else x[2][KNEE:KNEE + 3]) for x in tr[1:])
                    margin = WMAX - value if diff == 0 else -diff
                out.append(Case(f"{where} |w| = {w:g}, {W.cfg.substeps} substep(s)", W, st, "free",
                                f"{where} clamp {'taken' if taken else 'not taken'}", value, WMAX, margin))
    return out


def limit_cases():
    """one DOF below lo, above hi and inside, on that side at the start of every substep (the limit branch is chosen there)"""
    out = []
    for W, d, lo_d, hi_d in ((workload("federer", "ball"), 64, 64, 63), (workload("amass", "tight"), 0, 0, 0)):
        b = base_state(W, 3)
        lo, hi = float(W.ms.lim_lo[lo_d]), float(W.ms.lim_hi[hi_d])
        body_d0 = (d // 3) * 3
        for side, dof, val in (("below lo", lo_d, lo - 0.15), ("above hi", hi_d, hi + 0.15), ("inside", d, 0.5 * (float(W.ms.lim_lo[d]) + float(W.ms.lim_hi[d])))):
            st = {k: (v.copy() if v is not None else None) for k, v in b.items()}
            vec = np.zeros(3)
            vec[dof - body_d0] = val
            st = _with_joint(st, body_d0, vec)
            tr = substep_trace(W, st)
            qs = np.array([x[1][dof] for x in tr[:-1]])
            l, h = float(W.ms.lim_lo[dof]), float(W.ms.lim_hi[dof])
            m = {"below lo": (l - qs).min(), "above hi": (qs - h).min(), "inside": np.minimum(qs - l, h - qs).min()}[side]
            out.append(Case(f"{W.name} DOF {dof} {side}", W, st, "free", f"limit {side}", qs[0], {"below lo": l, "above hi": h, "inside": l}[side], m))
    return out


def _flat_poses(W, n, seed):
    """lying humanoids (identity root: face down), small joint angles: bodies reach the ground at nearby heights"""
    from scipy.spatial.transform import Rotation
    rng = np.random.default_rng(seed)
    root = np.zeros((n, 13))
    root[:, 2] = 1.0
    root[:, 3:7] = Rotation.from_rotvec(rng.normal(0, 0.03, (n, 3))).as_quat()
    q = rng.normal(0, 0.1, (n, W.nd)) * rng.uniform(0, 1, (n, 1))
    return root, q


def _placed(W, root, q, dz):
    st = dict(root=root.copy(), q=q.copy(), qd=np.zeros(W.nd), tar=q.copy(), ext=np.zeros(6), ball=None)
    st["root"][2] += dz
    return st


def contact_cases():
    """bodies with penetrating vertices: counted on the restatement's contact rows at sim_dt = 1e-12 (at rest, a body has a
    non-zero normal force iff a vertex is below z = 0); the margin is the gap between the ground and the nearest vertex that would
    change the count (or the mask / sphere property)"""
    W = workload("amass", "sub2")
    out = []
    root, q = _flat_poses(W, 600, 1)
    rb, _ = poses(W, root, q)
    z = vertex_z(W, rb)
    bm = np.sort(z.min(2), 1)
    rad = np.array(list(W.ms.radius)[:W.nb])

    def count(st):
        _, cf = poses(W, st["root"][None], st["q"][None])
        return int((cf[0, :, 2] > 0).sum())

    for K in (0, 1, 8, 9, 16, 17, 20):
        if K == 0:       # the lowest vertex 4 mm above the ground; some bounding spheres (body origin, radius) cross z = 0
            i = 0
            dz, margin = -bm[i, 0] + 0.004, 0.004
        else:
            gap = bm[:, K] - bm[:, K - 1]
            depth = bm[:, K - 1] - bm[:, 0] + gap / 2
            ok = np.flatnonzero(gap > 0.006)
            i = int(ok[np.argmin(depth[ok])])
            dz, margin = -(bm[i, K - 1] + bm[i, K]) / 2, gap[i] / 2
        st = _placed(W, root[i], q[i], dz)
        k = count(st)
        rnd = -(-k // 8)
        out.append(Case(f"{K} bodies in contact", W, st, "contact", f"contact hand-out, {rnd} round(s)", k, K, margin if k == K else -1.0))
        if K == 0:
            zz = rb[i, :, 2] + dz - rad
            out.append(Case("bounding sphere across z = 0, no vertex", W, st, "contact", "sphere test passes, mask empty", zz.min(), 0.0,
                            min(-zz.min(), margin) if k == 0 else -1.0))
    # a body whose penetrating vertices all have index >= 32: random orientations, the lowest vertex of the whole humanoid has index
    # >= 32 and every vertex of index < 32 (of any body) is 3 mm higher
    from scipy.spatial.transform import Rotation
    rng = np.random.default_rng(5)
    n = 400
    r2 = np.zeros((n, 13))
    r2[:, 2] = 2.0
    r2[:, 3:7] = Rotation.random(n, random_state=6).as_quat()
    q2 = rng.normal(0, 0.3, (n, W.nd))
    rb2, _ = poses(W, r2, q2)
    z2 = vertex_z(W, rb2)
    lowest = z2.reshape(n, -1).min(1)
    lo_word = z2[:, :, :32].reshape(n, -1).min(1)
    hi_first = np.sort(z2[:, :, 32:].reshape(n, -1), 1)
    best = np.argmax(lo_word - lowest)
    gap = lo_word[best] - lowest[best]
    st = _placed(W, r2[best], q2[best], -lowest[best] - min(0.001, gap / 3))
    zz = z2[best] + st["root"][2] - r2[best, 2]
    pen = np.argwhere(zz < 0)
    ok = len(pen) > 0 and (pen[:, 1] >= 32).all() and len(np.unique(pen[:, 0])) == 1 and count(st) == 1
    out.append(Case("penetrating vertices all at index >= 32", W, st, "contact", "high mask word only", len(pen), 32,
                    (lo_word[best] - lowest[best] - min(0.001, gap / 3)) if ok else -1.0))
    # every vertex of a body in the ground: a flat humanoid pressed 0.35 m into it
    st = _placed(W, root[0], q[0], -bm[0, 0] - 0.35)
    zz = z[0] - bm[0, 0] - 0.35
    top = np.where(np.isinf(zz), -np.inf, zz).max(1)
    b = int(np.argmin(top))
    out.append(Case("every vertex of a body in the ground", W, st, "contact", f"full mask ({W.names[b]})", top[b], 0.0, -top[b]))
    return out


def ball_cases():
    """federer at rest in free flight (ball and humanoid fall together, so the ball's approach is its velocity relative to the
    racket); hits counted by the restatement"""
    W = workload("federer", "ball")
    b = base_state(W, 4)
    rb, _ = poses(W, b["root"][None], b["q"][None])
    c = W.cfg
    R = float(c.ball_radius)
    rk = rb[0, c.racket_body]
    Rr = _rot(rk[3:7]) @ _rot(np.array(list(c.racket_head_quat)))
    ctr = rk[0:3] + Rr @ np.array(list(c.racket_head_center))
    H, Rad = float(c.racket_head_halfthick) + R, float(c.racket_head_radius) + R
    ny = Rr[:, 1]
    out = []

    def with_ball(p, v):
        st = {k: (x.copy() if x is not None else None) for k, x in b.items()}
        st["ball"][:] = 0
        st["ball"][0:3], st["ball"][7:10] = p, v
        return st

    # the ground test after the first substep, on the restatement run for one substep (a control step of one substep of length h):
    # it puts a bouncing ball at z = R exactly; the same substep with R = 0 (no bounce for z > 0; the ball is 4 m from the player,
    # so nothing else sees R) gives the unbounced height, whose distance to R is the margin
    one = dict(sim_dt=W.h, substeps=1, control_freq_inv=1)
    for f in (1 + 1e-3, 1 - 1e-3):
        for vz, name in ((-1.0, "down"), (2.0, "up")):
            st = with_ball(b["root"][0:3] + [3.0, 3.0, R * f - b["root"][2]], [0.5, 0.0, vz])
            z_ref = float(restate(W, [st], cfg=W.cfg_with(**one))["ball"][0, 2])
            z_free = float(restate(W, [st], cfg=W.cfg_with(ball_radius=0.0, **one))["ball"][0, 2])
            taken = name == "down"
            ok = (z_ref == R and z_free < R) if taken else (z_ref == z_free > R)
            out.append(Case(f"ball z = R (1 {'+' if f > 1 else '-'} 1e-3) moving {name}", W, st, "free",
                            f"ground bounce {'taken' if taken else 'not taken'}", z_free, R, abs(z_free - R) if ok else -1.0))
    for dr, name in ((-1e-3, "inside"), (1e-3, "outside")):
        p = ctr + Rr @ np.array([Rad + dr, H + 0.01, 0.0])
        st = with_ball(p, rk[7:10] - 20.0 * ny)
        hits = int(restate(W, [st])["hits"][0])
        out.append(Case(f"racket head rim at Rad {'-' if dr < 0 else '+'} 1e-3", W, st, "free", f"head rim, {name}", hits,
                        1 if dr < 0 else 0, 1e-3 if hits == (dr < 0) else -1.0))
    st = with_ball(ctr + (H + 0.1) * ny, rk[7:10] - 70.0 * ny)
    hits = int(restate(W, [st])["hits"][0])
    out.append(Case("70 m/s ball through the head", W, st, "free", "swept head hit", 0.1 / 70.0, W.h, (W.h - 0.1 / 70.0) if hits == 1 else -1.0))
    # ball centre inside the chest hull (hull centroid): the exact query's inside branch (max face distance <= 0)
    chest = W.names.index("Chest")
    nv = int(W.ms.nverts[chest])
    cl = W.verts[chest, :nv].astype(np.float64).mean(0)
    st = with_ball(rb[0, chest, 0:3] + _rot(rb[0, chest, 3:7]) @ cl, np.zeros(3))
    physics_ref.set_hull_faces(*W.faces)
    try:
        hit, pen, _ = physics_ref.hull_sphere(W.ms, W.verts, chest, cl, R)
    finally:
        physics_ref.clear_hull_faces()
    out.append(Case("ball centre inside the chest hull", W, st, "free", "hull query, centre inside", pen, R, (pen - R) if hit else -1.0))
    # the handle capsule (racket frame, axis a -> b, radius r): the ball 1 mm into each end cap, off the axis beyond its end
    hd = np.array(list(c.racket_handle), np.float64)
    a_, b_, r_ = hd[0:3], hd[3:6], hd[6]
    ax = (b_ - a_) / np.linalg.norm(b_ - a_)
    Rk = _rot(rk[3:7])
    nohandle = W.cfg_with()
    nohandle.racket_handle[6] = 0.0
    import copy
    handle_only = copy.deepcopy(W.ms)               # no body hulls: the forearm's hull reaches past end a and is the deeper contact
    for k in range(W.nb):                           # there in the full model (the humanoid flies: no ground contact either)
        handle_only.nverts[k] = 0
    for end, sgn, name in ((a_, -1.0, "a"), (b_, 1.0, "b")):
        # off the axis beyond the end; the capsule's contact is confirmed on the restatement with the handle as the only obstacle:
        # its ball differs from the same step with the handle removed
        dvec = sgn * 0.8 * ax + 0.6 * np.array([0.0, 1.0, 0.0])
        dvec /= np.linalg.norm(dvec)
        pl = end + (r_ + R - 1e-3) * dvec
        t = float(np.dot(pl - a_, b_ - a_) / np.dot(b_ - a_, b_ - a_))
        st = with_ball(rk[0:3] + Rk @ pl, rk[7:10] - 1.0 * (Rk @ dvec))      # 1 m/s into the cap, relative to the racket
        dv = float(np.abs(restate(W, [st], ms=handle_only)["ball"][0] - restate(W, [st], cfg=nohandle, ms=handle_only)["ball"][0]).max())
        out.append(Case(f"ball at the handle's end cap {name}", W, st, "free", "capsule end cap", t, 0.0 if sgn < 0 else 1.0,
                        min(-t if sgn < 0 else t - 1.0, 1e-3) if dv > 0 else -1.0))
    return out


NONFINITE_FIELDS = (("root position", "root", 1), ("root quaternion", "root", 4), ("joint q", "q", KNEE + 1), ("joint qd", "qd", KNEE + 1),
                    ("PD target", "tar", KNEE + 1), ("residual wrench", "ext", 3), ("ball position", "ball", 2), ("ball velocity", "ball", 8))


def nonfinite_cases():
    """(case, field, index, value) for NaN and +Inf in each field; the ball fields on federer only"""
    out = []
    for wl, var in (("amass", "sub2"), ("federer", "ball")):
        W = workload(wl, var)
        for i, (name, key, idx) in enumerate(NONFINITE_FIELDS):
            if key == "ball" and not W.has_ball:
                continue
            for val in (np.nan, np.inf):
                st = base_state(W, 10 + i)
                st["root"][2] = 1.0                        # feet near the ground: the contact path runs as well
                st[key] = st[key].copy()
                st[key][idx] = val
                out.append(Case(f"{wl}: {'NaN' if np.isnan(val) else '+Inf'} in {name}", W, st, "nonfinite", "non-finite input", val, 0, 1.0))
    return out


def catalogue():
    return rotation_cases() + clamp_cases() + limit_cases() + contact_cases() + ball_cases()


# ------------------------------------------------------------------------------------------------ emulator and comparators
_keep = []


def emu(W, sts, f32=False):
    """the sensor instantiation of the packed step on the lane emulator (float64, or float32: the product arithmetic) on a list of
    states; returns dict(root, q, qd, rb, cf, ball, hits, tau)"""
    lib = emu_lib()
    if W.faces is not None:
        planes, tris, ntris, tmax = W.faces
        arrs = (np.ascontiguousarray(planes, np.float32), np.ascontiguousarray(tris, np.uint8), np.ascontiguousarray(ntris, np.int32))
        _keep[:] = arrs
        lib.emu_set_hull_faces(_p(arrs[0]), _p(arrs[1]), _p(arrs[2]), C.c_int(int(tmax)))
    dt = np.float32 if f32 else np.float64
    n = len(sts)
    S = lambda k: np.ascontiguousarray(np.stack([s[k] for s in sts]), dt)  # noqa: E731
    root, q, qd, tar, ext = S("root"), S("q"), S("qd"), S("tar"), S("ext")
    ball = S("ball") if W.has_ball else None
    hits = np.zeros(n, np.int32) if W.has_ball else None
    rb, cf, tau = np.zeros((n, W.nb, 13), dt), np.zeros((n, W.nb, 3), dt), np.full((n, W.nd), np.nan, dt)
    fn = lib.emu_dof_force_physics_f32 if f32 else lib.emu_dof_force_physics
    rc = fn(C.byref(W.ms), _p(np.ascontiguousarray(W.verts, np.float32)), C.byref(W.cfg), C.c_int(n), C.c_int(1), _p(root), _p(q), _p(qd),
            _p(tar), _p(ext), _p(rb), _p(cf), _p(ball), _p(hits), _p(tau))
    lib.emu_set_hull_faces(None, None, None, C.c_int(0))
    assert rc == 0
    return dict(root=root, q=q, qd=qd, rb=rb, cf=cf, ball=ball, hits=hits, tau=tau)


def restate_sensor(W, sts, ms=None, cfg=None):
    """the restatement and the sensor of its last substep (test_dof_force.restatement_dof_force)"""
    n = len(sts)
    S = lambda k: np.ascontiguousarray(np.stack([s[k] for s in sts]), np.float64)  # noqa: E731
    root, q, qd, tar, ext = S("root"), S("q"), S("qd"), S("tar"), S("ext")
    ball = S("ball") if W.has_ball else None
    hits = np.zeros(n, np.int32) if W.has_ball else None
    if W.faces is not None:
        physics_ref.set_hull_faces(*W.faces)
    try:
        tau = restatement_dof_force(ms or W.ms, W.verts, cfg or W.cfg, root, q, qd, tar, ext, ball=ball, hits=hits)
    finally:
        physics_ref.clear_hull_faces()
    return dict(root=root, q=q, qd=qd, ball=ball, hits=hits, tau=tau)


def f64_failures(names, got, ref, keys=("root", "q", "qd", "rb", "cf", "ball", "tau"), tol=1e-9):
    """every env within tol of its own scale (largest magnitude of the reference row, at least 1), per field"""
    fails = []
    for k in keys:
        if k not in ref or ref[k] is None or got.get(k) is None:
            continue
        a, b = got[k].reshape(len(names), -1).astype(np.float64), ref[k].reshape(len(names), -1)
        scale = np.maximum(1.0, np.abs(b).max(1))
        err = np.abs(a - b).max(1) / scale
        for i in np.flatnonzero(~(err < tol)):
            fails.append(f"{names[i]}: {k} error {err[i]:.3e} of its scale > {tol:g}")
    return fails


def joint_errors(qk, qo):
    """per env, the largest joint error: |q_k - q_o| per component, or, both within PI_BAND of pi, the geodesic angle between exp(q_k)
    and exp(q_o); and whether a joint vector flipped (q_k . q_o < 0) outside that band"""
    from scipy.spatial.transform import Rotation
    n, nd = qk.shape
    a, b = qk.reshape(n, -1, 3).astype(np.float64), qo.reshape(n, -1, 3).astype(np.float64)
    na, nb_ = np.linalg.norm(a, axis=-1), np.linalg.norm(b, axis=-1)
    band = np.minimum(na, nb_) > np.pi - PI_BAND
    plain = np.abs(a - b).max(-1)
    geo = (Rotation.from_rotvec(a.reshape(-1, 3)).inv() * Rotation.from_rotvec(b.reshape(-1, 3))).magnitude().reshape(n, -1)
    err = np.where(band, geo, plain)
    flip = ((a * b).sum(-1) < -1e-12) & ~band
    return err.max(1), flip.any(1)


def f32_failures(cases, got, ref):
    """the float32 bounds of the module docstring"""
    fails = []
    eq, flip = joint_errors(got["q"], ref["q"])
    er = np.abs(got["root"].astype(np.float64) - ref["root"]).max(1)
    ev = np.abs(got["qd"].astype(np.float64) - ref["qd"]).max(1)
    for i, c in enumerate(cases):
        st = c.st
        S = max(1.0, max(np.linalg.norm(st["root"][10:13]), np.abs(st["qd"]).max()) / 10.0)
        bq, bv = (1e-5, 1e-3) if c.kind == "free" else (1e-4, 2e-3)
        if flip[i]:
            fails.append(f"{c.name}: a joint vector flipped outside the band around pi")
        if not (max(eq[i], er[i]) <= bq * S):
            fails.append(f"{c.name}: q / root error {max(eq[i], er[i]):.3e} > {bq * S:.3e}")
        if not (ev[i] <= bv * S):
            fails.append(f"{c.name}: qd error {ev[i]:.3e} > {bv * S:.3e}")
    return fails


def _groups(cases):
    out = {}
    for c in cases:
        out.setdefault(c.key, []).append(c)
    return out.values()


@pytest.fixture(scope="module")
def cases():
    return catalogue()


# ------------------------------------------------------------------------------------------------ tests
def test_catalogue_lands_on_its_branches(cases):
    """every constructor's state lies on its branch on the restatement, with a positive margin; the coverage table names them"""
    print(f"\n{'case':44s} {'workload':16s} {'branch':36s} {'value':>11s} {'threshold':>10s} {'margin':>9s}")
    for c in cases:
        print(f"{c.name:44s} {c.W.name + '/' + c.W.variant:16s} {c.branch:36s} {c.value:11.4g} {c.threshold:10.4g} {c.margin:9.3g}")
    bad = [c.name for c in cases if not c.margin > 0]
    assert not bad, bad
    branches = {c.branch for c in cases}
    for need in ("contact hand-out, 0 round(s)", "contact hand-out, 1 round(s)", "contact hand-out, 2 round(s)", "contact hand-out, 3 round(s)",
                 "high mask word only", "root clamp taken", "root clamp not taken", "joint clamp taken", "joint clamp not taken",
                 "limit below lo", "limit above hi", "limit inside", "qexp series, qlog series", "qexp sin/cos, qlog series",
                 "qexp sin/cos, qlog atan2", "qexp sin/cos, qlog at its switch", "qlog wrap at pi", "ground bounce taken", "ground bounce not taken", "head rim, inside",
                 "head rim, outside", "hull query, centre inside", "capsule end cap"):
        assert need in branches, need
    assert sum(c.branch == "capsule end cap" for c in cases) == 2


def test_float64_emulator_matches_restatement(cases):
    """every finite case, with the DOF force sensor: within 1e-9 of each env's scale (the sensor is left out where a joint's
    velocity is clamped at the end of the step: its definition runs the last substep backwards and needs the unclamped velocity)"""
    fails = []
    for grp in _groups(cases):
        W = grp[0].W
        names = [c.name for c in grp]
        got = emu(W, [c.st for c in grp])
        ref = restate(W, [c.st for c in grp])
        fails += f64_failures(names, got, ref, keys=("root", "q", "qd", "rb", "cf", "ball"))
        free = [i for i in range(len(grp)) if np.linalg.norm(ref["qd"][i].reshape(-1, 3), axis=-1).max() < WMAX * (1 - 1e-9)]
        sen = restate_sensor(W, [grp[i].st for i in free])
        fails += f64_failures([names[i] for i in free], dict(tau=got["tau"][free]), sen, keys=("tau",))
        if W.has_ball:
            assert np.array_equal(got["hits"], ref["hits"])
    assert not fails, "\n".join(fails)


def test_float32_emulator_within_bounds(cases):
    fails = []
    for grp in _groups(cases):
        W = grp[0].W
        got = emu(W, [c.st for c in grp], f32=True)
        ref = restate(W, [c.st for c in grp])
        fails += f32_failures(grp, got, ref)
    assert not fails, "\n".join(fails)


def _bits_equal(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return np.array_equal(a.view(np.uint8), b.view(np.uint8))


def isolation_failures(W, finite, bad, slot, f32):
    """8 envs (two warps) of finite states; env 4 + slot holds `bad` in one run and its finite state in the other: the other envs'
    rows must be bit-identical between the runs.  Returns (failures, the rows of the run with the bad env)"""
    sts = list(finite)
    e = EPW + slot
    ref = emu(W, sts, f32)
    sts[e] = bad
    got = emu(W, sts, f32)
    return neighbour_failures(ref, got, e), got, e


def neighbour_failures(ref, got, e):
    others = [i for i in range(len(ref["root"])) if i != e]
    return [f"{k} of a neighbour env changed" for k in ("root", "q", "qd", "rb", "cf", "ball", "hits", "tau")
            if ref[k] is not None and not _bits_equal(ref[k][others], got[k][others])]


@pytest.mark.parametrize("f32", [False, True], ids=["float64", "float32"])
def test_nonfinite_env_is_isolated_and_not_repaired(f32):
    """each non-finite case in every env slot of the second warp: the loops of the step are count-bounded (the run returns), the
    other seven envs are bit-identical to the run where that env is finite, and the env itself keeps a non-finite value where the
    restatement fails on it or goes non-finite"""
    fails = []
    for i, c in enumerate(nonfinite_cases()):
        W = c.W
        finite = [base_state(W, 40 + k) for k in range(2 * EPW)]
        for s in finite:
            s["root"][2] = 1.0
        f, got, e = isolation_failures(W, finite, c.st, i % EPW, f32)
        fails += [f"{c.name}: {x}" for x in f]
        try:
            ref = restate(W, [c.st])
            ref_bad = not all(np.isfinite(ref[k]).all() for k in ("root", "q", "qd"))
        except RuntimeError:
            ref_bad = True
        mine_finite = all(np.isfinite(got[k][e]).all() for k in ("root", "q", "qd"))
        if ref_bad and mine_finite:
            fails.append(f"{c.name}: the env was repaired to a finite state")
    assert not fails, "\n".join(fails)


def test_comparators_reject_the_mistakes(cases):
    """negative controls: a joint vector flipped to its equivalent outside the band around pi, a restatement without the clamp, one
    limit branch inverted in the restatement, one NaN leaked into a neighbour env's row"""
    by = {c.name: c for c in cases}
    # the wrap case ends at |q| = 1.53: the same rotation as the opposite vector of angle 2 pi - 1.53, outside the band
    c = by["|q| carried across pi (wrap)"]
    ref = restate(c.W, [c.st])
    got = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in ref.items()}
    v = got["q"][0, KNEE:KNEE + 3]
    got["q"][0, KNEE:KNEE + 3] = -v / np.linalg.norm(v) * (2 * np.pi - np.linalg.norm(v))
    assert f32_failures([c], ref, ref) == []
    assert any("flipped outside the band" in f for f in f32_failures([c], got, ref))
    # the clamp removed from the restatement
    for name in ("root |w| = 150, 2 substep(s)", "joint |w| = 150, 6 substep(s)"):
        c = by[name]
        got = emu(c.W, [c.st])
        assert f64_failures([name], got, restate(c.W, [c.st]), keys=("root", "q", "qd")) == []
        assert f64_failures([name], got, restate(c.W, [c.st], cfg=c.W.cfg_with(max_ang_vel=1e6)), keys=("root", "q", "qd")) != []
    # one limit branch inverted: the restatement's DOF past its limit is treated as inside
    import copy
    for name, dof, attr in (("federer DOF 64 below lo", 64, "lim_lo"), ("amass DOF 0 above hi", 0, "lim_hi")):
        c = by[name]
        ms = copy.deepcopy(c.W.ms)
        getattr(ms, attr)[dof] = -1e9 if attr == "lim_lo" else 1e9
        got = emu(c.W, [c.st])
        assert f64_failures([name], got, restate(c.W, [c.st], ms=ms), keys=("q", "qd")) != []
    # a NaN leaked into the neighbour of the non-finite env
    W = workload("amass", "sub2")
    sts = [base_state(W, 40 + k) for k in range(2 * EPW)]
    ref = emu(W, sts)
    got = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in ref.items()}
    assert neighbour_failures(ref, got, 5) == []
    got["qd"][6, 10] = np.nan
    assert neighbour_failures(ref, got, 5) == ["qd of a neighbour env changed"]


@pytest.mark.parametrize("f32", [False, True], ids=["float64", "float32"])
def test_negated_root_quaternion_on_the_emulator(cases, f32):
    """-Q for Q: every formula of the step that reads the root quaternion is even in it (qmat, qrot) or linear (qmul, qnormalize), so
    the rigid-body quaternions come out negated and every other row bit-identical: root position and velocities, q, qd, body
    positions and velocities, contact forces and sensor rows.  The pair of the catalogue (free flight) and a pair in contact with 17
    bodies.  (The observation and reward come from the task launches around the physics step; the GPU test checks those.)"""
    by = {c.name: c for c in cases}
    pairs = [(by["root w < 0"].st, by["root w < 0 at -Q"].st)]
    c = by["17 bodies in contact"].st
    neg = {k: (v.copy() if v is not None else None) for k, v in c.items()}
    neg["root"][3:7] *= -1
    pairs.append((c, neg))
    W = workload("amass", "sub2")
    a = emu(W, [p[0] for p in pairs], f32)
    b = emu(W, [p[1] for p in pairs], f32)
    assert _bits_equal(a["rb"][..., 3:7], -b["rb"][..., 3:7])
    assert _bits_equal(a["root"][:, 3:7], -b["root"][:, 3:7])
    for k, cols in (("root", np.r_[0:3, 7:13]), ("rb", np.r_[0:3, 7:13])):
        assert _bits_equal(a[k][..., cols], b[k][..., cols]), k
    for k in ("q", "qd", "cf", "tau"):
        assert _bits_equal(a[k], b[k]), k
    assert by["17 bodies in contact"].margin > 0                  # 17 bodies penetrate at the start of the step (the contact rows
                                                                  # are those of the last substep, after the bodies lifted off)
