"""ctypes mirror of include/b200env.h (structs + packing helpers).  Product code: the native
binding (native.py) and the tests' oracle wrapper both build their arguments from these."""
import ctypes as C

import numpy as np

MAX_BODIES, MAX_DOF, MAX_KEY = 32, 96, 8
ABI_VERSION = 6


class Model(C.Structure):
    _fields_ = [
        ("nb", C.c_int32), ("nd", C.c_int32), ("vmax", C.c_int32), ("max_depth", C.c_int32),
        ("parent", C.c_int32 * MAX_BODIES), ("depth", C.c_int32 * MAX_BODIES),
        ("dof_of_body", C.c_int32 * MAX_BODIES), ("fixed", C.c_int32 * MAX_BODIES),
        ("nverts", C.c_int32 * MAX_BODIES),
        ("offset", (C.c_float * 3) * MAX_BODIES), ("mass", C.c_float * MAX_BODIES),
        ("com", (C.c_float * 3) * MAX_BODIES), ("inertia", (C.c_float * 6) * MAX_BODIES),
        ("radius", C.c_float * MAX_BODIES),
        ("kp", C.c_float * MAX_DOF), ("kd", C.c_float * MAX_DOF), ("armature", C.c_float * MAX_DOF),
        ("lim_lo", C.c_float * MAX_DOF), ("lim_hi", C.c_float * MAX_DOF),
    ]


class Cfg(C.Structure):
    _fields_ = [
        ("sim_dt", C.c_float), ("substeps", C.c_int32), ("control_freq_inv", C.c_int32), ("gravity_z", C.c_float),
        ("contact_kn", C.c_float), ("contact_cn", C.c_float), ("friction_mu", C.c_float), ("friction_vs", C.c_float),
        ("ang_damping", C.c_float), ("max_ang_vel", C.c_float), ("limit_k", C.c_float), ("limit_c", C.c_float),
        ("pd_tar_lim", C.c_float), ("res_force_scale", C.c_float), ("res_torque_scale", C.c_float),
        ("max_episode_length", C.c_int32), ("enable_early_termination", C.c_int32),
        ("termination_height", C.c_float * MAX_BODIES), ("contact_body", C.c_int32 * MAX_BODIES),
        ("body_pos_weight", C.c_float * MAX_BODIES),
        ("k_dof", C.c_float), ("k_vel", C.c_float), ("k_pos", C.c_float), ("k_rot", C.c_float),
        ("w_dof", C.c_float), ("w_vel", C.c_float), ("w_pos", C.c_float), ("w_rot", C.c_float),
        ("num_key", C.c_int32), ("key_body", C.c_int32 * MAX_KEY), ("shape_dim", C.c_int32),
        ("ground_tolerance", C.c_float),
        ("task_mode", C.c_int32), ("pd_mode", C.c_int32), ("has_ball", C.c_int32), ("racket_body", C.c_int32),
        ("ball_mass", C.c_float), ("ball_inertia", C.c_float), ("ball_radius", C.c_float), ("spin_scale", C.c_float),
        ("ball_e_ground", C.c_float), ("ball_mu_ground", C.c_float), ("ball_e_racket", C.c_float), ("ball_mu_racket", C.c_float),
        ("bounce_threshold_velocity", C.c_float),
        ("racket_head_center", C.c_float * 3), ("racket_head_halfthick", C.c_float), ("racket_head_radius", C.c_float),
        ("racket_head_quat", C.c_float * 4),
        ("ball_body_contact", C.c_int32), ("ball_e_body", C.c_float), ("ball_mu_body", C.c_float), ("racket_handle", C.c_float * 7),
    ]


class MotionLibView(C.Structure):
    _fields_ = [
        ("gts", C.c_void_p), ("grs", C.c_void_p), ("lrs", C.c_void_p), ("grvs", C.c_void_p), ("gravs", C.c_void_p),
        ("dvs", C.c_void_p), ("motion_lengths", C.c_void_p), ("num_frames", C.c_void_p), ("motion_dt", C.c_void_p),
        ("length_starts", C.c_void_p), ("min_verts_h", C.c_void_p),
        ("num_motions", C.c_int32), ("num_lib_bodies", C.c_int32), ("total_frames", C.c_int64),
    ]


class Buffers(C.Structure):
    _fields_ = [
        ("root_states", C.c_void_p), ("actors_per_env", C.c_int32),
        ("dof_state", C.c_void_p), ("rigid_body_state", C.c_void_p), ("contact_forces", C.c_void_p),
        ("bodies_per_env", C.c_int32),
        ("obs_buf", C.c_void_p), ("num_obs", C.c_int32),
        ("rew_buf", C.c_void_p), ("sub_rewards", C.c_void_p), ("reset_buf", C.c_void_p), ("progress_buf", C.c_void_p),
        ("terminate_buf", C.c_void_p), ("motion_ids", C.c_void_p), ("ref_motion_times", C.c_void_p),
        ("motion_bodies", C.c_void_p),
        ("t_root_pos", C.c_void_p), ("t_root_rot", C.c_void_p), ("t_dof_pos", C.c_void_p), ("t_root_vel", C.c_void_p),
        ("t_root_ang_vel", C.c_void_p), ("t_dof_vel", C.c_void_p), ("t_key_pos", C.c_void_p), ("t_rb_pos", C.c_void_p),
        ("t_rb_rot", C.c_void_p),
        ("p_dof_pos", C.c_void_p), ("p_dof_vel", C.c_void_p), ("p_rb_pos", C.c_void_p), ("p_rb_rot", C.c_void_p),
        ("pd_targets", C.c_void_p), ("actions_used", C.c_void_p), ("num_actions", C.c_int32),
        ("has_bounce", C.c_void_p), ("has_bounce_now", C.c_void_p), ("bounce_pos", C.c_void_p), ("racket_hit_now", C.c_void_p),
    ]


def _fill(arr, values):
    for i, v in enumerate(values):
        arr[i] = v


def pack_model(model, pd_scale=1.0, kd_scale=None):
    """model: dict from model_compiler.  pd_scale = humanoid_mass/90 * kp_scale
    (humanoid_smpl_im.py:376-383).  Returns (Model, verts float32 [nb,vmax,3])."""
    kd_scale = pd_scale if kd_scale is None else kd_scale
    nb, nd = len(model["parent"]), len(model["kp"])
    assert nb <= MAX_BODIES and nd <= MAX_DOF
    m = Model()
    m.nb, m.nd = nb, nd
    vmax = int(max(4, (int(model["nverts"].max()) + 3) // 4 * 4))
    m.vmax = vmax
    m.max_depth = int(model["depth"].max())
    _fill(m.parent, [int(x) for x in model["parent"]])
    _fill(m.depth, [int(x) for x in model["depth"]])
    _fill(m.dof_of_body, [int(x) for x in model["dof_of_body"]])
    _fill(m.fixed, [int(x) for x in model["fixed"]])
    _fill(m.nverts, [int(x) for x in model["nverts"]])
    for i in range(nb):
        _fill(m.offset[i], [float(x) for x in model["offset"][i]])
        _fill(m.com[i], [float(x) for x in model["dyn_com"][i]])
        I = model["dyn_inertia"][i]
        _fill(m.inertia[i], [float(I[0, 0]), float(I[1, 1]), float(I[2, 2]), float(I[0, 1]), float(I[0, 2]), float(I[1, 2])])
    _fill(m.mass, [float(x) for x in model["dyn_mass"]])
    _fill(m.radius, [float(x) for x in model["radius"]])
    _fill(m.kp, [float(x) * pd_scale for x in model["kp"]])
    _fill(m.kd, [float(x) * kd_scale for x in model["kd"]])
    _fill(m.armature, [float(x) for x in model["armature"]])
    _fill(m.lim_lo, [float(x) for x in model["limits"][:, 0]])
    _fill(m.lim_hi, [float(x) for x in model["limits"][:, 1]])
    verts = np.ascontiguousarray(model["verts"][:, :vmax], dtype=np.float32)
    return m, verts


def pack_faces(model, verts):
    """hull faces of a compiled model for b200env_set_hull_faces: planes float32 [nb, TMAX, 4] (outward unit normal, offset: n.x <= d
    inside), tris uint8 [nb, TMAX, 4] (vertex indices + pad), ntris int32 [MAX_BODIES].  `verts` = the float32 array pack_model returns
    (the planes are computed from exactly the vertex values the kernels see).  Models compiled before round 2 have no faces: ntris = 0."""
    nb = verts.shape[0]
    ntris = np.zeros(MAX_BODIES, np.int32)
    if "tris" not in model:
        return np.zeros((nb, 4, 4), np.float32), np.zeros((nb, 4, 4), np.uint8), ntris, 4
    t3 = np.asarray(model["tris"])
    tmax = int(t3.shape[1])
    tris = np.zeros((nb, tmax, 4), np.uint8)
    tris[..., :3] = t3
    planes = np.zeros((nb, tmax, 4), np.float32)
    for b in range(nb):
        k = int(model["ntris"][b])
        ntris[b] = k
        if k == 0:
            continue
        V = verts[b].astype(np.float64)
        a, bb, c = V[t3[b, :k, 0]], V[t3[b, :k, 1]], V[t3[b, :k, 2]]
        n = np.cross(bb - a, c - a)
        n /= np.maximum(np.linalg.norm(n, axis=1, keepdims=True), 1e-30)
        planes[b, :k, :3] = n
        planes[b, :k, 3] = np.max(V[:int(model["nverts"][b])] @ n.T, axis=0)    # support value: every vertex satisfies n.x <= d
    return planes, tris, ntris, tmax


DEFAULT_PHYSICS = dict(contact_kn=6.0e4, contact_cn=6.0e2, friction_mu=1.0, friction_vs=0.05,
                       ang_damping=0.01, max_ang_vel=100.0, limit_k=2000.0, limit_c=20.0)


def make_cfg(model, *, sim_dt=1.0 / 60.0, substeps=2, control_freq_inv=2, gravity_z=-9.81, pd_tar_lim=0.5 * np.pi,
             res_force_scale=31.85, res_torque_scale=None, max_episode_length=300, enable_early_termination=True,
             termination_body_height=-0.5, termination_head_height=1.0, contact_bodies=("R_Ankle", "L_Ankle"),
             key_bodies=("R_Ankle", "L_Ankle", "L_Hand", "R_Hand"), body_pos_weights=None, reward_specs=None,
             shape_dim=11, ground_tolerance=0.0, task_mode=0, pd_mode=0, ball=None, **physics):
    names = [str(x) for x in model["body_names"]]
    nb = len(names)
    c = Cfg()
    c.sim_dt, c.substeps, c.control_freq_inv, c.gravity_z = sim_dt, substeps, control_freq_inv, gravity_z
    ph = dict(DEFAULT_PHYSICS)
    ph.update(physics)
    for k, v in ph.items():
        setattr(c, k, v)
    c.pd_tar_lim = pd_tar_lim
    c.res_force_scale = res_force_scale
    c.res_torque_scale = res_force_scale if res_torque_scale is None else res_torque_scale
    c.max_episode_length = int(max_episode_length)
    c.enable_early_termination = int(bool(enable_early_termination))
    th = [termination_body_height] * nb  # humanoid_smpl_im.py:217-224
    if "Head" in names:
        hid = names.index("Head")
        th[hid] = max(termination_head_height, th[hid])
    _fill(c.termination_height, th)
    _fill(c.contact_body, [1 if n in contact_bodies else 0 for n in names])
    w = [1.0] * nb
    for val, bodies in (body_pos_weights or {}).items():
        for b in bodies:
            w[names.index(b)] = float(val)
    _fill(c.body_pos_weight, w)
    rs = {'k_dof': 60, 'k_vel': 0.2, 'k_pos': 100, 'k_rot': 40, 'w_dof': 0.6, 'w_vel': 0.1, 'w_pos': 0.2, 'w_rot': 0.1}
    rs.update(reward_specs or {})
    for k, v in rs.items():
        setattr(c, k, float(v))
    c.num_key = len(key_bodies)
    _fill(c.key_body, [names.index(k) for k in key_bodies])
    c.shape_dim = shape_dim
    c.ground_tolerance = ground_tolerance
    c.task_mode, c.pd_mode = task_mode, pd_mode
    c.racket_body = names.index("Racket") if "Racket" in names else -1
    c.has_ball = 0
    _fill(c.racket_head_quat, (0.0, 0.0, 0.0, 1.0))
    if ball is not None:
        b = dict(DEFAULT_BALL)
        b.update(racket_head_from_prims(model))
        b.update(ball)
        _fill(c.racket_head_quat, b["racket_head_quat"])
        c.has_ball = 1
        for k in ("ball_mass", "ball_inertia", "ball_radius", "spin_scale", "ball_e_ground", "ball_mu_ground", "ball_e_racket",
                  "ball_mu_racket", "bounce_threshold_velocity", "racket_head_halfthick", "racket_head_radius"):
            setattr(c, k, b[k])
        _fill(c.racket_head_center, b["racket_head_center"])
        # optional ball contacts with the bodies / the racket handle (include/b200env.h; default off)
        c.ball_body_contact = int(bool(b.get("ball_body_contact", 0)))
        c.ball_e_body, c.ball_mu_body = float(b.get("ball_e_body", 0.45)), float(b.get("ball_mu_body", 0.6))
        _fill(c.racket_handle, racket_handle_from_prims(model))
    return c


def racket_handle_from_prims(model):
    """the thin cylinder of the Racket body (the grip, e.g. federer.xml fromto="0.5 0 0 0.15 0 0" size 0.016) as p0, p1, radius;
    zeros when the asset has none"""
    names = [str(x) for x in model["body_names"]]
    if "Racket" not in names or len(model["prims"]) == 0:
        return [0.0] * 7
    rows = [r for r in np.asarray(model["prims"]) if int(r[0]) == names.index("Racket")]
    if not rows:
        return [0.0] * 7
    r = min(rows, key=lambda x: x[7])            # the head slab is the wide one (radius 0.15), the handle the thin one
    if r[7] > 0.05:
        return [0.0] * 7
    return [float(x) for x in r[1:8]]


def racket_head_from_prims(model):
    """Racket head slab from the asset's geom primitives (model_compiler `prims` rows: body, p0, p1, radius): the head is the
    widest cylinder of the Racket body; its axis is the string-bed normal.  Returns {} when the model has no Racket."""
    names = [str(x) for x in model["body_names"]]
    if "Racket" not in names or "prims" not in model or len(model["prims"]) == 0:
        return {}
    rows = [r for r in np.asarray(model["prims"], np.float64) if int(r[0]) == names.index("Racket")]
    if not rows:
        return {}
    r = max(rows, key=lambda x: x[7])
    p0, p1 = r[1:4], r[4:7]
    axis = (p1 - p0) / np.linalg.norm(p1 - p0)
    y = np.array([0.0, 1.0, 0.0])                      # quaternion (xyzw) rotating +y onto the axis
    v, w = np.cross(y, axis), 1.0 + float(y @ axis)
    q = np.array([v[0], v[1], v[2], w])
    q /= np.linalg.norm(q)
    x, yq, z, w = q
    R = np.array([[1 - 2 * (yq * yq + z * z), 2 * (x * yq - z * w), 2 * (x * z + yq * w)],
                  [2 * (x * yq + z * w), 1 - 2 * (x * x + z * z), 2 * (yq * z - x * w)],
                  [2 * (x * z - yq * w), 2 * (yq * z + x * w), 1 - 2 * (x * x + yq * yq)]])
    return dict(racket_head_center=tuple(R.T @ (0.5 * (p0 + p1))), racket_head_halfthick=float(0.5 * np.linalg.norm(p1 - p0)),
                racket_head_radius=float(r[7]), racket_head_quat=tuple(q))


# tennis_ball.urdf (r 0.032, m 0.057, I 4e-5); restitution/friction: PhysX "average" combine of the material values the
# reference sets (humanoid_smpl_im_mvae.py:414-416,436-438: ball & racket 0.9 / 0.2 & 0.8; plane 0.5 / 1.0 from
# cfg/controller/federer.yaml:14-23); racket head = cylinder fromto "0 0 0 0 0.0425 0" size 0.15 (federer.xml:190)
DEFAULT_BALL = dict(ball_mass=0.057, ball_inertia=4e-5, ball_radius=0.032, spin_scale=5.0, ball_e_ground=0.7, ball_mu_ground=0.6,
                    ball_e_racket=0.9, ball_mu_racket=0.5, bounce_threshold_velocity=0.2, racket_head_center=(0.0, 0.02125, 0.0),
                    racket_head_halfthick=0.02125, racket_head_radius=0.15, racket_head_quat=(0.0, 0.0, 0.0, 1.0))


# ---------------------------------------------------------------- include/b200env_v2p.h
class V2PState(C.Structure):
    _fields_ = [
        ("n", C.c_int32), ("bodies_per_env", C.c_int32), ("ball_stride", C.c_int32), ("root_stride", C.c_int32),
        ("racket_body", C.c_int32), ("wrist_body", C.c_int32), ("grip_normal", C.c_float * 3),
        ("dual", C.c_int32), ("racket_body2", C.c_int32), ("wrist_body2", C.c_int32), ("grip_normal2", C.c_float * 3),
        ("rigid_body_state", C.c_void_p), ("root_states", C.c_void_p), ("ball_states", C.c_void_p),
        ("has_contact", C.c_void_p), ("has_contact_now", C.c_void_p),
        ("root_pos", C.c_void_p), ("root_vel", C.c_void_p), ("racket_pos", C.c_void_p), ("racket_vel", C.c_void_p),
        ("racket_normal", C.c_void_p), ("ball_pos", C.c_void_p), ("ball_vel", C.c_void_p), ("ball_vspin", C.c_void_p),
        ("only_mask", C.c_void_p),
    ]


class V2PCtrl(C.Structure):
    _fields_ = [
        ("n", C.c_int32), ("bodies_per_env", C.c_int32), ("ball_stride", C.c_int32), ("racket_body", C.c_int32),
        ("num_obs", C.c_int32), ("obs_traj_len", C.c_int32), ("use_target", C.c_int32), ("reward_type", C.c_int32),
        ("early_termination", C.c_int32), ("max_episode_length", C.c_int32), ("est_nx", C.c_int32), ("est_ny", C.c_int32),
        ("obs_only", C.c_int32), ("dual", C.c_int32), ("use_history", C.c_int32), ("advance", C.c_int32),
        ("scale_pos", C.c_float), ("scale_phase", C.c_float), ("scale_bounce_pos", C.c_float), ("scale_bounce_time", C.c_float),
        ("w_pos", C.c_float), ("w_ball_pos", C.c_float),
        ("court_min", C.c_float * 2), ("court_max", C.c_float * 2), ("est_params", C.c_float * 15),
        ("rigid_body_state", C.c_void_p), ("ball_states", C.c_void_p),
        ("root_pos", C.c_void_p), ("root_vel", C.c_void_p), ("racket_pos", C.c_void_p), ("racket_normal", C.c_void_p),
        ("ball_pos", C.c_void_p),
        ("has_contact", C.c_void_p), ("has_contact_now", C.c_void_p), ("has_bounce", C.c_void_p), ("has_bounce_now", C.c_void_p),
        ("bounce_pos", C.c_void_p), ("ball_traj", C.c_void_p), ("target_bounce_pos", C.c_void_p), ("phase", C.c_void_p),
        ("swing_type", C.c_void_p), ("swing_type_cycle", C.c_void_p), ("tar_action", C.c_void_p), ("tar_time", C.c_void_p),
        ("tar_time_total", C.c_void_p), ("progress_buf", C.c_void_p),
        ("est_x", C.c_void_p), ("est_y", C.c_void_p),
        ("bounce_in", C.c_void_p), ("est_bounce_in", C.c_void_p), ("reset_reaction", C.c_void_p), ("reset_recovery", C.c_void_p),
        ("est_bounce_pos", C.c_void_p), ("est_bounce_time", C.c_void_p), ("est_max_height", C.c_void_p), ("distance", C.c_void_p),
        ("obs_buf", C.c_void_p), ("rew_buf", C.c_void_p), ("sub_rewards", C.c_void_p),
        ("reset_buf", C.c_void_p), ("terminate_buf", C.c_void_p), ("ball_obs", C.c_void_p), ("touch_mask", C.c_void_p),
    ]


class V2PPreStep(C.Structure):
    _fields_ = [
        ("n", C.c_int32), ("num_actions", C.c_int32), ("num_latent", C.c_int32), ("num_res_dof", C.c_int32),
        ("random_walk_in_recovery", C.c_int32), ("vae_action_scale", C.c_float), ("residual_dof_scale", C.c_float), ("seed", C.c_uint64),
        ("actions", C.c_void_p), ("tar_action", C.c_void_p), ("step_counter", C.c_void_p), ("done_counter", C.c_void_p),
        ("mvae_actions", C.c_void_p), ("res_dof_actions", C.c_void_p),
    ]


class V2PStream(C.Structure):
    _fields_ = [
        ("n", C.c_int32), ("frames", C.c_int32), ("advance", C.c_int32), ("pad_", C.c_int32),
        ("clock", C.c_void_p), ("done_counter", C.c_void_p), ("offset", C.c_void_p), ("reseed_mask", C.c_void_p), ("seed", C.c_uint64),
        ("ring_rotmat", C.c_void_p), ("rotmat", C.c_void_p), ("ring_root_pos", C.c_void_p), ("root_pos", C.c_void_p),
        ("ring_racket_pos", C.c_void_p), ("racket_pos", C.c_void_p), ("ring_phase", C.c_void_p), ("phase", C.c_void_p),
        ("ring_swing_type", C.c_void_p), ("swing_type", C.c_void_p), ("ring_swing_type_cycle", C.c_void_p), ("swing_type_cycle", C.c_void_p),
    ]


class V2PTaskReset(C.Structure):
    _fields_ = [
        ("n", C.c_int32), ("pool_size", C.c_int32), ("ball_stride", C.c_int32), ("bodies_per_env", C.c_int32),
        ("reaction_nframes", C.c_int32), ("target_mode", C.c_int32), ("target_min", C.c_float * 3), ("target_max", C.c_float * 3),
        ("reset_reaction", C.c_void_p), ("reset_recovery", C.c_void_p),
        ("pool_rand", C.c_void_p), ("side_rand", C.c_void_p), ("frame_rand", C.c_void_p), ("target_seed", C.c_void_p),
        ("pool", C.c_void_p), ("ball_states", C.c_void_p), ("rigid_body_state", C.c_void_p),
        ("ball_pos", C.c_void_p), ("ball_vel", C.c_void_p), ("bounce_pos", C.c_void_p), ("ball_traj", C.c_void_p),
        ("est_bounce_pos", C.c_void_p), ("est_bounce_time", C.c_void_p), ("est_max_height", C.c_void_p), ("target_bounce_pos", C.c_void_p),
        ("has_bounce", C.c_void_p), ("has_contact", C.c_void_p), ("bounce_in", C.c_void_p), ("est_bounce_in", C.c_void_p),
        ("tar_time", C.c_void_p), ("tar_time_total", C.c_void_p), ("tar_action", C.c_void_p), ("num_reset_reaction", C.c_void_p),
        ("swing_type_cycle", C.c_void_p), ("ball_obs", C.c_void_p), ("obs_traj_len", C.c_int32), ("pad_", C.c_int32),
    ]


class V2PActorReset(C.Structure):
    _fields_ = [
        ("n", C.c_int32), ("num_dof", C.c_int32), ("bodies_per_env", C.c_int32), ("root_stride", C.c_int32),
        ("racket_body", C.c_int32), ("racket_parent", C.c_int32), ("racket_offset", C.c_float * 3),
        ("dual", C.c_int32), ("racket_offset2", C.c_float * 3), ("racket_parent2", C.c_int32), ("pad_", C.c_int32),
        ("env_ids", C.c_void_p),
        ("src_root_pos", C.c_void_p), ("src_root_rot", C.c_void_p), ("src_dof_pos", C.c_void_p), ("src_rb_pos", C.c_void_p),
        ("src_rb_rot", C.c_void_p),
        ("root_states", C.c_void_p), ("dof_state", C.c_void_p), ("rigid_body_state", C.c_void_p),
        ("prev_target_root_pos", C.c_void_p), ("prev_target_rb_rot", C.c_void_p), ("root_pos", C.c_void_p), ("root_vel", C.c_void_p),
        ("pd_target_dof_pos", C.c_void_p), ("target_root_pos", C.c_void_p),
        ("progress_buf", C.c_void_p), ("reset_buf", C.c_void_p), ("terminate_buf", C.c_void_p), ("mask", C.c_void_p),
    ]
