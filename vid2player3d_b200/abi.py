"""ctypes mirror of include/b200env.h, include/b200env_v2p.h and include/b200ball.h (structs, entry-point signatures, packing
helpers).  Product code: the native binding (native.py) and the tests' oracle wrapper both build their arguments from these."""
import ctypes as C

import numpy as np

MAX_BODIES, MAX_DOF, MAX_KEY = 32, 96, 8
ABI_VERSION = 11


# Pointer fields of the descriptor structs below carry the element type the header points at; native.fill refuses a tensor of any
# other dtype, tests/test_descriptor_fill.py holds the pointee types to the headers.  void* fields (and pointers to host structs)
# stay c_void_p.  Each struct also names the pointers that may be NULL (_nullable_) and the scalars a caller may omit, which stay 0
# (_defaults_).
class F32P(C.c_void_p):
    pointee = C.c_float


class I64P(C.c_void_p):
    pointee = C.c_int64


class U8P(C.c_void_p):
    pointee = C.c_uint8


class U32P(C.c_void_p):
    pointee = C.c_uint32


class I32P(C.c_void_p):
    pointee = C.c_int32


class F64P(C.c_void_p):
    pointee = C.c_double


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
        ("gts", F32P), ("grs", F32P), ("lrs", F32P), ("grvs", F32P), ("gravs", F32P),
        ("dvs", F32P), ("motion_lengths", F32P), ("num_frames", I64P), ("motion_dt", F32P),
        ("length_starts", I64P), ("min_verts_h", F32P),
        ("num_motions", C.c_int32), ("num_lib_bodies", C.c_int32), ("total_frames", C.c_int64),
    ]
    _nullable_, _defaults_ = (), ()


class Buffers(C.Structure):
    _fields_ = [
        ("root_states", F32P), ("actors_per_env", C.c_int32),
        ("dof_state", F32P), ("rigid_body_state", F32P), ("contact_forces", F32P),
        ("bodies_per_env", C.c_int32),
        ("obs_buf", F32P), ("num_obs", C.c_int32),
        ("rew_buf", F32P), ("sub_rewards", F32P), ("reset_buf", I64P), ("progress_buf", I64P),
        ("terminate_buf", I64P), ("motion_ids", I64P), ("ref_motion_times", F32P),
        ("motion_bodies", F32P),
        ("t_root_pos", F32P), ("t_root_rot", F32P), ("t_dof_pos", F32P), ("t_root_vel", F32P),
        ("t_root_ang_vel", F32P), ("t_dof_vel", F32P), ("t_key_pos", F32P), ("t_rb_pos", F32P),
        ("t_rb_rot", F32P),
        ("p_dof_pos", F32P), ("p_dof_vel", F32P), ("p_rb_pos", F32P), ("p_rb_rot", F32P),
        ("pd_targets", F32P), ("actions_used", F32P), ("num_actions", C.c_int32),
        ("has_bounce", U8P), ("has_bounce_now", U8P), ("bounce_pos", F32P), ("racket_hit_now", U8P),
        ("dof_force", F32P),
    ]
    _nullable_ = ("has_bounce", "has_bounce_now", "bounce_pos", "racket_hit_now", "dof_force")
    _defaults_ = ()


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


class ImPolicy(C.Structure):
    """b200_im_policy_t: the imitation policy's operand launch (b200env_im_policy_rows)"""
    _fields_ = [
        ("n", C.c_int32), ("num_obs", C.c_int32), ("num_frames", C.c_int32), ("feat_width", C.c_int32),
        ("context_padding", C.c_int32), ("context_length", C.c_int32), ("ld", C.c_int32), ("clip_obs", C.c_float), ("clip", C.c_float),
        ("pad_", C.c_int32),
        ("obs_buf", F32P), ("context_feat", F32P), ("step", I64P), ("mean", F32P), ("rstd", F32P), ("x", C.c_void_p), ("resid", F32P),
    ]
    _nullable_, _defaults_ = ("mean", "rstd"), ("clip", "pad_")


class LinearDesc(C.Structure):
    """b200nn_linear_desc_t (include/b200nn.h): one wgmma GEMM layer of libb200nn.so; nn.Linear fills it.  The noise fields (the
    sampled action: sigma per output column, seed, device step counter, done ticket) are NULL / 0 for a deterministic layer."""
    _fields_ = [("a", C.c_void_p), ("lda", C.c_int32), ("w", C.c_void_p), ("ldw", C.c_int32), ("bias", F32P), ("coef", F32P),
                ("out", C.c_void_p), ("ldo", C.c_int32), ("out_col0", C.c_int32), ("rows", C.c_int32), ("n", C.c_int32),
                ("n_padded", C.c_int32), ("k_padded", C.c_int32), ("num_experts", C.c_int32), ("act", C.c_int32), ("out_bf16", C.c_int32),
                ("out_min", C.c_float), ("out_max", C.c_float), ("resid", F32P), ("ld_resid", C.c_int32), ("resid_cols", C.c_int32),
                ("noise_sigma", F32P), ("noise_seed", C.c_uint64), ("noise_step", I64P), ("noise_done", U32P)]
    _nullable_ = ("coef", "resid", "noise_sigma", "noise_step", "noise_done")
    _defaults_ = ("out_min", "out_max", "ld_resid", "resid_cols", "noise_seed")


class PlayStats(C.Structure):
    """b200_play_stats_t: ImitatorPlayer.run's bookkeeping of one step (b200env_play_stats)"""
    _fields_ = [
        ("n", C.c_int32), ("max_log", C.c_int32), ("n_games", C.c_int64),
        ("rew", F32P), ("reset_buf", I64P), ("cr", F32P), ("steps", F32P), ("prev_dones", F32P), ("totals", F64P), ("log", F64P),
        ("games", I64P), ("step", I64P), ("queue_games", C.c_int64),
    ]
    _nullable_, _defaults_ = (), ("queue_games",)


class ImMotionQueue(C.Structure):
    """b200_im_motion_queue_t: the motion queue of an imitation test run (b200env_im_motion_queue)"""
    _fields_ = [
        ("n", C.c_int32), ("num_motions", C.c_int32), ("queue_len", C.c_int64), ("shape_dim", C.c_int32), ("pad_", C.c_int32),
        ("reset_buf", I64P), ("lib_motion_bodies", F32P), ("motion_ids", I64P), ("motion_bodies", F32P), ("entry", I64P), ("mask", U8P),
        ("idle", U8P), ("cursor", I64P), ("game_env", I64P), ("game_start_step", I64P), ("step", I64P), ("games", I64P),
        ("prev_dones", F32P), ("env_flags", I32P), ("motion_asset", I32P), ("env_asset", I32P),
    ]
    _nullable_, _defaults_ = ("games", "env_flags", "motion_asset", "env_asset"), ("pad_",)


class ResampleMotions(C.Structure):
    """b200_resample_motions_t: the training resample of the finished envs' motions (b200env_resample_motions)"""
    _fields_ = [
        ("n", C.c_int32), ("num_motions", C.c_int32), ("shape_dim", C.c_int32), ("pad_", C.c_int32), ("seed", C.c_uint64),
        ("mask", U8P), ("progress_buf", I64P), ("terminate_buf", I64P), ("cdf", F64P), ("lib_motion_bodies", F32P), ("motion_ids", I64P),
        ("motion_bodies", F32P), ("counter", I64P), ("done", U32P), ("tries", I64P), ("fails", I64P), ("motion_asset", I32P),
        ("env_asset", I32P),
    ]
    _nullable_, _defaults_ = ("tries", "fails", "motion_asset", "env_asset"), ("pad_",)


class MotionWeights(C.Structure):
    """b200_motion_weights_t: the resample's motion distribution rebuilt from the failure counts (b200env_motion_weights)"""
    _fields_ = [("num_motions", C.c_int32), ("pad_", C.c_int32), ("h", C.c_double), ("base", F32P), ("tries", I64P), ("fails", I64P),
                ("rate", F64P), ("cdf", F64P)]
    _nullable_, _defaults_ = ("base", "tries", "fails", "rate"), ("pad_",)


class SetEnvAssets(C.Structure):
    """b200_set_env_assets_t: the assets of a mixed-plan handle's envs, re-pointed on the device (b200env_set_env_assets)"""
    _fields_ = [("n", C.c_int32), ("pad_", C.c_int32), ("env_asset", I32P), ("error", I32P)]
    _nullable_, _defaults_ = (), ("pad_",)


class ImRecord(C.Structure):
    """b200_im_record_t: one recorded viewer frame of HumanoidSMPLIMVis (b200env_im_record)"""
    _fields_ = [
        ("n_rec", C.c_int32), ("num_envs", C.c_int32), ("num_bodies", C.c_int32), ("num_lib_bodies", C.c_int32), ("nd", C.c_int32),
        ("cap", C.c_int32), ("init", C.c_int32), ("pad_", C.c_int32),
        ("env_ids", I64P), ("rigid_body_state", F32P), ("dof_state", F32P), ("p_dof_pos", F32P), ("p_rb_pos", F32P), ("p_rb_rot", F32P),
        ("reset_buf", I64P), ("motion_ids", I64P), ("qpos", F32P), ("rec_motion_ids", I64P), ("rec_reset", I64P), ("frame", I64P),
        ("done", U32P), ("games", I64P),
    ]
    _nullable_, _defaults_ = ("games",), ("pad_",)


class ImMotionStats(C.Structure):
    """b200_im_motion_stats_t: the per-motion meters of one test step of HumanoidSMPLIMVis (b200env_im_motion_stats)"""
    _fields_ = [
        ("n", C.c_int32), ("num_motions", C.c_int32), ("num_bodies", C.c_int32), ("num_lib_bodies", C.c_int32),
        ("rew", F32P), ("sub_rewards", F32P), ("reset_buf", I64P), ("terminate_buf", I64P), ("rigid_body_state", F32P),
        ("target_rb_pos", F32P), ("motion_start", I64P), ("motion_envs", I64P), ("env_sums", F64P), ("env_flags", I32P),
        ("counts", I64P), ("sums", F64P), ("games", I64P),
        ("env_pose", F64P), ("pose_hist", F32P), ("pose_fill", I32P), ("pose_sums", F64P), ("success", I64P),
        ("success_threshold", C.c_double),
    ]
    _nullable_ = ("games", "env_pose", "pose_hist", "pose_fill", "pose_sums", "success")
    _defaults_ = ("success_threshold",)


class ImMotionQueueStats(C.Structure):
    """b200_im_motion_queue_stats_t: the per-motion meters folded by queue entry (b200env_im_motion_queue_stats); the fields of
    b200_im_motion_stats_t (its first member) and env_entry"""
    _fields_ = ImMotionStats._fields_ + [("env_entry", I64P)]
    _nullable_ = ImMotionStats._nullable_ + ("motion_start", "motion_envs")
    _defaults_ = ImMotionStats._defaults_


# the context window's transform program (include/b200env.h: b200_motion_context_t), appended to b200_reset_masked_t and
# b200_motion_context_t; zero = no transforms
XF_MASK_JOINTS, XF_NOISY_JOINTS, XF_MASK_RANDOM_JOINTS = 1, 2, 3
_XF_FIELDS = [("xf_ops", C.c_int32 * 3), ("xf_joint_mask", C.c_uint32), ("xf_noisy_prob", C.c_float), ("xf_noise_std", C.c_float),
              ("xf_conf_std", C.c_float), ("xf_min_conf", C.c_float), ("xf_random_prob", C.c_float), ("feat_width", C.c_int32)]
_XF_DEFAULTS = tuple(name for name, _ in _XF_FIELDS)
TRANSFORMS = {"mask_joints": XF_MASK_JOINTS, "noisy_joints": XF_NOISY_JOINTS, "mask_random_joints": XF_MASK_RANDOM_JOINTS}


def transform_program(transform_specs, body_names, num_bodies):
    """the xf_* fields of cfg.env.transform_specs (HumanoidSMPLIM._transform_target, humanoid_smpl_im.py:565-592), ops in the dict's
    order; body_names[:num_bodies] are the bodies of joint_conf.  Raises ValueError on an unknown or repeated transform, a joint that
    is not one of those bodies, a prob outside [0, 1], noise_std < 0, conf_std <= 0 or a missing key; the refusals of the C side."""
    ops, p = [], dict(xf_joint_mask=0, xf_noisy_prob=0.0, xf_noise_std=0.0, xf_conf_std=0.0, xf_min_conf=0.0, xf_random_prob=0.0)
    if num_bodies > 32:
        raise ValueError(f"transform_specs: {num_bodies} bodies, the device transforms serve at most 32")
    for name, specs in (transform_specs or {}).items():
        if name not in TRANSFORMS:
            raise ValueError(f"transform_specs: unknown transform {name!r} (known: {', '.join(TRANSFORMS)})")
        ops.append(TRANSFORMS[name])
        try:
            if name == "mask_joints":
                for j in specs["joints"]:
                    if j not in body_names[:num_bodies]:
                        raise ValueError(f"transform_specs.mask_joints: {j!r} is not a body of the humanoid")
                    p["xf_joint_mask"] |= 1 << body_names.index(j)
            elif name == "noisy_joints":
                p.update(xf_noisy_prob=float(specs["prob"]), xf_noise_std=float(specs["noise_std"]), xf_conf_std=float(specs["conf_std"]),
                         xf_min_conf=float(specs["min_conf"]))
                if not p["xf_noise_std"] >= 0:
                    raise ValueError(f"transform_specs.noisy_joints: noise_std {specs['noise_std']} < 0")
                if not p["xf_conf_std"] > 0:
                    raise ValueError(f"transform_specs.noisy_joints: conf_std {specs['conf_std']} must be > 0")
            else:
                p["xf_random_prob"] = float(specs["prob"])
        except KeyError as ex:
            raise ValueError(f"transform_specs.{name}: missing {ex.args[0]!r}") from None
        prob = p["xf_noisy_prob"] if name == "noisy_joints" else p["xf_random_prob"]
        if name != "mask_joints" and not 0.0 <= prob <= 1.0:
            raise ValueError(f"transform_specs.{name}: prob {prob} outside [0, 1]")
    return dict(p, xf_ops=ops + [0] * (3 - len(ops)))


class ResetMasked(C.Structure):
    """b200_reset_masked_t: the mask-driven reset of the imitation task (b200env_reset_masked)"""
    _fields_ = [
        ("sample_time", C.c_int32), ("truncate", C.c_float), ("ref_prob", C.c_float), ("num_frames", C.c_int32),
        ("first_frame", C.c_int32), ("dt", C.c_float), ("seed", C.c_uint64),
        ("mask", U8P), ("counter", I64P), ("init_root", F32P), ("init_dof_pos", F32P), ("init_dof_vel", F32P), ("reset_times", F32P),
        ("context_feat", F32P), ("context_mask", U8P), ("work", I32P),
    ] + _XF_FIELDS + [("step", I64P), ("context_length", C.c_int32), ("pad_", C.c_int32)]
    _nullable_, _defaults_ = ("init_root", "init_dof_pos", "init_dof_vel", "step"), _XF_DEFAULTS + ("context_length", "pad_")


class MotionState(C.Structure):
    """b200_motion_state_t: MoCap states of (id, time) pairs (b200env_motion_state)"""
    _fields_ = [
        ("n", C.c_int32), ("pad_", C.c_int32), ("motion_ids", I64P), ("motion_times", F32P),
        ("root_pos", F32P), ("root_rot", F32P), ("dof_pos", F32P), ("root_vel", F32P), ("root_ang_vel", F32P), ("dof_vel", F32P),
        ("key_pos", F32P), ("rb_pos", F32P), ("rb_rot", F32P),
    ]
    _nullable_ = ("root_pos", "root_rot", "dof_pos", "root_vel", "root_ang_vel", "dof_vel", "key_pos", "rb_pos", "rb_rot")
    _defaults_ = ("pad_",)


class MotionContext(C.Structure):
    """b200_motion_context_t: the MoCap context window of listed envs (b200env_motion_context)"""
    _fields_ = [
        ("n", C.c_int32), ("num_frames", C.c_int32), ("first_frame", C.c_int32), ("dt", C.c_float),
        ("env_ids", I64P), ("motion_ids", I64P), ("motion_times", F32P), ("context_feat", F32P), ("context_mask", U8P),
    ] + _XF_FIELDS + [("seed", C.c_uint64), ("counter", I64P)]
    _nullable_, _defaults_ = ("env_ids", "counter"), _XF_DEFAULTS + ("seed",)


class ObsImitation(C.Structure):
    """b200_obs_imitation_t: the imitation observation from contiguous gathers (b200env_obs_imitation)"""
    _fields_ = [
        ("n", C.c_int32), ("local_root_obs", C.c_int32), ("root_height_obs", C.c_int32), ("jpos", C.c_int32),
        ("body_pos", F32P), ("body_rot", F32P), ("target_pos", F32P), ("target_rot", F32P), ("dof_pos", F32P), ("dof_vel", F32P),
        ("target_dof_pos", F32P), ("body_vel", F32P), ("body_ang_vel", F32P), ("motion_bodies", F32P), ("obs", F32P),
    ]
    _nullable_, _defaults_ = (), ()


class ObsRows(C.Structure):
    """b200_obs_rows_t: the imitation observation from the state rows, and the policy's bf16 operand row (b200env_obs_imitation_rows;
    b200env_obs_imitation_rows_dual: one block of rows per player, clamp1 = player 1's clamp)"""
    _fields_ = [
        ("n", C.c_int32), ("bodies_per_env", C.c_int32), ("local_root_obs", C.c_int32), ("root_height_obs", C.c_int32),
        ("jpos", C.c_int32), ("ld_bf16", C.c_int32), ("clamp", C.c_float), ("clamp1", C.c_float),
        ("rigid_body_state", F32P), ("dof_state", F32P), ("target_pos", F32P), ("target_rot", F32P), ("target_dof_pos", F32P),
        ("motion_bodies", F32P), ("obs", F32P), ("obs_bf16", C.c_void_p), ("mean", F32P), ("rstd", F32P),
    ]
    _nullable_, _defaults_ = ("obs_bf16", "mean", "rstd"), ("clamp1",)


# ---------------------------------------------------------------- include/b200env_v2p.h
class V2PSmpl(C.Structure):
    _fields_ = [
        ("n", C.c_int32), ("num_rest", C.c_int32), ("dt", C.c_float), ("pad_", C.c_int32),
        ("root_pos", F32P), ("joint_rotmat", F32P), ("rest", F32P), ("parents", I32P), ("smpl_2_mujoco", I32P),
        ("prev_root_pos", F32P), ("prev_rb_rot", F32P),
        ("root_rot", F32P), ("dof_pos", F32P), ("root_vel", F32P), ("root_ang_vel", F32P), ("dof_vel", F32P), ("rb_pos", F32P),
        ("rb_rot", F32P), ("prev_root_pos_update", F32P), ("target_root_pos_out", F32P), ("only_mask", U8P),
    ]
    _nullable_ = ("prev_root_pos", "prev_rb_rot", "prev_root_pos_update", "target_root_pos_out", "only_mask")
    _defaults_ = ("pad_",)


class V2PHead(C.Structure):
    _fields_ = [
        ("n", C.c_int32), ("head_body", C.c_int32),
        ("rb_pos", F32P), ("rb_rot", F32P), ("ball_pos", F32P), ("root_pos", F32P), ("joint_rotmat", F32P),
    ]
    _nullable_, _defaults_ = (), ()


class V2PAero(C.Structure):
    _fields_ = [
        ("n", C.c_int32), ("stride", C.c_int32), ("substeps", C.c_int32), ("spin_scale", C.c_float),
        ("ball_states", F32P), ("has_bounce", U8P), ("has_bounce_now", U8P), ("bounce_pos", F32P), ("force", F32P),
    ]
    _nullable_, _defaults_ = (), ()


class V2PBallReset(C.Structure):
    _fields_ = [
        ("n", C.c_int32), ("stride", C.c_int32),
        ("env_ids", I64P), ("pool_index", I64P), ("pool", F32P), ("ball_states", F32P), ("ball_pos", F32P), ("ball_vel", F32P),
        ("has_bounce", U8P), ("bounce_pos", F32P), ("has_contact", U8P), ("traj", F32P),
    ]
    _nullable_, _defaults_ = (), ()


class V2PCtrlReset(C.Structure):
    _fields_ = [
        ("n", C.c_int32), ("pad_", C.c_int32),
        ("mask", U8P), ("progress_buf", I64P), ("reset_buf", I64P), ("terminate_buf", I64P), ("num_reset_reaction", I64P),
        ("distance", F32P), ("num_reset", I64P),
    ]
    _nullable_, _defaults_ = (), ("pad_",)


class V2PInEst(C.Structure):
    _fields_ = [
        ("n", C.c_int32), ("stride", C.c_int32), ("table_rows", C.c_int64), ("params", C.c_double * 12),
        ("contact_ids", I64P), ("ball_states", F32P), ("table", F32P), ("traj", F32P), ("states_in", F32P), ("states_out", F32P),
    ]
    _nullable_, _defaults_ = (), ()


class V2PState(C.Structure):
    _fields_ = [
        ("n", C.c_int32), ("bodies_per_env", C.c_int32), ("ball_stride", C.c_int32), ("root_stride", C.c_int32),
        ("racket_body", C.c_int32), ("wrist_body", C.c_int32), ("grip_normal", C.c_float * 3),
        ("dual", C.c_int32), ("racket_body2", C.c_int32), ("wrist_body2", C.c_int32), ("grip_normal2", C.c_float * 3),
        ("rigid_body_state", F32P), ("root_states", F32P), ("ball_states", F32P),
        ("has_contact", U8P), ("has_contact_now", U8P),
        ("root_pos", F32P), ("root_vel", F32P), ("racket_pos", F32P), ("racket_vel", F32P),
        ("racket_normal", F32P), ("ball_pos", F32P), ("ball_vel", F32P), ("ball_vspin", F32P),
        ("only_mask", U8P),
    ]
    _nullable_, _defaults_ = ("only_mask",), ()


class V2PCtrl(C.Structure):
    _fields_ = [
        ("n", C.c_int32), ("bodies_per_env", C.c_int32), ("ball_stride", C.c_int32), ("racket_body", C.c_int32),
        ("num_obs", C.c_int32), ("obs_traj_len", C.c_int32), ("use_target", C.c_int32), ("reward_type", C.c_int32),
        ("early_termination", C.c_int32), ("max_episode_length", C.c_int32), ("est_nx", C.c_int32), ("est_ny", C.c_int32),
        ("obs_only", C.c_int32), ("dual", C.c_int32), ("use_history", C.c_int32), ("advance", C.c_int32),
        ("scale_pos", C.c_float), ("scale_phase", C.c_float), ("scale_bounce_pos", C.c_float), ("scale_bounce_time", C.c_float),
        ("w_pos", C.c_float), ("w_ball_pos", C.c_float),
        ("court_min", C.c_float * 2), ("court_max", C.c_float * 2), ("est_params", C.c_float * 15),
        ("rigid_body_state", F32P), ("ball_states", F32P),
        ("root_pos", F32P), ("root_vel", F32P), ("racket_pos", F32P), ("racket_normal", F32P),
        ("ball_pos", F32P),
        ("has_contact", U8P), ("has_contact_now", U8P), ("has_bounce", U8P), ("has_bounce_now", U8P),
        ("bounce_pos", F32P), ("ball_traj", F32P), ("target_bounce_pos", F32P), ("phase", F32P),
        ("swing_type", I64P), ("swing_type_cycle", I64P), ("tar_action", I64P), ("tar_time", I64P),
        ("tar_time_total", I64P), ("progress_buf", I64P),
        ("est_x", F32P), ("est_y", F32P),
        ("bounce_in", U8P), ("est_bounce_in", U8P), ("reset_reaction", U8P), ("reset_recovery", U8P),
        ("est_bounce_pos", F32P), ("est_bounce_time", F32P), ("est_max_height", F32P), ("distance", F32P),
        ("obs_buf", F32P), ("rew_buf", F32P), ("sub_rewards", F32P),
        ("reset_buf", I64P), ("terminate_buf", I64P), ("ball_obs", F32P), ("touch_mask", U8P),
        ("eval", C.c_int32), ("eval_episode_length", C.c_int32), ("ball_vel", F32P),
        ("meter_sum", F32P), ("meter_avg", F32P), ("meter_max", F32P), ("meter_count", I64P),
        ("policy_x", C.c_void_p), ("policy_mean", F32P), ("policy_rstd", F32P), ("policy_ld", C.c_int32),
        ("policy_dual", C.c_int32), ("policy_clip_obs", C.c_float), ("policy_clip", C.c_float * 2), ("pad_", C.c_int32),
    ]
    _nullable_ = ("est_x", "est_y", "ball_obs", "touch_mask", "ball_vel", "meter_sum", "meter_avg", "meter_max", "meter_count",
                  "policy_x", "policy_mean", "policy_rstd")
    _defaults_ = ("obs_only", "dual", "use_history", "advance", "eval", "eval_episode_length", "policy_ld", "policy_dual",
                  "policy_clip_obs", "policy_clip", "pad_")


class V2PPreStep(C.Structure):
    _fields_ = [
        ("n", C.c_int32), ("num_actions", C.c_int32), ("num_latent", C.c_int32), ("num_res_dof", C.c_int32),
        ("random_walk_in_recovery", C.c_int32), ("vae_action_scale", C.c_float), ("residual_dof_scale", C.c_float), ("seed", C.c_uint64),
        ("actions", F32P), ("tar_action", I64P), ("step_counter", I64P), ("done_counter", U32P),
        ("mvae_actions", F32P), ("res_dof_actions", F32P),
    ]
    _nullable_, _defaults_ = ("res_dof_actions",), ()


class V2PStream(C.Structure):
    _fields_ = [
        ("n", C.c_int32), ("frames", C.c_int32), ("advance", C.c_int32), ("pad_", C.c_int32),
        ("clock", I64P), ("done_counter", U32P), ("offset", I64P), ("reseed_mask", U8P), ("seed", C.c_uint64),
        ("ring_rotmat", F32P), ("rotmat", F32P), ("ring_root_pos", F32P), ("root_pos", F32P),
        ("ring_racket_pos", F32P), ("racket_pos", F32P), ("ring_phase", F32P), ("phase", F32P),
        ("ring_swing_type", I64P), ("swing_type", I64P), ("ring_swing_type_cycle", I64P), ("swing_type_cycle", I64P),
    ]
    _nullable_, _defaults_ = ("reseed_mask",), ("pad_",)


class V2PTaskReset(C.Structure):
    _fields_ = [
        ("n", C.c_int32), ("pool_size", C.c_int32), ("ball_stride", C.c_int32), ("bodies_per_env", C.c_int32),
        ("reaction_nframes", C.c_int32), ("target_mode", C.c_int32), ("target_min", C.c_float * 3), ("target_max", C.c_float * 3),
        ("reset_reaction", U8P), ("reset_recovery", U8P),
        ("pool_rand", I64P), ("side_rand", I64P), ("frame_rand", I64P), ("target_seed", F32P),
        ("pool", F32P), ("ball_states", F32P), ("rigid_body_state", F32P),
        ("ball_pos", F32P), ("ball_vel", F32P), ("bounce_pos", F32P), ("ball_traj", F32P),
        ("est_bounce_pos", F32P), ("est_bounce_time", F32P), ("est_max_height", F32P), ("target_bounce_pos", F32P),
        ("has_bounce", U8P), ("has_contact", U8P), ("bounce_in", U8P), ("est_bounce_in", U8P),
        ("tar_time", I64P), ("tar_time_total", I64P), ("tar_action", I64P), ("num_reset_reaction", I64P),
        ("swing_type_cycle", I64P), ("ball_obs", F32P), ("obs_traj_len", C.c_int32), ("pad_", C.c_int32),
        ("pool_cursor", I64P),
    ]
    _nullable_, _defaults_ = ("ball_obs", "pool_cursor"), ("obs_traj_len", "pad_")


BSTATS_COLS = 5                   # B200V2P_BSTATS_COLS: recoveries, hits, forehands, bounce_in, bounce-in error in 2^-24 m
BSTATS_FIX_SCALE = float(1 << 24)  # B200V2P_BSTATS_FIX_SCALE


class V2PBallStats(C.Structure):
    """b200v2p_bstats_t: the per-row results of the fixed test set (b200v2p_eval_ball_stats), in its draws form (reset_reaction,
    row_served) or its events form (reset_recovery and the fields after it); the entry point refuses a form with a field missing"""
    _fields_ = [
        ("n", C.c_int32), ("pool_size", C.c_int32), ("pool_cursor", I64P), ("reset_reaction", U8P), ("row_served", I64P),
        ("reset_recovery", U8P), ("has_contact", U8P), ("swing_type_cycle", I64P), ("est_bounce_in", U8P), ("est_bounce_pos", F32P),
        ("target_bounce_pos", F32P), ("buckets", I64P),
    ]
    _nullable_ = ("reset_reaction", "row_served", "reset_recovery", "has_contact", "swing_type_cycle", "est_bounce_in", "est_bounce_pos",
                  "target_bounce_pos", "buckets")
    _defaults_ = ()


RSTATS_HIST = 65                  # B200V2P_RSTATS_HIST: shots per rally 0..63, then 64 or more
RSTATS_CAUSES = ("behind", "double_bounce", "out")   # B200V2P_RSTATS_CAUSES, in the order of the ends columns
RSTATS_PLAYER = ("faced", "hits", "forehands")       # columns of the player counts


class V2PRallyStats(C.Structure):
    """b200v2p_rstats_t: the rally results of the dual test run (b200v2p_eval_rally_stats): the post launch's flags, the per-pair state
    and the int64 accumulators; every pointer is required"""
    _fields_ = [
        ("n", C.c_int32), ("pad_", C.c_int32), ("tar_action", I64P), ("has_contact", U8P), ("has_bounce", U8P), ("bounce_in", U8P),
        ("ball_pos", F32P), ("root_pos", F32P), ("swing_type_cycle", I64P), ("progress_buf", I64P), ("pair_open", U8P),
        ("pair_hits", I64P), ("totals", I64P), ("ends", I64P), ("player", I64P), ("shots_hist", I64P),
    ]
    _nullable_ = ()
    _defaults_ = ("pad_",)


class V2PActorReset(C.Structure):
    _fields_ = [
        ("n", C.c_int32), ("num_dof", C.c_int32), ("bodies_per_env", C.c_int32), ("root_stride", C.c_int32),
        ("racket_body", C.c_int32), ("racket_parent", C.c_int32), ("racket_offset", C.c_float * 3),
        ("dual", C.c_int32), ("racket_offset2", C.c_float * 3), ("racket_parent2", C.c_int32), ("pad_", C.c_int32),
        ("env_ids", I64P),
        ("src_root_pos", F32P), ("src_root_rot", F32P), ("src_dof_pos", F32P), ("src_rb_pos", F32P),
        ("src_rb_rot", F32P),
        ("root_states", F32P), ("dof_state", F32P), ("rigid_body_state", F32P),
        ("prev_target_root_pos", F32P), ("prev_target_rb_rot", F32P), ("root_pos", F32P), ("root_vel", F32P),
        ("pd_target_dof_pos", F32P), ("target_root_pos", F32P),
        ("progress_buf", I64P), ("reset_buf", I64P), ("terminate_buf", I64P), ("mask", U8P),
    ]
    _nullable_, _defaults_ = ("mask",), ("dual", "racket_offset2", "racket_parent2", "pad_")


class V2PRec(C.Structure):
    _fields_ = [
        ("n", C.c_int32), ("cap", C.c_int32), ("row_counter", I64P), ("done_counter", U32P), ("progress_buf", I64P),
        ("joint_rot", F32P), ("root_pos", F32P), ("ball_pos", F32P), ("target_pos", F32P), ("phase", F32P),
        ("swing_type", I64P), ("tar_action", I64P),
        ("rec_joint_rot", F32P), ("rec_root_pos", F32P), ("rec_ball_pos", F32P), ("rec_target_pos", F32P),
        ("rec_phase", F32P), ("rec_swing_type", I64P), ("rec_tar_action", I64P),
    ]
    _nullable_ = ("row_counter", "done_counter", "progress_buf", "target_pos", "tar_action", "rec_target_pos", "rec_tar_action")
    _defaults_ = ()


class V2PBest(C.Structure):
    _fields_ = [
        ("n", C.c_int32), ("cap", C.c_int32), ("num_eg", C.c_int32), ("pad_", C.c_int32),
        ("reset_buf", I64P), ("progress_buf", I64P), ("distance", F32P),
        ("list_len", I64P), ("order", I64P), ("best_distance", F32P), ("best_env", I64P),
        ("best_nframes", I64P), ("copy_slot", I64P),
        ("rec_joint_rot", F32P), ("rec_root_pos", F32P), ("rec_ball_pos", F32P), ("rec_phase", F32P),
        ("rec_swing_type", I64P), ("rec_tar_action", I64P),
        ("best_joint_rot", F32P), ("best_root_pos", F32P), ("best_ball_pos", F32P), ("best_phase", F32P),
        ("best_swing_type", I64P), ("best_tar_action", I64P),
    ]
    _nullable_, _defaults_ = (), ("pad_",)


class V2PBhProb(C.Structure):
    _fields_ = [
        ("joint_rot", C.c_void_p), ("phase", C.c_void_p), ("swing_type", I64P), ("rest", C.c_void_p), ("out", C.c_void_p),
        ("T", C.c_int64), ("swing_type_len", C.c_int64), ("righthand", C.c_int32), ("pad_", C.c_int32),
    ]


class V2PBhFix(C.Structure):
    _fields_ = [
        ("num_problems", C.c_int32), ("iters", C.c_int32), ("problems", C.c_void_p), ("scratch", C.c_void_p), ("scratch_bytes", C.c_int64),
        ("losses", C.c_void_p), ("precision", C.c_int32), ("pad_", C.c_int32),
    ]


BHFIX_FRAME_WORDS = 75    # B200V2P_BHFIX_FRAME_WORDS


def bhfix_scratch_bytes(Ts, scalar_bytes):
    """B200V2P_BHFIX_SCRATCH_BYTES for problems of T = Ts"""
    al = lambda x: (x + 255) // 256 * 256  # noqa: E731
    F = sum((int(t) + 31) // 32 * 32 for t in Ts)
    return al(len(Ts) * C.sizeof(V2PBhProb)) + al(4 * F) + F * BHFIX_FRAME_WORDS * scalar_bytes


# ---------------------------------------------------------------- entry points of libb200env.so
# name -> (restype, argtypes) of every function include/b200env.h, include/b200env_v2p.h and include/b200ball.h declare; native.lib()
# applies all of them when it loads the library, so an argument too many or too few, or one that does not convert to its C type,
# raises ctypes.ArgumentError at the call instead of reaching the library as an undefined register.  Pointers and opaque handles
# are c_void_p.  tests/test_host.py holds the table to the headers.
_i32, _i64, _p = C.c_int32, C.c_int64, C.c_void_p
SIGNATURES = {
    # include/b200env.h
    "b200env_abi_version": (C.c_int, []),
    "b200env_last_error": (C.c_char_p, []),
    "b200env_create": (C.c_int, [_p, _p, _p, _i32, _i32, _p]),
    "b200env_destroy": (C.c_int, [_p]),
    "b200env_bind": (C.c_int, [_p, _p]),
    "b200env_set_motion_lib": (C.c_int, [_p, _p]),
    "b200env_step": (C.c_int, [_p, _p, _p]),
    "b200env_reset": (C.c_int, [_p, _p, _p, _i32, _p]),
    "b200env_reset_masked": (C.c_int, [_p, _p, _p]),
    "b200env_motion_state": (C.c_int, [_p, _p, _p]),
    "b200env_obs_imitation": (C.c_int, [_p, _p, _p]),
    "b200env_obs_imitation_rows": (C.c_int, [_p, _p, _p]),
    "b200env_obs_imitation_rows_dual": (C.c_int, [_p, _p, _p]),
    "b200env_physics_only": (C.c_int, [_p, _i32, _i32, _i32, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p]),
    "b200env_motion_context": (C.c_int, [_p, _p, _p]),
    "b200env_reset_masked_desc_size": (_i32, []),
    "b200env_motion_context_desc_size": (_i32, []),
    "b200env_im_policy_rows": (C.c_int, [_p, _p, _p]),
    "b200env_play_stats": (C.c_int, [_p, _p]),
    "b200env_play_stats_desc_size": (_i32, []),
    "b200env_im_motion_queue": (C.c_int, [_p, _p]),
    "b200env_im_motion_queue_desc_size": (_i32, []),
    "b200env_resample_motions": (C.c_int, [_p, _p]),
    "b200env_resample_motions_desc_size": (_i32, []),
    "b200env_motion_weights": (C.c_int, [_p, _p]),
    "b200env_motion_weights_desc_size": (_i32, []),
    "b200env_im_motion_queue_stats": (C.c_int, [_p, _p]),
    "b200env_im_motion_queue_stats_desc_size": (_i32, []),
    "b200env_im_record": (C.c_int, [_p, _p]),
    "b200env_im_record_desc_size": (_i32, []),
    "b200env_im_motion_stats": (C.c_int, [_p, _p]),
    "b200env_im_motion_stats_desc_size": (_i32, []),
    "b200env_set_env_slice": (C.c_int, [_p, _i32, _i32]),
    "b200env_set_hull_faces": (C.c_int, [_p, _p, _p, _p, _i32]),
    "b200env_kernel_form": (_i32, [_p]),
    "b200env_physics_launch_shape": (C.c_int, [_p, _p, _p]),
    "b200env_create_assets": (C.c_int, [_p, _p, _i32, _p, _p, _i32, _i32, _p]),
    "b200env_plan_assets": (C.c_int, [_p, _i32, _i32, _i32, _p, _p, _p, _p, _p]),
    "b200env_plan_assets_mixed": (C.c_int, [_p, _i32, _i32, _i32, _p, _p, _p, _p, _p]),
    "b200env_choose_asset_plan": (C.c_int, [_p, _i32, _i32, _i32, _p]),
    "b200env_asset_plan": (C.c_int, [_p, _p, _p, _p, _p, _p, _p, _p]),
    "b200env_fix_mixed_plan": (C.c_int, [_p]),
    "b200env_set_env_assets": (C.c_int, [_p, _p, _p]),
    "b200env_set_env_assets_desc_size": (_i32, []),
    "b200env_launch_count": (_i64, [_p]),
    "b200env_set_kernel_timing": (C.c_int, [_p, _i32]),
    "b200env_kernel_ms": (C.c_int, [_p, _p, _p]),
    # include/b200env_v2p.h
    "b200v2p_last_error": (C.c_char_p, []),
    "b200v2p_smpl_to_sim": (C.c_int, [_p, _p]),
    "b200v2p_fix_head": (C.c_int, [_p, _p]),
    "b200v2p_ball_aero": (C.c_int, [_p, _p]),
    "b200v2p_ball_reset": (C.c_int, [_p, _p]),
    "b200v2p_update_state": (C.c_int, [_p, _p]),
    "b200v2p_controller_post": (C.c_int, [_p, _p]),
    "b200v2p_pre_step": (C.c_int, [_p, _p]),
    "b200v2p_ctrl_reset": (C.c_int, [_p, _p]),
    "b200v2p_stream_gather": (C.c_int, [_p, _p]),
    "b200v2p_ball_in_estimate": (C.c_int, [_p, _p]),
    "b200v2p_task_reset": (C.c_int, [_p, _p]),
    "b200v2p_task_reset_desc_size": (_i32, []),
    "b200v2p_eval_ball_stats": (C.c_int, [_p, _p]),
    "b200v2p_eval_ball_stats_desc_size": (_i32, []),
    "b200v2p_eval_rally_stats": (C.c_int, [_p, _p]),
    "b200v2p_eval_rally_stats_desc_size": (_i32, []),
    "b200v2p_actor_reset": (C.c_int, [_p, _p]),
    "b200v2p_eval_record": (C.c_int, [_p, _p]),
    "b200v2p_eval_best": (C.c_int, [_p, _p]),
    "b200v2p_backhand_fix": (C.c_int, [_p, _p]),
    # include/b200ball.h
    "b200ball_simulate": (C.c_int, [_p, _i64, _i32, _p, _p, _p, _p, _p, _p, _p, _p]),
    "b200ball_out_rows": (C.c_int, [_p, _i64, _i32, _p, _p, _p, _p, _p, _i32, _i32, _p, _p, _i32, _i32, _p, _p, _p]),
}
