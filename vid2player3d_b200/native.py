"""ctypes binding of libb200env.so (C ABI: include/b200env.h).

There is deliberately NO fallback: if the CUDA library is missing or no GPU is visible the
product path raises.  (CPU restatements live in oracle/ and are test infrastructure.)
"""
import ctypes as C
import os

from . import abi
from .build import LIB

_lib = None

ENVS_PER_BATCH = 32   # envs per CTA batch of the default physics launch (step_kernel_packed<true>): the batch size of the asset plan


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB):
            raise RuntimeError(f"{LIB} not built - run `python -c 'import __graft_entry__ as g; g.build()'` "
                               "(the environment has no CPU fallback)")
        L = C.CDLL(LIB)
        for name, (restype, argtypes) in abi.SIGNATURES.items():
            fn = getattr(L, name)
            fn.restype, fn.argtypes = restype, argtypes
        if L.b200env_abi_version() != abi.ABI_VERSION:
            raise RuntimeError("libb200env.so ABI version mismatch - rebuild")
        for S, size in ((abi.ResetMasked, L.b200env_reset_masked_desc_size()), (abi.MotionContext, L.b200env_motion_context_desc_size()),
                        (abi.ImRecord, L.b200env_im_record_desc_size()), (abi.V2PTaskReset, L.b200v2p_task_reset_desc_size()),
                        (abi.ImMotionStats, L.b200env_im_motion_stats_desc_size()),
                        (abi.PlayStats, L.b200env_play_stats_desc_size()), (abi.ImMotionQueue, L.b200env_im_motion_queue_desc_size()),
                        (abi.ImMotionQueueStats, L.b200env_im_motion_queue_stats_desc_size()),
                        (abi.SetEnvAssets, L.b200env_set_env_assets_desc_size()),
                        (abi.ResampleMotions, L.b200env_resample_motions_desc_size()),
                        (abi.MotionWeights, L.b200env_motion_weights_desc_size()),
                        (abi.V2PBallStats, L.b200v2p_eval_ball_stats_desc_size()),
                        (abi.V2PRallyStats, L.b200v2p_eval_rally_stats_desc_size())):
            if size != C.sizeof(S):    # these descriptors grow by appended fields within one version
                raise RuntimeError(f"libb200env.so takes a {size}-byte {S.__name__} descriptor, the binding fills {C.sizeof(S)} - rebuild")
        _lib = L
    return _lib


def _check(rc):
    if rc != 0:
        raise RuntimeError(f"b200env error {rc}: {lib().b200env_last_error().decode()}")


def _ptr(t):
    return t.data_ptr() if t is not None else None


_layouts = {}


def _layout(S):
    """(scalar fields as (name, array length or None), pointer fields as (name, accepted dtypes or None)) of S"""
    lay = _layouts.get(S)
    if lay is None:
        import torch
        dtypes = {abi.F32P: (torch.float32,), abi.I64P: (torch.int64,), abi.U8P: (torch.uint8, torch.bool),
                  abi.U32P: (torch.int32, torch.uint32), abi.I32P: (torch.int32,), abi.F64P: (torch.float64,)}
        scalars = [(name, ct._length_ if issubclass(ct, C.Array) else None) for name, ct in S._fields_ if not issubclass(ct, C.c_void_p)]
        ptrs = [(name, dtypes.get(ct)) for name, ct in S._fields_ if issubclass(ct, C.c_void_p)]
        lay = _layouts[S] = (scalars, ptrs)
    return lay


def fill(S, scalars, tensors):
    """a launch descriptor S (a struct of abi.py) filled from `scalars` (field -> number, a sequence for an array field) and `tensors`
    (field -> tensor or None).  Every scalar field must be given except those of S._defaults_, which stay 0 when left out or None; a
    pointer may be None only in S._nullable_.  A tensor must have the dtype of its field's pointee (any for void*), be contiguous and
    lie on the one CUDA device of all of them.  Keys that name no field are ignored.  Refusals raise ValueError naming the field."""
    scalar_fields, ptr_fields = _layout(S)
    s = S()
    for name, length in scalar_fields:
        v = scalars.get(name)
        if v is None:
            if name not in S._defaults_:
                raise ValueError(f"{S.__name__}.{name}: missing")
        elif length is None:
            setattr(s, name, v)
        elif len(v) != length:
            raise ValueError(f"{S.__name__}.{name}: {len(v)} values for {length}")
        else:
            getattr(s, name)[:] = v
    dev, off_device = None, None
    for name, dtypes in ptr_fields:
        x = tensors.get(name)
        if x is None:
            if name not in S._nullable_:
                raise ValueError(f"{S.__name__}.{name}: None, but the header allows no NULL here")
            continue
        if dtypes is not None and x.dtype not in dtypes:
            raise ValueError(f"{S.__name__}.{name}: {x.dtype}, the header's pointee needs {' or '.join(map(str, dtypes))}")
        if not x.is_contiguous():
            raise ValueError(f"{S.__name__}.{name}: not contiguous")
        d = x.get_device()
        dev = d if dev is None else dev
        if off_device is None and (d < 0 or d != dev):
            off_device = name
        setattr(s, name, x.data_ptr())
    if off_device is not None:
        raise ValueError(f"{S.__name__}.{off_device}: not on the CUDA device of the other tensors")
    return s


def _stream():
    import torch
    return torch.cuda.current_stream().cuda_stream


def play_stats(scalars, tensors):
    """one step of ImitatorPlayer.run's bookkeeping on the device (include/b200env.h: b200env_play_stats); the fields of abi.PlayStats"""
    d = fill(abi.PlayStats, scalars, tensors)
    _check(lib().b200env_play_stats(C.byref(d), _stream()))


def im_record(scalars, tensors):
    """one recorded viewer frame of HumanoidSMPLIMVis on the device (include/b200env.h: b200env_im_record); the fields of abi.ImRecord"""
    d = fill(abi.ImRecord, scalars, tensors)
    _check(lib().b200env_im_record(C.byref(d), _stream()))


def im_motion_stats(scalars, tensors):
    """the per-motion meters of one test step on the device (include/b200env.h: b200env_im_motion_stats); the fields of
    abi.ImMotionStats"""
    d = fill(abi.ImMotionStats, scalars, tensors)
    _check(lib().b200env_im_motion_stats(C.byref(d), _stream()))


def im_motion_queue_stats(scalars, tensors):
    """the per-motion meters of one test step folded by queue entry (include/b200env.h: b200env_im_motion_queue_stats); the fields of
    abi.ImMotionQueueStats"""
    d = fill(abi.ImMotionQueueStats, scalars, tensors)
    _check(lib().b200env_im_motion_queue_stats(C.byref(d), _stream()))


def im_motion_queue(scalars, tensors):
    """one assignment of the motion queue on the device (include/b200env.h: b200env_im_motion_queue); the fields of abi.ImMotionQueue"""
    d = fill(abi.ImMotionQueue, scalars, tensors)
    _check(lib().b200env_im_motion_queue(C.byref(d), _stream()))


def resample_motions(scalars, tensors):
    """new motions for the masked envs that played a step, drawn on the device (include/b200env.h: b200env_resample_motions); the
    fields of abi.ResampleMotions"""
    d = fill(abi.ResampleMotions, scalars, tensors)
    _check(lib().b200env_resample_motions(C.byref(d), _stream()))


def motion_weights(scalars, tensors):
    """the resample's motion CDF rebuilt on the device (include/b200env.h: b200env_motion_weights); the fields of abi.MotionWeights"""
    d = fill(abi.MotionWeights, scalars, tensors)
    _check(lib().b200env_motion_weights(C.byref(d), _stream()))


def plan_assets(env_asset, num_assets, envs_per_batch=ENVS_PER_BATCH, mixed=False):
    """the batch plan of a handle of several assets (include/b200env.h: b200env_plan_assets; host only): (rows [N] = envs grouped by
    asset, batches [num_batches, 3] of (asset, first row, count)).  mixed: the mixed plan (b200env_plan_assets_mixed): rows in env
    order, batches of consecutive envs whatever their asset (asset -1 for a batch of several)"""
    import numpy as np
    ea = np.ascontiguousarray(env_asset, np.int32)
    n = len(ea)
    rows, ba, bf, bc = (np.zeros(max(n, 1), np.int32) for _ in range(4))
    nb = C.c_int32(0)
    p = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    fn = lib().b200env_plan_assets_mixed if mixed else lib().b200env_plan_assets
    _check(fn(p(ea), n, num_assets, envs_per_batch, p(rows), p(ba), p(bf), p(bc), C.byref(nb)))
    k = nb.value
    return rows[:n], np.stack([ba[:k], bf[:k], bc[:k]], 1)


def choose_asset_plan(env_asset, num_assets, grid):
    """True when b200env_create_assets runs the mixed plan on a persistent grid of `grid` CTAs (include/b200env.h:
    b200env_choose_asset_plan; host only)"""
    import numpy as np
    ea = np.ascontiguousarray(env_asset, np.int32)
    m = C.c_int32(0)
    _check(lib().b200env_choose_asset_plan(ea.ctypes.data_as(C.c_void_p), len(ea), num_assets, grid, C.byref(m)))
    return bool(m.value)


class Env:
    """Owns one b200env handle.  All tensors passed in must live on `device` and be contiguous.

    One asset: Env(model_struct, verts, cfg, N, dev).  Several assets of one topology (include/b200env.h: b200env_create_assets):
    Env([model_struct, ...], [verts, ...], cfg, N, dev, env_asset=[asset of env 0, ...])."""

    def __init__(self, model_struct, verts, cfg_struct, num_envs, device_index, env_asset=None):
        self._h = C.c_void_p()
        self._keep = []
        import numpy as np
        if env_asset is None:
            verts = np.ascontiguousarray(verts, np.float32)
            _check(lib().b200env_create(C.byref(model_struct), verts.ctypes.data_as(C.c_void_p), C.byref(cfg_struct), num_envs, device_index,
                                        C.byref(self._h)))
        else:
            models, vs = list(model_struct), [np.ascontiguousarray(v, np.float32) for v in verts]
            ea = np.ascontiguousarray(env_asset, np.int32)
            if len(models) != len(vs) or len(ea) != num_envs:
                raise ValueError(f"{len(models)} models, {len(vs)} vertex arrays and {len(ea)} env_asset entries for {num_envs} envs")
            marr = (abi.Model * len(models))(*models)
            varr = (C.c_void_p * len(vs))(*[v.ctypes.data for v in vs])
            _check(lib().b200env_create_assets(marr, varr, len(models), ea.ctypes.data_as(C.c_void_p), C.byref(cfg_struct), num_envs,
                                               device_index, C.byref(self._h)))
            model_struct = models[0]
        self.model, self.cfg, self.num_envs = model_struct, cfg_struct, num_envs

    def close(self):
        if self._h:
            lib().b200env_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def bind(self, tensors, actors_per_env, bodies_per_env, num_obs):
        """tensors: name -> CUDA tensor of every b200_buffers_t pointer; the ball flag buffers only for the vid2player player env, and
        "dof_force" ([rows, nd] float32) only with DOF force sensors"""
        self.num_actions = int(tensors["actions_used"].shape[-1])      # row width of `actions` in step()
        self.num_envs_bound = int(tensors["actions_used"].shape[0])    # rows of the bound tensors (>= num_envs with an env slice)
        f = tensors.get("dof_force")
        assert f is None or tuple(f.shape) == (self.num_envs_bound, int(self.model.nd)), \
            f"dof_force must be [{self.num_envs_bound}, {int(self.model.nd)}], got {tuple(f.shape)}"
        b = fill(abi.Buffers, dict(actors_per_env=actors_per_env, bodies_per_env=bodies_per_env, num_obs=num_obs,
                                   num_actions=self.num_actions), tensors)
        self._keep.append(tensors)
        _check(lib().b200env_bind(self._h, C.byref(b)))

    def set_motion_lib(self, t, num_lib_bodies):
        v = fill(abi.MotionLibView, dict(num_motions=t["motion_lengths"].shape[0], num_lib_bodies=num_lib_bodies,
                                         total_frames=t["gts"].shape[0]), t)
        self._keep.append(t)
        _check(lib().b200env_set_motion_lib(self._h, C.byref(v)))
        self._num_lib_bodies = int(num_lib_bodies)

    @property
    def lib_bodies(self):
        """humanoid bodies of the observation: the motion library's body count, else the model's bodies without a welded last one"""
        nb = int(self.model.nb)
        return getattr(self, "_num_lib_bodies", nb - 1 if self.model.fixed[nb - 1] else nb)

    def set_hull_faces(self, planes, tris, ntris, tmax):
        """hull faces for the exact ball / convex-hull contact (abi.pack_faces); host numpy arrays, copied by the library"""
        import numpy as np
        planes = np.ascontiguousarray(planes, np.float32)
        tris = np.ascontiguousarray(tris, np.uint8)
        ntris = np.ascontiguousarray(ntris, np.int32)
        _check(lib().b200env_set_hull_faces(self._h, planes.ctypes.data_as(C.c_void_p), tris.ctypes.data_as(C.c_void_p),
                                            ntris.ctypes.data_as(C.c_void_p), tmax))

    def set_env_slice(self, first, stride):
        """this handle steps rows first, first+stride, ... of the bound tensors (one handle per asset in dual mode)"""
        _check(lib().b200env_set_env_slice(self._h, first, stride))

    def step(self, actions):
        if not (actions.is_cuda and actions.is_contiguous() and actions.dtype.is_floating_point):
            raise ValueError("actions must be a contiguous floating-point CUDA tensor")
        if tuple(actions.shape) != (self.num_envs_bound, self.num_actions):
            raise ValueError(f"actions must be [{self.num_envs_bound}, {self.num_actions}], got {tuple(actions.shape)}")
        _check(lib().b200env_step(self._h, _ptr(actions), _stream()))

    def reset(self, env_ids, motion_times):
        n = int(env_ids.shape[0])
        if n:
            _check(lib().b200env_reset(self._h, _ptr(env_ids), _ptr(motion_times), n, _stream()))

    def reset_masked(self, mask, sample_time, truncate, ref_prob, seed, counter, init_root, init_dof_pos, init_dof_vel, reset_times,
                     num_frames, first_frame, dt, feat, feat_mask, work, transforms=None, step=None, context_length=None):
        """reset of the envs whose mask [N] bool is set, context window included (include/b200env.h: b200env_reset_masked);
        transforms: the window's transform program (abi.transform_program), with feat rows W + bodies wide; step ([1] int64, the
        bookkeeping's step counter) with context_length: each window starts step % context_length frames earlier"""
        assert mask.shape[0] == self.num_envs and work.shape[0] >= self.num_envs + 2
        xf = dict(transforms, feat_width=int(feat.shape[-1])) if transforms is not None else {}
        d = fill(abi.ResetMasked, dict(xf, sample_time=int(bool(sample_time)), truncate=truncate, ref_prob=ref_prob, num_frames=num_frames,
                                       first_frame=first_frame, dt=dt, seed=int(seed), context_length=context_length),
                 dict(mask=mask, counter=counter, init_root=init_root, init_dof_pos=init_dof_pos, init_dof_vel=init_dof_vel,
                      reset_times=reset_times, context_feat=feat, context_mask=feat_mask, work=work, step=step))
        _check(lib().b200env_reset_masked(self._h, C.byref(d), _stream()))

    def motion_state(self, ids, times, out):
        """out: dict name -> tensor or None for root_pos, root_rot, dof_pos, root_vel, root_ang_vel, dof_vel, key_pos,
        rb_pos, rb_rot."""
        d = fill(abi.MotionState, dict(n=ids.shape[0]), dict(out, motion_ids=ids, motion_times=times))
        _check(lib().b200env_motion_state(self._h, C.byref(d), _stream()))

    def motion_context(self, env_ids, motion_ids, motion_times, num_frames, first_frame, dt, feat, mask, transforms=None, seed=0,
                       counter=None):
        """feat [N, num_frames, W] float32, mask [N, num_frames] bool; rows env_ids (None: rows 0..n-1).  transforms: the transform
        program (abi.transform_program) with feat [N, num_frames, W + bodies], drawing from (seed, counter [1] int64, not advanced)"""
        xf = dict(transforms, feat_width=int(feat.shape[-1]), seed=int(seed)) if transforms is not None else {}
        d = fill(abi.MotionContext, dict(xf, n=motion_ids.shape[0], num_frames=num_frames, first_frame=first_frame, dt=dt),
                 dict(env_ids=env_ids, motion_ids=motion_ids, motion_times=motion_times, context_feat=feat, context_mask=mask,
                      counter=counter))
        _check(lib().b200env_motion_context(self._h, C.byref(d), _stream()))

    def obs_row_width(self, jpos=False):
        """columns of the row the observation launches write: 734 (513 with jpos) for the 24-body humanoid, 69 dofs, shape_dim 11"""
        nbl = self.lib_bodies
        nd, sd = int(self.model.nd), int(self.cfg.shape_dim)
        w = 1 + (nbl - 1) * 3 + nbl * 6 + nbl * 6 + nd + sd
        return w + ((3 + nbl * 3) if jpos else (11 + nd + nbl * 9))

    def obs_imitation(self, body_pos, body_rot, target_pos, target_rot, dof_pos, dof_vel, target_dof_pos, body_vel,
                      body_ang_vel, motion_bodies, local_root_obs, root_height_obs, obs, jpos=False):
        n = int(body_pos.shape[0])
        assert obs.dim() == 2 and obs.shape[0] >= n and obs.shape[1] == self.obs_row_width(jpos), (tuple(obs.shape), self.obs_row_width(jpos))
        d = fill(abi.ObsImitation, dict(n=n, local_root_obs=int(bool(local_root_obs)), root_height_obs=int(root_height_obs), jpos=int(bool(jpos))),
                 dict(body_pos=body_pos, body_rot=body_rot, target_pos=target_pos, target_rot=target_rot, dof_pos=dof_pos, dof_vel=dof_vel,
                      target_dof_pos=target_dof_pos, body_vel=body_vel, body_ang_vel=body_ang_vel, motion_bodies=motion_bodies, obs=obs))
        _check(lib().b200env_obs_imitation(self._h, C.byref(d), _stream()))

    def obs_imitation_rows(self, n, rigid_body_state, bodies_per_env, dof_state, target_pos, target_rot, target_dof_pos, motion_bodies,
                           local_root_obs, root_height_obs, obs, obs_bf16=None, mean=None, rstd=None, clamp=5.0, jpos=False, dual=False,
                           clamp1=None):
        """the 734-d observation (513-d with jpos) straight from the state rows (no gathers); obs_bf16: padded bf16 operand buffer of
        the policy's first layer, written in the same launch (normalised by mean / rstd when given, clamped to +-clamp).  dual: the two
        players' policies of a rally (b200env_obs_imitation_rows_dual) - env e's operand row is (e & 1) * n/2 + (e >> 1), with row
        e & 1 of mean / rstd [2, W] and clamp (player 0) or clamp1 (player 1)"""
        W = self.obs_row_width(jpos)
        assert obs.dim() == 2 and obs.shape[0] >= n and obs.shape[1] == W, (tuple(obs.shape), W)
        assert obs_bf16 is None or (obs_bf16.dim() == 2 and obs_bf16.shape[0] >= n), tuple(obs_bf16.shape)
        if dual and mean is not None:
            assert tuple(mean.shape) == (2, W) and tuple(rstd.shape) == (2, W), (tuple(mean.shape), tuple(rstd.shape))
        d = fill(abi.ObsRows, dict(n=n, bodies_per_env=bodies_per_env, local_root_obs=int(bool(local_root_obs)),
                                   root_height_obs=int(root_height_obs), jpos=int(bool(jpos)),
                                   ld_bf16=obs_bf16.shape[1] if obs_bf16 is not None else 0, clamp=clamp, clamp1=clamp1),
                 dict(rigid_body_state=rigid_body_state, dof_state=dof_state, target_pos=target_pos, target_rot=target_rot,
                      target_dof_pos=target_dof_pos, motion_bodies=motion_bodies, obs=obs, obs_bf16=obs_bf16, mean=mean, rstd=rstd))
        fn = lib().b200env_obs_imitation_rows_dual if dual else lib().b200env_obs_imitation_rows
        _check(fn(self._h, C.byref(d), _stream()))

    def im_policy_rows(self, scalars, tensors):
        """the imitation policy's bf16 operand rows and residual from obs_buf and the context slot of the device step counter
        (include/b200env.h: b200env_im_policy_rows); scalars / tensors: the fields of abi.ImPolicy"""
        d = fill(abi.ImPolicy, scalars, tensors)
        _check(lib().b200env_im_policy_rows(self._h, C.byref(d), _stream()))

    def physics_only(self, root, dof_pos, dof_vel, pd_tar, ext_wrench, rb_out, contact_out, n_steps=1, ball=None, ball_hits=None,
                     dof_force=None):
        """dof_force: [n, nd] of root's dtype, receives the DOF force sensor of the last control step (include/b200env.h)"""
        import torch
        prec = {torch.float32: 0, torch.float64: 1}[root.dtype]
        for t in (dof_pos, dof_vel, pd_tar, rb_out) + ((dof_force,) if dof_force is not None else ()):
            assert t.dtype == root.dtype and t.is_cuda and t.is_contiguous()
        _check(lib().b200env_physics_only(self._h, prec, root.shape[0], n_steps, _ptr(root), _ptr(dof_pos), _ptr(dof_vel), _ptr(pd_tar),
                                          _ptr(ext_wrench), _ptr(rb_out), _ptr(contact_out), _ptr(ball), _ptr(ball_hits), _stream(),
                                          _ptr(dof_force)))

    @property
    def kernel_form(self):
        """'lane' | 'packed' | 'packed3' | 'tmem' (include/b200env.h: b200env_kernel_form)"""
        return ("lane", "packed", "packed3", "tmem")[lib().b200env_kernel_form(self._h)]

    @property
    def physics_launch_shape(self):
        """(envs per CTA batch, resident CTA slots of the persistent grid) of the step's physics launch (include/b200env.h:
        b200env_physics_launch_shape); a step of n envs runs batch b in round b // grid"""
        b, g = C.c_int32(0), C.c_int32(0)
        _check(lib().b200env_physics_launch_shape(self._h, C.byref(b), C.byref(g)))
        return b.value, g.value

    @property
    def asset_plan(self):
        """(num_assets, rows [N], batches [num_batches, 3] of (asset, first row, count)) of a handle of several assets
        (include/b200env.h: b200env_asset_plan): batch b of rows[first:first + count] runs in round b // grid"""
        import numpy as np
        na, nb = C.c_int32(0), C.c_int32(0)
        _check(lib().b200env_asset_plan(self._h, C.byref(na), C.byref(nb), None, None, None, None, None))
        rows = np.zeros(self.num_envs, np.int32)
        b = np.zeros((3, max(nb.value, 1)), np.int32)
        p = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
        _check(lib().b200env_asset_plan(self._h, C.byref(na), C.byref(nb), p(rows), p(b[0]), p(b[1]), p(b[2]), None))
        return na.value, rows, b[:, :nb.value].T.copy()

    @property
    def asset_plan_mixed(self):
        """True when a handle of several assets runs the mixed plan (batches of consecutive envs whatever their asset), False for the
        grouped one (include/b200env.h: b200env_asset_plan)"""
        na, nb, m = C.c_int32(0), C.c_int32(0), C.c_int32(0)
        _check(lib().b200env_asset_plan(self._h, C.byref(na), C.byref(nb), None, None, None, None, C.byref(m)))
        return bool(m.value)

    def fix_mixed_plan(self):
        """a handle of several assets runs the mixed plan for its lifetime, so set_env_assets may move envs to other assets
        (include/b200env.h: b200env_fix_mixed_plan; setup work, before the first step)"""
        _check(lib().b200env_fix_mixed_plan(self._h))

    def set_env_assets(self, env_asset, error):
        """env e is simulated with asset env_asset[e] ([N] int32, device) from the next physics launch on; an index outside the
        handle's assets keeps the env's asset and sets error ([1] int32, device) to env + 1 when it is 0 (include/b200env.h:
        b200env_set_env_assets; graph-safe, no host synchronisation)"""
        d = fill(abi.SetEnvAssets, dict(n=self.num_envs), dict(env_asset=env_asset, error=error))
        _check(lib().b200env_set_env_assets(self._h, C.byref(d), _stream()))

    @property
    def launch_count(self):
        return lib().b200env_launch_count(self._h)

    def set_kernel_timing(self, on=True):
        """event pairs around the physics launch of every step (measurement aid, include/b200env.h)"""
        _check(lib().b200env_set_kernel_timing(self._h, 1 if on else 0))

    def kernel_ms(self):
        """(mean ms, count) of the physics launches since the last call"""
        ms, n = C.c_double(0.0), C.c_int32(0)
        _check(lib().b200env_kernel_ms(self._h, C.byref(ms), C.byref(n)))
        return ms.value, n.value
