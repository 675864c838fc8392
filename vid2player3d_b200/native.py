"""ctypes binding of libb200env.so (C ABI: include/b200env.h).

There is deliberately NO fallback: if the CUDA library is missing or no GPU is visible the
product path raises.  (CPU restatements live in oracle/ and are test infrastructure.)
"""
import ctypes as C
import os

from . import abi
from .build import LIB

_lib = None

SYMBOLS = ["b200env_abi_version", "b200env_last_error", "b200env_create", "b200env_destroy", "b200env_bind",
           "b200env_set_motion_lib", "b200env_step", "b200env_reset", "b200env_motion_state", "b200env_obs_imitation",
           "b200env_physics_only", "b200env_launch_count", "b200env_set_env_slice", "b200env_motion_context", "b200env_set_kernel_timing",
           "b200env_kernel_ms", "b200env_obs_imitation_rows", "b200env_set_hull_faces", "b200env_kernel_form",
           "b200env_physics_launch_shape", "b200env_create_assets", "b200env_plan_assets", "b200env_asset_plan"]

ENVS_PER_BATCH = 32   # envs per CTA batch of the default physics launch (step_kernel_packed<true>): the batch size of the asset plan


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB):
            raise RuntimeError(f"{LIB} not built - run `python -c 'import __graft_entry__ as g; g.build()'` "
                               "(the environment has no CPU fallback)")
        L = C.CDLL(LIB)
        L.b200env_last_error.restype = C.c_char_p
        L.b200env_launch_count.restype = C.c_int64
        L.b200env_launch_count.argtypes = [C.c_void_p]
        for name in SYMBOLS:
            getattr(L, name)
        if L.b200env_abi_version() != abi.ABI_VERSION:
            raise RuntimeError("libb200env.so ABI version mismatch - rebuild")
        _lib = L
    return _lib


def _check(rc):
    if rc != 0:
        raise RuntimeError(f"b200env error {rc}: {lib().b200env_last_error().decode()}")


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _stream():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def plan_assets(env_asset, num_assets, envs_per_batch=ENVS_PER_BATCH):
    """the batch plan of a handle of several assets (include/b200env.h: b200env_plan_assets; host only): (rows [N] = envs grouped by
    asset, batches [num_batches, 3] of (asset, first row, count))"""
    import numpy as np
    ea = np.ascontiguousarray(env_asset, np.int32)
    n = len(ea)
    rows, ba, bf, bc = (np.zeros(max(n, 1), np.int32) for _ in range(4))
    nb = C.c_int32(0)
    p = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    _check(lib().b200env_plan_assets(p(ea), C.c_int32(n), C.c_int32(int(num_assets)), C.c_int32(int(envs_per_batch)), p(rows), p(ba), p(bf),
                                     p(bc), C.byref(nb)))
    k = nb.value
    return rows[:n], np.stack([ba[:k], bf[:k], bc[:k]], 1)


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
            _check(lib().b200env_create(C.byref(model_struct), verts.ctypes.data_as(C.c_void_p), C.byref(cfg_struct),
                                        C.c_int32(num_envs), C.c_int32(device_index), C.byref(self._h)))
        else:
            models, vs = list(model_struct), [np.ascontiguousarray(v, np.float32) for v in verts]
            ea = np.ascontiguousarray(env_asset, np.int32)
            if len(models) != len(vs) or len(ea) != num_envs:
                raise ValueError(f"{len(models)} models, {len(vs)} vertex arrays and {len(ea)} env_asset entries for {num_envs} envs")
            marr = (abi.Model * len(models))(*models)
            varr = (C.c_void_p * len(vs))(*[v.ctypes.data for v in vs])
            _check(lib().b200env_create_assets(marr, varr, C.c_int32(len(models)), ea.ctypes.data_as(C.c_void_p), C.byref(cfg_struct),
                                               C.c_int32(num_envs), C.c_int32(device_index), C.byref(self._h)))
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
        b = abi.Buffers()
        for name, _ in abi.Buffers._fields_:
            if name in ("actors_per_env", "bodies_per_env", "num_obs", "num_actions"):
                continue
            if name in ("has_bounce", "has_bounce_now", "bounce_pos", "racket_hit_now") and name not in tensors:
                continue  # ball flag buffers: only for the vid2player player env
            t = tensors[name]
            assert t.is_cuda and t.is_contiguous(), name
            setattr(b, name, t.data_ptr())
        b.actors_per_env, b.bodies_per_env, b.num_obs = actors_per_env, bodies_per_env, num_obs
        b.num_actions = self.num_actions = int(tensors["actions_used"].shape[-1])   # row width of `actions` in step()
        self.num_envs_bound = int(tensors["actions_used"].shape[0])   # rows of the bound tensors (>= num_envs with an env slice)
        self._keep.append(tensors)
        _check(lib().b200env_bind(self._h, C.byref(b)))

    def set_motion_lib(self, t, num_lib_bodies):
        v = abi.MotionLibView()
        for k in ("gts", "grs", "lrs", "grvs", "gravs", "dvs", "motion_lengths", "num_frames", "motion_dt", "length_starts",
                  "min_verts_h"):
            assert t[k].is_cuda and t[k].is_contiguous(), k
            setattr(v, k, t[k].data_ptr())
        v.num_motions = t["motion_lengths"].shape[0]
        v.num_lib_bodies = num_lib_bodies
        v.total_frames = t["gts"].shape[0]
        self._keep.append(t)
        _check(lib().b200env_set_motion_lib(self._h, C.byref(v)))

    def set_hull_faces(self, planes, tris, ntris, tmax):
        """hull faces for the exact ball / convex-hull contact (abi.pack_faces); host numpy arrays, copied by the library"""
        import numpy as np
        planes = np.ascontiguousarray(planes, np.float32)
        tris = np.ascontiguousarray(tris, np.uint8)
        ntris = np.ascontiguousarray(ntris, np.int32)
        _check(lib().b200env_set_hull_faces(self._h, planes.ctypes.data_as(C.c_void_p), tris.ctypes.data_as(C.c_void_p),
                                            ntris.ctypes.data_as(C.c_void_p), C.c_int32(int(tmax))))

    def set_env_slice(self, first, stride):
        """this handle steps rows first, first+stride, ... of the bound tensors (one handle per asset in dual mode)"""
        _check(lib().b200env_set_env_slice(self._h, C.c_int32(int(first)), C.c_int32(int(stride))))

    def step(self, actions):
        if not (actions.is_cuda and actions.is_contiguous() and actions.dtype.is_floating_point):
            raise ValueError("actions must be a contiguous floating-point CUDA tensor")
        if tuple(actions.shape) != (self.num_envs_bound, self.num_actions):
            raise ValueError(f"actions must be [{self.num_envs_bound}, {self.num_actions}], got {tuple(actions.shape)}")
        _check(lib().b200env_step(self._h, _ptr(actions), _stream()))

    def reset(self, env_ids, motion_times):
        n = int(env_ids.shape[0])
        if n:
            _check(lib().b200env_reset(self._h, _ptr(env_ids), _ptr(motion_times), C.c_int32(n), _stream()))

    def motion_state(self, ids, times, out):
        """out: dict name -> tensor or None for root_pos, root_rot, dof_pos, root_vel, root_ang_vel, dof_vel, key_pos,
        rb_pos, rb_rot."""
        names = ("root_pos", "root_rot", "dof_pos", "root_vel", "root_ang_vel", "dof_vel", "key_pos", "rb_pos", "rb_rot")
        _check(lib().b200env_motion_state(self._h, _ptr(ids), _ptr(times), C.c_int32(int(ids.shape[0])),
                                          *[_ptr(out.get(k)) for k in names], _stream()))

    def motion_context(self, env_ids, motion_ids, motion_times, num_frames, first_frame, dt, feat, mask):
        """feat [N, num_frames, W] float32, mask [N, num_frames] bool; rows env_ids (None: rows 0..n-1)"""
        assert feat.is_cuda and feat.is_contiguous() and mask.is_contiguous() and motion_ids.is_contiguous() and motion_times.is_contiguous()
        _check(lib().b200env_motion_context(self._h, _ptr(env_ids), _ptr(motion_ids), _ptr(motion_times), C.c_int32(int(motion_ids.shape[0])),
                                            C.c_int32(int(num_frames)), C.c_int32(int(first_frame)), C.c_float(float(dt)), _ptr(feat),
                                            _ptr(mask), _stream()))

    def obs_imitation(self, body_pos, body_rot, target_pos, target_rot, dof_pos, dof_vel, target_dof_pos, body_vel,
                      body_ang_vel, motion_bodies, local_root_obs, root_height_obs, obs, jpos=False):
        n = int(body_pos.shape[0])
        _check(lib().b200env_obs_imitation(self._h, C.c_int32(n), _ptr(body_pos), _ptr(body_rot), _ptr(target_pos),
                                           _ptr(target_rot), _ptr(dof_pos), _ptr(dof_vel), _ptr(target_dof_pos),
                                           _ptr(body_vel), _ptr(body_ang_vel), _ptr(motion_bodies),
                                           C.c_int32(int(bool(local_root_obs)) | (2 if jpos else 0)), C.c_int32(int(root_height_obs)), _ptr(obs),
                                           _stream()))

    def obs_imitation_rows(self, n, rigid_body_state, bodies_per_env, dof_state, target_pos, target_rot, target_dof_pos, motion_bodies,
                           local_root_obs, root_height_obs, obs, obs_bf16=None, mean=None, rstd=None, clamp=5.0):
        """the 734-d observation straight from the state rows (no gathers); obs_bf16: padded bf16 operand buffer of the policy's
        first layer, written in the same launch (normalised by mean / rstd when given, clamped to +-clamp)"""
        _check(lib().b200env_obs_imitation_rows(self._h, C.c_int32(int(n)), _ptr(rigid_body_state), C.c_int32(int(bodies_per_env)), _ptr(dof_state),
                                                _ptr(target_pos), _ptr(target_rot), _ptr(target_dof_pos), _ptr(motion_bodies),
                                                C.c_int32(int(bool(local_root_obs))), C.c_int32(int(root_height_obs)), _ptr(obs), _ptr(obs_bf16),
                                                C.c_int32(int(obs_bf16.shape[1]) if obs_bf16 is not None else 0), _ptr(mean), _ptr(rstd),
                                                C.c_float(float(clamp)), _stream()))

    def physics_only(self, root, dof_pos, dof_vel, pd_tar, ext_wrench, rb_out, contact_out, n_steps=1, ball=None, ball_hits=None):
        import torch
        prec = {torch.float32: 0, torch.float64: 1}[root.dtype]
        for t in (dof_pos, dof_vel, pd_tar, rb_out):
            assert t.dtype == root.dtype and t.is_cuda and t.is_contiguous()
        _check(lib().b200env_physics_only(self._h, C.c_int32(prec), C.c_int32(int(root.shape[0])), C.c_int32(n_steps),
                                          _ptr(root), _ptr(dof_pos), _ptr(dof_vel), _ptr(pd_tar), _ptr(ext_wrench),
                                          _ptr(rb_out), _ptr(contact_out), _ptr(ball), _ptr(ball_hits), _stream()))

    @property
    def kernel_form(self):
        """'lane' | 'packed' | 'packed3' | 'tmem' (include/b200env.h: b200env_kernel_form)"""
        return ("lane", "packed", "packed3", "tmem")[int(lib().b200env_kernel_form(self._h))]

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
        _check(lib().b200env_asset_plan(self._h, C.byref(na), C.byref(nb), None, None, None, None))
        rows = np.zeros(self.num_envs, np.int32)
        b = np.zeros((3, max(nb.value, 1)), np.int32)
        p = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
        _check(lib().b200env_asset_plan(self._h, C.byref(na), C.byref(nb), p(rows), p(b[0]), p(b[1]), p(b[2])))
        return na.value, rows, b[:, :nb.value].T.copy()

    @property
    def launch_count(self):
        return int(lib().b200env_launch_count(self._h))

    def set_kernel_timing(self, on=True):
        """event pairs around the physics launch of every step (measurement aid, include/b200env.h)"""
        _check(lib().b200env_set_kernel_timing(self._h, C.c_int32(1 if on else 0)))

    def kernel_ms(self):
        """(mean ms, count) of the physics launches since the last call"""
        ms, n = C.c_double(0.0), C.c_int32(0)
        _check(lib().b200env_kernel_ms(self._h, C.byref(ms), C.byref(n)))
        return ms.value, n.value
