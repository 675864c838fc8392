"""Offline tennis-ball data generators on the GPU (SURVEY.md 8f-2): host-side mirror of the reference's

  simulate / TennisBallGeneratorIsaac / generate_incoming_trajectory      vid2player/utils/tennis_ball.py:113-394
  traj_out_params / simulate_without_bounce / generate_outgoing_trajectory vid2player/utils/tennis_ball_out_estimator.py:13-121,208-258
  traj_in_params / generate_incoming_trajectory                            vid2player/utils/tennis_ball_in_estimator.py:10-14,82-140

with the same names, argument meaning and on-disk `.npy` layouts:

  pool       [P, 307]            launch_pos 3 | launch_vel 3 | vspin 1 | traj 100 x 3 @ 30 Hz, sorted by launch x
  in-table   [rows, 50, 2]       (y, z) of a ball launched straight out, rows over (height, vel_x, vel_y, vspin) in C order
  out-tables [rows, 60] / [rows, 30, 2]  rows over (vel_x, vel_y, vspin) in C order

The reference steps 10 000 balls at a time through Isaac Gym from Python (two FFI calls + ~25 torch kernels per sim step, 825
batches for the out tables); here each function is ONE kernel launch over all rows (csrc/ballgen.cuh through the C ABI of
include/b200ball.h), integrating the same ball model as the env step kernel.  There is no CPU fallback: tensors live on the
CUDA device (the numpy twin in oracle/ref_port_ballgen.py is test infrastructure).
"""
import ctypes as C
import math

import numpy as np
import torch

from . import native


class BallSim(C.Structure):
    """b200ball_sim_t"""
    _fields_ = [("num_frames", C.c_int32), ("control_freq_inv", C.c_int32), ("substeps", C.c_int32), ("first_comp", C.c_int32),
                ("sim_dt", C.c_float), ("spin_scale", C.c_float), ("gravity_z", C.c_float), ("ball_mass", C.c_float),
                ("ball_inertia", C.c_float), ("ball_radius", C.c_float), ("e_ground", C.c_float), ("mu_ground", C.c_float),
                ("bounce_threshold_velocity", C.c_float)]


# tennis_ball.urdf + the material values of TennisBallGeneratorIsaac (:256-258, plane :93-96) under PhysX' "average" combine:
# restitution (0.9 + 0.5) / 2, friction (0.2 + 1.0) / 2 - the same numbers abi.make_cfg gives the env step kernel
BALL = dict(ball_mass=0.057, ball_inertia=4e-5, ball_radius=0.032, e_ground=0.7, mu_ground=0.6, bounce_threshold_velocity=0.2,
            gravity_z=-9.81, sim_dt=1.0 / 60.0)


class traj_out_params:   # tennis_ball_out_estimator.py:13-18
    VEL_X_RANGE = (10, 65, 0.1)
    VEL_Y_RANGE = (-5, 10, 0.1)
    VSPIN_RANGE = (-10, 10, 0.2)
    TRAJ_X_RANGE = (0, 30, 0.5)
    TRAJ_Y_RANGE = (0, 3, 0.1)


class traj_in_params:    # tennis_ball_in_estimator.py:10-14
    VEL_X_RANGE = (25, 30, 0.1)
    VEL_Y_RANGE = (5, 8, 0.1)
    VSPIN_RANGE = (5, 10, 0.1)
    HEIGHT_RANGE = (0.5, 2, 0.1)


def _cfg(num_frames, control_freq_inv, substeps, spin_scale, first_comp=0, **over):
    kw = dict(BALL)
    kw.update(over)
    return BallSim(num_frames=num_frames, control_freq_inv=control_freq_inv, substeps=substeps, first_comp=first_comp,
                   spin_scale=float(spin_scale), **kw)


def _dev(t, dtype, device):
    return torch.as_tensor(t, dtype=dtype, device=device).contiguous()


def simulate(launch_pos, launch_vel, launch_vspin, control_freq_inv=2, num_frames=100, substeps=6, spin_scale=5, device="cuda:0",
             first_comp=0, dtype=torch.float32, **physics):
    """tennis_ball.py:113-218 (the gym/sim handles are gone: the balls are integrated by the kernel).
    Returns traj [n, num_frames, 3 - first_comp], bounce_pos [n,3], bounce_idx [n] int64, pass_net [n] bool on `device`."""
    lp, lv, ls = _dev(launch_pos, dtype, device), _dev(launch_vel, dtype, device), _dev(launch_vspin, dtype, device)
    n = int(lp.shape[0])
    assert lp.shape == (n, 3) and lv.shape == (n, 3) and ls.shape == (n,)
    traj = torch.empty(n, num_frames, 3 - first_comp, dtype=dtype, device=lp.device)
    bpos = torch.empty(n, 3, dtype=dtype, device=lp.device)
    bidx = torch.empty(n, dtype=torch.int64, device=lp.device)
    pnet = torch.empty(n, dtype=torch.uint8, device=lp.device)
    cfg = _cfg(num_frames, control_freq_inv, substeps, spin_scale, first_comp, **physics)
    with torch.cuda.device(lp.device):
        native._check(native.lib().b200ball_simulate(C.byref(cfg), n, 0 if dtype == torch.float32 else 1, native._ptr(lp),
                                                     native._ptr(lv), native._ptr(ls), native._ptr(traj), native._ptr(bpos), native._ptr(bidx),
                                                     native._ptr(pnet), native._stream()))
    return traj, bpos, bidx, pnet.bool()


def _grid(rng, scale):
    """values of torch.arange(*rng), the column `int(v * scale)` the reference writes each one to (:98, :110) with Python's
    index semantics (a negative column counts from the end of the row, one outside [-n, n) raises IndexError), and the row width n"""
    v = torch.arange(*rng)
    n = int((rng[1] - rng[0]) / rng[2])
    col = []
    for x in v:
        c = int(x * scale)
        if not -n <= c < n:
            raise IndexError(f"grid value {float(x)} maps to column {c} of a row of {n}")
        col.append(c % n)
    return v.to(torch.float32), torch.tensor(col, dtype=torch.int32), n


def simulate_without_bounce(launch_vel_h, launch_vel_v, launch_vspin, params=traj_out_params, control_freq_inv=2, num_frames=60,
                            substeps=6, spin_scale=5, device="cuda:0", dtype=torch.float32, **physics):
    """tennis_ball_out_estimator.py:21-121 for rows launched straight out with (horizontal, vertical) speed and spin.
    Returns traj_x [n, NX], traj_y [n, NY, 2] on `device` (heights relative to the launch height)."""
    vh, vv, vs = _dev(launch_vel_h, dtype, device), _dev(launch_vel_v, dtype, device), _dev(launch_vspin, dtype, device)
    n = int(vh.shape[0])
    gx, cx, nx = _grid(params.TRAJ_X_RANGE, 2)
    gy, cy, ny = _grid(params.TRAJ_Y_RANGE, 10)
    # columns no grid value maps to stay 0 like the reference's torch.zeros; when every column is written (true for the shipped
    # grids) the 3.96 GB zero fill of the full table is skipped
    covered = set(cx.tolist()) == set(range(nx)) and set(cy.tolist()) == set(range(ny))
    alloc = torch.empty if covered else torch.zeros
    gx, cx, gy, cy = gx.to(vh.device), cx.to(vh.device), gy.to(vh.device), cy.to(vh.device)
    out_x = alloc(n, nx, dtype=dtype, device=vh.device)
    out_y = alloc(n, ny, 2, dtype=dtype, device=vh.device)
    cfg = _cfg(num_frames, control_freq_inv, substeps, spin_scale, 0, **physics)
    with torch.cuda.device(vh.device):
        native._check(native.lib().b200ball_out_rows(C.byref(cfg), n, 0 if dtype == torch.float32 else 1, native._ptr(vh),
                                                     native._ptr(vv), native._ptr(vs), native._ptr(gx), native._ptr(cx), len(gx),
                                                     nx, native._ptr(gy), native._ptr(cy), len(gy), ny,
                                                     native._ptr(out_x), native._ptr(out_y), native._stream()))
    return out_x, out_y


def _mesh(*ranges, device):
    """C-order launch grid of the reference's nested `batch_*[i, :, :] = v` loops (np.arange values cast to float32)"""
    axes = [torch.from_numpy(np.arange(*r).astype(np.float32)).to(device) for r in ranges]
    return [g.reshape(-1) for g in torch.meshgrid(*axes, indexing="ij")]


def generate_outgoing_trajectory(traj_path=None, params=traj_out_params, device="cuda:0", spin_scale=5, substeps=6):
    """tennis_ball_out_estimator.py:208-258: the whole (vel_x, vel_y, vspin) grid in one launch.  Writes `<traj_path>` (x table) and
    the `_y` twin when a path is given; returns (traj_x, traj_y) device tensors."""
    vh, vv, vs = _mesh(params.VEL_X_RANGE, params.VEL_Y_RANGE, params.VSPIN_RANGE, device=device)
    tx, ty = simulate_without_bounce(vh, vv, vs, params, spin_scale=spin_scale, substeps=substeps, device=device)
    if traj_path is not None:
        np.save(traj_path, tx.cpu().numpy())
        np.save(traj_path.replace('_x', '_y'), ty.cpu().numpy())
    return tx, ty


def generate_incoming_table(traj_path=None, params=traj_in_params, device="cuda:0", spin_scale=5, substeps=6):
    """tennis_ball_in_estimator.py:82-140 (`generate_incoming_trajectory` there): rows over (height, vel_x, vel_y, vspin), 50 frames
    of (y, z) for a ball launched straight out from (0, 0, height)."""
    hh, vx, vz, vs = _mesh(params.HEIGHT_RANGE, params.VEL_X_RANGE, params.VEL_Y_RANGE, params.VSPIN_RANGE, device=device)
    n = hh.shape[0]
    pos = torch.stack([torch.zeros_like(hh), torch.zeros_like(hh), hh], 1)
    vel = torch.stack([torch.zeros_like(hh), vx, vz], 1)
    traj, _, _, _ = simulate(pos, vel, vs, num_frames=50, substeps=substeps, spin_scale=spin_scale, device=device, first_comp=1)
    assert traj.shape == (n, 50, 2)
    if traj_path is not None:
        np.save(traj_path, traj.cpu().numpy())
    return traj


def torch_sample_range(size, lo, hi, generator=None):   # tennis_ball.py:41-42
    return torch.rand(size, generator=generator) * (hi - lo) + lo


def pool_valid(traj, bounce_pos, bounce_idx, pass_net, bmin, bmax):
    """the pool's validity rule (tennis_ball.py:319-327): passes the net, first bounce inside the far box, rebound higher than 1 m.
    `bounce_pos.sum() != 0` is over the whole tensor, as in the reference."""
    valid = pass_net & (bounce_pos.sum() != 0) & (bounce_pos[:, 0] > bmin[0]) & (bounce_pos[:, 0] < bmax[0]) & \
        (bounce_pos[:, 1] > bmin[1]) & (bounce_pos[:, 1] < bmax[1])
    frame = torch.arange(traj.shape[1], device=traj.device)[None, :]
    after = torch.where(frame >= bounce_idx[:, None], traj[:, :, 2], torch.full_like(traj[:, :, 2], -math.inf))
    return valid & (after.max(dim=1).values > 1.0)      # `traj[i, bounce_idx[i]:, 2].max() > 1.0` without the Python loop over envs


class TennisBallGeneratorB200:
    """TennisBallGeneratorIsaac (tennis_ball.py:221-356) without Isaac Gym: `num_env` launches per reset() drawn from the same
    ranges, simulated by one kernel launch, filtered by the same validity rules."""

    def __init__(self, cfg, is_train=True, need_traj=True, need_reset=True, substeps=6, spin_scale=5, device="cuda:0", num_env=None,
                 generator=None):
        self.is_train, self.need_traj, self.substeps, self.spin_scale = is_train, need_traj, substeps, spin_scale
        self.device = torch.device(device)
        self.num_env = num_env if num_env is not None else (10000 if is_train else 1000)
        self.traj_pool = None
        self.generator = generator
        self.traj_length = cfg.get('ball_traj_length', 100)
        self.origin_min = torch.FloatTensor(cfg.get('origin_min', [-4, 12, 1]))
        self.origin_max = torch.FloatTensor(cfg.get('origin_max', [4, 13, 1.5]))
        self.bounce_min = torch.FloatTensor(cfg.get('bounce_min', [-3, -10, 0]))
        self.bounce_max = torch.FloatTensor(cfg.get('bounce_max', [3, -7, 0]))
        self.vel_range = torch.FloatTensor(cfg.get('vel_range', [28, 30]))
        self.vspin_range = torch.FloatTensor(cfg.get('vspin_range', [5, 10]))
        self.theta_range = torch.FloatTensor(cfg.get('theta_range', [5, 15]))
        if need_reset:
            self.reset()

    def reset(self):
        n, g = self.num_env, self.generator
        origin = torch_sample_range((n, 3), self.origin_min, self.origin_max, g)
        bounce = torch_sample_range((n, 3), self.bounce_min, self.bounce_max, g)
        d = torch.nn.functional.normalize(bounce[:, :2] - origin[:, :2], dim=1)
        speed = torch_sample_range((n,), self.vel_range[0], self.vel_range[1], g)
        theta = torch_sample_range((n,), self.theta_range[0], self.theta_range[1], g)
        vspin = torch_sample_range((n,), self.vspin_range[0], self.vspin_range[1], g)
        vel = torch.stack([speed * torch.cos(theta / 180 * np.pi) * d[:, 0], speed * torch.cos(theta / 180 * np.pi) * d[:, 1],
                           speed * torch.sin(theta / 180 * np.pi)]).T
        launch_pos, launch_vel, launch_vspin = origin.to(self.device), vel.contiguous().to(self.device), vspin.to(self.device)
        traj, bounce_pos, bounce_idx, pass_net = simulate(launch_pos, launch_vel, launch_vspin, num_frames=self.traj_length,
                                                          substeps=self.substeps, spin_scale=self.spin_scale, device=self.device)
        valid = pool_valid(traj, bounce_pos, bounce_idx, pass_net, self.bounce_min.to(self.device), self.bounce_max.to(self.device))
        assert valid.sum() > 0
        self.traj_pool = traj[valid].cpu()
        self.launch_pos, self.launch_vel, self.launch_vspin = launch_pos[valid].cpu(), launch_vel[valid].cpu(), launch_vspin[valid].cpu()
        return int(valid.sum())

    def generate(self, n_traj, need_init_state=False):
        idx = torch.randint(0, len(self.traj_pool), (n_traj,), generator=self.generator)
        if need_init_state:
            return self.traj_pool[idx].clone(), self.launch_pos[idx], self.launch_vel[idx], self.launch_vspin[idx]
        return self.traj_pool[idx].clone()

    def generate_init_state(self, n_ball):
        idx = torch.randint(0, len(self.launch_pos), (n_ball,), generator=self.generator)
        return self.launch_pos[idx], self.launch_vel[idx], self.launch_vspin[idx]

    def generate_all(self):
        return self.traj_pool, self.launch_pos, self.launch_vel, self.launch_vspin


def generate_incoming_trajectory(traj_path=None, substeps=6, rounds=100, max_rows=1000000, device="cuda:0", num_env=10000, seed=None,
                                 spin_scale=5):
    """tennis_ball.py:359-394: the trajectory pool file [P, 307], sorted by launch x."""
    g = torch.Generator().manual_seed(seed) if seed is not None else None
    gen = TennisBallGeneratorB200({}, is_train=True, need_reset=False, substeps=substeps, spin_scale=spin_scale, device=device,
                                  num_env=num_env, generator=g)
    chunks, rows = [], 0
    for _ in range(rounds):
        try:
            gen.reset()
        except AssertionError:
            continue
        traj, lp, lv, ls = gen.generate_all()
        chunks.append(torch.cat([lp, lv, ls.view(-1, 1), traj.reshape(-1, 300)], dim=1))
        rows += chunks[-1].shape[0]
        if rows > max_rows:
            break
    data = torch.cat(chunks, 0).numpy()
    data = data[np.argsort(data[:, 0])]
    if traj_path is not None:
        np.save(traj_path, data)
    return data
