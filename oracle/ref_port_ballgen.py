"""ORACLE (test infrastructure - never imported by the product path): numpy restatement of the reference's offline
tennis-ball data generators (SURVEY.md 8f-2).

  simulate                 vid2player/utils/tennis_ball.py:113-218   trajectory pool / incoming-ball table rows
  simulate_without_bounce  vid2player/utils/tennis_ball_out_estimator.py:21-121   outgoing-ball estimator rows
  launch_grid_out / launch_grid_in   the row order of generate_outgoing_trajectory (:208-258) and
                           tennis_ball_in_estimator.py:82-140

The reference drives Isaac Gym (`gym.simulate`) for the rigid-body part; Isaac Gym is absent (SURVEY.md 8c), so the
sim step is OUR ball model (`BallWorld.sim_step`, the float64 twin of csrc/b200env.cu::ball_substep without a racket:
semi-implicit Euler, h = 1/60/substeps, force held over the sim step, impulse bounce with restitution on the normal
part and Coulomb friction capped at the sticking impulse).  Everything AROUND the sim step - when forces are
evaluated, the signed-spin lift, bounce / net flags, the back-spin -> top-spin hack, the 30 Hz sampling, the grid
resampling with its index arithmetic - follows the reference line by line and is pinned by
tests/golden/v2p_ballgen.npz, which is produced by executing the reference's own two functions on a fake `gym`
whose simulate() is `BallWorld.sim_step` (tests/golden/make_golden_ballgen.py).

`state32=True` keeps the root-state tensor in float32 between sim steps and evaluates the forces in float32 like the
reference's torch code (this is the mode the golden file pins); `state32=False` is the float64 twin the CUDA kernel's
double instantiation is compared with.
"""
import math

import numpy as np

M_BALL, R_BALL, RHO = 0.057, 0.032, 1.21          # tennis_ball.py:15-18
KF = (RHO * math.pi * R_BALL * R_BALL) / 2        # :23
BASE_CD = 0.55                                    # :26
NET_HEIGHT = 1.07                                 # :20
I_BALL = 4e-5                                     # tennis_ball.urdf


class BallWorld:
    """N free balls over the plane z = 0 (our model; see module docstring).  state[N,13] = pos3 quat4 vel3 angvel3."""

    def __init__(self, n, substeps=6, sim_dt=1.0 / 60.0, e_ground=0.7, mu_ground=0.6, vth=0.2, gravity=-9.81, ground=True,
                 mass=M_BALL, radius=R_BALL, inertia=I_BALL):
        self.n, self.substeps, self.h = n, substeps, sim_dt / substeps
        self.e, self.mu, self.vth, self.g, self.ground = e_ground, mu_ground, vth, gravity, ground
        self.m, self.R, self.I = mass, radius, inertia

    def sim_step(self, state, force):
        """one gym.simulate(): `substeps` substeps with the applied force held constant; float64 arithmetic in place"""
        p, v, w = state[:, 0:3], state[:, 7:10], state[:, 10:13]
        h, m, R, I = self.h, self.m, self.R, self.I
        for _ in range(self.substeps):
            v[:, 0] += h * force[:, 0] / m
            v[:, 1] += h * force[:, 1] / m
            v[:, 2] += h * (self.g + force[:, 2] / m)
            p += h * v
            if not self.ground:
                continue
            hit = np.nonzero((p[:, 2] < R) & (v[:, 2] < 0))[0]
            if len(hit) == 0:
                continue
            # contact point -R z; u = v + w x (-R z); the balls in contact at once, row by row the same arithmetic
            r = np.array([0.0, 0.0, -R])
            u = v[hit] + np.cross(w[hit], r)
            i = hit[u[:, 2] < 0]
            u = u[u[:, 2] < 0]
            un = u[:, 2]
            jn = np.where(-un > self.vth, 1.0 + self.e, 1.0) * (-un) * m
            ut = np.stack([u[:, 0], u[:, 1], np.zeros(len(u))], 1)
            utn = np.sqrt(u[:, 0] * u[:, 0] + u[:, 1] * u[:, 1])
            slide = utn > 1e-9
            jt = np.where(slide, np.minimum(self.mu * jn, m * utn / (1.0 + m * R * R / I)), 0.0)
            ut[slide] /= utn[slide, None]
            J = np.stack([np.zeros(len(u)), np.zeros(len(u)), jn], 1) - jt[:, None] * ut
            v[i] += J / m
            w[i] += np.cross(r, J) / I
            p[hit, 2] = R


def _aero(vel, angvel, launch_vspin, spin_scale, dt):
    """forces of simulate() :160-183 / simulate_without_bounce :58-74 (signed spin)"""
    f = dt
    vel = vel.astype(f)
    vs = np.sqrt((vel * vel).sum(-1, dtype=f)).astype(f)[:, None]
    vn = vel / vs
    g = np.array([0.0, 0.0, -1.0], f)
    vt = np.cross(vn, g).astype(f)
    vspin = (np.sqrt((angvel.astype(f) ** 2).sum(-1, dtype=f)) / f(math.pi * 2)).astype(f)
    vspin = np.where(launch_vspin > 0, vspin, vspin * f(-1))[:, None].astype(f)
    vsc = vspin * f(spin_scale)
    cl = (f(1) / (f(2) + np.abs(vs / (vsc + f(1e-6))))).astype(f)
    cl = cl * np.where(vspin > 0, f(-1), f(1))
    drag = -f(KF) * f(BASE_CD) * vs * vel
    lift = -f(KF) * cl * vs ** 2 * np.cross(vt, vn).astype(f)
    return (drag + lift).astype(f)


def launch_state(launch_pos, launch_vel, launch_vspin, dt):
    """root state rows at launch: ang vel = vspin * 2pi * normalize(v x (0,0,-1))  (tennis_ball.py:134-139)"""
    n = len(launch_pos)
    st = np.zeros((n, 13), dt)
    st[:, 6] = 1
    c = np.cross(launch_vel.astype(dt), np.array([0.0, 0.0, -1.0], dt))
    nn = np.maximum(np.sqrt((c * c).sum(-1, keepdims=True)), dt(1e-12))
    st[:, 0:3], st[:, 7:10] = launch_pos, launch_vel
    st[:, 10:13] = launch_vspin.astype(dt)[:, None] * dt(math.pi * 2) * (c / nn)
    return st


def simulate(launch_pos, launch_vel, launch_vspin, control_freq_inv=2, num_frames=100, substeps=6, spin_scale=5,
             state32=True, world_kw=None):
    """tennis_ball.py:113-218 -> traj[n,num_frames,3], bounce_pos[n,3], bounce_idx[n] int64, pass_net[n] bool"""
    dt = np.float32 if state32 else np.float64
    n = len(launch_pos)
    world = BallWorld(n, substeps=substeps, **(world_kw or {}))
    st = launch_state(np.asarray(launch_pos), np.asarray(launch_vel), np.asarray(launch_vspin), dt)
    lvspin = np.array(launch_vspin, dt)
    traj = np.zeros((n, num_frames, 3), dt)
    bounce_pos = np.zeros((n, 3), dt)
    bounce_idx = np.zeros(n, np.int64) + num_frames - 1
    has_bounce, has_pass_net, pass_ok = np.zeros(n, bool), np.zeros(n, bool), np.zeros(n, bool)
    thr = world.R * 6 if substeps > 2 else world.R * 4
    for t in range(num_frames):
        traj[:, t] = st[:, 0:3]
        for _ in range(control_freq_inv):
            pos = st[:, 0:3]
            force = _aero(st[:, 7:10], st[:, 10:13], lvspin, spin_scale, dt)
            now = (~has_pass_net) & (pos[:, 1] < 0)                                  # :168-170
            pass_ok[now] = (~has_bounce[now]) & (pos[now, 2] > NET_HEIGHT)
            has_pass_net |= now
            bnow = ~has_bounce & (pos[:, 2] <= thr)                                  # :185-191
            bounce_pos[bnow] = pos[bnow]
            bounce_idx[bnow] = t
            has_bounce |= bnow
            lvspin[bnow] = np.where(lvspin[bnow] > 0, lvspin[bnow], -lvspin[bnow])   # :194-199 back-spin -> top-spin
            s64 = st.astype(np.float64)
            world.sim_step(s64, force.astype(np.float64))
            st = s64.astype(dt)
    return traj, bounce_pos, bounce_idx, pass_ok


def torch_arange(lo, hi, step):
    """values of torch.arange(lo, hi, step) (float32: start + i*step computed in double, rounded) and its length"""
    n = int(math.ceil((hi - lo) / step))
    return (lo + np.arange(n, dtype=np.float64) * step).astype(np.float32)


def grid(rng, scale):
    """values of torch.arange(*rng), the column int(v * scale) the reference writes each one to (:98, :110; negative = counted
    from the end of the row) and the row width"""
    v = torch_arange(*rng)
    return v, np.array([int(x * np.float32(scale)) for x in v], np.int64), int((rng[1] - rng[0]) / rng[2])


def simulate_without_bounce(launch_pos, launch_vel, launch_vspin, traj_x_range=(0, 30, 0.5), traj_y_range=(0, 3, 0.1),
                            control_freq_inv=2, num_frames=60, substeps=6, spin_scale=5, state32=True, world_kw=None, grid_x=None,
                            grid_y=None, table_dtype=np.float32, walk=None):
    """tennis_ball_out_estimator.py:21-121 -> traj_x[n, NX] (height over launch at horizontal distance x),
    traj_y[n, NY, 2] (distance, time at which the ball has dropped y below the launch height)

    grid_x / grid_y: explicit (values, columns, row width) instead of grid(traj_x_range, 2) / grid(traj_y_range, 10).  The columns
    are written in grid order with Python's index semantics (negative counts from the end, outside [-NX, NX) raises IndexError).
    table_dtype: the tables' storage type (the reference's float32 by default).  walk: a dict that receives the (y, z) samples
    [n, T, 2] and the sample index each grid value stopped at, t_x [n, ngx] / t_y [n, ngy] (the value interpolates samples t-1, t)."""
    dt = np.float32 if state32 else np.float64
    n = len(launch_pos)
    world = BallWorld(n, substeps=substeps, ground=False, **(world_kw or {}))
    st = launch_state(np.asarray(launch_pos), np.asarray(launch_vel), np.asarray(launch_vspin), dt)
    lvspin = np.array(launch_vspin, dt)
    samples = []
    for _ in range(num_frames + 1):
        for _ in range(control_freq_inv):
            samples.append(st[:, 0:3].copy())
            force = _aero(st[:, 7:10], st[:, 10:13], lvspin, spin_scale, dt)
            s64 = st.astype(np.float64)
            world.sim_step(s64, force.astype(np.float64))
            st = s64.astype(dt)
    traj = np.stack(samples, 1)[:, :, 1:].copy()          # (y, z)                       :82
    traj[:, :, 1] -= traj[0, 0, 1].copy()                # :83 height relative to the launch height (value taken ONCE: the reference's
                                                         # in-place op aliases its operand, see tests/golden/make_golden_ballgen.py)
    T = traj.shape[1]
    gx, cx, nx = grid(traj_x_range, 2) if grid_x is None else grid_x
    gy, cy, ny = grid(traj_y_range, 10) if grid_y is None else grid_y
    traj_x = np.zeros((n, nx), table_dtype)
    traj_y = np.zeros((n, ny, 2), table_dtype)
    ids = np.arange(n)
    t_x, t_y = np.zeros((n, len(gx)), np.int64), np.zeros((n, len(gy)), np.int64)
    t = np.zeros(n, np.int64)
    with np.errstate(divide="ignore", invalid="ignore"):    # two equal samples: inf / nan entries, like the reference
        for j, (x, c) in enumerate(zip(np.asarray(gx, np.float32), cx)):   # :90-98
            while True:
                adv = (t < T - 1) & (traj[ids, t, 0] < x)
                if adv.sum() > 0:
                    t[adv] += 1
                else:
                    break
            t_x[:, j] = t
            x1, x2 = traj[ids, t - 1, 0], traj[ids, t, 0]    # t - 1 == -1 wraps to the last sample, like torch
            w = (x - x1) / (x2 - x1)
            traj_x[:, int(c)] = traj[ids, t - 1, 1] * (1 - w) + traj[ids, t, 1] * w
        t = np.zeros(n, np.int64)
        for j, (y, c) in enumerate(zip(np.asarray(gy, np.float32), cy)):   # :101-110
            while True:
                adv = (t < T - 1) & (-traj[ids, t, 1] < y)
                if adv.sum() > 0:
                    t[adv] += 1
                else:
                    break
            t_y[:, j] = t
            y1, y2 = traj[ids, t - 1, 1], traj[ids, t, 1]
            w = (-y - y1) / (y2 - y1)
            traj_y[:, int(c), 0] = traj[ids, t - 1, 0] * (1 - w) + traj[ids, t, 0] * w
            tt = (t - 1).astype(dt) * (1 - w) + t.astype(dt) * w     # torch: int64 * float32 -> float32
            traj_y[:, int(c), 1] = tt / (control_freq_inv * 30)
    if walk is not None:
        walk.update(samples=traj, t_x=t_x, t_y=t_y)
    return traj_x, traj_y


def f32_physics():
    """the parameter block as the C ABI carries it (b200ball_sim_t holds floats): what the kernel's double instantiation integrates"""
    f = lambda x: float(np.float32(x))  # noqa: E731
    return dict(sim_dt=f(1.0 / 60.0), e_ground=f(0.7), mu_ground=f(0.6), vth=f(0.2), gravity=f(-9.81), mass=f(M_BALL), radius=f(R_BALL),
                inertia=f(I_BALL))


def launch_grid_out(vel_x=(10, 65, 0.1), vel_y=(-5, 10, 0.1), vspin=(-10, 10, 0.2)):
    """row order of generate_outgoing_trajectory (:208-232): C order over (horizontal speed, vertical speed, spin);
    np.arange values cast to float32 like `batch_vel_y[i, :, :] = vel_y`"""
    a, b, c = (np.arange(*r).astype(np.float32) for r in (vel_x, vel_y, vspin))
    A, Bv, Cv = np.meshgrid(a, b, c, indexing="ij")
    return A.ravel(), Bv.ravel(), Cv.ravel()


def launch_grid_in(height=(0.5, 2, 0.1), vel_x=(25, 30, 0.1), vel_y=(5, 8, 0.1), vspin=(5, 10, 0.1)):
    """row order of tennis_ball_in_estimator.generate_incoming_trajectory (:82-111)"""
    axes = [np.arange(*r).astype(np.float32) for r in (height, vel_x, vel_y, vspin)]
    G = np.meshgrid(*axes, indexing="ij")
    return tuple(g.ravel() for g in G)
