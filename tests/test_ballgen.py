"""Offline tennis-ball data generators (SURVEY.md 8f-2): oracle vs the golden file (CPU), CUDA kernels vs oracle / golden (GPU).

Tolerances: float32 kernel vs the float32-state golden trajectories 2e-3 m over 100 frames of flight and bounces (positions up
to 25 m; the kernel keeps the state in float32 through all 1200 substeps, the golden run rounds it once per sim step);
double instantiation of the same kernel vs the float64 twin of the oracle 1e-9; flags / indices exact."""
import os

import numpy as np
import pytest
import torch

from oracle import ref_port_ballgen as P

HERE = os.path.dirname(os.path.abspath(__file__))
Z = np.load(os.path.join(HERE, "golden", "v2p_ballgen.npz"))


def _out_launch():
    return Z["out_vel"][:, 1], Z["out_vel"][:, 2], Z["out_vspin"]


# ------------------------------------------------------------------ CPU: the oracle is pinned by the reference's own functions
def test_oracle_simulate_matches_reference_run():
    traj, bpos, bidx, pnet = P.simulate(Z["sim_pos"], Z["sim_vel"], Z["sim_vspin"])
    assert np.abs(traj - Z["sim_traj"]).max() < 5e-5
    assert np.abs(bpos - Z["sim_bounce_pos"]).max() < 5e-6
    assert (bidx == Z["sim_bounce_idx"]).all() and (pnet == Z["sim_pass_net"]).all()
    assert 0 < pnet.sum() < len(pnet) and (bidx < 99).any()          # the fixture covers both outcomes
    traj, _, _, _ = P.simulate(Z["in_pos"], Z["in_vel"], Z["in_vspin"], num_frames=50)
    assert np.abs(traj - Z["in_traj"]).max() < 5e-5
    traj, bpos, bidx, pnet = P.simulate(Z["sim_pos"][:16], Z["sim_vel"][:16], Z["sim_vspin"][:16], substeps=2)   # 4R threshold branch
    assert np.abs(traj - Z["sim2_traj"]).max() < 5e-5 and (bidx == Z["sim2_bounce_idx"]).all() and (pnet == Z["sim2_pass_net"]).all()


def test_oracle_out_rows_match_reference_run():
    vh, vv, vs = _out_launch()
    m = len(vs)
    lp = np.zeros((m, 3), np.float32)
    lv = np.stack([np.zeros(m), vh, vv], 1).astype(np.float32)
    tx, ty = P.simulate_without_bounce(lp, lv, vs)
    assert np.abs(tx - Z["out_x"]).max() < 1e-5
    assert (np.abs(ty - Z["out_y"]) <= 1e-5 + 1e-4 * np.abs(Z["out_y"])).all()   # extrapolated entries divide by a float32 difference
    assert (Z["out_x"][:, 0] == 0).all() and (Z["out_y"][:, 0] == 0).all()    # the x = 0 / y = 0 columns pair sample 0 with sample -1
    assert (Z["out_y"][:, 1:, 0] != 0).all()                                  # no unwritten column: int(y * 10) hits every index


def test_launch_grids_have_the_reference_row_counts():
    assert len(P.launch_grid_out()[0]) == 550 * 150 * 100      # SURVEY.md 8f: 8 250 000 rows
    assert len(P.launch_grid_in()[0]) == 15 * 50 * 30 * 50     # 1 125 000 rows


# ------------------------------------------------------------------ GPU
gpu = pytest.mark.gpu


@gpu
def test_simulate_kernel_double_equals_oracle_twin():
    from vid2player3d_b200 import ball_gen
    for substeps, frames in ((6, 100), (2, 60)):
        ref = P.simulate(Z["sim_pos"].astype(np.float64), Z["sim_vel"].astype(np.float64), Z["sim_vspin"].astype(np.float64),
                         num_frames=frames, substeps=substeps, state32=False, world_kw=P.f32_physics())
        got = ball_gen.simulate(Z["sim_pos"], Z["sim_vel"], Z["sim_vspin"], num_frames=frames, substeps=substeps, dtype=torch.float64)
        assert np.abs(got[0].cpu().numpy() - ref[0]).max() < 1e-9
        assert np.abs(got[1].cpu().numpy() - ref[1]).max() < 1e-6      # the oracle keeps bounce_pos in float32 like the reference
        assert (got[2].cpu().numpy() == ref[2]).all() and (got[3].cpu().numpy() == ref[3]).all()


@gpu
def test_simulate_kernel_float_matches_golden():
    from vid2player3d_b200 import ball_gen
    traj, bpos, bidx, pnet = ball_gen.simulate(Z["sim_pos"], Z["sim_vel"], Z["sim_vspin"])
    assert traj.dtype == torch.float32 and traj.shape == (48, 100, 3)
    assert np.abs(traj.cpu().numpy() - Z["sim_traj"]).max() < 2e-3
    assert np.abs(bpos.cpu().numpy() - Z["sim_bounce_pos"]).max() < 2e-3
    assert (bidx.cpu().numpy() == Z["sim_bounce_idx"]).all() and (pnet.cpu().numpy() == Z["sim_pass_net"]).all()
    # incoming-table rows: (y, z) only, 50 frames
    t2, _, _, _ = ball_gen.simulate(Z["in_pos"], Z["in_vel"], Z["in_vspin"], num_frames=50, first_comp=1)
    assert t2.shape == (40, 50, 2) and np.abs(t2.cpu().numpy() - Z["in_traj"][:, :, 1:]).max() < 2e-3
    t3, _, b3, p3 = ball_gen.simulate(Z["sim_pos"][:16], Z["sim_vel"][:16], Z["sim_vspin"][:16], substeps=2)
    assert np.abs(t3.cpu().numpy() - Z["sim2_traj"]).max() < 2e-3
    assert (b3.cpu().numpy() == Z["sim2_bounce_idx"]).all() and (p3.cpu().numpy() == Z["sim2_pass_net"]).all()


@gpu
def test_out_rows_kernel_vs_oracle_and_golden():
    from vid2player3d_b200 import ball_gen
    vh, vv, vs = _out_launch()
    m = len(vs)
    lv = np.stack([np.zeros(m), vh, vv], 1)
    rx, ry = P.simulate_without_bounce(np.zeros((m, 3)), lv, vs.astype(np.float64), state32=False, world_kw=P.f32_physics())
    gx, gy = ball_gen.simulate_without_bounce(vh, vv, vs, dtype=torch.float64)
    # the oracle interpolates in the dtype of its trajectory (float64 here) and stores float32 tables
    assert np.abs(gx.cpu().numpy() - rx).max() < 1e-5
    assert (np.abs(gy.cpu().numpy() - ry) <= 1e-5 + 1e-6 * np.abs(ry)).all()
    fx, fy = ball_gen.simulate_without_bounce(vh, vv, vs)
    assert fx.dtype == torch.float32 and fx.shape == (m, 60) and fy.shape == (m, 30, 2)
    assert np.abs(fx.cpu().numpy() - Z["out_x"]).max() < 2e-3
    # entries extrapolated beyond the 2 s of flight reach hundreds of metres: relative tolerance there
    assert (np.abs(fy.cpu().numpy() - Z["out_y"]) <= 2e-3 + 1e-3 * np.abs(Z["out_y"])).all()


@gpu
def test_generators_edge_cases_and_errors():
    from vid2player3d_b200 import ball_gen
    e = np.zeros((0, 3), np.float32)
    traj, bpos, bidx, pnet = ball_gen.simulate(e, e, np.zeros(0, np.float32))
    assert traj.shape == (0, 100, 3) and bidx.shape == (0,)
    one = ball_gen.simulate(Z["sim_pos"][:1], Z["sim_vel"][:1], Z["sim_vspin"][:1])
    many = ball_gen.simulate(Z["sim_pos"], Z["sim_vel"], Z["sim_vspin"])
    assert torch.equal(one[0][0], many[0][0])                                  # a ball's result does not depend on the batch
    with pytest.raises(RuntimeError, match="bad simulation parameters"):
        ball_gen.simulate(Z["sim_pos"], Z["sim_vel"], Z["sim_vspin"], substeps=0)
    # a ball at rest on the ground stays there (zero velocity: the reference's 0/0 force is NaN; the kernel's guarded norm gives 0)
    rest = ball_gen.simulate(np.array([[0, 0, 0.032]], np.float32), np.zeros((1, 3), np.float32), np.zeros(1, np.float32), num_frames=10)
    assert torch.isfinite(rest[0]).all() and abs(float(rest[0][0, -1, 2]) - 0.032) < 1e-4


@gpu
def test_full_size_tables_properties():
    """BASELINE-size products: the 8 250 000-row outgoing tables (3.96 GB) and the 1 125 000-row incoming table in one launch each;
    checked through size-independent properties + a strided sample against the float64 oracle."""
    from vid2player3d_b200 import ball_gen
    tx, ty = ball_gen.generate_outgoing_trajectory()
    assert tx.shape == (8250000, 60) and ty.shape == (8250000, 30, 2)
    vh, vv, vs = P.launch_grid_out()
    assert bool(torch.isfinite(tx).all()) and bool((tx[:, 0] == 0).all()) and bool((ty[:, 0] == 0).all())
    # A ball that is still above its launch height after the 2 s of flight has its drop columns EXTRAPOLATED from the last two
    # samples (the reference does the same, :101-110): meaningless values, non-finite when the two heights coincide (14 of the
    # 8.25 M rows on the GPU).  Balls launched flat or downwards without back-spin (whose lift exceeds gravity at 60 m/s) come down at
    # once: there every column is an interpolation.
    down = torch.from_numpy((vv <= 0) & (vs >= 0)).to(ty.device)
    assert bool(torch.isfinite(ty[down]).all())
    assert bool((ty[down][:, 2:, 1] >= ty[down][:, 1:-1, 1]).all())     # a larger drop is never reached earlier
    assert bool((ty[down][:, 1:, 0] > 0).all())                         # ... and the ball has moved forward by then
    assert int((~torch.isfinite(ty)).any(2).any(1).sum()) < 100
    pick = np.arange(0, len(vh), 350003)
    sx, sy = ball_gen.simulate_without_bounce(vh[pick], vv[pick], vs[pick])
    assert torch.equal(sx, tx[pick]) and torch.equal(sy, ty[pick])              # rows do not depend on the batch they were in
    m = len(pick)
    rx, ry = P.simulate_without_bounce(np.zeros((m, 3)), np.stack([np.zeros(m), vh[pick], vv[pick]], 1).astype(np.float64),
                                       vs[pick].astype(np.float64), state32=False)
    assert np.abs(sx.cpu().numpy() - rx).max() < 2e-3
    assert (np.abs(sy.cpu().numpy() - ry) <= 2e-3 + 1e-3 * np.abs(ry)).all()
    del tx, ty
    tab = ball_gen.generate_incoming_table()
    assert tab.shape == (1125000, 50, 2) and bool(torch.isfinite(tab).all())
    hh, ivx, ivz, isp = P.launch_grid_in()
    assert np.abs(tab[:, 0, 1].cpu().numpy() - hh).max() < 1e-6 and bool((tab[:, 0, 0] == 0).all())   # frame 0 = the launch point
    assert bool((tab[:, :, 1] >= 0.032 - 1e-4).all())                                                 # never below the ground
    pick = np.arange(0, len(hh), 37501)
    m = len(pick)
    lp = np.stack([np.zeros(m), np.zeros(m), hh[pick]], 1).astype(np.float32)
    lv = np.stack([np.zeros(m), ivx[pick], ivz[pick]], 1).astype(np.float32)
    again, _, _, _ = ball_gen.simulate(lp, lv, isp[pick], num_frames=50, first_comp=1)
    assert torch.equal(again, tab[pick])                                                              # rows do not depend on the batch
    ref = P.simulate(lp.astype(np.float64), lv.astype(np.float64), isp[pick].astype(np.float64), num_frames=50, state32=False,
                     world_kw=P.f32_physics())[0]
    assert np.abs(tab[pick].cpu().numpy() - ref[:, :, 1:]).max() < 2e-3


@gpu
def test_pool_generator_follows_the_reference_rules():
    from vid2player3d_b200 import ball_gen
    data = ball_gen.generate_incoming_trajectory(rounds=2, num_env=4096, seed=3)
    assert data.ndim == 2 and data.shape[1] == 307 and data.dtype == np.float32 and len(data) > 100
    assert (np.diff(data[:, 0]) >= 0).all()                                     # sorted by launch x (:378-382)
    traj = data[:, 7:].reshape(-1, 100, 3)
    assert np.abs(traj[:, 0] - data[:, 0:3]).max() == 0                         # frame 0 = launch position
    assert (traj[:, :, 1].min(1) < 0).all()                                     # every kept ball crosses the net line
    again = ball_gen.generate_incoming_trajectory(rounds=2, num_env=4096, seed=3)
    assert np.array_equal(data, again)                                          # seeded -> reproducible
