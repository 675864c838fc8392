"""Pin oracle/ref_port_v2p.py against fixtures produced by executing the reference's vid2player code (CPU only)."""
import numpy as np

from conftest import golden
from oracle import ref_port_v2p as V


def close(a, b, tol=1e-5, msg=""):
    np.testing.assert_allclose(a, b, rtol=0, atol=tol, err_msg=msg)


def test_smpl_to_sim():
    g = golden("v2p_smpl_to_sim.npz")
    names = ("root_pos", "root_rot", "dof_pos", "root_vel", "root_ang_vel", "dof_vel", "rb_pos", "rb_rot")
    a = V.smpl_to_sim(g["root0"], g["rotmat0"], g["rest"], g["parents"], g["smpl_2_mujoco"], float(g["dt"]))
    for n, x in zip(names, a):
        close(x, g["a_" + n], 2e-5, n)
    b = V.smpl_to_sim(g["root1"], g["rotmat1"], g["rest"], g["parents"], g["smpl_2_mujoco"], float(g["dt"]),
                      prev_root_pos=g["a_root_pos"], prev_rb_rot=g["a_rb_rot"])
    for n, x in zip(names, b):
        tol = {"dof_vel": 2e-3, "root_ang_vel": 6e-2}.get(n, 2e-5)  # finite differences divide by dt (and dt^2 for the root)
        close(x, g["b_" + n], tol, n)


def test_ball_aero_and_reset():
    g = golden("v2p_ball.npz")
    for s in (2, 6):
        force, hb, now = V.ball_aero(g[f"s{s}_ball_states"], g[f"s{s}_has_bounce_in"], s, 5.0)
        close(force, g[f"s{s}_force"], 1e-6)
        assert np.array_equal(hb, g[f"s{s}_has_bounce"]) and np.array_equal(now, g[f"s{s}_has_bounce_now"])
        close(np.where(now[:, None], g[f"s{s}_ball_states"][:, 0:3], 0), g[f"s{s}_bounce_pos"], 0)
    traj, pos, vel, angvel = V.ball_reset(g["pool"], g["reset_pool_index"])
    ids = g["reset_ids"]
    close(traj, g["reset_traj"], 0)
    close(pos, g["reset_ball_states"][ids, 0:3], 0)
    close(vel, g["reset_ball_states"][ids, 7:10], 0)
    close(angvel, g["reset_ball_states"][ids, 10:13], 2e-5)
    assert not g["reset_has_bounce"][ids].any() and not g["reset_contact"][ids].any() and g["reset_has_bounce"].sum() == 64 - len(ids)


def test_update_state_from_sim():
    g = golden("v2p_update_state.npz")
    for grip in ("eastern", "semi_western"):
        o = V.update_state_from_sim(g[f"{grip}_rbs"], g[f"{grip}_root_states"], g[f"{grip}_ball_states"], g[f"{grip}_prev_ball_vel"],
                                    g[f"{grip}_contact_in"], grip)
        for k, v in o.items():
            if v.dtype == bool:
                assert np.array_equal(v, g[f"{grip}_{k}"]), k
            else:
                close(v, g[f"{grip}_{k}"], 2e-6, k)
        assert o["contact_now"].sum() > 0


def test_controller_obs_rewards_estimator_reset():
    g = golden("v2p_controller.npz")
    obs = V.controller_obs(g["rbs"], g["p_root_pos"], g["p_root_vel"], g["p_racket_normal"], g["ball_traj"], g["target_bounce_pos"], 10)
    close(obs, g["obs"], 2e-6)
    scales = {'pos': 5.0, 'phase': 10.0, 'bounce_pos': 0.05, 'bounce_time': 0.1}
    w = {'pos': 0.5, 'ball_pos': 0.5}
    # estimator + bounce-in bookkeeping of _update_state (:271-314)
    upd = (g["tar_action"] == 0) & g["p_has_bounce_now"]
    assert np.array_equal(np.where(upd, V.in_court(g["p_bounce_pos"]), False), g["bounce_in"])
    now = g["p_has_racket_ball_contact_now"]
    valid, bp, bt, mh = V.estimator_estimate(g["ball_states"], g["est_x"], g["est_y"], g["est_params"])
    use = now & valid
    assert use.sum() >= 3
    est_pos = np.zeros((len(now), 3), np.float32)
    est_pos[use, :2] = bp[use]
    close(est_pos, g["est_bounce_pos"], 1e-5)
    close(np.where(use, bt, 0), g["est_bounce_time"], 1e-6)
    close(np.where(use, mh, 0), g["est_max_height"], 1e-5)
    assert np.array_equal(np.where(use, V.in_court(est_pos), False), g["est_bounce_in"])
    r, s = V.reward_reach(g["phase"], g["tar_action"], g["p_racket_pos"], g["p_ball_pos"], g["swing_type"], scales, w)
    close(r, g["rew_reach"]); close(s, g["sub_reach"])
    r, s = V.reward_return(g["phase"], g["p_racket_pos"], g["p_ball_pos"], g["p_has_racket_ball_contact"], g["p_has_bounce"],
                           g["p_bounce_pos"], g["target_bounce_pos"], g["swing_type"], scales, w)
    close(r, g["rew_return"]); close(s, g["sub_return"])
    r, s = V.reward_return_w_estimate(g["p_racket_pos"], g["phase"], g["swing_type_cycle"], g["p_ball_pos"], g["p_has_racket_ball_contact"],
                                      g["est_bounce_pos"], g["est_bounce_time"], g["est_bounce_in"], g["target_bounce_pos"], scales, w)
    close(r, g["rew_return_w_estimate"]); close(s, g["sub_return_w_estimate"])
    assert str(g["names_return_w_estimate"]) == "pos_reward,ball_pos_reward" and str(g["names_reach"]) == "pos_reward"
    assert np.array_equal(V.check_out_of_court(g["p_root_pos"], g["court_min"], g["court_max"]), g["out_of_court"])
    reset, term, rea, rec = V.controller_reset(g["p_root_pos"], g["court_min"], g["court_max"], np.isnan(g["obs_for_reset"]).any(axis=1),
                                               g["progress"], 300, g["tar_time"], g["tar_time_total"], g["tar_action"],
                                               g["p_has_racket_ball_contact"], g["p_ball_pos"], g["est_bounce_in"])
    assert np.array_equal(reset, g["reset"]) and np.array_equal(term, g["terminate"])
    assert np.array_equal(rea, g["reset_reaction"]) and np.array_equal(rec, g["reset_recovery"])
    assert 0 < reset.sum() < len(reset)


def test_fix_head_orientation():
    g = golden("v2p_fix_head.npz")
    a = V.smpl_to_sim(g["player_root_pos"], g["rotmat_in"], g["rest"], g["parents"], g["smpl_2_mujoco"], float(g["dt"]))
    out = V.fix_head_orientation(g["rotmat_in"], a[7][:, 13], a[6][:, 13], g["ball_pos"], g["root_pos"])
    close(out, g["rotmat_out"], 2e-6)
    assert np.abs(out - g["rotmat_in"]).max() > 0.05          # a correction happened ...
    assert np.array_equal(out[1], g["rotmat_in"][1]) or np.abs(out[1] - g["rotmat_in"][1]).max() < 2e-6   # ... except for the "miss" rows
    b = V.smpl_to_sim(g["player_root_pos"], out, g["rest"], g["parents"], g["smpl_2_mujoco"], float(g["dt"]),
                      prev_root_pos=g["prev_target_root_pos"], prev_rb_rot=g["prev_target_rb_rot"])
    close(b[2], g["target_dof_pos"], 2e-5); close(b[6], g["target_rb_pos"], 2e-5); close(b[7], g["target_rb_rot"], 2e-5)


def test_dual_golden():
    """dual mode: in-estimator (index math on the small AND the shipped grid), _reset_balls, _compute_reset vs the reference"""
    g = golden("v2p_dual.npz")
    idx, snapped = V.in_estimator_index(g["full_h"], g["full_vx"], g["full_vy"], g["full_vs"], g["in_params_full"])
    assert np.array_equal(idx, g["full_index"])
    np.testing.assert_array_equal(np.stack(snapped, -1), g["full_snapped"])
    bs = g["in_states"]
    vspin = np.sqrt((bs[:, 10:13] ** 2).sum(-1)) / np.float32(2 * np.pi)
    idx, _ = V.in_estimator_index(bs[:, 2], np.sqrt((bs[:, 7:9] ** 2).sum(-1)), bs[:, 9], vspin, g["in_params"])
    assert np.array_equal(idx, g["in_index"])
    traj, s_in, s_out = V.in_estimator_estimate(bs, g["in_table"], g["in_params"])
    np.testing.assert_allclose(traj, g["in_traj"], rtol=0, atol=1e-5)
    np.testing.assert_allclose(s_in, g["in_states_in"], rtol=0, atol=2e-5)
    np.testing.assert_allclose(s_out, g["in_states_out"], rtol=0, atol=2e-5)
    # _reset_balls (mixed parities in the id list)
    traj, after, extra = V.dual_reset_balls(g["rb_states_before"], g["rb_racket_pos"], g["rb_recovery_ids"], g["rb_ball_ids"], g["rb_rand"],
                                            g["in_table"], g["in_params"])
    np.testing.assert_allclose(traj, g["rb_traj"], rtol=0, atol=1e-5)
    np.testing.assert_allclose(after, g["rb_states_after"], rtol=0, atol=2e-5)
    np.testing.assert_allclose(extra["ball_pos"], g["rb_ball_pos"][g["rb_ball_ids"]], rtol=0, atol=2e-6)
    np.testing.assert_allclose(extra["ball_vel"], g["rb_ball_vel"][g["rb_ball_ids"]], rtol=0, atol=2e-5)
    ids = g["rb_ball_ids"]
    assert not g["rb_has_bounce"][ids].any() and not g["rb_has_contact"][ids].any() and not g["rb_bounce_pos"][ids].any()
    rest = np.setdiff1d(np.arange(32), ids)
    assert g["rb_has_bounce"][rest].all() and g["rb_has_contact"][rest].all()
    # _compute_reset
    reset, reaction, recovery, dist = V.dual_controller_reset(g["cr_tar_action"], g["cr_has_contact"], g["cr_has_bounce"], g["cr_ball_pos"],
                                                              g["cr_root_pos"], g["cr_root_vel"], g["cr_bounce_in"], g["cr_distance"],
                                                              g["crreset_buf"])
    assert np.array_equal(reset, g["cr_out_reset"]) and np.array_equal(reaction, g["cr_out_reaction"])
    assert np.array_equal(recovery, g["cr_out_recovery"])
    np.testing.assert_allclose(dist, g["cr_out_distance"], rtol=0, atol=1e-6)
    assert g["cr_out_reset"].sum() > g["crreset_buf"].sum() and g["cr_out_reaction"].any() and g["cr_out_recovery"].any()


def test_history_ball_obs_variant():
    """use_history_ball_obs (physics_mvae_controller.py:213-214, 345-351): fill on a reaction reset, roll + append at every
    observation, partial refresh touches the listed rows only"""
    g = golden("v2p_controller.npz")
    assert np.array_equal(g["hist_in"], g["ball_obs_after"])
    h = V.reset_ball_obs(g["hist_in"], g["hist_ball_pos0"], g["hist_reset_ids"])
    assert np.array_equal(h, g["hist_after_reset"])
    part = g["hist_part_ids"]
    h = V.roll_ball_obs(h, g["hist_ball_pos0"], part)
    assert np.array_equal(h, g["hist_after_partial"])
    args = (g["rbs"], g["p_root_pos"], g["p_root_vel"], g["p_racket_normal"], g["ball_traj"], g["hist_target_bounce_pos"], 10)
    close(V.controller_obs(*args, ball_obs=h)[part], g["hist_obs_partial"][part], 2e-6)
    for k in (1, 2):
        h = V.roll_ball_obs(h, g[f"hist_ball_pos{k}"])
        assert np.array_equal(h, g[f"hist_after_full{k}"])
        close(V.controller_obs(*args, ball_obs=h), g[f"hist_obs_full{k}"], 2e-6)



def test_task_reset():
    """pool_index against TennisBallGeneratorOffline.generate with start_pos (x edges at -4, 4, +-8 / P, outside the court; ball_y at 0
    and +-1 ulp), and task_reset's recovery / reaction bookkeeping against _reset_recovery_tasks / _reset_reaction_tasks in both
    target modes (discrete seeds at 0.33 and 0.67), history rows included; the fixture's recorded draws are fed back in"""
    g = golden("v2p_task_reset.npz")
    P = int(g["tr_pool_size"])
    got = V.pool_index(g["tr_start"], g["tr_pool_rand"], g["tr_side_rand"], P)
    assert np.array_equal(got, g["tr_index"]), np.flatnonzero(got != g["tr_index"])
    for mode in ("continuous", "discrete"):
        i = lambda k: g[f"{mode}_in_{k}"].copy()  # noqa: E731
        n = len(i("ball_pos"))
        rea, rec = np.zeros(n, bool), np.zeros(n, bool)
        rea[g[f"{mode}_rea_ids"]], rec[g[f"{mode}_rec_ids"]] = True, True
        # a pool whose row e is env e's ball position: the launch position the reaction rows' history is reset to
        pool = np.zeros((n, 307), np.float32)
        pool[:, 0:3] = i("ball_pos")
        ball_pos = i("ball_pos")
        ball_pos[:, 1] = -1          # near side: the draw pool_rand (= the env) picks the row
        s = dict(ball_pos=ball_pos, ball_vel=np.zeros((n, 3), np.float32), bounce_pos=i("bounce_pos"), ball_traj=np.zeros((n, 100, 3), np.float32),
                 est_bounce_pos=i("est_bounce_pos"), est_bounce_time=i("est_bounce_time"), est_max_height=i("est_max_height"),
                 target_bounce_pos=i("target_bounce_pos"), ball_states=np.zeros((n, 13), np.float32), rbs_ball=np.zeros((n, 13), np.float32),
                 has_bounce=i("has_bounce"), has_contact=np.zeros(n, bool), bounce_in=i("bounce_in"), est_bounce_in=i("est_bounce_in"),
                 tar_time=i("tar_time"), tar_time_total=i("tar_time_total"), tar_action=i("tar_action"), num_reset_reaction=i("num_reset_reaction"),
                 swing_type_cycle=i("cycle"), reset_reaction=rea, reset_recovery=rec, ball_obs=i("ball_obs"))
        frame = np.zeros(n, np.int64)
        frame[g[f"{mode}_rea_ids"]] = g[f"{mode}_frame_rand"]
        seed = g[f"{mode}_seed"]
        if mode == "discrete":
            seed = np.zeros(n, np.float32)
            seed[g[f"{mode}_rea_ids"]] = g[f"{mode}_seed"]
        out = V.task_reset(s, dict(pool=pool, reaction_nframes=70, target_mode=mode, target_min=(-3, 9, 0), target_max=(3, 11, 0)),
                           dict(pool_rand=np.arange(n), side_rand=np.zeros(n, np.int64), frame_rand=frame, target_seed=seed))
        for k, gk in (("ball_obs", "ball_obs"), ("tar_time", "tar_time"), ("tar_action", "tar_action"), ("num_reset_reaction", "num_reset_reaction"),
                      ("bounce_in", "bounce_in"), ("est_bounce_in", "est_bounce_in"), ("est_bounce_pos", "est_bounce_pos"),
                      ("est_bounce_time", "est_bounce_time"), ("est_max_height", "est_max_height"), ("tar_time_total", "tar_time_total"),
                      ("target_bounce_pos", "target_bounce_pos"), ("swing_type_cycle", "cycle")):
            assert np.array_equal(out[k], g[f"{mode}_out_{gk}"]), (mode, k)
        # has_bounce / bounce_pos: the reference's _reset_balls (not in this fixture) clears them for the reaction rows too
        for k in ("has_bounce", "bounce_pos"):
            assert np.array_equal(out[k][~rea], g[f"{mode}_out_{k}"][~rea]), (mode, k)
