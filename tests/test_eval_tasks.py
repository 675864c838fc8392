"""CPU checks of the test-time tasks (MVAEControllerVis, MVAEControllerVisDual): the float restatement oracle/ref_port_eval.py against
the fixture made by executing the reference (tests/golden/make_golden_eval.py), task lookup, refused cfgs, the new bindings."""
import ctypes as C
import importlib

import numpy as np
import pytest

from conftest import golden
from oracle import ref_port_eval as R

RESET_IN = ("progress", "tar_time", "tar_time_total", "tar_action", "swing_type_cycle", "has_contact", "has_bounce", "est_bounce_in",
            "ball_pos", "root_pos", "ball_vel", "est_bounce_pos", "target_bounce_pos")


def test_reset_rule_and_meters_match_reference():
    z = golden("v2p_eval.npz")
    T, N = z["reset_progress"].shape
    M = R.new_meters(N)
    for t in range(T):
        s = {k: z["reset_" + k][t] for k in RESET_IN}
        term, rea, rec = R.eval_reset(s, int(z["reset_episode_length"]), M)
        np.testing.assert_array_equal(term, z["reset_out_terminate"][t])
        np.testing.assert_array_equal(rea, z["reset_out_reaction"][t])
        np.testing.assert_array_equal(rec, z["reset_out_recovery"][t])
        np.testing.assert_array_equal(M["count"], z["reset_out_meter_count"][t])
        np.testing.assert_array_equal(M["sum"][:3], z["reset_out_meter_sum"][t][:3])
        np.testing.assert_allclose(M["sum"][3], z["reset_out_meter_sum"][t][3], rtol=1e-6)
        np.testing.assert_allclose(M["avg"], z["reset_out_meter_avg"][t], rtol=1e-6)
        np.testing.assert_allclose(M["max"], z["reset_out_meter_max"][t], rtol=1e-6)


def test_select_best_matches_reference():
    z = golden("v2p_eval.npz")
    order = R.select_best(z["single_root_pos"], z["single_bounce_in_avg"], z["single_fh_avg"])
    eg = int(z["single_num_eg"])
    np.testing.assert_array_equal(order[:eg], z["single_best_env_ids"])
    np.testing.assert_array_equal(z["single_all_env_ids"], np.arange(eg))


def test_dual_recording_and_best_list_match_reference():
    z = golden("v2p_eval.npz")
    cap, eg = int(z["dual_capacity"]), int(z["dual_num_eg"])
    S, N = z["dual_progress"].shape
    fields = ("joint_rot", "root_pos", "ball_pos", "phase", "swing_type", "tar_action")
    rec = {k: np.zeros((N, cap) + z["dual_" + k].shape[2:], z["dual_" + k].dtype) for k in fields}
    best = []
    for s in range(S):
        R.record(rec, z["dual_progress"][s], {k: z["dual_" + k][s] for k in fields})
        R.best_update(best, z["dual_reset"][s], z["dual_distance"][s], z["dual_progress"][s], rec, eg)
    np.testing.assert_array_equal([b["distance"] for b in best], z["dual_best_distance"])
    np.testing.assert_array_equal([b["nframes"] for b in best], z["dual_best_nframes"])
    assert max(b["nframes"] for b in best) == cap - 1        # the rally that filled the buffer
    for k in fields:
        np.testing.assert_array_equal(np.concatenate([b["arrays"][k] for b in best], 1), z["dual_best_" + k])


def test_parse_task_resolves_the_test_time_tasks():
    pt = importlib.import_module("vid2player3d_b200.tasks.parse_task")
    from vid2player3d_b200.tasks import MVAEControllerVis, MVAEControllerVisDual
    assert pt.TASKS["MVAEControllerVis"] is MVAEControllerVis and pt.TASKS["MVAEControllerVisDual"] is MVAEControllerVisDual


@pytest.mark.parametrize("cls,env,headless,msg", [
    ("MVAEControllerVisDual", dict(numEnvs=7), True, "even number"),
    ("MVAEControllerVis", dict(numEnvs=8, num_eg=0), True, "num_eg"),
    ("MVAEControllerVisDual", dict(numEnvs=8, num_eg=0), True, "num_eg"),
    ("MVAEControllerVis", dict(numEnvs=8, num_rec_frames=0, record=True), True, "num_rec_frames"),
    ("MVAEControllerVis", dict(numEnvs=8), False, "viewer"),
    ("MVAEControllerVisDual", dict(numEnvs=8), False, "viewer"),
])
def test_malformed_cfgs_are_refused(cls, env, headless, msg):
    """refused before any device work, so this runs without a GPU"""
    from vid2player3d_b200 import tasks
    cfg = {"env": dict(episodeLength=300, vid2player={}, **env)}
    with pytest.raises(ValueError, match=msg):
        getattr(tasks, cls)(cfg, None, None, "cuda", 0, headless)


def test_eval_struct_layouts_match_header(tmp_path, monkeypatch):
    import test_host
    monkeypatch.setattr(test_host, "STRUCT_MIRRORS", [("abi", "V2PRec", "b200v2p_rec_t"), ("abi", "V2PBest", "b200v2p_best_t"),
                                                      ("abi", "V2PCtrl", "b200v2p_ctrl_t")])
    assert test_host.layout_mismatches(tmp_path) == []
    from vid2player3d_b200 import abi
    assert abi.SIGNATURES["b200v2p_eval_record"] == (C.c_int, [C.c_void_p, C.c_void_p])
