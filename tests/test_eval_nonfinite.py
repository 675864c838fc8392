"""CPU checks of the test-time restatements on the inputs of a failing policy: oracle/ref_port_record.py against
tests/golden/im_record_nonfinite.npz (the reference's _sync_ref_motion on rotation vectors with NaN components, +-Inf, +-1e30 and
non-finite roots, tests/golden/make_golden_record.py) and oracle/ref_port_eval.best_update against tests/golden/v2p_eval_nonfinite.npz
(the reference's dual render_vis with NaN pair distances into an empty, a short and a full list, several NaN pairs on one step and a NaN
already in the list, tests/golden/make_golden_eval.py), and the NaN-aware comparator the GPU tests of these launches use."""
import numpy as np
import pytest

from conftest import golden
from oracle import ref_port_eval as E
from oracle import ref_port_record as R

REC_FIELDS = ("joint_rot", "root_pos", "ball_pos", "phase", "swing_type", "tar_action")


def assert_nonfinite_close(got, want, atol=0.0, rtol=0.0, what=""):
    """NaN where want is NaN and only there, +-Inf where want has the same infinity and only there, the finite values within
    atol + rtol |want|"""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    assert got.shape == want.shape, f"{what}: shape {got.shape} != {want.shape}"
    gn, wn = np.isnan(got), np.isnan(want)
    assert np.array_equal(gn, wn), f"{what}: NaN at {np.argwhere(gn != wn)[:8].tolist()} in one only"
    gi, wi = np.isinf(got), np.isinf(want)
    assert np.array_equal(gi, wi) and np.array_equal(got[gi], want[wi]), f"{what}: infinities differ at {np.argwhere(gi != wi)[:8].tolist()}"
    f = np.isfinite(want)
    err = np.abs(got[f] - want[f])
    bad = err > atol + rtol * np.abs(want[f])
    assert not bad.any(), f"{what}: {int(bad.sum())} finite values off, largest {err.max()}"


def test_comparator_accepts_equal_non_finite_values():
    w = np.array([1.0, np.nan, np.inf, -np.inf, -2.5])
    assert_nonfinite_close(w + np.array([1e-9, 0, 0, 0, -1e-9]), w, atol=1e-8)


@pytest.mark.parametrize("i,v", [(1, 0.0), (0, np.nan), (2, -np.inf), (3, np.inf), (2, np.nan), (0, np.inf), (4, -2.5 + 1e-6)])
def test_comparator_rejects_a_different_value(i, v):
    """a finite value in place of a NaN, a NaN in place of a finite value, a sign-flipped Inf, a NaN for an Inf, an Inf for a finite
    value, a finite value past the tolerance"""
    w = np.array([1.0, np.nan, np.inf, -np.inf, -2.5])
    g = w.copy()
    g[i] = v
    with pytest.raises(AssertionError):
        assert_nonfinite_close(g, w, atol=1e-8)


@pytest.mark.parametrize("init", [0, 1])
def test_record_restatement_is_the_reference_on_non_finite_joints(init):
    """a NaN in any component of a joint's rotation vector, or an infinity, makes all three of its angles NaN, the pitch included
    (torch.clamp keeps a NaN); a non-finite root is copied as it is"""
    Z = golden("im_record_nonfinite.npz")
    n = len(Z["dof_pos"])
    got = R.sync_ref_motion(Z["rb_pos"], Z["rb_rot"], Z["dof_pos"], Z["p_rb_pos"], Z["p_rb_rot"], Z["p_dof_pos"], list(range(n)), init)
    want = Z[f"qpos_init{init}"]
    assert_nonfinite_close(got, want, atol=1e-12, what=f"init {init}")
    nq = want.shape[1] // 3
    src = Z["dof_pos"].reshape(n, -1, 3)
    bad = ~np.isfinite(src).all(-1)
    angles = want[:, 7:nq].reshape(n, -1, 3)
    assert bad.any() and np.isnan(angles[bad]).all() and np.isfinite(angles[~bad]).all()
    assert np.isinf(want).any()


def test_best_list_restatement_is_the_reference_on_nan_distances():
    """a NaN pair is the argmax (the first NaN of several), enters only an empty list, and once there no later pair passes it"""
    Z = golden("v2p_eval_nonfinite.npz")
    cap, eg = int(Z["capacity"]), int(Z["num_eg"])
    for s in range(int(Z["scenarios"])):
        z = {k[len(f"s{s}_"):]: v for k, v in Z.items() if k.startswith(f"s{s}_")}
        S, N = z["progress"].shape
        rec = {k: np.zeros((N, cap) + z[k].shape[2:], z[k].dtype) for k in REC_FIELDS}
        best = []
        for t in range(S):
            E.record(rec, z["progress"][t], {k: z[k][t] for k in REC_FIELDS})
            E.best_update(best, z["reset"][t], z["distance"][t], z["progress"][t], rec, eg)
        assert_nonfinite_close([b["distance"] for b in best], z["best_distance"], what=f"scenario {s}")
        np.testing.assert_array_equal([b["nframes"] for b in best], z["best_nframes"])
        for k in REC_FIELDS:
            np.testing.assert_array_equal(np.concatenate([b["arrays"][k] for b in best], 1), z["best_" + k], f"scenario {s} {k}")
    assert np.isnan(Z["s0_best_distance"]).all() and np.isnan(Z["s3_best_distance"]).all()
    assert not np.isnan(Z["s1_best_distance"]).any() and not np.isnan(Z["s2_best_distance"]).any()
