"""CPU checks of the two-hand backhand fix: the torch restatement oracle/ref_port_backhand.py, run through the callers' selection and
write-back, against the fixture made by executing the reference's optimize_two_hand_backhand (tests/golden/make_golden_backhand.py),
and the binding of b200v2p_backhand_fix against include/b200env_v2p.h.

Agreement bound.  The restatement and the reference are both float32 but round differently (konia conversions, FK association).
After the first step each fitted component sits at about +-lr, and a neighbour's component differs from it by far less than that, so
the sign of an L1 term (target, reg or smoothness) can come out differently under a different rounding.  One such flip moves that
component by at most about 2 lr in the step (Adam normalises the step to about lr) and its effect on later steps through the moment
estimates adds up to no more than that again.  So after k steps a fitted angle-axis component differs by at most 2 lr k; the other
joints see only the float32 round trip.  At k = 1 no smoothness or reg sign is evaluated away from zero, and the two agree to rounding.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from conftest import golden
from oracle import ref_port_backhand as B

Z = golden("v2p_backhand.npz")
CASES = range(int(Z["num_cases"]))


def case(c):
    t = lambda k: torch.tensor(Z[f"c{c}_{k}"])  # noqa: E731
    return t("joint_rot"), t("phase"), t("swing_type"), t("rest"), bool(Z[f"c{c}_righthand"])


@pytest.mark.parametrize("k", [1, 10, 500])
@pytest.mark.parametrize("c", CASES)
def test_restatement_matches_reference(c, k):
    jr, ph, sw, rest, rh = case(c)
    torch.set_num_threads(1)
    out, losses = B.fix_episode(jr, ph, sw, rest, rh, k)
    want, want_loss = Z[f"c{c}_out_{k}"], Z[f"c{c}_loss_{k}"]
    need = B.select(sw, ph).numpy()
    np.testing.assert_array_equal(out.numpy()[~need], jr.numpy()[~need])          # rows not selected: untouched
    np.testing.assert_array_equal(want[~need], jr.numpy()[~need])
    ik = B.arm_joints(rh)[0]
    other = [j for j in range(24) if j not in ik]
    np.testing.assert_allclose(out.numpy()[need][:, other], want[need][:, other], atol=2e-5)
    tol = 2 * B.LR * k if k > 1 else 1e-5
    np.testing.assert_allclose(out.numpy()[need][:, ik], want[need][:, ik], atol=tol, rtol=0)
    if k == 1:
        np.testing.assert_allclose(losses, want_loss, rtol=1e-5, atol=1e-7)
        assert losses[1] == 0 and (np.isnan(losses[2]) == (need.sum() == 1))         # reg 0 at the first step; no smoothness at M = 1
    else:
        assert losses[0] < Z[f"c{c}_loss_1"][0] and want_loss[0] < Z[f"c{c}_loss_1"][0]


def test_fixture_covers_the_issue_cases():
    Ms = [int(B.select(torch.tensor(Z[f"c{c}_swing_type"]), torch.tensor(Z[f"c{c}_phase"])).sum()) for c in CASES]
    assert 1 in Ms and 2 in Ms and max(Ms) >= 60
    assert {bool(Z[f"c{c}_righthand"]) for c in CASES} == {True, False}


def test_backhand_struct_layouts_and_scratch_size_match_header(tmp_path, monkeypatch):
    import subprocess

    import test_host
    from vid2player3d_b200 import abi
    monkeypatch.setattr(test_host, "STRUCT_MIRRORS", [("abi", "V2PBhProb", "b200v2p_bhprob_t"), ("abi", "V2PBhFix", "b200v2p_bhfix_t")])
    assert test_host.layout_mismatches(tmp_path) == []
    assert abi.SIGNATURES["b200v2p_backhand_fix"] == (C.c_int, [C.c_void_p, C.c_void_p])
    Ts = [[0], [1], [31, 32, 33], [1800, 1800, 300]]
    src, exe = tmp_path / "scratch.c", tmp_path / "scratch"
    lines = []
    for ts in Ts:
        F = sum((t + 31) // 32 * 32 for t in ts)
        lines += [f'printf("%lld\\n", (long long)B200V2P_BHFIX_SCRATCH_BYTES({len(ts)}, {F}, {s}));' for s in (4, 8)]
    src.write_text('#include <stdio.h>\n#include "b200env_v2p.h"\nint main(void) {\n' + "\n".join(lines) + "\nreturn 0;\n}\n")
    subprocess.check_call(["gcc", "-I", test_host.os.path.join(test_host.ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)], text=True).split()]
    assert got == [abi.bhfix_scratch_bytes(ts, s) for ts in Ts for s in (4, 8)]
