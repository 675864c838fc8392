"""CPU checks of the tennis controller's high-level policy at test time: the float64 restatement oracle/ref_port_v2p_policy.py against the
fixture made by executing the reference (tests/golden/make_golden_v2p_policy.py), the checkpoint reader of nn.V2PPolicy against the
restatement, the refusal of a stochastic player, and b200v2p_ctrl_t's layout with the policy fields."""
import os
import re

import numpy as np
import pytest
import torch

from conftest import golden
from oracle import ref_port_v2p_policy as R

SINGLE = ("single_full", "single_padded")
DUAL = ("dual_running", "dual_n0", "dual_padded")
D = 257


def ckpt(z, prefix):
    """the checkpoint dict the fixture's case was made from"""
    ck = {"model": {k.split(":", 1)[1]: torch.from_numpy(z[k]) for k in z if k.startswith(prefix + "_model:")}}
    rms = {k.split(":", 1)[1]: torch.from_numpy(z[k]) for k in z if k.startswith(prefix + "_rms:")}
    if rms:
        ck["running_mean_std"] = rms
    return ck


def t64(a):
    return torch.from_numpy(np.asarray(a)).to(torch.float64)


@pytest.mark.parametrize("case", SINGLE)
def test_single_restore_normaliser_and_actor_match_reference(case):
    z = golden("v2p_policy.npz")
    ck = ckpt(z, case)
    net = R.load_single(ck, D)
    w0 = z.get(case + "_w0", ck["model"]["a2c_network.actor_mlp.0.weight"].numpy())    # zero-padded first layer, or the checkpoint's
    np.testing.assert_array_equal(net["layers"][0][0].numpy(), w0)
    np.testing.assert_array_equal(net["mean"].numpy(), z[case + "_rms_mean"])          # prefix of a fresh mean 0 / var 1
    np.testing.assert_array_equal(net["var"].numpy(), z[case + "_rms_var"])
    mu = R.act(t64(z[case + "_obs"]), [net])
    np.testing.assert_allclose(mu.numpy(), z[case + "_mu"], rtol=1e-4, atol=1e-5)


@pytest.mark.parametrize("case", DUAL)
def test_dual_load_running_norm_and_interleave_match_reference(case):
    z = golden("v2p_policy.npz")
    cks = [ckpt(z, case + "0"), ckpt(z, case + "1")]
    nets = R.load_dual(cks, D)
    x = t64(z[case + "_obs"])
    for i, net in enumerate(nets):
        assert net["n"] == int(z[f"{case}{i}_ro_n"])
        np.testing.assert_allclose(net["mean"].numpy(), z[f"{case}{i}_ro_mean"], rtol=1e-7)
        np.testing.assert_allclose(net["std"].numpy(), z[f"{case}{i}_ro_std"], rtol=1e-6)
        w0 = z.get(f"{case}{i}_w0", cks[i]["model"]["a2c_network.actor_mlp.0.weight"].numpy())
        np.testing.assert_array_equal(net["layers"][0][0].numpy(), w0)
        np.testing.assert_allclose(R.normalize(x[i::2], net).numpy(), z[f"{case}{i}_norm"], rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(R.act(x, nets).numpy(), z[case + "_mu"], rtol=1e-4, atol=1e-5)


def test_fixture_covers_the_edges():
    z = golden("v2p_policy.npz")
    assert int(z["dual_n00_ro_n"]) > 0 and int(z["dual_n01_ro_n"]) == 0                 # one network still at n == 0: identity
    np.testing.assert_array_equal(z["dual_n01_norm"], z["dual_n0_obs"][1::2])
    for case in ("single_padded", "dual_padded"):
        w0 = z[case + "_w0"] if case.startswith("single") else z[case + "0_w0"]
        assert not w0[:, 250:].any() and w0[:, :250].any()                               # the padded columns
    assert np.all(z["dual_padded0_ro_std"][250:] == 0)                                  # prefix: rstd 1e8 behind it
    for case in SINGLE + DUAL:
        rows = np.flatnonzero(z[case + "_reset_rows"])
        assert (rows % 2 == 0).any() and (rows % 2 == 1).any() and np.abs(z[case + "_obs"][rows]).max() > 5


@pytest.mark.parametrize("case", SINGLE + DUAL)
def test_checkpoint_reader_matches_restatement(case):
    """nn.v2p_networks_from_checkpoint (what V2PPolicy.from_checkpoint builds its layers and operand normaliser from) against the
    restatement's loaders: the same weights, mean, rstd and clamps, and through a float64 forward the same action"""
    from vid2player3d_b200 import nn
    z = golden("v2p_policy.npz")
    dual = case.startswith("dual")
    cks = [ckpt(z, case + "0"), ckpt(z, case + "1")] if dual else ckpt(z, case)
    got = nn.v2p_networks_from_checkpoint(cks, obs_dim=D, dual=dual)
    want = R.load_dual(cks, D) if dual else [R.load_single(cks, D)]
    x = t64(z[case + "_obs"])
    for g, w in zip(got, want):
        for (gw, gb), (ww, wb) in zip(g["layers"], w["layers"]):
            np.testing.assert_array_equal(gw.double().numpy(), ww.numpy())
            np.testing.assert_array_equal(gb.double().numpy(), wb.numpy())
    acts = []
    for i, g in enumerate(got):
        xi = x[i::2] if dual else x
        if g["mean"] is not None:
            xi = torch.clamp((xi - g["mean"].double()) * g["rstd"].double(), -g["clip"], g["clip"])
        acts.append(R.eval_actor(xi, [(w.double(), b.double()) for w, b in g["layers"]]))
    mu = torch.stack(acts, 1).reshape(-1, acts[0].shape[1]) if dual else acts[0]
    np.testing.assert_allclose(mu.numpy(), R.act(x, want).numpy(), rtol=1e-5, atol=1e-5)
    if case == "dual_n0":
        assert got[1]["mean"] is None and got[1]["clip"] == float("inf")


def test_stochastic_player_is_refused():
    from vid2player3d_b200 import nn
    with pytest.raises(ValueError, match="deterministic"):
        nn.V2PPolicy.from_checkpoint({"model": {}}, 8, "cpu", deterministic=False)


def test_ctrl_struct_layout_and_abi_version_match_header(tmp_path, monkeypatch):
    import test_host
    monkeypatch.setattr(test_host, "STRUCT_MIRRORS", [("abi", "V2PCtrl", "b200v2p_ctrl_t")])
    assert test_host.layout_mismatches(tmp_path) == []
    from vid2player3d_b200 import abi
    text = open(os.path.join(test_host.ROOT, "include", "b200env.h")).read()
    assert int(re.search(r"#define B200_ABI_VERSION (\d+)", text).group(1)) == abi.ABI_VERSION
    names = [f for f, _ in abi.V2PCtrl._fields_]
    assert names[-8:] == ["policy_x", "policy_mean", "policy_rstd", "policy_ld", "policy_dual", "policy_clip_obs", "policy_clip", "pad_"]
