"""CPU checks of the tennis controller's trained low-level imitation policy: nn.low_level_networks_from_cfg (what PhysicsMVAEController
loads from physics.pretrained_model_cp / dual_model_cp) and the float64 restatement (oracle/ref_port_low_level_policy.py loaders,
oracle/ref_port_v2p_policy.act) against the fixture made by executing the reference (tests/golden/make_golden_low_level_policy.py),
the loader's refusals, and b200_obs_rows_t's layout with player 1's clamp."""
import os
import re

import numpy as np
import pytest
import torch

from conftest import golden
from oracle import ref_port_low_level_policy as L
from oracle import ref_port_v2p_policy as R
from vid2player3d_b200 import nn

SINGLE = ("single_running", "single_n0", "single_rms", "single_inmodel", "single_both", "single_lightning")
DUAL = ("dual_running_n0", "dual_rms_inmodel", "dual_both_running")
D, A = 734, 75


def ckpt(z, prefix):
    """the checkpoint dict the fixture's network was loaded from"""
    model = {k.split(":", 1)[1]: torch.from_numpy(z[k]) for k in z if k.startswith(prefix + "_model:")}
    if prefix + "_lightning" in z:
        return {"pytorch-lightning_version": "1.5.0", "state_dict": {k[len("a2c_network."):]: v for k, v in model.items()}}
    ck = {"model": model}
    rms = {k.split(":", 1)[1]: torch.from_numpy(z[k]) for k in z if k.startswith(prefix + "_rms:")}
    if rms:
        ck["running_mean_std"] = rms
    return ck


def case_ckpts(z, case):
    return [ckpt(z, case + "0"), ckpt(z, case + "1")] if case.startswith("dual") else [ckpt(z, case)]


def physics(tmp_path, case, cks):
    paths = []
    for i, ck in enumerate(cks):
        paths.append(str(tmp_path / f"{case}_{i}.pth"))
        torch.save(ck, paths[-1])
    return dict(dual_model_cp=paths) if case.startswith("dual") else dict(pretrained_model_cp=paths[0])


def t64(a):
    return torch.from_numpy(np.asarray(a)).to(torch.float64)


def close(got, want, rel=1e-6):
    """|got - want| <= rel * max|want| elementwise"""
    want = np.asarray(want)
    assert np.abs(np.asarray(got) - want).max() <= rel * max(np.abs(want).max(), 1e-30)


@pytest.mark.parametrize("case", SINGLE + DUAL)
def test_loader_reproduces_the_reference_loaded_networks(case, tmp_path):
    """the layers and statistics ImitatorPlayer.load_pretrained / load_dual_cp leave in the reference's networks"""
    z = golden("v2p_low_level_policy.npz")
    dual = case.startswith("dual")
    cks = case_ckpts(z, case)
    nets = nn.low_level_networks_from_cfg(physics(tmp_path, case, cks), D, A, dual)
    assert len(nets) == (2 if dual else 1)
    for i, net in enumerate(nets):
        p = f"{case}{i}" if dual else case
        for (w, b), k in zip(net["layers"], nn.V2P_ACTOR_KEYS):
            np.testing.assert_array_equal(w.numpy(), z[f"{p}_model:a2c_network.{k}.weight"])
            np.testing.assert_array_equal(b.numpy(), z[f"{p}_model:a2c_network.{k}.bias"])
        if int(z[p + "_ro_n"]) == 0:
            assert net["mean"] is None and net["rstd"] is None and net["clip"] == float("inf")
        else:
            assert net["clip"] == 5.0
            np.testing.assert_array_equal(net["mean"].numpy(), z[p + "_ro_mean"].astype(np.float32))
            np.testing.assert_allclose(net["rstd"].numpy(), 1.0 / (z[p + "_ro_std"] + 1e-8), rtol=1e-6)


@pytest.mark.parametrize("case", SINGLE + DUAL)
def test_restatement_matches_reference_eval_actor(case):
    """oracle loaders + ref_port_v2p_policy.act (RunningNorm, eval_actor, the dual interleave) against the reference's outputs"""
    z = golden("v2p_low_level_policy.npz")
    dual = case.startswith("dual")
    cks = case_ckpts(z, case)
    nets = L.load_dual(cks, D) if dual else [L.load_single(cks[0], D)]
    x = t64(z[case + "_obs"])
    for i, net in enumerate(nets):
        p = f"{case}{i}" if dual else case
        assert net["n"] == int(z[p + "_ro_n"])
        close(net["mean"].numpy(), z[p + "_ro_mean"])
        close(net["std"].numpy(), z[p + "_ro_std"])
        close(R.normalize((x[i::2] if dual else x)[:3], net).numpy(), z[p + "_norm"], 1e-6)
    close(R.act(x, nets).numpy(), z[case + "_mu"])


@pytest.mark.parametrize("case", SINGLE + DUAL)
def test_loaded_networks_act_as_the_restatement(case, tmp_path):
    """the loader's dicts (mean, rstd, clip: what V2PPolicy and the operand launch use) through a float64 forward give the action of
    the restatement"""
    z = golden("v2p_low_level_policy.npz")
    dual = case.startswith("dual")
    cks = case_ckpts(z, case)
    nets = nn.low_level_networks_from_cfg(physics(tmp_path, case, cks), D, A, dual)
    x = t64(z[case + "_obs"])
    acts = []
    for i, g in enumerate(nets):
        xi = x[i::2] if dual else x
        if g["mean"] is not None:
            xi = torch.clamp((xi - g["mean"].double()) * g["rstd"].double(), -g["clip"], g["clip"])
        acts.append(R.eval_actor(xi, [(w.double(), b.double()) for w, b in g["layers"]]))
    mu = torch.stack(acts, 1).reshape(-1, A) if dual else acts[0]
    close(mu.numpy(), z[case + "_mu"])


def test_fixture_covers_the_edges():
    z = golden("v2p_low_level_policy.npz")
    assert int(z["single_n0_ro_n"]) == 0 and int(z["dual_running_n01_ro_n"]) == 0 and int(z["dual_running_n00_ro_n"]) > 0
    np.testing.assert_array_equal(z["dual_running_n01_norm"], z["dual_running_n0_obs"][1::2][:3])     # n == 0: identity
    assert "single_lightning_lightning" in z
    assert "single_rms_rms:running_mean" in z and "single_rms_model:a2c_network.running_obs.n" not in z
    assert "single_inmodel_model:a2c_network.running_obs.running_mean" in z and "single_inmodel_rms:running_mean" not in z
    assert "single_both_rms:running_mean" in z and "single_both_model:a2c_network.running_obs.n" in z
    assert not np.array_equal(z["single_both_ro_mean"], z["single_both_rms:running_mean"])            # RunningNorm wins
    for case in SINGLE + DUAL:
        rows = np.flatnonzero(z[case + "_reset_rows"])
        assert (rows % 2 == 0).any() and (rows % 2 == 1).any() and np.abs(z[case + "_obs"][rows]).max() > 5


def fake_ckpt(obs_dim=D, actions=A, units=8, stat_dim=None, seed=0):
    g = torch.Generator().manual_seed(seed)
    dims = [obs_dim, units, units, units, actions]
    model = {}
    for k, i, o in zip(nn.V2P_ACTOR_KEYS, dims[:-1], dims[1:]):
        model[f"a2c_network.{k}.weight"] = torch.randn(o, i, generator=g)
        model[f"a2c_network.{k}.bias"] = torch.randn(o, generator=g)
    ck = {"model": model}
    if stat_dim:
        ck["running_mean_std"] = {"running_mean": torch.zeros(stat_dim, dtype=torch.float64), "running_var": torch.ones(stat_dim, dtype=torch.float64),
                                  "count": torch.tensor(8.0, dtype=torch.float64)}
    return ck


MISSING = "/nonexistent/never_read.pth"        # the structural refusals come before any checkpoint is read


@pytest.mark.parametrize("phys, dual, msg", [
    (dict(pretrained_model_cp=MISSING, checkpoint="best"), False, "physics.checkpoint"),
    (dict(dual_model_cp=[MISSING, MISSING], checkpoint="epoch10"), True, "physics.checkpoint"),
    (dict(pretrained_model_cp=[MISSING, MISSING]), False, "is a list"),
    (dict(dual_model_cp=[MISSING, MISSING]), False, "single-player task"),
    (dict(pretrained_model_cp=MISSING), True, "dual-player task"),
    (dict(dual_model_cp=[MISSING]), True, "exactly two"),
    (dict(dual_model_cp=[MISSING, MISSING, MISSING]), True, "exactly two"),
    (dict(dual_model_cp=MISSING), True, "exactly two"),
], ids=["checkpoint", "checkpoint-dual", "list", "dual-key-on-single", "single-key-on-dual", "one", "three", "not-a-list"])
def test_loader_refusals_before_reading(phys, dual, msg):
    with pytest.raises(ValueError, match=msg):
        nn.low_level_networks_from_cfg(phys, D, A, dual)


@pytest.mark.parametrize("kw, dual, msg", [
    (dict(obs_dim=730), False, "first layer takes 730"),
    (dict(obs_dim=730), True, "first layer takes 730"),
    (dict(actions=69), False, "mu gives 69"),
    (dict(actions=69), True, "mu gives 69"),
    (dict(stat_dim=730), True, "statistics are 730 wide"),
    (dict(stat_dim=740), True, "statistics are 740 wide"),
])
def test_loader_refuses_networks_of_another_shape(kw, dual, msg, tmp_path, monkeypatch):
    """a checkpoint of the wrong width is refused by the loader itself: no V2PPolicy (and none of its device buffers) is built"""
    monkeypatch.setattr(nn, "V2PPolicy", None)
    monkeypatch.setattr(nn, "Linear", None)
    p = str(tmp_path / "bad.pth")
    torch.save(fake_ckpt(**kw), p)
    good = str(tmp_path / "good.pth")
    torch.save(fake_ckpt(stat_dim=D), good)
    phys = dict(dual_model_cp=[good, p]) if dual else dict(pretrained_model_cp=p)
    with pytest.raises(ValueError, match=msg):
        nn.low_level_networks_from_cfg(phys, D, A, dual)


def test_no_key_no_policy():
    assert nn.low_level_networks_from_cfg({}, D, A, False) is None
    assert nn.low_level_networks_from_cfg(dict(pretrained_model_cp=None, dual_model_cp=None, checkpoint="best"), D, A, True) is None


def test_obs_rows_layout_and_dual_entry_point_match_header(tmp_path, monkeypatch):
    """b200_obs_rows_t keeps the layout of ABI version 11 (the former pad_ is clamp1), and the dual launch is an entry point of its own"""
    import ctypes as C

    import test_host
    from vid2player3d_b200 import abi
    monkeypatch.setattr(test_host, "STRUCT_MIRRORS", [("abi", "ObsRows", "b200_obs_rows_t")])
    assert test_host.layout_mismatches(tmp_path) == []
    text = open(os.path.join(test_host.ROOT, "include", "b200env.h")).read()
    assert int(re.search(r"#define B200_ABI_VERSION (\d+)", text).group(1)) == abi.ABI_VERSION
    names = [f for f, _ in abi.ObsRows._fields_]
    assert names[6:8] == ["clamp", "clamp1"] and C.sizeof(abi.ObsRows) == 32 + 10 * 8
    assert "int b200env_obs_imitation_rows_dual(b200env_handle h, const b200_obs_rows_t* d, void* stream);" in text
    assert abi.SIGNATURES["b200env_obs_imitation_rows_dual"] == abi.SIGNATURES["b200env_obs_imitation_rows"]
