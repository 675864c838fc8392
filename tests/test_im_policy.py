"""CPU checks of the embodied_pose imitation policy at test time: the float64 restatement oracle/ref_port_im_policy.py against
tests/golden/im_policy.npz (made by executing the reference's own eval_actor, RunningNorm, load_pretrained and ImitatorPlayer.run,
tests/golden/make_golden_im_policy.py), nn.im_networks_from_checkpoint against the same checkpoints, the C ABI mirrors of the new
descriptors, the GEMM layer's residual refusals (made before any driver call) and the task's registration."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

import test_host
from conftest import golden
from oracle import ref_port_im_policy as R
from vid2player3d_b200 import abi, native, nn

Z = golden("im_policy.npz")
NB, ND, PAD, L = 24, 69, 2, 4


def checkpoint(case):
    """the checkpoint of a fixture case as the generator saved it (actor and normaliser keys)"""
    model = {k.split(":", 1)[1]: torch.from_numpy(v) for k, v in Z.items() if k.startswith(f"{case}_model:")}
    ck = {"model": model}
    rms = {k.split(":", 1)[1]: torch.from_numpy(v) for k, v in Z.items() if k.startswith(f"{case}_rms:")}
    if rms:
        ck["running_mean_std"] = rms
    return ck


@pytest.mark.parametrize("case", ["n0", "running", "rlgame"])
def test_loader_matches_load_pretrained(case):
    net = R.load(checkpoint(case))
    assert net["n"] == int(Z[f"{case}_ro_n"])
    np.testing.assert_array_equal(net["mean"], Z[f"{case}_ro_mean"].astype(np.float64))
    np.testing.assert_allclose(net["std"], Z[f"{case}_ro_std"], rtol=1e-7, atol=0)
    dev = nn.im_networks_from_checkpoint(checkpoint(case))
    if case == "n0":
        assert dev["mean"] is None and dev["rstd"] is None and dev["clip"] == float("inf")
    else:
        torch.testing.assert_close(dev["mean"], torch.from_numpy(Z[f"{case}_ro_mean"]))
        torch.testing.assert_close(dev["rstd"], 1.0 / (torch.from_numpy(Z[f"{case}_ro_std"]) + 1e-8))
        assert dev["clip"] == 5.0


@pytest.mark.parametrize("case", ["n0", "running", "rlgame"])
def test_actions_match_eval_actor(case):
    net = R.load(checkpoint(case))
    for t in (0, 1, L - 1):
        h, _ = R.human_obs(Z["obs"], Z["feat"], NB, ND, PAD, t)
        # the reference computes in float32: a few ulp of its largest terms (|x| <= 60 with the rows far outside the clamps)
        np.testing.assert_allclose(h, Z[f"human_obs_t{t}"], rtol=2e-4, atol=2e-5)
        if t == 0:
            np.testing.assert_allclose(R.normalize(Z["human_obs_t0"].astype(np.float64), net), Z[f"{case}_norm"], rtol=1e-5, atol=2e-5)
        mu = R.act(Z["obs"], Z["feat"], net, NB, ND, PAD, t)
        np.testing.assert_allclose(mu, Z[f"{case}_mu_t{t}"], rtol=0, atol=1e-4 * max(1.0, np.abs(mu).max()))


def test_bookkeeping_prints_the_reference_lines():
    N, games_num, max_steps, life = (int(x) for x in Z["run_args"])
    games, i = [], 0
    while f"run_game{i}_rew" in Z:
        games.append(list(zip(Z[f"run_game{i}_rew"], Z[f"run_game{i}_done"])))
        i += 1
    lines, sr, ss, gp = R.run_stats(games, games_num, max_steps, life)
    want = [f"reward: {r / c} steps: {s / c}" for c, r, s in lines] + [str(sr), f"av reward: {sr / gp * life} av steps: {ss / gp * life}"]
    assert want == [str(x) for x in Z["run_printed"]]


def test_parse_task_knows_the_test_task():
    import importlib
    from vid2player3d_b200.tasks import HumanoidSMPLIMVis
    assert importlib.import_module("vid2player3d_b200.tasks.parse_task").TASKS["HumanoidSMPLIMVis"] is HumanoidSMPLIMVis


@pytest.mark.parametrize("kw, msg", [(dict(normalize_input=True), "normalize_input"), (dict(use_ik=True), "use_ik"),
                                     (dict(deterministic=False), "deterministic")])
def test_loader_refusals(kw, msg):
    with pytest.raises(ValueError, match=msg):
        nn.im_networks_from_checkpoint(checkpoint("running"), **kw)


def test_abi_version_11_and_layouts(tmp_path):
    assert abi.ABI_VERSION == 11 and nn.ABI_VERSION == 2
    text = open(os.path.join(test_host.ROOT, "include", "b200env.h")).read()
    assert "#define B200_ABI_VERSION 11" in text
    assert "#define B200NN_ABI_VERSION 2" in open(os.path.join(test_host.ROOT, "include", "b200nn.h")).read()
    mirrors = [(abi.ImPolicy, "b200_im_policy_t"), (abi.PlayStats, "b200_play_stats_t"), (nn.LinearDesc, "b200nn_linear_desc_t")]
    lines, want = [], []
    for S, ctype in mirrors:
        lines.append(f'printf("{ctype} %zu\\n", sizeof({ctype}));')
        want.append(f"{ctype} {C.sizeof(S)}")
        for f, _ in S._fields_:
            lines.append(f'printf("{ctype}.{f} %zu %zu\\n", offsetof({ctype}, {f}), sizeof((({ctype}*)0)->{f}));')
            want.append(f"{ctype}.{f} {getattr(S, f).offset} {getattr(S, f).size}")
    # the pointee type of every typed pointer field
    names = {C.c_float: "float", C.c_int64: "int64_t", C.c_double: "double"}
    for S, ctype in mirrors[:2]:
        for f, ct in S._fields_:
            if issubclass(ct, C.c_void_p) and ct is not C.c_void_p:
                lines.append(f'printf("{ctype}.{f} %d\\n", __builtin_types_compatible_p(__typeof__(*(({ctype}*)0)->{f}), {names[ct.pointee]}));')
                want.append(f"{ctype}.{f} 1")
    src, exe = tmp_path / "layout.c", tmp_path / "layout"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "b200env.h"\n#include "b200nn.h"\nint main(void) {\n' +
                   "\n".join(lines) + "\nreturn 0;\n}\n")
    subprocess.check_call(["gcc", "-w", "-I", os.path.join(test_host.ROOT, "include"), str(src), "-o", str(exe)])
    got = subprocess.check_output([str(exe)], text=True).splitlines()
    assert got == want


def test_signatures_cover_the_new_entry_points():
    assert test_host.signature_mismatches(abi.SIGNATURES, test_host.ENV_HEADERS) == []
    assert "b200env_im_policy_rows" in abi.SIGNATURES and "b200env_play_stats" in abi.SIGNATURES


def test_fill_holds_the_new_descriptors_to_their_types():
    t = dict(obs_buf=torch.zeros(4), context_feat=torch.zeros(4), step=torch.zeros(1, dtype=torch.int32), mean=None, rstd=None,
             x=torch.zeros(4, dtype=torch.bfloat16), resid=torch.zeros(4))
    s = dict(n=1, num_obs=461, num_frames=48, feat_width=378, context_padding=8, context_length=32, ld=768, clip_obs=5.0)
    with pytest.raises(ValueError, match="ImPolicy.step: torch.int32"):
        native.fill(abi.ImPolicy, s, t)
    with pytest.raises(ValueError, match="ImPolicy.obs_buf: None"):
        native.fill(abi.ImPolicy, s, dict(t, obs_buf=None))
    with pytest.raises(ValueError, match="ImPolicy.ld: missing"):
        native.fill(abi.ImPolicy, dict(s, ld=None), t)
    p = dict(rew=torch.zeros(2), reset_buf=torch.zeros(2, dtype=torch.long), cr=torch.zeros(2), steps=torch.zeros(2), prev_dones=torch.zeros(2),
             totals=torch.zeros(2, dtype=torch.float32), log=torch.zeros(3, dtype=torch.float64), games=torch.zeros(3, dtype=torch.long),
             step=torch.zeros(1, dtype=torch.long))
    with pytest.raises(ValueError, match="PlayStats.totals: torch.float32"):
        native.fill(abi.PlayStats, dict(n=2, max_log=1, n_games=4), p)


def _create(**over):
    """b200nn_linear_create on fake, aligned device addresses: every refusal below is made before the first driver call"""
    d = dict(a=0x10000, lda=64, w=0x20000, ldw=64, bias=0x30000, coef=None, out=0x40000, ldo=128, out_col0=0, rows=128, n=75, n_padded=128,
             k_padded=64, num_experts=1, act=0, out_bf16=0, out_min=0.0, out_max=0.0, resid=0x50000, ld_resid=69, resid_cols=69)
    d.update(over)
    h = C.c_void_p()
    rc = nn.lib().b200nn_linear_create(C.byref(nn.LinearDesc(**d)), 0, C.byref(h))
    return rc, nn.lib().b200nn_last_error().decode()


@pytest.mark.parametrize("over, msg", [
    (dict(num_experts=2, coef=0x60000, n_padded=96), "single-expert"),
    (dict(out_bf16=1), "float output"),
    (dict(resid_cols=76), "resid_cols must be in 1..n"),
    (dict(ld_resid=60), "ld_resid < resid_cols"),
    (dict(resid=0x50002), "4-byte aligned"),
    (dict(resid=None), "without resid"),
])
def test_residual_refusals(over, msg):
    rc, err = _create(**over)
    assert rc == -2 and msg in err, err
