"""CPU checks of the sampled action of a stochastic test-time player: sigma = exp(a2c_network.sigma) read from the checkpoints the
reference's players load (the controller fixture tests/golden/v2p_policy.npz made by executing V2PPlayer.restore / load_dual_cp, the
imitation fixture tests/golden/im_policy.npz of load_pretrained, plus a Lightning state_dict), the refusals (learned sigma head, no
sigma), the noise fields of b200nn_linear_desc_t (layout, pointee types, fill, create's refusals made before any driver call) and the
float64 restatement of the noise, oracle/ref_port_sampled_policy.py."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest
import torch

import test_host
from conftest import golden
from oracle import ref_port_sampled_policy as S
from oracle import ref_port_v2p as V
from vid2player3d_b200 import abi, native, nn

D = 257                                                   # the controller fixture's observation width


def v2p_ckpt(z, prefix):
    ck = {"model": {k.split(":", 1)[1]: torch.from_numpy(z[k]) for k in z if k.startswith(prefix + "_model:")}}
    rms = {k.split(":", 1)[1]: torch.from_numpy(z[k]) for k in z if k.startswith(prefix + "_rms:")}
    if rms:
        ck["running_mean_std"] = rms
    return ck


def im_ckpt(sigma=None, lightning=False, head=False):
    """the fixture's `running` imitation checkpoint, with a fixed sigma parameter (or a learned sigma head) added the way the
    reference's network saves it (`a2c_network.sigma`, or `sigma` in a Lightning state_dict)"""
    z = golden("im_policy.npz")
    model = {k.split(":", 1)[1]: torch.from_numpy(v) for k, v in z.items() if k.startswith("running_model:")}
    if sigma is not None:
        model["a2c_network.sigma"] = sigma
    if head:
        model["a2c_network.sigma.weight"] = torch.zeros(75, 512)
        model["a2c_network.sigma.bias"] = torch.zeros(75)
    if lightning:
        return {"pytorch-lightning_version": "1.5.10", "state_dict": {k[len("a2c_network."):]: v for k, v in model.items()}}
    return {"model": model}


@pytest.mark.parametrize("case", ["single_full", "single_padded"])
def test_single_sigma_is_exp_of_the_restored_parameter(case):
    z = golden("v2p_policy.npz")
    ck = v2p_ckpt(z, case)
    (net,) = nn.v2p_networks_from_checkpoint(ck, obs_dim=D, deterministic=False)
    want = np.exp(z[case + "_model:a2c_network.sigma"].astype(np.float32))
    np.testing.assert_allclose(net["sigma"].numpy(), want, rtol=1e-6)
    assert net["sigma"].dtype == torch.float32 and net["sigma"].shape == (net["layers"][-1][0].shape[0],)
    (det,) = nn.v2p_networks_from_checkpoint(ck, obs_dim=D)
    assert "sigma" not in det


@pytest.mark.parametrize("case", ["dual_running", "dual_n0", "dual_padded"])
def test_dual_sigma_per_network(case):
    z = golden("v2p_policy.npz")
    nets = nn.v2p_networks_from_checkpoint([v2p_ckpt(z, case + "0"), v2p_ckpt(z, case + "1")], obs_dim=D, dual=True, deterministic=False)
    for p, net in enumerate(nets):
        np.testing.assert_allclose(net["sigma"].numpy(), np.exp(z[f"{case}{p}_model:a2c_network.sigma"].astype(np.float32)), rtol=1e-6)
    assert not torch.equal(nets[0]["sigma"], nets[1]["sigma"])


@pytest.mark.parametrize("lightning", [False, True])
def test_imitation_sigma_from_load_pretrained_checkpoints(lightning):
    logstd = torch.linspace(-2.5, -0.5, 75)
    net = nn.im_networks_from_checkpoint(im_ckpt(logstd, lightning=lightning), deterministic=False)
    torch.testing.assert_close(net["sigma"], torch.exp(logstd), rtol=0, atol=0)
    assert "sigma" not in nn.im_networks_from_checkpoint(im_ckpt(logstd, lightning=lightning))


def test_learned_sigma_head_and_missing_sigma_are_refused():
    z = golden("v2p_policy.npz")
    ck = v2p_ckpt(z, "single_full")
    ck["model"]["a2c_network.sigma.weight"] = torch.zeros(35, 512)
    with pytest.raises(ValueError, match="learned sigma head"):
        nn.v2p_networks_from_checkpoint(ck, obs_dim=D, deterministic=False)
    with pytest.raises(ValueError, match="learned sigma head"):
        nn.V2PPolicy.from_checkpoint(ck, 8, "cpu", obs_dim=D, deterministic=False)
    for lightning in (False, True):
        with pytest.raises(ValueError, match="learned sigma head"):
            nn.im_networks_from_checkpoint(im_ckpt(torch.zeros(75), lightning=lightning, head=True), deterministic=False)
        with pytest.raises(ValueError, match="no fixed sigma"):
            nn.im_networks_from_checkpoint(im_ckpt(None, lightning=lightning), deterministic=False)
    nets = nn.v2p_networks_from_checkpoint(v2p_ckpt(z, "single_full"), obs_dim=D)
    with pytest.raises(ValueError, match="needs every network's sigma"):
        nn.V2PPolicy(nets, 8, "cpu", deterministic=False)


def test_abi_version_and_descriptor_layout(tmp_path):
    """libb200env ABI 11, libb200nn ABI 2 with the noise fields appended to b200nn_linear_desc_t (the built library reports the
    descriptor size the binding fills); the layout of b200_im_policy_t, b200_play_stats_t and b200nn_linear_desc_t and the pointee
    type of every typed pointer field, from gcc on the headers"""
    assert abi.ABI_VERSION == 11 and nn.ABI_VERSION == 2
    assert "#define B200_ABI_VERSION 11" in open(os.path.join(test_host.ROOT, "include", "b200env.h")).read()
    assert "#define B200NN_ABI_VERSION 2" in open(os.path.join(test_host.ROOT, "include", "b200nn.h")).read()
    assert nn.lib().b200nn_linear_desc_size() == C.sizeof(abi.LinearDesc)
    assert nn.LinearDesc is abi.LinearDesc
    mirrors = [(abi.ImPolicy, "b200_im_policy_t"), (abi.PlayStats, "b200_play_stats_t"), (abi.LinearDesc, "b200nn_linear_desc_t")]
    lines, want = [], []
    names = {C.c_float: "float", C.c_int64: "int64_t", C.c_double: "double", C.c_uint32: "uint32_t"}
    for S_, ctype in mirrors:
        lines.append(f'printf("{ctype} %zu\\n", sizeof({ctype}));')
        want.append(f"{ctype} {C.sizeof(S_)}")
        for f, ct in S_._fields_:
            lines.append(f'printf("{ctype}.{f} %zu %zu\\n", offsetof({ctype}, {f}), sizeof((({ctype}*)0)->{f}));')
            want.append(f"{ctype}.{f} {getattr(S_, f).offset} {getattr(S_, f).size}")
            if issubclass(ct, C.c_void_p) and ct is not C.c_void_p:
                lines.append(f'printf("{ctype}.{f} %d\\n", __builtin_types_compatible_p(__typeof__(*(({ctype}*)0)->{f}), {names[ct.pointee]}));')
                want.append(f"{ctype}.{f} 1")
    src, exe = tmp_path / "layout.c", tmp_path / "layout"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "b200env.h"\n#include "b200nn.h"\nint main(void) {\n' +
                   "\n".join(lines) + "\nreturn 0;\n}\n")
    subprocess.check_call(["gcc", "-w", "-I", os.path.join(test_host.ROOT, "include"), str(src), "-o", str(exe)])
    assert subprocess.check_output([str(exe)], text=True).splitlines() == want
    assert [f for f, _ in abi.LinearDesc._fields_][-4:] == ["noise_sigma", "noise_seed", "noise_step", "noise_done"]


def test_fill_holds_the_noise_fields_to_their_types():
    t = dict(a=torch.zeros(4, dtype=torch.bfloat16), w=torch.zeros(4, dtype=torch.bfloat16), bias=torch.zeros(4), out=torch.zeros(4),
             noise_sigma=torch.zeros(4), noise_step=torch.zeros(1, dtype=torch.long), noise_done=torch.zeros(1, dtype=torch.int32))
    s = dict(lda=64, ldw=64, ldo=4, out_col0=0, rows=1, n=4, n_padded=128, k_padded=64, num_experts=1, act=0, out_bf16=0)
    for f, bad in (("noise_sigma", torch.float64), ("noise_step", torch.int32), ("noise_done", torch.int64), ("bias", torch.float16)):
        with pytest.raises(ValueError, match=rf"^LinearDesc\.{f}: {bad}"):
            native.fill(abi.LinearDesc, s, dict(t, **{f: torch.zeros(1, dtype=bad)}))
    with pytest.raises(ValueError, match="not on the CUDA device"):          # valid host tensors: only the device is wrong
        native.fill(abi.LinearDesc, s, t)
    with pytest.raises(ValueError, match=r"^LinearDesc\.rows: missing"):
        native.fill(abi.LinearDesc, dict(s, rows=None), t)


def _create(**over):
    """b200nn_linear_create on fake, aligned device addresses: every refusal below is made before the first driver call"""
    d = dict(a=0x10000, lda=64, w=0x20000, ldw=64, bias=0x30000, coef=None, out=0x40000, ldo=128, out_col0=0, rows=128, n=75, n_padded=128,
             k_padded=64, num_experts=1, act=0, out_bf16=0, out_min=-1.0, out_max=1.0, resid=None, ld_resid=0, resid_cols=0,
             noise_sigma=0x60000, noise_seed=7, noise_step=0x70000, noise_done=0x70008)
    d.update(over)
    h = C.c_void_p()
    rc = nn.lib().b200nn_linear_create(C.byref(nn.LinearDesc(**d)), 0, C.byref(h))
    if h:
        nn.lib().b200nn_linear_destroy(h)
    return rc, nn.lib().b200nn_last_error().decode()


@pytest.mark.parametrize("over, msg", [
    (dict(num_experts=2, coef=0x50000, n_padded=96), "single-expert"),
    (dict(out_bf16=1), "float output"),
    (dict(noise_step=None), "needs the device step counter"),
    (dict(noise_done=None), "needs the done ticket"),
    (dict(noise_sigma=None), "without noise_sigma"),
    (dict(noise_sigma=None, noise_step=None), "without noise_sigma"),
    (dict(noise_sigma=0x60002), "aligned"),
    (dict(noise_step=0x70004), "aligned"),
    (dict(noise_done=0x70002), "aligned"),
])
def test_noise_refusals(over, msg):
    nn.lib()
    rc, err = _create(**over)
    assert rc == -2 and msg in err, (rc, err)


def test_valid_noise_descriptors_pass_validation():
    want = 0 if torch.cuda.is_available() else -3
    for over in (dict(), dict(resid=0x50000, ld_resid=69, resid_cols=69), dict(n=40), dict(noise_seed=2 ** 64 - 1),
                 dict(noise_sigma=None, noise_step=None, noise_done=None, noise_seed=5)):
        rc, err = _create(**over)
        assert rc == want, (over, rc, err)


def test_restatement_is_the_counter_hash_box_muller():
    """the restatement's index is the flat output index, its uniforms those of the kernel's float32 formulas, and eps is finite"""
    seed, step = 1234567, 9
    rows, cols, ldo = np.arange(5), np.arange(3), 70
    idx = S.element_index(rows[:, None], cols[None, :], ldo, 35)
    assert idx.tolist() == [[r * 70 + 35 + c for c in range(3)] for r in range(5)]
    np.testing.assert_allclose(V.counter_normal(seed, step, idx.reshape(-1)).reshape(5, 3), S.counter_normal(seed, step, rows, cols, ldo, 35),
                               rtol=0, atol=1e-6)                # the float32 restatement of pre_step: same draws to float32 rounding
    # dual: network p's row r of its [H, 2A] view is env 2 r + p of the [N, A] output
    A = 35
    for p in (0, 1):
        np.testing.assert_array_equal(S.element_index(np.arange(4)[:, None], np.arange(A)[None, :], 2 * A, p * A),
                                      S.element_index((2 * np.arange(4) + p)[:, None], np.arange(A)[None, :], A))
    eps = S.counter_normal(seed, step, np.arange(4096), np.arange(64), 64)
    assert np.isfinite(eps).all() and np.abs(eps).max() <= np.sqrt(48 * np.log(2)) + 1e-12
    assert abs(eps.mean()) < 5 / np.sqrt(eps.size) and abs(eps.var() - 1) < 5 * np.sqrt(2 / eps.size)
    assert not np.array_equal(eps, S.counter_normal(seed, step + 1, np.arange(4096), np.arange(64), 64))
    assert not np.array_equal(eps, S.counter_normal(seed + 1, step, np.arange(4096), np.arange(64), 64))
    # negative seeds (the cfgs' default seed -1) are taken mod 2^64, as the descriptor's uint64 holds them
    np.testing.assert_array_equal(S.counter_normal(-1, 0, rows, cols, 3), S.counter_normal(2 ** 64 - 1, 0, rows, cols, 3))
    a = S.sample(np.zeros((3, 2)), [0.0, 2.0], seed, 0, clip=1.0)
    assert (a[:, 0] == 0).all() and np.abs(a[:, 1]).max() <= 1.0
    assert re.search(r"counter_hash", S.__doc__)


def test_binding_refuses_a_library_of_another_descriptor_size(monkeypatch):
    """the descriptor grew by appended fields within ABI version 2: nn.lib() compares the library's b200nn_linear_desc_size() with the
    binding's struct, so a library built before the noise fields (which would ignore them and serve mu) is refused"""
    nn.lib()
    old = type("LinearDesc", (C.Structure,), {"_fields_": abi.LinearDesc._fields_[:-4]})   # the parent's layout
    monkeypatch.setattr(nn, "LinearDesc", old)
    monkeypatch.setattr(nn, "_lib", None)
    with pytest.raises(RuntimeError, match="b200nn_linear_desc_t.*rebuild"):
        nn.lib()
