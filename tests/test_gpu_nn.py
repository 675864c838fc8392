"""GPU tests of libb200nn.so (wgmma GEMM layers, include/b200nn.h) through its C ABI.

Tolerances.  Operands are bf16 (8 significant bits), accumulation fp32.  Against a torch computation that rounds the SAME
operands to bf16 the kernel must agree to accumulation-order noise (`TIGHT`); against the fp32 reference module (the
reference's own MixedDecoder.forward fixture, or a plain fp32 torch MLP) the bound is the bf16 operand rounding: each product
carries a relative error of 2^-8 twice, a K-term dot product of O(1) entries about 2^-8 sqrt(K) / sqrt(K) relative to the
result's scale, i.e. ~1 % of max|y| after three layers (`LOOSE`)."""
import numpy as np
import pytest
import torch

from conftest import golden
from helpers import mixed_decoder_params

pytestmark = pytest.mark.gpu
TIGHT = 2e-3
LOOSE = 2.5e-2
DEV = "cuda:0"


def bf(x):
    return x.to(torch.bfloat16).to(torch.float32)


def act_fn(name):
    return {None: lambda x: x, "relu": torch.relu, "elu": torch.nn.functional.elu}[name]


@pytest.mark.parametrize("M,K,N,act,out_bf16", [(300, 734, 1024, "relu", True), (128, 64, 64, "elu", True), (1000, 1024, 75, None, False),
                                                (8192, 512, 512, "relu", True), (77, 1024, 1024, None, False)])
def test_linear_matches_torch(M, K, N, act, out_bf16):
    from vid2player3d_b200 import nn
    g = torch.Generator(device=DEV).manual_seed(M + K + N)
    a = torch.randn(M, K, device=DEV, generator=g)
    w = torch.randn(N, K, device=DEV, generator=g) / K ** 0.5
    b = torch.randn(N, device=DEV, generator=g)
    abuf = nn.padded_bf16(M, K, DEV)
    nn.cast_rows(a, abuf, K)
    assert torch.equal(abuf[:M, :K].float(), bf(a)) and float(abuf[:, K:].abs().max() if abuf.shape[1] > K else 0) == 0
    out = nn.padded_bf16(M, N, DEV) if out_bf16 else torch.zeros(M, N, device=DEV)
    lin = nn.Linear(abuf, w, b, out, M, act=act)
    lin.run()
    torch.cuda.synchronize()
    ref = act_fn(act)(bf(a).double() @ bf(w).double().T + b.double()).float()
    got = out[:M, :N].float()
    tol = TIGHT * float(ref.abs().max()) + (2 ** -8 * ref.abs() if out_bf16 else 0)
    assert bool(((got - ref).abs() <= tol).all()), float((got - ref).abs().max())
    if out_bf16:   # nothing outside the [rows, N] block was written
        assert float(out[M:].abs().max() if out.shape[0] > M else 0) == 0 and float(out[:, N:].abs().max() if out.shape[1] > N else 0) == 0


def test_policy_mlp_matches_fp32_torch():
    """PolicyMLP (734 -> 1024 -> 1024 -> 512 -> 75, ReLU, input normalisation + clamp) vs the same network in fp32 torch
    (embodied_pose/models/im_network_builder.py:191-230 actor path)"""
    from vid2player3d_b200 import nn
    M = 1000
    g = torch.Generator().manual_seed(1)
    dims = [734, 1024, 1024, 512, 75]
    layers = [((torch.rand(dims[i + 1], dims[i], generator=g) * 2 - 1) / dims[i] ** 0.5 * 1.7, (torch.rand(dims[i + 1], generator=g) * 2 - 1) * 0.1)
              for i in range(4)]
    mean, var = torch.randn(734, generator=g) * 0.3, torch.rand(734, generator=g) + 0.5
    obs = (torch.randn(M, 734, generator=g) * 2.5).to(DEV)
    net = nn.PolicyMLP(layers, M, DEV, obs_mean=mean, obs_var=var)
    mu = net(obs).clone()
    torch.cuda.synchronize()
    x = torch.clamp((obs - mean.to(DEV)) / torch.sqrt(var.to(DEV) + 1e-5), -5, 5)
    x32, xb = x, bf(x)
    for i, (w, b) in enumerate(layers):
        w, b = w.to(DEV), b.to(DEV)
        x32 = x32 @ w.T + b
        xb = xb @ bf(w).T + b
        if i < 3:
            x32, xb = torch.relu(x32), bf(torch.relu(xb))
    scale = float(x32.abs().max())
    assert float((mu - xb).abs().max()) <= TIGHT * scale, "vs bf16-operand emulation"
    assert float((mu - x32).abs().max()) <= LOOSE * scale, "vs fp32 network"
    # launches only: capturable, and the replay reproduces the eager result bit for bit
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        net(obs)
    torch.cuda.current_stream().wait_stream(s)
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        net(obs)
    net.out.zero_()
    gr.replay()
    torch.cuda.synchronize()
    assert torch.equal(net.out, mu)


def test_mixed_decoder_matches_reference_fixture():
    """MixedDecoder vs the reference's own MixedDecoder.forward executed in fp32 (tests/golden/make_golden_nn.py,
    vid2player/motion_vae/model.py:237-252); parameters rebuilt from the same numpy draw."""
    from vid2player3d_b200 import nn
    gd = golden("nn_mixed_decoder.npz")
    ws, bs, gate = mixed_decoder_params(seed=int(gd["seed"]))
    t = torch.from_numpy
    n = gd["z"].shape[0]
    dec = nn.MixedDecoder([t(w) for w in ws], [t(b) for b in bs], [(t(w), t(b)) for w, b in gate], n, DEV)
    out = dec(t(gd["z"]).to(DEV), t(gd["c"]).to(DEV))
    torch.cuda.synchronize()
    np.testing.assert_allclose(dec.coef.cpu().numpy(), gd["coef"], rtol=0, atol=1e-2)
    assert abs(float(dec.coef.sum(1).mean()) - 1.0) < 1e-5
    scale = float(np.abs(gd["out"]).max())
    err = np.abs(out.cpu().numpy() - gd["out"]).max()
    assert err <= LOOSE * scale, (err, scale)
    # same computation with bf16-rounded operands and the kernel's own coefficients: accumulation-order noise only
    z, c = t(gd["z"]).to(DEV), t(gd["c"]).to(DEV)
    coef = dec.coef
    h = c
    for i in range(3):
        x = bf(torch.cat([z, h], 1))
        y = torch.einsum("nk,eko->neo", x, bf(t(ws[i]).to(DEV))) + t(bs[i]).to(DEV)[None]
        y = (coef[:, :, None] * y).sum(1)
        h = torch.nn.functional.elu(y) if i < 2 else y
    assert float((out - h).abs().max()) <= TIGHT * scale + 2 ** -8 * scale
