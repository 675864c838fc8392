"""GPU tests of libb200nn.so (wgmma GEMM layers, include/b200nn.h) through its C ABI.

Tolerances.  Operands are bf16 (8 significant bits), accumulation fp32.

Layer comparator (`check_layer`).  The reference is computed in float64 from the SAME bf16-rounded A and W the kernel reads:
ref = clamp(act(sum_e coef_e (A W_e^T + b_e))).  A product of two bf16 numbers is exact in fp32 (8 + 8 <= 24 significant bits), so
every error of the kernel is a rounding of a sum: the K-term dot product (wgmma accumulates in fp32; its adder is not specified to
round to nearest, so take one unit of 2^-23 per addition instead of half a unit), the bias add, the E fused multiply-adds of the
expert blend.  The standard bound for a recursive sum of n terms, |fl(sum) - sum| <= gamma_n sum |terms|, gamma_n = n u / (1 - n u),
with u = 2^-23 and n = k_padded + E + 2 gives, for every element,

    |got - ref| <= c * sum_e |coef_e| (sum_k |a_k w_ek| + |b_e|) + 2 u |ref|  (+ 2^-8 |ref| for bf16 output)

with c = gamma_{k_padded + E + 2}; ELU (expm1f, <= 2 ulp) contributes the 2 u |ref|; ReLU, ELU and the clamp are 1-Lipschitz, so
the bound carries through them; bf16 output rounding to nearest is at most half a bf16 ulp, 2^-8 |ref| (8 significant bits), so
for bf16 outputs the measured ratio can come close to 1 from the rounding alone; the fp32 outputs show the accumulation error.  The bound is per element:
outputs far below max|ref| are held to their own magnitude sum.  `test_comparator_rejects_plausible_kernel_bugs` shows that it
catches the bugs it is there for.

Against the fp32 reference module (the reference's own MixedDecoder.forward fixture, or a plain fp32 torch MLP) the bound is the
bf16 operand rounding: each product carries a relative error of 2^-8 twice, a K-term dot product of O(1) entries about
2^-8 sqrt(K) / sqrt(K) relative to the result's scale, i.e. ~1 % of max|y| after three layers (`LOOSE`).  `TIGHT` is the older,
whole-matrix bound kept by the fixed-shape tests."""
import ctypes as C

import numpy as np
import pytest
import torch

from conftest import golden
from helpers import mixed_decoder_params

pytestmark = pytest.mark.gpu
TIGHT = 2e-3
LOOSE = 2.5e-2
DEV = "cuda:0"
U = 2.0 ** -23
SENTINEL = -7.75          # exact in bf16 and fp32: a stray write of any computed value (0 included) changes it


def bf(x):
    return x.to(torch.bfloat16).to(torch.float32)


def act_fn(name):
    return {None: lambda x: x, "relu": torch.relu, "elu": torch.nn.functional.elu}[name]


def up(x, m):
    return (x + m - 1) // m * m


# ------------------------------------------------------------------------------------------------ comparator
def reference(a, w, b, coef=None, act=None, clamp=None):
    """float64 layer on the operands the kernel reads: a [M, K], w [E, N, K], b [E, N] (bf16-valued or fp32), coef [M, E] or None.
    Returns (ref [M, N], magnitude sum_e |coef_e| (sum_k |a_k w_ek| + |b_e|) [M, N])."""
    a64, w64, b64 = a.double(), w.double(), b.double()
    pre = torch.einsum("mk,enk->men", a64, w64) + b64[None]
    mag = torch.einsum("mk,enk->men", a64.abs(), w64.abs()) + b64.abs()[None]
    c64 = torch.ones(a.shape[0], 1, dtype=torch.float64, device=a.device) if coef is None else coef.double()
    y = (c64[:, :, None] * pre).sum(1)
    m = (c64.abs()[:, :, None] * mag).sum(1)
    y = act_fn(act)(y)
    if clamp is not None:
        y = torch.clamp(y, clamp[0], clamp[1])
    return y, m


def bound(mag, ref, k_padded, E, out_bf16):
    n = k_padded + E + 2
    c = n * U / (1 - n * U)
    return c * mag + 2 * U * ref.abs() + (2.0 ** -8 * ref.abs() if out_bf16 else 0.0)


def layer_errors(got, ref, mag, k_padded, E, out_bf16):
    """(ok, worst |got - ref| / bound).  Where ref is NaN the kernel must give NaN, where it is +-Inf the same Inf; the finite
    elements are held to the per-element bound."""
    got = got.double()
    nan = torch.isnan(ref)
    inf = torch.isinf(ref)
    fin = ~(nan | inf)
    ok = bool((torch.isnan(got) == nan).all()) and bool((got[inf] == ref[inf]).all())
    err = (got[fin] - ref[fin]).abs()
    bnd = bound(mag[fin], ref[fin], k_padded, E, out_bf16)
    ok = ok and bool(torch.isfinite(got[fin]).all()) and bool((err <= bnd).all())
    ratio = float((err / bnd.clamp_min(1e-300)).max()) if err.numel() else 0.0
    return ok, ratio


WORST = {}


def check_layer(got, ref, mag, k_padded, E, out_bf16, what=""):
    ok, ratio = layer_errors(got, ref, mag, k_padded, E, out_bf16)
    key = (E, "bf16" if out_bf16 else "fp32")
    WORST[key] = max(WORST.get(key, 0.0), ratio)
    if not ok:
        d = (got.double() - ref).abs()
        i = int(torch.nan_to_num(d / bound(mag, ref, k_padded, E, out_bf16).clamp_min(1e-300), nan=1e300).argmax())
        r, c = divmod(i, ref.shape[1])
        raise AssertionError(f"{what}: worst err/bound {ratio:.3g} at ({r}, {c}): got {float(got[r, c])} ref {float(ref[r, c])}")
    return ratio


@pytest.fixture(scope="module", autouse=True)
def report_worst_ratio():
    yield
    if WORST:
        print("\nworst |got - ref| / bound per expert count and output type: " +
              ", ".join(f"E={e} {t}: {r:.3g}" for (e, t), r in sorted(WORST.items())))


# ------------------------------------------------------------------------------------------------ inputs
def coef_rows(M, E, g):
    """blend coefficients: rows cycle through one-hot (rotating expert), uniform, all-zero and distinct random softmax rows"""
    c = torch.softmax(torch.randn(M, E, device=DEV, generator=g) * 2, 1)
    r = torch.arange(M, device=DEV)
    onehot = torch.nn.functional.one_hot(r % E, E).float()
    c = torch.where((r % 4 == 0)[:, None], onehot, c)
    c = torch.where((r % 4 == 1)[:, None], torch.full_like(c, 1.0 / E), c)
    c = torch.where((r % 4 == 2)[:, None], torch.zeros_like(c), c)
    return c.contiguous()


def layer_inputs(M, K, N, E, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    a = torch.randn(M, K, device=DEV, generator=g)
    w = torch.randn(E, N, K, device=DEV, generator=g) / K ** 0.5
    b = torch.randn(E, N, device=DEV, generator=g)
    coef = coef_rows(M, E, g) if E > 1 else None
    return a, w, b, coef


def operand(a):
    """padded bf16 operand buffer holding a (written by torch: the cast kernel is tested on its own)"""
    from vid2player3d_b200 import nn
    M, K = a.shape
    buf = nn.padded_bf16(M, K, DEV)
    buf[:M, :K] = a.to(torch.bfloat16)
    return buf


def run_layer(abuf, w, b, out, M, act, coef, col0, clamp):
    from vid2player3d_b200 import nn
    lin = nn.Linear(abuf, w if w.shape[0] > 1 else w[0], b if b.shape[0] > 1 else b[0], out, M, act=act, coef=coef, out_col0=col0,
                    out_clamp=clamp)
    lin.run()
    torch.cuda.synchronize()
    return lin


def sentinel_out(M, ncols, out_bf16):
    from vid2player3d_b200 import nn
    if out_bf16:
        return torch.full((nn.padded_rows(M) + 8, up(ncols, 8) + 8), SENTINEL, device=DEV, dtype=torch.bfloat16)
    return torch.full((M + 3, ncols + 5), SENTINEL, device=DEV)


def assert_untouched_outside(out, M, col0, N):
    inside = torch.zeros(out.shape, dtype=torch.bool, device=DEV)
    inside[:M, col0:col0 + N] = True
    outside = out[~inside]
    assert bool((outside == SENTINEL).all()), f"{int((outside != SENTINEL).sum())} elements outside the written block changed"


# shapes: every expert count sees a single k block (K = 1, 63), ragged K (63, 65, 288, 734), a ring of stages that wraps at least
# twice (734 = 12 k blocks), rows 1 / 127 / 128 / 129 / ~8192, last tiles ending in either warpgroup's half (rows % 128 in (0, 64]:
# 1, 129; in (64, 128): 127, 200, 8191), ragged last N tiles (1, 31, 33, 75, 129, 290) and several N tiles
SHAPES = [(1, 1, 1), (127, 63, 31), (128, 65, 33), (129, 288, 75), (200, 734, 129), (8191, 320, 290)]
ACTS = [None, "relu", "elu"]
CLAMPS = [None, (-1.0, 1.0), (-0.25, 0.6)]
CASES = []
for _E in range(1, 7):
    for _i, (_M, _K, _N) in enumerate(SHAPES):
        _bf16 = (_i + _E) % 2 == 0
        _col0 = [0, 8, 32][(_i // 2 + _E) % 3] if _bf16 else [3, 0, 32][(_i // 2 + _E) % 3]
        CASES.append(pytest.param(_E, _M, _K, _N, ACTS[(_i + _E) % 3], _bf16, _col0, CLAMPS[(_i + 2 * _E) % 3],
                                  id=f"E{_E}-M{_M}-K{_K}-N{_N}-{ACTS[(_i + _E) % 3]}-{'bf16' if _bf16 else 'f32'}-col{_col0}-clamp{(_i + 2 * _E) % 3}"))


@pytest.mark.parametrize("E,M,K,N,act,out_bf16,col0,clamp", CASES)
def test_linear_layer_matrix(E, M, K, N, act, out_bf16, col0, clamp):
    """one layer vs the float64 reference on the same bf16 operands, element by element; nothing outside [0, rows) x [col0, col0 + N)
    of a sentinel-filled buffer changes; in a padded_bf16 buffer (the next layer's operand) the K padding stays exactly zero and the
    block written is bitwise the same as in the other buffer"""
    from vid2player3d_b200 import nn
    a, w, b, coef = layer_inputs(M, K, N, E, seed=1000 * E + M + K + N)
    abuf = operand(a)
    out = sentinel_out(M, col0 + N, out_bf16)
    lin = run_layer(abuf, w, b, out, M, act, coef, col0, clamp)
    ref, mag = reference(abuf[:M, :K], lin.w[:, :N, :K], lin.b[:, :N], coef, act, clamp)
    check_layer(out[:M, col0:col0 + N], ref, mag, lin.k_padded, E, out_bf16, "layer")
    assert_untouched_outside(out, M, col0, N)
    if clamp is not None:                                   # the bounds as the output type represents them
        lo, hi = (float(torch.tensor(v).to(out.dtype)) for v in clamp)
        assert float(out[:M, col0:col0 + N].min()) >= lo and float(out[:M, col0:col0 + N].max()) <= hi
    if out_bf16:
        z = nn.padded_bf16(M, col0 + N, DEV)
        z[:M, :col0] = SENTINEL                             # the latent block of a MixedDecoder operand
        run_layer(abuf, w, b, z, M, act, coef, col0, clamp)
        assert torch.equal(z[:M, col0:col0 + N], out[:M, col0:col0 + N])
        assert bool((z[:M, :col0] == SENTINEL).all())
        assert int(z[M:].count_nonzero()) == 0 and int(z[:, col0 + N:].count_nonzero()) == 0, "K padding of the next operand written"


def test_comparator_rejects_plausible_kernel_bugs():
    """torch math only: the comparator accepts an honest fp32 computation and rejects a reference altered by each bug a wgmma
    epilogue / pipeline plausibly has: one column's bias missing, experts 0 and 1 swapped in one row's coefficients, the last 16-wide
    K slice (one MMA_K step) dropped, one row's output read from row + 8 (the other half of a wgmma accumulator fragment)"""
    M, K, N, E = 200, 288, 75, 6
    a, w, b, coef = layer_inputs(M, K, N, E, seed=7)
    a, w = bf(a), bf(w)
    k_padded = up(K, 64)
    ref, mag = reference(a, w, b, coef, "elu")
    honest = torch.nn.functional.elu((coef[:, :, None] * (torch.einsum("mk,enk->men", a, w) + b[None])).sum(1))
    ok, ratio = layer_errors(honest, ref, mag, k_padded, E, True)
    assert ok, ratio
    r = int(((coef[:, 0] - coef[:, 1]).abs() * (torch.arange(M, device=DEV) % 4 == 3))[:M - 8].argmax())
    assert float((coef[r, 0] - coef[r, 1]).abs()) > 0.05
    b_missing = b.clone()
    j = int(b.abs().sum(0).argmax())
    b_missing[:, j] = 0
    swapped = coef.clone()
    swapped[r, 0], swapped[r, 1] = coef[r, 1], coef[r, 0]
    dropped = a.clone()
    dropped[:, 16 * ((K - 1) // 16):] = 0
    bugs = {"bias of one column missing": reference(a, w, b_missing, coef, "elu")[0],
            "experts 0 and 1 swapped in one row": reference(a, w, b, swapped, "elu")[0],
            "last MMA_K slice dropped": reference(dropped, w, b, coef, "elu")[0]}
    row8 = ref.clone()
    row8[r] = ref[r + 8]
    bugs["row taken from row + 8"] = row8
    for name, bad in bugs.items():
        assert not layer_errors(bad, ref, mag, k_padded, E, True)[0], f"comparator accepts: {name}"


@pytest.mark.parametrize("E", range(1, 7))
def test_linear_isolation_and_determinism(E):
    """rows are independent and the result does not depend on where a row sits in a tile: permuting the rows of A (and coef)
    permutes the output bitwise, changing one row of A changes that output row only; two runs and a CUDA-graph replay are
    bit-identical"""
    from vid2player3d_b200 import nn
    M, K, N = 300, 288, 75
    a, w, b, coef = layer_inputs(M, K, N, E, seed=40 + E)
    abuf = operand(a)
    out = nn.padded_bf16(M, N, DEV)
    lin = run_layer(abuf, w, b, out, M, "elu", coef, 0, None)
    y0 = out.clone()
    lin.run()
    torch.cuda.synchronize()
    assert torch.equal(out, y0)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        lin.run()
    torch.cuda.current_stream().wait_stream(s)
    with torch.cuda.graph(gr):
        lin.run()
    out.fill_(SENTINEL)
    gr.replay()
    torch.cuda.synchronize()
    assert torch.equal(out[:M, :N], y0[:M, :N])
    perm = torch.randperm(M, device=DEV, generator=torch.Generator(device=DEV).manual_seed(E))
    pbuf = operand(a[perm])
    pout = nn.padded_bf16(M, N, DEV)
    run_layer(pbuf, w, b, pout, M, "elu", coef[perm].contiguous() if coef is not None else None, 0, None)
    d = (pout[:M, :N].float() - y0[:M, :N][perm].float()).abs()
    assert torch.equal(pout[:M, :N], y0[:M, :N][perm]), f"row permutation changes values: max diff {float(d.max())}"
    a2 = a.clone()
    a2[137] = torch.randn(K, device=DEV)
    cbuf = operand(a2)
    cout = nn.padded_bf16(M, N, DEV)
    run_layer(cbuf, w, b, cout, M, "elu", coef, 0, None)
    diff = (cout != y0).any(1)
    assert diff[137] and int(diff.sum()) == 1


@pytest.mark.parametrize("E", range(1, 7))
@pytest.mark.parametrize("act,clamp,out_bf16", [("relu", (-1.0, 1.0), False), (None, (-0.25, 0.6), True), ("elu", None, False)])
def test_linear_non_finite_inputs(E, act, clamp, out_bf16):
    """NaN / +Inf / -Inf in rows of A and NaN in a row of coef: those rows match torch's float64 result (NaN where torch gives NaN,
    after ReLU and after the clamp too), every other row is bit-identical to the run without them"""
    from vid2player3d_b200 import nn
    M, K, N = 200, 288, 75
    a, w, b, coef = layer_inputs(M, K, N, E, seed=90 + E)
    clean = nn.padded_bf16(M, N, DEV) if out_bf16 else torch.zeros(M, N, device=DEV)
    run_layer(operand(a), w, b, clean, M, act, coef, 0, clamp)
    bad_rows = [3, 70, 129, 130]
    a2 = a.clone()
    a2[3, 5] = float("nan")
    a2[70, 11] = float("inf")
    a2[129, 200] = float("-inf")
    a2[130, 0], a2[130, 1] = float("inf"), float("-inf")
    c2 = None
    if coef is not None:
        c2 = coef.clone()
        c2[187, E - 1] = float("nan")
        bad_rows.append(187)
    abuf = operand(a2)
    out = nn.padded_bf16(M, N, DEV) if out_bf16 else torch.zeros(M, N, device=DEV)
    lin = run_layer(abuf, w, b, out, M, act, c2, 0, clamp)
    ref, mag = reference(abuf[:M, :K], lin.w[:, :N, :K], lin.b[:, :N], c2, act, clamp)
    rows = torch.tensor(bad_rows, device=DEV)
    assert bool(torch.isnan(ref[rows]).any()) and bool(torch.isnan(ref[3]).all())
    check_layer(out[:M, :N][rows], ref[rows], mag[rows], lin.k_padded, E, out_bf16, "non-finite rows")
    keep = torch.ones(M, dtype=torch.bool, device=DEV)
    keep[rows] = False
    assert torch.equal(out[:M, :N][keep], clean[:M, :N][keep])


# ------------------------------------------------------------------------------------------------ gate softmax
def gate_softmax(h, k, w, b, coef, rows):
    from vid2player3d_b200 import nn
    nn._check(nn.lib().b200nn_gate_softmax(C.c_void_p(h.data_ptr()), C.c_int32(h.shape[1]), C.c_int32(k), C.c_void_p(w.data_ptr()),
                                           C.c_void_p(b.data_ptr()), C.c_int32(w.shape[0]), C.c_void_p(coef.data_ptr()), C.c_int32(rows),
                                           nn._stream()))


@pytest.mark.parametrize("E", range(1, 9))
def test_gate_softmax_matches_float64(E):
    """coef = softmax(h W^T + b) vs float64 on the same bf16 h, k = 1 .. 256, logits around +-80 and tied logits.  Each fp32 logit
    is within delta = gamma_(k/32 + 7) (sum_j |h_j w_j| + |b|) (u = 2^-24: per-lane fma chain, 5 shuffle adds, the bias); a softmax
    moves by at most a factor e^(2 delta) under such logit errors, expf and the normalisation add a few ulp."""
    from vid2player3d_b200 import nn
    M = 300
    for k in (1, 31, 64, 100, 256):
        g = torch.Generator(device=DEV).manual_seed(E * 1000 + k)
        hf = torch.randn(M, k, device=DEV, generator=g)
        w = (torch.randn(E, k, device=DEV, generator=g) / k ** 0.5).contiguous()
        b = torch.randn(E, device=DEV, generator=g)
        hf[: M // 3] *= 80.0 / k ** 0.5 * 1.5                 # logits of size ~80: exp overflows unless the max is subtracted
        hf[M // 3: M // 3 + 20] = 0                             # logits = b: tied logits where b ties
        if E > 1:
            b[1] = b[0]
            b[E - 1] = 80.0 if E > 2 else b[E - 1]
        h = nn.padded_bf16(M, k, DEV)
        h[:M, :k] = hf.to(torch.bfloat16)
        coef = torch.full((M, E), SENTINEL, device=DEV)
        gate_softmax(h, k, w, b, coef, M)
        torch.cuda.synchronize()
        h64 = h[:M, :k].double()
        logit = h64 @ w.double().T + b.double()
        ref = torch.softmax(logit, 1)
        mag = h64.abs() @ w.double().abs().T + b.double().abs()
        n = k // 32 + 8
        delta = (n * 2.0 ** -24 / (1 - n * 2.0 ** -24) * mag).max(1, keepdim=True).values
        tol = ref * (2.5 * delta + (E + 4) * 2.0 ** -23) + 1e-38
        err = (coef.double() - ref).abs()
        assert bool((err <= tol).all()), (k, float((err / tol).max()))
        assert float((coef.double().sum(1) - 1).abs().max()) <= 1e-6, k
        if E > 1:
            tied = slice(M // 3, M // 3 + 20)
            assert torch.equal(coef[tied, 0], coef[tied, 1])


# ------------------------------------------------------------------------------------------------ cast kernels
def same_bf16(got, want):
    """bitwise equal, any NaN equal to any NaN"""
    gn, wn = torch.isnan(got.float()), torch.isnan(want.float())
    return bool((gn == wn).all()) and torch.equal(got.view(torch.int16)[~gn], want.view(torch.int16)[~wn])


def cast_src(rows, cols, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(rows, cols + 5, device=DEV, generator=g) * 4          # ld_src > cols; values beyond the clamp
    x[1, 0], x[2, 3 % cols], x[4, cols - 1] = float("nan"), float("inf"), float("-inf")
    return x


@pytest.mark.parametrize("rows,cols", [(5, 1), (97, 63), (300, 288), (1000, 734)])
def test_cast_rows_exact(rows, cols):
    """cast_rows == bf16(clamp((x - mean) * rstd, lo, hi)) in torch fp32, exactly (NaN propagated), with and without mean / rstd;
    columns [cols, ld) and the rows below `rows` untouched"""
    from vid2player3d_b200 import nn
    x = cast_src(rows, cols, rows + cols)
    g = torch.Generator(device=DEV).manual_seed(cols)
    mean, rstd = torch.randn(cols, device=DEV, generator=g), torch.rand(cols, device=DEV, generator=g) + 0.5
    ld = up(cols, 64) + 64
    for mr, lo, hi in (((mean, rstd), -5.0, 5.0), (None, -3.0e38, 3.0e38), (None, -1.5, 2.0)):
        dst = torch.full((rows + 8, ld), SENTINEL, device=DEV, dtype=torch.bfloat16)
        nn.cast_rows(x, dst, cols, *(mr or (None, None)), lo=lo, hi=hi)
        torch.cuda.synchronize()
        y = x[:, :cols]
        if mr:
            y = (y - mean) * rstd
        want = torch.clamp(y, lo, hi).to(torch.bfloat16)
        assert same_bf16(dst[:rows, :cols], want)
        assert bool(torch.isnan(dst[1, 0].float()))
        assert bool((dst[:, cols:] == SENTINEL).all()) and bool((dst[rows:] == SENTINEL).all())


def test_cast_rows3_and_masked():
    """cast_rows3 writes the same bf16(clamp(x)) into all three destinations; cast_rows_masked writes the masked rows only (through a
    column offset, as MixedDecoder.set_condition does) and leaves every other row bitwise untouched"""
    from vid2player3d_b200 import nn
    rows, cols = 300, 32
    x = cast_src(rows, cols, 3)
    ld = 384
    dsts = [torch.full((rows + 8, ld), SENTINEL + i, device=DEV, dtype=torch.bfloat16) for i in range(3)]
    nn._check(nn.lib().b200nn_cast_rows3(C.c_void_p(x.data_ptr()), C.c_int32(x.stride(0)), *[C.c_void_p(d.data_ptr()) for d in dsts],
                                         C.c_int32(ld), C.c_int32(rows), C.c_int32(cols), nn._stream()))
    torch.cuda.synchronize()
    want = torch.clamp(x[:, :cols], -3.0e38, 3.0e38).to(torch.bfloat16)
    for i, d in enumerate(dsts):
        assert same_bf16(d[:rows, :cols], want)
        assert bool((d[:, cols:] == SENTINEL + i).all()) and bool((d[rows:] == SENTINEL + i).all())
    mask = torch.rand(rows, device=DEV, generator=torch.Generator(device=DEV).manual_seed(4)) < 0.3
    mask[1] = mask[4] = True                                     # the NaN and -Inf rows
    col0, n = 32, 288
    xs = cast_src(rows, n, 5)
    dst = torch.full((rows + 8, ld), SENTINEL, device=DEV, dtype=torch.bfloat16)
    nn._cast_cols(xs, dst, col0, n, -3.0, 3.0, row_mask=mask)
    torch.cuda.synchronize()
    want = torch.clamp(xs[:, :n], -3.0, 3.0).to(torch.bfloat16)
    assert same_bf16(dst[:rows][mask][:, col0:col0 + n], want[mask])
    keep = torch.ones(rows + 8, dtype=torch.bool, device=DEV)
    keep[:rows] = ~mask
    assert bool((dst[keep] == SENTINEL).all()) and bool((dst[:, :col0] == SENTINEL).all()) and bool((dst[:, col0 + n:] == SENTINEL).all())


# ------------------------------------------------------------------------------------------------ networks
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


def test_policy_mlp_action_clamp_and_prepared_operand():
    """clamp_actions = 1.0 (the action clamp folded into the last layer): every layer vs the float64 layer on the kernel's own
    operand buffers, the last one including the clamp, and the whole network vs the float64 network; forward_prepared after the
    operand row is written == forward, bitwise"""
    from vid2player3d_b200 import nn
    M = 333
    g = torch.Generator().manual_seed(2)
    mean, var = torch.randn(734, generator=g) * 0.3, torch.rand(734, generator=g) + 0.5
    dims = [734, 1024, 1024, 512, 75]
    layers = [((torch.rand(dims[i + 1], dims[i], generator=g) * 2 - 1) / dims[i] ** 0.5 * (1.7 if i < 3 else 3.0),
               (torch.rand(dims[i + 1], generator=g) * 2 - 1) * 0.1) for i in range(4)]
    net = nn.PolicyMLP(layers, M, DEV, obs_mean=mean, obs_var=var, clamp_actions=1.0)
    obs = (torch.randn(M, 734, generator=g) * 3).to(DEV)
    mu = net(obs).clone()
    torch.cuda.synchronize()
    assert 0.05 < float((mu.abs() == 1.0).float().mean()) < 0.95, "the clamp must be active on some actions and not on all"
    x = torch.clamp((obs - net.mean) * net.rstd, -5, 5)
    assert same_bf16(net.x[:M, :734], x.to(torch.bfloat16))
    a = net.x
    for i, l in enumerate(net.layers):
        last = i == len(net.layers) - 1
        N = dims[i + 1]
        ref, mag = reference(a[:M, :l.k_padded], l.w[:, :N, :l.k_padded], l.b[:, :N], None, None if last else "relu",
                             (-1.0, 1.0) if last else None)
        got = l.out[:M, :N]
        check_layer(got, ref, mag, l.k_padded, 1, not last, f"policy layer {i}")
        a = l.out
    h = x.double()
    for i, l in enumerate(net.layers):
        h = h @ l.w[0, :dims[i + 1], :dims[i]].double().T + l.b[0, :dims[i + 1]].double()
        h = torch.relu(h) if i < 3 else torch.clamp(h, -1, 1)
    assert float((mu.double() - h).abs().max()) <= LOOSE * float(h.abs().max())
    net.out.fill_(SENTINEL)
    nn.cast_rows(obs, net.x, 734, net.mean, net.rstd, -5.0, 5.0)
    assert torch.equal(net.forward_prepared(), mu)


def check_decoder_step(dec, z, hid):
    """every launch of one forward vs the float64 layer on the kernel's own operand buffers and coefficients (no compounding)"""
    M, L = dec.rows, dec.L
    zb = z.to(torch.bfloat16)
    for buf in (dec.x0, dec.x1, dec.x2):
        assert torch.equal(buf[:M, :L], zb), "latent block"
    gh = dec.gw.shape[1]                                     # the last gate layer's input is gate2's output
    layers = [("gate1", dec.x0, dec.gate1, dec.g1, 1, "elu", 0, gh), ("gate2", dec.g1, dec.gate2, dec.g2, 1, "elu", 0, gh),
              ("l1", dec.x0, dec.l1, dec.x1, dec.E, "elu", L, hid), ("l2", dec.x1, dec.l2, dec.x2, dec.E, "elu", L, hid),
              ("l3", dec.x2, dec.l3, dec.out, dec.E, None, 0, dec.out_dim)]
    for name, a, lin, out, E, act, col0, N in layers:
        kp = lin.k_padded
        ref, mag = reference(a[:M, :kp], lin.w[:, :N, :kp], lin.b[:, :N], dec.coef if E > 1 else None, act)
        check_layer(out[:M, col0:col0 + N], ref, mag, kp, E, name != "l3", f"decoder {name}")
    logit = dec.g2[:M, :dec.gw.shape[1]].double() @ dec.gw.double().T + dec.gb.double()
    assert float((dec.coef.double() - torch.softmax(logit, 1)).abs().max()) < 1e-5
    for buf in (dec.x1, dec.x2):
        assert int(buf[M:].count_nonzero()) == 0 and int(buf[:, L + hid:].count_nonzero()) == 0
    assert int(dec.x0[M:].count_nonzero()) == 0 and int(dec.x0[:, L + dec.cond:].count_nonzero()) == 0


@pytest.mark.parametrize("E", range(2, 7))
def test_mixed_decoder_layers_and_autoregression(E):
    """MixedDecoder at E experts, 300 rows (not a multiple of 128): every layer vs float64 with the kernel's own coefficients; the
    latent block is in all three operands and no layer writes over it; set_condition(row_mask) writes the masked rows of the condition
    block only; feed_back(3) writes exactly bf16(clamp(out[:, :cond], +-3)); a three-step autoregressive loop, each step checked
    from the kernel's own condition buffer"""
    from vid2player3d_b200 import nn
    ws, bs, gate = mixed_decoder_params(seed=11 + E, experts=E)
    t = torch.from_numpy
    M = 300
    dec = nn.MixedDecoder([t(w) for w in ws], [t(b) for b in bs], [(t(w), t(b)) for w, b in gate], M, DEV)
    g = torch.Generator(device=DEV).manual_seed(E)
    z, c = torch.randn(M, 32, device=DEV, generator=g), torch.randn(M, dec.cond, device=DEV, generator=g)
    dec(z, c)
    torch.cuda.synchronize()
    assert same_bf16(dec.x0[:M, 32:32 + dec.cond], c.to(torch.bfloat16))
    check_decoder_step(dec, z, ws[0].shape[2])
    # set_condition on a row mask
    before = dec.x0.clone()
    mask = torch.rand(M, device=DEV, generator=g) < 0.25
    c2 = torch.randn(M, dec.cond, device=DEV, generator=g) * 5
    dec.set_condition(c2, 3.0, row_mask=mask)
    torch.cuda.synchronize()
    want = before.clone()
    want[:M][mask, 32:32 + dec.cond] = torch.clamp(c2[mask], -3, 3).to(torch.bfloat16)
    assert torch.equal(dec.x0, want)
    # autoregression
    for step in range(3):
        z = torch.randn(M, 32, device=DEV, generator=g)
        dec(z)
        torch.cuda.synchronize()
        check_decoder_step(dec, z, ws[0].shape[2])
        dec.feed_back(clamp=3.0)
        torch.cuda.synchronize()
        want = torch.clamp(dec.out[:, :dec.cond], -3, 3).to(torch.bfloat16)
        assert torch.equal(dec.x0[:M, 32:32 + dec.cond], want), step
        assert torch.equal(dec.x0[:M, :32], z.to(torch.bfloat16))


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
