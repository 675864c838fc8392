"""GPU tests of the residual and sampled-action epilogues of the GEMM layer (csrc/b200nn.cu `linear_kernel<E, BN, RES, NOISE>`), of the
narrow `<1, 64>` form and of the mixtures past one tile per CTA, against the float64 layer.

`b200nn_linear_create` picks one of 13 forms: BN = 32 for a mixture (E > 1), else 64 when n <= 64, else 128; RES when a residual is
given, NOISE when sigma is.  The grid is the device's resident CTA slots and CTA c takes tiles c, c + grid, ..., with the shared-memory
ring's (stage, phase) carried from one tile to the next.  The tests here run every residual and sampled form

  * over rows / K / n / out_col0 / ldo / resid_cols / act / clamp edges (`test_epilogue_matrix`);
  * at G - 1 ... 2G + 1 tiles for G = the SM count and twice it, so a CTA takes up to five tiles (`test_persistent_epilogue_forms`);
  * at every k-block count around the ring depth, so the ring crosses a tile boundary at each stage offset (`test_ring_offsets_across_tiles`);
  * with the device step counter of the sampled action over eager launches and graph replays (`test_noise_counter_under_persistent_grid`);
  * in the imitation and tennis policy chains past one round of tiles, with and without programmatic dependent launch (`test_policy_chains_*`).

Reference: y = clamp(act(A W^T + b + resid + sigma * eps64)) in float64 on the bf16 operands the kernel reads, eps64 the float64
restatement of the counter-based normal (oracle/ref_port_sampled_policy.py) at the launch's step and the layer's ldo / out_col0.  Bound:
`test_gpu_nn.bound` with |resid| + |sigma eps| added to the magnitude and one rounding step more (the residual add and the fused noise
add), plus sigma (1e-5 + 4 * 2^-23 / sqrt(-2 ln u1)) for the kernel's float32 Box-Muller (the rule of tests/test_gpu_sampled_policy.py)."""

import numpy as np
import pytest
import torch

from oracle import ref_port_sampled_policy as S
from test_gpu_nn import DEV, SENTINEL, U, assert_untouched_outside, bound, check_layer, layer_inputs, operand, reference, sentinel_out

SEED = 0xD6E8FEB86659FD93          # the high bit set: the seed is a full 64-bit value on both sides
TOL = 1e-5                         # float32 logf / sqrtf / cosf of the kernel's Box-Muller against float64


# ------------------------------------------------------------------------------------------------ the forms and the cases
def form(E, n, res, noise):
    """the (E, BN, RES, NOISE) instantiation b200nn_linear_create dispatches for a layer"""
    return (E, 32 if E > 1 else (64 if n <= 64 else 128), bool(res), bool(noise))


FORMS = ([(1, 128, False, False), (1, 64, False, False)] + [(E, 32, False, False) for E in range(2, 7)] +
         [(1, bn, res, noise) for res, noise in ((True, False), (False, True), (True, True)) for bn in (128, 64)])
STAGES = {128: 3, 64: 4, 32: 5}    # stages<E, BN>(): the depth of the ring
EPILOGUE_FORMS = [f for f in FORMS if f[2] or f[3]]


def tile_counts(g):
    """G - 1, G, G + 1, 2G - 1, 2G + 1 for G = g SMs and G = 2g: one or two CTAs per SM, partial and full rounds"""
    return sorted({t for G in (g, 2 * g) for t in (G - 1, G, G + 1, 2 * G - 1, 2 * G + 1)})


def rows_for(t, n_tiles):
    """a row count whose launch has at least t tiles, the last row tile ending in the second warpgroup's half"""
    return 128 * -(-t // n_tiles) - 37


def n_tiles(E, n):
    return -(-n // form(E, n, False, False)[1])


def sm_count():
    return torch.cuda.get_device_properties(DEV).multi_processor_count


def coprime_tiles(g):
    """a column-tile count that divides neither g nor 2g, so a CTA's consecutive tiles (grid apart) fall on different columns"""
    return next(p for p in (3, 5, 7, 11, 13) if g % p)


# epilogue matrix: rows 1 / 127 / 129 / 8191 (last tile ending in either warpgroup's half), K = 1, 63, 65, 288, 734 (one k block,
# ragged K, a ring that wraps), n ragged in its last tile and one n of three column tiles, out_col0 odd and even, ldo > out_col0 + n
SHAPES = {128: [(1, 1, 65), (127, 63, 75), (129, 65, 129), (8191, 288, 290), (8191, 734, 100)],
          64: [(1, 1, 1), (127, 63, 35), (129, 65, 63), (8191, 288, 33), (8191, 734, 64)]}
ACTS = [None, "relu", "elu"]
CLAMPS = [None, (-1.0, 1.0), (-0.3, 0.5)]
EPI_CASES = []
for _f, (_E, _bn, _res, _noise) in enumerate(EPILOGUE_FORMS):
    for _i, (_M, _K, _N) in enumerate(SHAPES[_bn]):
        _act, _clamp, _col0 = ACTS[(_i + _f) % 3], CLAMPS[(_i + 2 * _f) % 3], [0, 3, 8, 1][(_i + _f) % 4]
        _rc = [1, max(1, _N - 6), _N][(_i + _f) % 3] if _res else 0
        EPI_CASES.append(pytest.param(_res, _noise, _M, _K, _N, _act, _clamp, _col0, _rc,
                                      id=f"{'res' if _res else ''}{'+' if _res and _noise else ''}{'noise' if _noise else ''}-"
                                         f"M{_M}-K{_K}-N{_N}-{_act}-clamp{CLAMPS.index(_clamp)}-col{_col0}-rc{_rc}"))

# persistence: (E, n, res, noise, several column tiles).  The several-column-tile case takes n = 128 * p - 40 at run time, p = coprime_tiles
PERSIST_CASES = ([(1, 35, False, False, False)] + [(E, 32, False, False, False) for E in range(2, 6)] +
                 [(1, n, res, noise, False) for res, noise in ((True, False), (False, True), (True, True)) for n in (100, 35)] +
                 [(1, None, True, False, True)])
RING_KBLOCKS = {S_: (1, S_ - 1, S_, S_ + 1, 2 * S_ + 1) for S_ in STAGES.values()}


def case_n(E, n, several, g):
    return 128 * coprime_tiles(g) - 40 if several else n


def test_form_table_covers_every_form():
    """CPU only: the cases below reach each of the 13 forms by the library's own rule, and every residual and sampled form is run past
    2G + 1 tiles (some CTA takes a third tile) for the SM counts of the H100 SXM (132) and PCIe (114) parts and a few others"""
    assert len(set(FORMS)) == 13
    epi = {form(1, c.values[4], c.values[0], c.values[1]) for c in EPI_CASES}
    persist = {form(E, case_n(E, n, sev, 132), res, noise) for E, n, res, noise, sev in PERSIST_CASES}
    ring = {f for f in FORMS}
    noise = {form(1, n, res, True) for n, res in NOISE_CASES}
    chains = {form(1, 75, True, False), form(1, 75, True, True), form(1, 35, False, True)}
    assert epi == set(EPILOGUE_FORMS)
    assert persist | {(1, 128, False, False), (6, 32, False, False)} == set(FORMS)   # those two: tests/test_gpu_nn_persistent.py
    assert ring == set(FORMS) and noise == {f for f in FORMS if f[3]} and chains <= set(EPILOGUE_FORMS)
    for S_ in STAGES.values():
        assert set(RING_KBLOCKS[S_]) >= {1, S_ - 1, S_, S_ + 1, 2 * S_ + 1}
    for g in (132, 114, 78, 100, 144):
        for E, n, res, noise, sev in PERSIST_CASES:
            nn_ = case_n(E, n, sev, g)
            nt = n_tiles(E, nn_)
            tiles = -(-rows_for(tile_counts(g)[-1], nt) // 128) * nt
            assert tiles >= 2 * (2 * g) + 1, (g, E, nn_, res, noise)
            if sev:
                assert nt > 1 and g % nt and (2 * g) % nt
        assert -(-ring_rows(g) // 128) >= 2 * (2 * g) + 1


# ------------------------------------------------------------------------------------------------ reference and comparator
EPS_CACHE = {}


def eps64(step, rows, n, ldo, col0):
    """(eps, 1 / sqrt(-2 ln u1)) of every output element, float64 on the device; one draw table per launch geometry"""
    key = (step, rows, n, ldo, col0)
    if key not in EPS_CACHE:
        if len(EPS_CACHE) > 8:
            EPS_CACHE.clear()
        r, c = np.arange(rows), np.arange(n)
        EPS_CACHE[key] = (torch.from_numpy(S.counter_normal(SEED, step, r, c, ldo, col0)).to(DEV),
                          torch.from_numpy(S.log_amplification(SEED, step, r, c, ldo, col0)).to(DEV))
    return EPS_CACHE[key]


def epilogue_reference(abuf, lin, rows, n, act, clamp, resid=None, resid_cols=0, sigma=None, step=0, ldo=None, col0=0):
    """(ref, magnitude, extra) of clamp(act(A W^T + b + resid + sigma eps64)) in float64; extra = the Box-Muller allowance"""
    kp = lin.k_padded
    y, mag = reference(abuf[:rows, :kp], lin.w[:, :n, :kp], lin.b[:, :n])
    extra = torch.zeros_like(y)
    if resid is not None:
        r = resid[:rows, :resid_cols].double()
        y[:, :resid_cols] += r
        mag[:, :resid_cols] += r.abs()
    if sigma is not None:
        e, amp = eps64(step, rows, n, ldo, col0)
        se = sigma.double()[None] * e
        y += se
        mag += se.abs()
        extra = sigma.double()[None] * (TOL + 4 * U * amp)
    y = {None: lambda x: x, "relu": torch.relu, "elu": torch.nn.functional.elu}[act](y)
    if clamp is not None:
        y = torch.clamp(y, clamp[0], clamp[1])
    return y, mag, extra


def check_epilogue(got, ref, mag, extra, k_padded, what):
    got = got.double()
    err = (got - ref).abs()
    bnd = bound(mag, ref, k_padded + 1, 1, False) + extra
    if not (bool(torch.isfinite(got).all()) and bool((err <= bnd).all())):
        i = int(torch.nan_to_num(err / bnd, nan=1e300).argmax())
        r, c = divmod(i, ref.shape[1])
        raise AssertionError(f"{what}: worst err/bound {float(torch.nan_to_num(err / bnd, nan=1e300).max()):.3g} at ({r}, {c}): "
                             f"got {float(got[r, c])} ref {float(ref[r, c])}")


# ------------------------------------------------------------------------------------------------ inputs and launches
def resid_buffer(rows, cols, seed):
    """float residual [padded rows, cols + 3]: finite in [0, rows) x [0, cols), NaN elsewhere, so a read past the last row or the last
    residual column (still inside the buffer) turns an output into NaN"""
    from vid2player3d_b200 import nn
    r = torch.full((nn.padded_rows(rows), cols + 3), float("nan"), device=DEV)
    g = torch.Generator(device=DEV).manual_seed(seed)
    r[:rows, :cols] = torch.randn(rows, cols, device=DEV, generator=g) * 0.5
    return r


def sigma_vector(n, seed, zeros=True):
    """sigma = exp(U(-2, 0)); with zeros, columns 0, 7, 14, ... have sigma 0 (no draw at all)"""
    g = torch.Generator().manual_seed(seed)
    s = torch.exp(torch.rand(n, generator=g) * 2 - 2)
    if zeros:
        s[::7] = 0
    return s.to(DEV)


def launch(abuf, w, b, rows, out, act=None, clamp=None, col0=0, resid=None, resid_cols=0, sigma=None, coef=None):
    """a fresh layer (its noise counter at 0) run once on `out`"""
    from vid2player3d_b200 import nn
    E = w.shape[0]
    lin = nn.Linear(abuf, w if E > 1 else w[0], b if E > 1 else b[0], out, rows, act=act, coef=coef, out_col0=col0, out_clamp=clamp,
                    residual=(resid, resid_cols) if resid is not None else None, noise=(sigma, SEED) if sigma is not None else None)
    lin.run()
    torch.cuda.synchronize()
    return lin


# ------------------------------------------------------------------------------------------------ 2. epilogue matrix
@pytest.mark.gpu
@pytest.mark.parametrize("res,noise,M,K,N,act,clamp,col0,resid_cols", EPI_CASES)
def test_epilogue_matrix(res, noise, M, K, N, act, clamp, col0, resid_cols):
    """every residual and sampled form vs the float64 layer, element by element, nothing outside [0, M) x [col0, col0 + N) written;
    act None: the residual form is bitwise (plain + resid).clamp; a sampled layer's sigma-0 columns are bitwise the layer without noise"""
    a, w, b, _ = layer_inputs(M, K, N, 1, seed=3 * M + 5 * K + 7 * N + res + 2 * noise)
    abuf = operand(a)
    resid = resid_buffer(M, resid_cols, seed=M + N) if res else None
    sigma = sigma_vector(N, seed=K + N) if noise else None
    out = sentinel_out(M, col0 + N, False)
    lin = launch(abuf, w, b, M, out, act, clamp, col0, resid, resid_cols, sigma)
    ref, mag, extra = epilogue_reference(abuf, lin, M, N, act, clamp, resid, resid_cols, sigma, 0, out.shape[1], col0)
    got = out[:M, col0:col0 + N]
    check_epilogue(got, ref, mag, extra, lin.k_padded, "epilogue")
    assert_untouched_outside(out, M, col0, N)
    if noise:
        assert int(lin.noise_step) == 1 and int(lin.noise_done) == 0
        det = sentinel_out(M, col0 + N, False)
        launch(abuf, w, b, M, det, act, clamp, col0, resid, resid_cols)
        z = (sigma == 0).nonzero().flatten() + col0
        assert torch.equal(out[:M, z].view(torch.int32), det[:M, z].view(torch.int32)), "sigma 0 columns differ from the layer without noise"
        if bool((sigma != 0).any()):
            assert not torch.equal(out[:M, col0:col0 + N], det[:M, col0:col0 + N])
    if res and act is None:
        plain = sentinel_out(M, col0 + N, False)
        launch(abuf, w, b, M, plain, col0=col0)
        want = plain[:M, col0:col0 + N].clone()
        want[:, :resid_cols] += resid[:M, :resid_cols]
        if clamp is not None:
            want = torch.clamp(want, clamp[0], clamp[1])
        mine = det if noise else out
        assert torch.equal(mine[:M, col0:col0 + N].view(torch.int32), want.view(torch.int32)), "residual layer != (plain + resid).clamp"


# ------------------------------------------------------------------------------------------------ 3. persistence
@pytest.mark.gpu
@pytest.mark.parametrize("E,N,res,noise,several", PERSIST_CASES,
                         ids=[f"E{c[0]}-N{c[1] or 'coprime'}{'-res' if c[2] else ''}{'-noise' if c[3] else ''}" for c in PERSIST_CASES])
def test_persistent_epilogue_forms(E, N, res, noise, several):
    """G - 1 ... 2G + 1 tiles (G = SMs, 2 SMs): rows [0, r) of the largest launch bitwise equal to a launch of r rows (every sampled
    launch at step 0, same ldo), nothing outside the block written, every element within the float64 bound"""
    g = sm_count()
    N = case_n(E, N, several, g)
    nt = n_tiles(E, N)
    K, col0, act = 288, 5, ("relu", "elu", None)[(E + N) % 3]
    clamp = (-1.0, 1.0) if res or noise else None
    counts = tile_counts(g)
    rows = {t: rows_for(t, nt) for t in counts}
    big = rows[counts[-1]]
    a, w, b, coef = layer_inputs(big, K, N, E, seed=700 + E + N + 2 * res + 4 * noise)
    rc = max(1, N - 6) if res else 0
    resid = resid_buffer(big, rc, seed=N) if res else None
    sigma = sigma_vector(N, seed=N) if noise else None
    abuf = operand(a)
    y_big = sentinel_out(big, col0 + N, False)
    lin = launch(abuf, w, b, big, y_big, act, clamp, col0, resid, rc, sigma, coef)
    ldo = y_big.shape[1]
    if E > 1:
        ref, mag = reference(abuf[:big, :K], lin.w[:, :N, :K], lin.b[:, :N], coef, act, clamp)
        extra = torch.zeros_like(ref)
    else:
        ref, mag, extra = epilogue_reference(abuf, lin, big, N, act, clamp, resid, rc, sigma, 0, ldo, col0)
    kp = lin.k_padded + E - 1                    # bound() of an E-expert blend: E - 1 more roundings than one expert
    check_epilogue(y_big[:big, col0:col0 + N], ref, mag, extra, kp, f"{big} rows")
    assert_untouched_outside(y_big, big, col0, N)
    for t in counts[:-1]:
        M = rows[t]
        y = sentinel_out(M, col0 + N, False)
        assert y.shape[1] == ldo
        launch(operand(a[:M]), w, b, M, y, act, clamp, col0, resid, rc, sigma, coef[:M].contiguous() if coef is not None else None)
        assert torch.equal(y[:M, col0:col0 + N].view(torch.int32), y_big[:M, col0:col0 + N].view(torch.int32)), \
            f"{t} tiles ({M} rows) differ from rows of the {big}-row launch"
        assert_untouched_outside(y, M, col0, N)
        check_epilogue(y[:M, col0:col0 + N], ref[:M], mag[:M], extra[:M], kp, f"{t} tiles ({M} rows)")


# ------------------------------------------------------------------------------------------------ 4. ring offsets
def ring_rows(g):
    """2G + 1 row tiles for G = 2g: every CTA takes at least two tiles whether the form holds one or two CTAs per SM"""
    return rows_for(4 * g + 1, 1)


@pytest.mark.gpu
@pytest.mark.parametrize("E,BN,res,noise", FORMS, ids=[f"E{f[0]}-BN{f[1]}{'-res' if f[2] else ''}{'-noise' if f[3] else ''}" for f in FORMS])
def test_ring_offsets_across_tiles(E, BN, res, noise):
    """K of 1, S - 1, S, S + 1 and 2S + 1 k blocks (S = the ring depth of the form) at two or more tiles per CTA: the ring's (stage,
    phase) enters each tile at every offset; every element within the float64 bound, nothing outside the block written"""
    M = ring_rows(sm_count())
    N = {128: 75, 64: 35, 32: 32}[BN]
    assert form(E, N, res, noise) == (E, BN, res, noise)
    col0, act, clamp = 3, ("elu", "relu", None)[E % 3], (-1.5, 1.5)
    rc = 69 if N == 75 else N
    for nkb in RING_KBLOCKS[STAGES[BN]]:
        K = 1 if nkb == 1 else 64 * nkb - 9
        a, w, b, coef = layer_inputs(M, K, N, E, seed=900 + 10 * nkb + E + BN + 2 * res + 4 * noise)
        resid = resid_buffer(M, rc, seed=nkb) if res else None
        sigma = sigma_vector(N, seed=nkb) if noise else None
        abuf = operand(a)
        out = sentinel_out(M, col0 + N, False)
        lin = launch(abuf, w, b, M, out, act, clamp, col0, resid, rc, sigma, coef)
        assert lin.k_padded // 64 == nkb
        if E > 1:
            ref, mag = reference(abuf[:M, :K], lin.w[:, :N, :K], lin.b[:, :N], coef, act, clamp)
            extra = torch.zeros_like(ref)
        else:
            ref, mag, extra = epilogue_reference(abuf, lin, M, N, act, clamp, resid, rc, sigma, 0, out.shape[1], col0)
        check_epilogue(out[:M, col0:col0 + N], ref, mag, extra, lin.k_padded + E - 1, f"{nkb} k blocks")
        assert_untouched_outside(out, M, col0, N)


# ------------------------------------------------------------------------------------------------ 5. the noise counter
NOISE_CASES = [(75, False), (35, False), (75, True), (35, True)]


@pytest.mark.gpu
@pytest.mark.parametrize("N,res", NOISE_CASES, ids=[f"N{n}{'-res' if r else ''}" for n, r in NOISE_CASES])
def test_noise_counter_under_persistent_grid(N, res):
    """2G + 1 row tiles (G = 2 SMs): two eager launches, then two replays of a graph capture of the layer.  After launch j the step
    counter is j + 1 and the done ticket 0; eps = (action - mu) / sigma of every row (a CTA's second and third tiles included) is the
    restatement's draw j, mu from the same layer built without noise"""
    from vid2player3d_b200 import nn
    M = ring_rows(sm_count())
    K, col0 = 288, 1
    a, w, b, _ = layer_inputs(M, K, N, 1, seed=1300 + N + res)
    abuf = operand(a)
    rc = N - 6 if res else 0
    resid = resid_buffer(M, rc, seed=N) if res else None
    sigma = sigma_vector(N, seed=N, zeros=False)
    mu = sentinel_out(M, col0 + N, False)
    launch(abuf, w, b, M, mu, col0=col0, resid=resid, resid_cols=rc)
    out = sentinel_out(M, col0 + N, False)
    lin = nn.Linear(abuf, w[0], b[0], out, M, out_col0=col0, residual=(resid, rc) if res else None, noise=(sigma, SEED))
    mu64, s64 = mu[:M, col0:col0 + N].double(), sigma.double()[None]

    def check(j):
        torch.cuda.synchronize()
        assert int(lin.noise_step) == j + 1 and int(lin.noise_done) == 0, (j, int(lin.noise_step), int(lin.noise_done))
        act = out[:M, col0:col0 + N].double()
        want, amp = eps64(j, M, N, out.shape[1], col0)
        err = ((act - mu64) / s64 - want).abs()
        tol = TOL + 4 * U * amp + 2.0 ** -24 * act.abs() / s64
        bad = (err > tol).any(1).nonzero().flatten()
        assert bad.numel() == 0, f"launch {j}: eps off the restatement's draw on {bad.numel()} rows, first {int(bad[0])}, max err {float(err.max()):.3g}"
        assert_untouched_outside(out, M, col0, N)

    for j in range(2):
        lin.run()
        check(j)
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        lin.run()
    torch.cuda.synchronize()
    assert int(lin.noise_step) == 2, "the capture launched the layer"
    for j in range(2, 4):
        out.fill_(SENTINEL)
        gr.replay()
        check(j)


# ------------------------------------------------------------------------------------------------ 6. production chains
def check_chain(layers, x, M, dims, last):
    """every layer of a chain vs the float64 layer on the kernel's own operand buffers (no compounding): the hidden layers (ReLU,
    bf16 output) by check_layer, the last one (n = dims[-1], float output) with its clamp, residual and noise at step 0"""
    a = x
    for i, l in enumerate(layers):
        N = dims[i + 1]
        if i == len(layers) - 1:
            ref, mag, extra = epilogue_reference(a, l, M, N, None, last["clamp"], last.get("resid"), last.get("rc", 0), last.get("sigma"),
                                                 0, N, 0)
            check_epilogue(l.out[:M, :N], ref, mag, extra, l.k_padded, f"layer {i}")
        else:
            ref, mag = reference(a[:M, :l.k_padded], l.w[:, :N, :l.k_padded], l.b[:, :N], None, "relu")
            check_layer(l.out[:M, :N], ref, mag, l.k_padded, 1, True, f"layer {i}")
        a = l.out


def assert_same_buffers(chain, serial):
    for i, (l, s) in enumerate(zip(chain, serial)):
        it = torch.int16 if l.out.dtype == torch.bfloat16 else torch.int32
        assert torch.equal(l.out.view(it), s.out.view(it)), f"layer {i}: the chain without programmatic dependent launch differs"


IM_DIMS = (734, 1024, 1024, 512, 75)


def im_layers(seed):
    g = torch.Generator().manual_seed(seed)
    d = IM_DIMS
    return [((torch.rand(d[i + 1], d[i], generator=g) * 2 - 1) / d[i] ** 0.5 * 1.7, (torch.rand(d[i + 1], generator=g) * 2 - 1) * 0.1)
            for i in range(4)]


@pytest.mark.gpu
@pytest.mark.parametrize("N", [16897, 33000])
@pytest.mark.parametrize("sampled", [False, True], ids=["mu", "sampled"])
def test_policy_chains_imitation(N, sampled, monkeypatch):
    """the imitation PolicyMLP with residual (resid, 69) and the ±1 action clamp, deterministic and sampled, at more envs than one round
    of tiles: each layer vs float64 on its own operand buffers; the chain built with B200NN_PDL=0 gives bitwise the same buffers"""
    from vid2player3d_b200 import nn
    layers = im_layers(N + sampled)
    g = torch.Generator().manual_seed(N)
    mean, var = torch.randn(734, generator=g) * 0.3, torch.rand(734, generator=g) + 0.5
    resid = (torch.randn(N, 69, generator=g) * 0.3).to(DEV)
    sigma = sigma_vector(75, seed=N) if sampled else None
    obs = (torch.randn(N, 734, generator=g) * 2.5).to(DEV)
    kw = dict(obs_mean=mean, obs_var=var, clamp_actions=1.0, residual=(resid, 69), noise_sigma=sigma, seed=SEED)
    net = nn.PolicyMLP(layers, N, DEV, **kw)
    net(obs)
    torch.cuda.synchronize()
    check_chain(net.layers, net.x, N, IM_DIMS, dict(clamp=(-1.0, 1.0), resid=resid, rc=69, sigma=sigma))
    monkeypatch.setenv("B200NN_PDL", "0")
    serial = nn.PolicyMLP(layers, N, DEV, **kw)
    serial(obs)
    torch.cuda.synchronize()
    assert_same_buffers(net.layers, serial.layers)


@pytest.mark.gpu
def test_policy_chains_sampled_v2p(monkeypatch):
    """a sampled single-network V2PPolicy (35 actions) at 16 897 envs: each layer vs float64 on its own operand buffers, the action with
    the draw of step 0; B200NN_PDL=0 gives bitwise the same buffers"""
    from vid2player3d_b200 import nn
    N, OBS, A = 16897, 257, 35
    g = torch.Generator().manual_seed(5)
    dims = (OBS, 1024, 1024, 512, A)
    layers = [((torch.rand(dims[i + 1], dims[i], generator=g) * 2 - 1) / dims[i] ** 0.5,
               (torch.rand(dims[i + 1], generator=g) * 2 - 1) / dims[i] ** 0.5) for i in range(4)]
    sigma = sigma_vector(A, seed=6)
    net = dict(layers=layers, mean=torch.randn(OBS, generator=g) * 0.5, rstd=torch.rand(OBS, generator=g) + 0.5, clip=5.0, sigma=sigma.cpu())
    obs = torch.randn(N, OBS, device=DEV, generator=torch.Generator(device=DEV).manual_seed(7)) * 3
    pol = nn.V2PPolicy([net], N, DEV, clip_obs=6.0, clip_actions=1.0, deterministic=False, seed=SEED)
    pol(obs)
    torch.cuda.synchronize()
    assert [int(s) for s in pol.noise_steps] == [1]
    check_chain(pol.layers, pol.x, N, dims, dict(clamp=(-1.0, 1.0), sigma=sigma))
    monkeypatch.setenv("B200NN_PDL", "0")
    serial = nn.V2PPolicy([net], N, DEV, clip_obs=6.0, clip_actions=1.0, deterministic=False, seed=SEED)
    serial(obs)
    torch.cuda.synchronize()
    assert_same_buffers(pol.layers, serial.layers)
