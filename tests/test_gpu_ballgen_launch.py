"""The two launches of csrc/ballgen.cuh through the C ABI (include/b200ball.h) at every size, frame chunk, grid and column edge:
b200ball_simulate (ball_simulate_kernel: the trajectory pool and the incoming-ball table) and b200ball_out_rows
(ball_out_rows_kernel: the outgoing-ball estimator tables), against the float64 twin of the oracle (oracle/ref_port_ballgen.py,
pinned to the reference by tests/test_ballgen.py).

1. Every output starts as a sentinel (SENT = -12345.5, exact in both precisions; bounce_idx -777, pass_net 0xA5) and has SLACK = 128
   rows after row n - a whole 128-thread block, and more than the 7 frames a chunk can overrun.  Rows past n and table columns no
   grid value maps to stay bit-identical.
2. b200ball_simulate at n in SIZES (the ragged last block on both sides of 128 and 256) for every num_frames in FRAMES (<= 8, a
   multiple of BALLGEN_CHUNK = 8 and the ragged last chunk), control_freq_inv in {1, 2, 3}, substeps in {1, 2, 3, 6} (both sides of
   the 4R / 6R bounce-flag threshold) and first_comp in {0, 1, 2}, on random pool-style launches plus constructed edges at the block
   boundaries: inside the bounce threshold at t = 0 (under 4R, and between 4R and 6R), never bouncing, bouncing before the net (with
   the back-spin to top-spin flip), crossing y = 0 0.7 mm above and 2.8 mm below the net height, vspin 0 / + / -, vertical
   velocity only (the clamped |v x z|).
   - double instantiation vs the float64 twin: trajectory and bounce position within TOL64 = 1e-9 m, bounce_idx and pass_net exact;
   - float: each row bitwise equal to the same row of the largest launch and of a one-row launch; the first_comp = k output bitwise
     equal to columns k: of the first_comp = 0 output;
   - float vs the float64 twin: trajectory and bounce position within TOL32 = 2e-3 m * max(1, S / 1200), S = num_frames *
     control_freq_inv * substeps substeps (the float state carries ~1 ulp per substep; 2e-3 m is the golden bound at S = 1200).
     A ball whose float64 run passes within rounding of a discontinuity - the bounce flag threshold, the net-height test at y = 0,
     the contact test z < R at a substep end (a contact one substep earlier moves the ball by v h ~ 3 cm) - may differ by more or
     flip a flag: such rows are counted, at most 1 % of a launch.
3. b200ball_out_rows on the grids of GRIDS: the shipped ones; ngx = 0 / ngy = 0 (that table stays at the sentinel); values <= 0
   including negatives (the sample-0 pairing with sample "-1"); the duplicate columns across the sample-0 boundary of
   TRAJ_X_RANGE = (-0.25, 30, 0.25); unsorted grids; columns that do not cover the row; values far beyond the flight
   (extrapolated from the last two samples); ngx = ngy = 4096 (more than 48 KB of shared memory), for every num_frames in FRAMES and
   control_freq_inv in {1, 2, 3} at every n in SIZES.  Negative columns are wrapped the way Python indexes; columns outside [0, nx)
   are skipped by the kernel, never stored.
   - double vs the float64 oracle.  The kernel integrates the closed form of the oracle's substep loop: their samples differ by
     rounding, D = 1e-9 m * (1 + M / 30 m) with M the largest coordinate involved.  An x-table entry interpolates samples
     a = (ya, za), b = (yb, zb) at x: w = (x - ya) / (yb - ya), v = za (1 - w) + zb w.  Moving each coordinate by D moves v by at
     most D (|1 - w| + |w|) (1 + |s|), s = (zb - za) / (yb - ya); the rounding of the formula (w to 3 eps, the products and the sum)
     adds less than 8 eps M per unit of that factor.  So bound_x = (D + 8 eps M) (|1 - w| + |w|) (1 + |s|), per entry, from the
     oracle's own samples.  The drop distance of the y table is the same with y and z exchanged; its time (t - 1 + w) / tscale
     moves by dw / tscale with dw <= (D + 8 eps M) (|1 - w| + |w|) / |zb - za|, plus 8 eps (t + 1) (1 + |w|) / tscale of rounding.
     A non-finite entry (two equal samples) must be non-finite in both, at the same position.
   - float, vector stores vs scalar stores: nx + 1 columns and an odd ny force the scalar path; the shared columns are bitwise
     equal and the extra column stays at the sentinel.  Tables whose base address is 4 bytes off 16-byte alignment (scalar path)
     are bitwise equal to the aligned ones.
   - float rows bitwise independent of the launch, as in 2.
4. The pool's validity rule (ball_gen.pool_valid) on kernel outputs equals a per-row restatement of tennis_ball.py:319-327,
   including its whole-tensor `bounce_pos.sum() != 0`.
5. CPU: the public wrapper's column arithmetic (Python index semantics, IndexError outside [-n, n)), and negative controls: each
   comparator rejects a mutated oracle output (a frame shifted by one chunk, a sample-0 column rewritten last, a bounce index off
   by one, one element just outside its bound) and accepts one just inside.

The module prints the worst error-to-bound ratio of each comparator."""
import ctypes as C

import numpy as np
import pytest

from oracle import ref_port_ballgen as P

f32, f64 = np.float32, np.float64
EPS = 2.0 ** -52
DEV = "cuda:0"
SIZES = (1, 127, 128, 129, 255, 257, 1000, 4097)
BIG = SIZES[-1]
SLACK = 128
SENT = -12345.5
SENT_IDX = -777
SENT_U8 = 0xA5
FRAMES = (1, 7, 8, 9, 17, 100)
CFI = (1, 2, 3)
SUBSTEPS = (1, 2, 3, 6)
TOL64 = 1e-9
TOL32 = 2e-3
SPIN_SCALE = 5
EDGE_ROWS = (0, 1, 2, 3, 126, 127, 128, 129, 254, 255, 256, 999, 1000, 4094, 4095, 4096)
ONE_ROW = EDGE_ROWS + (17, 640, 2048)
WORST = {}

gpu = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def report_worst_ratio():
    yield
    if WORST:
        print("\nworst |got - ref| / bound per comparator: " + ", ".join(f"{k}: {r:.3g}" for k, r in sorted(WORST.items())))


def note(key, ratio):
    WORST[key] = max(WORST.get(key, 0.0), float(ratio))


# ------------------------------------------------------------------------------------------------ inputs (CPU)
def sim_inputs(n=BIG, seed=11):
    """pool-style launches (TennisBallGeneratorIsaac's ranges, widened) with the constructed edges at EDGE_ROWS; float32 [n,3] x2, [n]"""
    rng = np.random.default_rng(seed)
    origin = rng.uniform([-4, 11, 0.5], [4, 13, 2.5], (n, 3))
    target = rng.uniform([-3, -10], [3, -3], (n, 2))
    d = target - origin[:, :2]
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    speed, theta = rng.uniform(15, 32, n), np.radians(rng.uniform(-5, 20, n))
    vel = np.stack([speed * np.cos(theta) * d[:, 0], speed * np.cos(theta) * d[:, 1], speed * np.sin(theta)], 1)
    spin = rng.uniform(-10, 10, n)
    edges = [((0, 3, 0.1), (0, -20, -2), 5),          # inside 4R and 6R at t = 0
             ((0, 3, 0.15), (0, -20, -1), -5),        # between 4R and 6R at t = 0: flagged for substeps > 2 only
             ((1, 4, 0.15), (0, -20, 3), 0),          # between, rising, no spin
             ((0, 5, 20), (1, -3, 15), 7),            # never bounces
             ((1, 12, 1.2), (0, -10, -8), 8),         # bounces before the net
             ((-1, 12, 1.2), (0, -10, -8), -8),       # ... with back-spin: top-spin after the bounce
             ((0, 0.05, 1.0734), (0, -30, 0), 0),     # y < 0 after one sim step, z 0.7 mm over the net (substeps 1: least margin)
             ((0, 0.05, 1.0694), (0, -30, 0), 0),     # ... z under the net
             ((2, 6, 1.0), (0, -25, 4), 0),           # vspin 0
             ((2, 6, 1.0), (0, -25, 4), 10),          # top-spin
             ((2, 6, 1.0), (0, -25, 4), -10),         # back-spin
             ((0, 3, 1.0), (0, 0, 8), 5),             # vertical velocity only: v x z = 0, the clamped norm
             ((0, 3, 2.0), (0, 0, 9), -3),            # vertical, back-spin; still bouncing after 5 s (at rest, v = 0, the
                                                      # reference's force is 0/0 where the kernel's guard gives 0)
             ((-3, 12, 2.2), (2, -60, 2), -10),       # fast
             ((0, 3, 0.1), (0, -20, -2), -5),         # inside at t = 0 with back-spin: the flip at t = 0
             ((0.5, 10, 0.5), (0, -1, 0), 2)]         # slow: rolls on the ground
    assert len(edges) == len(EDGE_ROWS)
    for r, (p, v, s) in zip(EDGE_ROWS, edges):
        if r < n:
            origin[r], vel[r], spin[r] = p, v, s
    return origin.astype(f32), vel.astype(f32), spin.astype(f32)


def out_inputs(n=BIG, seed=12):
    """outgoing-table launches over traj_out_params' ranges with edges at EDGE_ROWS; float32 [n] x3 (horizontal, vertical, spin)"""
    rng = np.random.default_rng(seed)
    vh, vv, vs = rng.uniform(10, 65, n), rng.uniform(-5, 10, n), rng.uniform(-10, 10, n)
    edges = [(10, -5, -10), (65, 10, -10), (65, -5, 10), (30, 0, 0), (10, 10, 10), (40, 10, -10), (0.5, 3, 0), (20, -5, 0),
             (60, 5, -0.2), (10, 0, 0.2), (64.9, 9.9, -9.8), (12, 2, 3), (50, -1, -5), (25, 8, 10), (35, 0.1, -10), (1, -0.5, 1)]
    assert len(edges) == len(EDGE_ROWS)
    for r, e in zip(EDGE_ROWS, edges):
        if r < n:
            vh[r], vv[r], vs[r] = e
    return vh.astype(f32), vv.astype(f32), vs.astype(f32)


def explicit(values, cols, width):
    return np.asarray(values, f32), np.asarray(cols, np.int64), int(width)


def _grid_big(lo, hi, scale, width):
    v = np.linspace(lo, hi, 4096, endpoint=False).astype(f32)
    return explicit(v, [int(x * f32(scale)) for x in v], width)


def _unsorted(rng, scale, seed):
    v, c, w = P.grid(rng, scale)
    perm = np.random.default_rng(seed).permutation(len(v))
    return v[perm], c[perm], w


def _reversed(rng, scale):
    v, c, w = P.grid(rng, scale)
    return v[::-1].copy(), c[::-1].copy(), w


EMPTY_X, EMPTY_Y = explicit([], [], 60), explicit([], [], 30)
GRIDS = {   # id: (x grid, y grid) as (values float32, columns with Python index semantics, row width)
    "shipped": lambda: (P.grid((0, 30, 0.5), 2), P.grid((0, 3, 0.1), 10)),
    "ngx0": lambda: (EMPTY_X, P.grid((0, 3, 0.1), 10)),
    "ngy0": lambda: (P.grid((0, 30, 0.5), 2), EMPTY_Y),
    "nonpos": lambda: (P.grid((-2, 30, 0.5), 2), P.grid((-0.3, 3, 0.1), 10)),
    "dup": lambda: (P.grid((-0.25, 30, 0.25), 2), P.grid((-0.05, 3, 0.05), 10)),
    "unsorted": lambda: (_unsorted((0, 30, 0.5), 2, 5), _reversed((0, 3, 0.1), 10)),
    "sparse": lambda: (explicit(np.arange(0, 30, 1.5), np.arange(0, 60, 3), 60), explicit(np.arange(0, 3, 0.3), np.arange(0, 30, 3) + 1, 30)),
    "beyond": lambda: (explicit(np.arange(0, 200, 4), np.arange(50), 50), explicit(np.arange(0, 60, 2), np.arange(30), 30)),
    "big": lambda: (_grid_big(0, 40, 2, 80), _grid_big(0, 4, 10, 40)),
}


def wrap(cols, width):
    """Python's index semantics, as ball_gen._grid applies them"""
    cols = np.asarray(cols, np.int64)
    assert ((cols >= -width) & (cols < width)).all()
    return (cols % max(width, 1)).astype(np.int32)


def covered(cols, width):
    m = np.zeros(width, bool)
    m[wrap(cols, width)] = True
    return m


# ------------------------------------------------------------------------------------------------ bounds (CPU)
def out_bounds(walk, gx, cx, nx, gy, cy, ny, tscale):
    """per-entry bounds of the double tables (module docstring 3), scattered in grid order like the values"""
    S = walk["samples"].astype(f64)
    n = S.shape[0]
    ids = np.arange(n)[:, None]
    bx, by = np.full((n, nx), np.nan), np.full((n, ny, 2), np.nan)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        if len(gx):
            t = walk["t_x"]
            a, b = S[ids, t - 1], S[ids, t]            # t - 1 = -1: the last sample, like the walk
            x = np.asarray(gx, f64)[None]
            w = (x - a[..., 0]) / (b[..., 0] - a[..., 0])
            s = (b[..., 1] - a[..., 1]) / (b[..., 0] - a[..., 0])
            M = np.maximum(np.maximum(np.abs(a).max(-1), np.abs(b).max(-1)), np.abs(x))
            e = (1e-9 * (1 + M / 30) + 8 * EPS * M) * (np.abs(1 - w) + np.abs(w)) * (1 + np.abs(s))
            for j, c in enumerate(cx):
                bx[:, int(c)] = e[:, j]
        if len(gy):
            t = walk["t_y"]
            a, b = S[ids, t - 1], S[ids, t]
            y = np.asarray(gy, f64)[None]
            dz = b[..., 1] - a[..., 1]
            w = (-y - a[..., 1]) / dz
            s = (b[..., 0] - a[..., 0]) / dz
            M = np.maximum(np.maximum(np.abs(a).max(-1), np.abs(b).max(-1)), np.abs(y))
            Dp = 1e-9 * (1 + M / 30) + 8 * EPS * M
            ed = Dp * (np.abs(1 - w) + np.abs(w)) * (1 + np.abs(s))
            et = (Dp * (np.abs(1 - w) + np.abs(w)) / np.abs(dz) + 8 * EPS * (t + 1) * (1 + np.abs(w))) / tscale
            for j, c in enumerate(cy):
                by[:, int(c), 0], by[:, int(c), 1] = ed[:, j], et[:, j]
    return bx, by


def out_oracle(inp, n, grids, F, cfi, substeps=6):
    vh, vv, vs = (np.asarray(a[:n], f64) for a in inp)
    (gx, cx, nx), (gy, cy, ny) = grids
    walk = {}
    tx, ty = P.simulate_without_bounce(np.zeros((n, 3)), np.stack([np.zeros(n), vh, vv], 1), vs, control_freq_inv=cfi, num_frames=F,
                                       substeps=substeps, spin_scale=SPIN_SCALE, state32=False, world_kw=P.f32_physics(),
                                       grid_x=(gx, cx, nx), grid_y=(gy, cy, ny), table_dtype=f64, walk=walk)
    bx, by = out_bounds(walk, gx, cx, nx, gy, cy, ny, cfi * 30)
    return tx, ty, bx, by


# ------------------------------------------------------------------------------------------------ comparators (CPU)
def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view({1: np.uint8, 4: np.uint32, 8: np.uint64}[a.dtype.itemsize])


def assert_sentinel(a, what):
    a = np.asarray(a)
    s = {np.dtype(f32): f32(SENT), np.dtype(f64): f64(SENT), np.dtype(np.int64): np.int64(SENT_IDX),
         np.dtype(np.uint8): np.uint8(SENT_U8)}[a.dtype]
    bad = np.nonzero((_bits(a.reshape(-1)) != _bits(np.array([s], a.dtype))[0]))[0]
    assert len(bad) == 0, f"{what}: {len(bad)} sentinel elements overwritten, first at flat index {bad[0]}: {a.reshape(-1)[bad[0]]}"


def _bounded(got, ref, bound, key, what):
    got, ref, bound = np.asarray(got, f64), np.asarray(ref, f64), np.broadcast_to(np.asarray(bound, f64), np.shape(ref))
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    fg, fr = np.isfinite(got), np.isfinite(ref)
    if (fg != fr).any():
        i = tuple(int(k) for k in np.argwhere(fg != fr)[0])
        raise AssertionError(f"{what}: finite in one only at {i}: got {got[i]}, ref {ref[i]}")
    with np.errstate(invalid="ignore", divide="ignore"):
        ratio = np.where(fr, np.abs(got - ref) / bound, 0.0)
    if ratio.size == 0:
        return
    ratio = np.where(np.isnan(ratio), np.inf, ratio)
    i = np.unravel_index(int(np.argmax(ratio)), ratio.shape)
    note(key, ratio[i])
    assert ratio[i] <= 1, f"{what}: at {tuple(int(k) for k in i)} got {got[i]!r}, ref {ref[i]!r}, |diff| {abs(got[i] - ref[i]):.3g} > bound {bound[i]:.3g}"


def check_sim_double(got, ref, fc, what):
    """double launch (traj [n,F,3-fc], bounce_pos, bounce_idx, pass_net uint8) vs the float64 twin (full xyz traj)"""
    traj, bpos, bidx, pnet = got
    rt, rb, ri, rp = ref
    _bounded(traj, rt[:, :, fc:], TOL64, "simulate f64 traj", what + " traj")
    _bounded(bpos, rb, TOL64, "simulate f64 bounce_pos", what + " bounce_pos")
    bad = np.nonzero(bidx != ri)[0]
    assert len(bad) == 0, f"{what}: bounce_idx of row {bad[0]}: {bidx[bad[0]]} vs {ri[bad[0]]}"
    bad = np.nonzero(pnet != np.asarray(rp).astype(np.uint8))[0]
    assert len(bad) == 0, f"{what}: pass_net of row {bad[0]}: {pnet[bad[0]]} vs {rp[bad[0]]}"


def check_sim_float(got, ref, S, what):
    """float launch (fc = 0) vs the float64 twin: rows off TOL32 (or with a different flag) counted, at most 1 % of the launch"""
    traj, bpos, bidx, pnet = got
    rt, rb, ri, rp = ref
    tol = TOL32 * max(1.0, S / 1200)
    et = np.abs(traj.astype(f64) - rt).reshape(len(rt), -1).max(1)
    eb = np.abs(bpos.astype(f64) - rb).max(1)
    off = ~(et <= tol) | ~(eb <= tol) | (bidx != ri) | (pnet != np.asarray(rp).astype(np.uint8))
    assert off.sum() <= len(rt) // 100, f"{what}: {int(off.sum())} of {len(rt)} rows off the float32 bound {tol:.3g} (first {np.nonzero(off)[0][:8]})"
    if (~off).any():
        note("simulate f32 vs f64 (rows not counted)", max(et[~off].max(), eb[~off].max()) / tol)
    WORST["simulate f32 rows counted (max per launch)"] = max(WORST.get("simulate f32 rows counted (max per launch)", 0), int(off.sum()))


def check_tables_double(got, ref, what):
    """double tables (out_x [n,nx], out_y [n,ny,2]) vs the float64 oracle with its bounds; uncovered columns at the sentinel"""
    gx_, gy_ = got
    tx, ty, bx, by, cov_x, cov_y = ref
    _bounded(gx_[:, cov_x], tx[:, cov_x], bx[:, cov_x], "out_rows f64 x", what + " out_x")
    _bounded(gy_[:, cov_y, 0], ty[:, cov_y, 0], by[:, cov_y, 0], "out_rows f64 y distance", what + " out_y distance")
    _bounded(gy_[:, cov_y, 1], ty[:, cov_y, 1], by[:, cov_y, 1], "out_rows f64 y time", what + " out_y time")
    assert_sentinel(gx_[:, ~cov_x], what + " uncovered out_x columns")
    assert_sentinel(gy_[:, ~cov_y], what + " uncovered out_y columns")


# ------------------------------------------------------------------------------------------------ launches (GPU)
def _lib():
    from vid2player3d_b200 import native
    return native


def _dev(a, dtype):
    import torch
    return torch.as_tensor(np.ascontiguousarray(a), dtype=dtype, device=DEV)


def run_simulate(inp, n, F, cfi, sub, fc, prec):
    """b200ball_simulate through ctypes on sentinel-filled outputs with SLACK rows; returns the first n rows, checks the rest"""
    import torch
    from vid2player3d_b200 import ball_gen as G
    N = _lib()
    td = torch.float32 if prec == 0 else torch.float64
    nc = 3 - fc
    lp, lv, ls = (_dev(a[:n], td) for a in inp)
    traj = torch.full(((n + SLACK) * F * nc,), SENT, dtype=td, device=DEV)
    bpos = torch.full(((n + SLACK) * 3,), SENT, dtype=td, device=DEV)
    bidx = torch.full((n + SLACK,), SENT_IDX, dtype=torch.int64, device=DEV)
    pnet = torch.full((n + SLACK,), SENT_U8, dtype=torch.uint8, device=DEV)
    cfg = G._cfg(F, cfi, sub, SPIN_SCALE, fc)
    N._check(N.lib().b200ball_simulate(C.byref(cfg), C.c_int64(n), C.c_int32(prec), N._ptr(lp), N._ptr(lv), N._ptr(ls), N._ptr(traj),
                                       N._ptr(bpos), N._ptr(bidx), N._ptr(pnet), N._stream()))
    torch.cuda.synchronize()
    traj, bpos, bidx, pnet = (t.cpu().numpy() for t in (traj, bpos, bidx, pnet))
    what = f"simulate n={n} F={F} cfi={cfi} substeps={sub} first_comp={fc} prec={prec}"
    assert_sentinel(traj[n * F * nc:], what + " traj slack")
    assert_sentinel(bpos[n * 3:], what + " bounce_pos slack")
    assert_sentinel(bidx[n:], what + " bounce_idx slack")
    assert_sentinel(pnet[n:], what + " pass_net slack")
    return traj[:n * F * nc].reshape(n, F, nc), bpos[:n * 3].reshape(n, 3), bidx[:n], pnet[:n]


def run_out_rows(inp, n, grids, F, cfi, prec, nx=None, ny=None, offset=0, lo=0, substeps=6):
    """b200ball_out_rows through ctypes on sentinel-filled tables with SLACK rows (optionally wider rows, or base addresses `offset`
    floats past a 16-byte boundary); the columns are passed as given (wrapped by the caller unless a test says otherwise).
    Rows lo ... n - 1 of the inputs are launched; returns their tables."""
    import torch
    from vid2player3d_b200 import ball_gen as G
    N = _lib()
    (gx, cx, nx0), (gy, cy, ny0) = grids
    nx, ny = nx or nx0, ny or ny0
    m = n - lo
    td = torch.float32 if prec == 0 else torch.float64
    vh, vv, vs = (_dev(a[lo:n], td) for a in inp)
    dummy = np.zeros(1)
    gxd, gyd = _dev(gx if len(gx) else dummy, torch.float32), _dev(gy if len(gy) else dummy, torch.float32)
    cxd, cyd = _dev(cx if len(cx) else dummy, torch.int32), _dev(cy if len(cy) else dummy, torch.int32)
    bx = torch.full(((m + SLACK) * nx + 4,), SENT, dtype=td, device=DEV)
    by = torch.full(((m + SLACK) * ny * 2 + 4,), SENT, dtype=td, device=DEV)
    assert bx.data_ptr() % 16 == 0 and by.data_ptr() % 16 == 0
    es = bx.element_size()
    cfg = G._cfg(F, cfi, substeps, SPIN_SCALE, 0)
    N._check(N.lib().b200ball_out_rows(C.byref(cfg), C.c_int64(m), C.c_int32(prec), N._ptr(vh), N._ptr(vv), N._ptr(vs), N._ptr(gxd),
                                       N._ptr(cxd), C.c_int32(len(gx)), C.c_int32(nx), N._ptr(gyd), N._ptr(cyd), C.c_int32(len(gy)),
                                       C.c_int32(ny), C.c_void_p(bx.data_ptr() + offset * es), C.c_void_p(by.data_ptr() + offset * es),
                                       N._stream()))
    torch.cuda.synchronize()
    bx, by = bx.cpu().numpy(), by.cpu().numpy()
    what = f"out_rows n={m} F={F} cfi={cfi} prec={prec} nx={nx} ny={ny} offset={offset}"
    assert_sentinel(bx[:offset], what + " before out_x")
    assert_sentinel(by[:offset], what + " before out_y")
    assert_sentinel(bx[offset + m * nx:], what + " out_x slack")
    assert_sentinel(by[offset + m * ny * 2:], what + " out_y slack")
    return bx[offset:offset + m * nx].reshape(m, nx), by[offset:offset + m * ny * 2].reshape(m, ny, 2)


def _raw(g, scale):
    """(values, int(v * scale) before any wrapping, width) of a grid the wrapper made"""
    v = np.asarray(g[0], f32)
    return v, np.array([int(x * f32(scale)) for x in v], np.int64), int(g[2])


def _wrapped(grids):
    return tuple((g, wrap(c, w), w) for g, c, w in grids)


# ------------------------------------------------------------------------------------------------ b200ball_simulate (GPU)
SIM_CONFIGS = [(F, cfi, sub) for F in FRAMES for cfi in CFI for sub in SUBSTEPS]


@gpu
@pytest.mark.parametrize("F,cfi,sub", SIM_CONFIGS, ids=[f"F{F}-cfi{c}-sub{s}" for F, c, s in SIM_CONFIGS])
def test_simulate_launch(F, cfi, sub):
    inp = sim_inputs()
    ref = P.simulate(*(a.astype(f64) for a in inp), control_freq_inv=cfi, num_frames=F, substeps=sub, spin_scale=SPIN_SCALE,
                     state32=False, world_kw=P.f32_physics())
    big32 = run_simulate(inp, BIG, F, cfi, sub, 0, 0)
    check_sim_float(big32, ref, F * cfi * sub, f"simulate F={F} cfi={cfi} substeps={sub} float")
    for n in SIZES:
        pre = tuple(a[:n] for a in ref)
        check_sim_double(run_simulate(inp, n, F, cfi, sub, 0, 1), pre, 0, f"simulate n={n} F={F} cfi={cfi} substeps={sub} double")
        if n < BIG:
            got = run_simulate(inp, n, F, cfi, sub, 0, 0)
            for k in range(4):
                assert np.array_equal(_bits(got[k]), _bits(big32[k][:n])), f"float n={n}: output {k} differs from the {BIG}-row launch"
    for n in (129, BIG):
        pre = tuple(a[:n] for a in ref)
        for fc in (1, 2):
            check_sim_double(run_simulate(inp, n, F, cfi, sub, fc, 1), pre, fc, f"simulate n={n} F={F} first_comp={fc} double")
            got = run_simulate(inp, n, F, cfi, sub, fc, 0)
            assert np.array_equal(_bits(got[0]), _bits(big32[0][:n, :, fc:])), f"float first_comp={fc} n={n}: traj != columns {fc}: of xyz"
            for k in (1, 2, 3):
                assert np.array_equal(_bits(got[k]), _bits(big32[k][:n])), f"float first_comp={fc} n={n}: output {k} differs"
    for r in ONE_ROW:
        one = run_simulate(tuple(a[r:r + 1] for a in inp), 1, F, cfi, sub, 0, 0)
        for k in range(4):
            assert np.array_equal(_bits(one[k]), _bits(big32[k][r:r + 1])), f"float row {r}: output {k} of a one-row launch differs"


def test_simulate_edges_reach_their_branches():
    """the constructed rows take the branches they were built for (on the float64 twin, which the launches are held to)"""
    inp = sim_inputs()
    e = {k: EDGE_ROWS[i] for i, k in enumerate(("in4R", "in6R", "in6R_up", "never", "before_net", "before_net_back", "net_over",
                                                 "net_under"))}
    for sub, thr_rows in ((2, ("in4R",)), (3, ("in4R", "in6R", "in6R_up"))):
        _, _, bidx, pnet = P.simulate(*(a.astype(f64) for a in inp), num_frames=100, substeps=sub, state32=False, world_kw=P.f32_physics())
        for k in thr_rows:
            assert bidx[e[k]] == 0, (sub, k)
        assert bidx[e["never"]] == 99 and pnet[e["never"]]              # crosses y = 0 high, never comes down
        assert not pnet[e["before_net"]] and not pnet[e["before_net_back"]] and bidx[e["before_net"]] < 20
        assert pnet[e["net_over"]] and not pnet[e["net_under"]]
    _, _, bidx, _ = P.simulate(*(a.astype(f64) for a in inp), num_frames=100, substeps=2, state32=False, world_kw=P.f32_physics())
    assert bidx[e["in6R"]] > 0                                       # 4R: not yet flagged at t = 0


@gpu
def test_simulate_launch_refuses_bad_first_comp():
    import torch
    from vid2player3d_b200 import ball_gen as G
    N = _lib()
    t = torch.zeros(16, dtype=torch.float32, device=DEV)
    for fc in (-1, 3):
        cfg = G._cfg(4, 2, 6, SPIN_SCALE, fc)
        rc = N.lib().b200ball_simulate(C.byref(cfg), C.c_int64(1), C.c_int32(0), *[N._ptr(t)] * 6, N._ptr(t), N._stream())
        assert rc == -2 and b"bad simulation parameters" in N.lib().b200env_last_error()


# ------------------------------------------------------------------------------------------------ b200ball_out_rows (GPU)
OUT_FRAMES = FRAMES + (60,)                                    # 60: the shipped tables
OUT_CONFIGS = [(g, F, cfi) for g in GRIDS if g != "big" for F in OUT_FRAMES for cfi in CFI]


def _out_ref(inp, grids, F, cfi):
    tx, ty, bx, by = out_oracle(inp, BIG, grids, F, cfi)
    return tx, ty, bx, by, covered(grids[0][1], grids[0][2]), covered(grids[1][1], grids[1][2])


def _pre(ref, n):
    tx, ty, bx, by, cx, cy = ref
    return tx[:n], ty[:n], bx[:n], by[:n], cx, cy


@gpu
@pytest.mark.parametrize("grid,F,cfi", OUT_CONFIGS, ids=[f"{g}-F{F}-cfi{c}" for g, F, c in OUT_CONFIGS])
def test_out_rows_launch(grid, F, cfi):
    inp = out_inputs()
    grids = GRIDS[grid]()
    ref = _out_ref(inp, grids, F, cfi)
    kg = _wrapped(grids)
    (_, _, nx), (_, _, ny) = kg
    big32 = run_out_rows(inp, BIG, kg, F, cfi, 0)
    for n in SIZES:
        what = f"out_rows grid={grid} n={n} F={F} cfi={cfi}"
        check_tables_double(run_out_rows(inp, n, kg, F, cfi, 1), _pre(ref, n), what + " double")
        if n < BIG:
            got = run_out_rows(inp, n, kg, F, cfi, 0)
            assert np.array_equal(_bits(got[0]), _bits(big32[0][:n])) and np.array_equal(_bits(got[1]), _bits(big32[1][:n])), \
                what + ": float rows differ from the largest launch"
    # scalar stores: a row one column wider, an odd number of (distance, time) pairs
    wx, wy = run_out_rows(inp, BIG, kg, F, cfi, 0, nx=nx + 1, ny=ny + 1 - ny % 2)
    assert np.array_equal(_bits(wx[:, :nx]), _bits(big32[0])) and np.array_equal(_bits(wy[:, :ny]), _bits(big32[1])), "scalar path != vector path"
    assert_sentinel(wx[:, nx:], "the extra out_x column")
    assert_sentinel(wy[:, ny:], "the extra out_y pairs")
    # base addresses 4 bytes past a 16-byte boundary
    mx, my = run_out_rows(inp, BIG, kg, F, cfi, 0, offset=1)
    assert np.array_equal(_bits(mx), _bits(big32[0])) and np.array_equal(_bits(my), _bits(big32[1])), "misaligned tables differ"
    for r in ONE_ROW:
        ox, oy = run_out_rows(inp, r + 1, kg, F, cfi, 0, lo=r)
        assert np.array_equal(_bits(ox), _bits(big32[0][r:r + 1])) and np.array_equal(_bits(oy), _bits(big32[1][r:r + 1])), \
            f"out_rows grid={grid} row {r}: a one-row launch differs"


@gpu
@pytest.mark.parametrize("F,cfi", [(60, 2), (9, 3)])
def test_out_rows_launch_grids_of_4096(F, cfi):
    """ngx = ngy = 4096: 80 KB of shared memory in the double instantiation (opt-in past 48 KB); 4097 refused"""
    inp = out_inputs()
    grids = GRIDS["big"]()
    ref = _out_ref(inp, grids, F, cfi)
    for n in (129, 1000):
        check_tables_double(run_out_rows(inp, n, grids, F, cfi, 1), _pre(ref, n), f"out_rows 4096-value grids n={n} double")
    big32 = run_out_rows(inp, 1000, grids, F, cfi, 0)
    small = run_out_rows(inp, 129, grids, F, cfi, 0)
    assert np.array_equal(_bits(small[0]), _bits(big32[0][:129])) and np.array_equal(_bits(small[1]), _bits(big32[1][:129]))
    (gx, cx, nx), (gy, cy, ny) = grids
    for over in ((np.append(gx, gx[-1]), np.append(cx, 0), nx), (gy, cy, ny)), ((gx, cx, nx), (np.append(gy, gy[-1]), np.append(cy, 0), ny)):
        with pytest.raises(RuntimeError, match="grid sizes out of range"):
            run_out_rows(inp, 1, over, F, cfi, 0)


@gpu
def test_out_rows_launch_skips_columns_outside_the_row():
    """raw columns -1, nx, nx + 5 (resp. for y) reach the kernel unwrapped: never stored; every other column as without them"""
    inp = out_inputs()
    (gx, cx, nx), (gy, cy, ny) = GRIDS["shipped"]()
    bad_x, bad_y = {7: -1, 20: nx, 41: nx + 5}, {3: -1, 12: ny, 25: ny + 5}
    raw = ((gx, np.array([bad_x.get(j, c) for j, c in enumerate(cx)], np.int32), nx),
           (gy, np.array([bad_y.get(j, c) for j, c in enumerate(cy)], np.int32), ny))
    keep_x, keep_y = np.array([j not in bad_x for j in range(len(gx))]), np.array([j not in bad_y for j in range(len(gy))])
    kept = ((gx[keep_x], cx[keep_x], nx), (gy[keep_y], cy[keep_y], ny))   # a sorted grid: dropping values does not move the others' walk
    ref = _out_ref(inp, kept, 60, 2)
    for prec in (0, 1):
        for n in (129, BIG):
            got = run_out_rows(inp, n, raw, 60, 2, prec)
            if prec == 1:
                check_tables_double(got, _pre(ref, n), f"out_rows raw columns n={n}")
            else:
                want = run_out_rows(inp, n, _wrapped(kept), 60, 2, 0)
                assert np.array_equal(_bits(got[0]), _bits(want[0])) and np.array_equal(_bits(got[1]), _bits(want[1]))


@gpu
def test_out_rows_wrapper_wraps_negative_columns():
    """ball_gen.simulate_without_bounce with ranges whose columns are negative (wrapped like Python) or duplicated across the
    sample-0 boundary, against the oracle on the same ranges; a column past the row raises IndexError before any launch"""
    import torch
    from vid2player3d_b200 import ball_gen as G
    inp = out_inputs(300)
    for xr, yr in (((-0.5, 30, 0.5), (0, 3, 0.1)), ((-0.25, 30, 0.25), (-0.3, 3, 0.1))):
        class params(G.traj_out_params):
            TRAJ_X_RANGE, TRAJ_Y_RANGE = xr, yr
        gx, gy = G.simulate_without_bounce(*inp, params=params, dtype=torch.float64)
        grids = (_raw(G._grid(xr, 2), 2), _raw(G._grid(yr, 10), 10))       # torch.arange's values (not always P.torch_arange's)
        tx, ty, bx, by = out_oracle(inp, 300, grids, 60, 2)
        cx, cy = covered(grids[0][1], grids[0][2]), covered(grids[1][1], grids[1][2])
        gx, gy = gx.cpu().numpy(), gy.cpu().numpy()
        assert (gx[:, ~cx] == 0).all() and (gy[:, ~cy] == 0).all()           # the wrapper zero-fills a row its grid does not cover
        gx[:, ~cx], gy[:, ~cy] = SENT, SENT
        check_tables_double((gx, gy), (tx, ty, bx, by, cx, cy), f"wrapper {xr} {yr}")

    class past(G.traj_out_params):
        TRAJ_X_RANGE = (0.5, 30, 0.5)
    with pytest.raises(IndexError):
        G.simulate_without_bounce(*inp, params=past)


# ------------------------------------------------------------------------------------------------ the pool filter (GPU)
def pool_valid_rows(traj, bounce_pos, bounce_idx, pass_net, bmin, bmax):
    """tennis_ball.py:319-327, row by row"""
    import torch
    valid = pass_net.bool() & (bounce_pos.sum() != 0) & (bounce_pos[:, 0] > bmin[0]) & (bounce_pos[:, 0] < bmax[0]) & \
        (bounce_pos[:, 1] > bmin[1]) & (bounce_pos[:, 1] < bmax[1])
    valid = valid.clone()
    for i in range(len(valid)):
        valid[i] &= bool(traj[i, bounce_idx[i]:, 2].max() > 1.0)
    return valid.to(torch.bool)


@gpu
def test_pool_filter_equals_the_per_row_rule():
    import torch
    from vid2player3d_b200 import ball_gen as G
    gen = G.TennisBallGeneratorB200({}, need_reset=False, device=DEV)
    bmin, bmax = gen.bounce_min.to(DEV), gen.bounce_max.to(DEV)
    inp = sim_inputs()
    for sub in (6, 2):
        out = G.simulate(*inp, substeps=sub, device=DEV)
        got = G.pool_valid(*out, bmin, bmax)
        want = pool_valid_rows(*out, bmin, bmax)
        assert torch.equal(got, want) and 0 < int(got.sum()) < BIG
    # no ball bounces: bounce_pos is zero everywhere, the whole-tensor sum rejects every row
    never = (np.tile(inp[0][EDGE_ROWS[3]], (64, 1)), np.tile(inp[1][EDGE_ROWS[3]], (64, 1)), np.full(64, 7, f32))
    out = G.simulate(*never, device=DEV)
    assert float(out[1].abs().sum()) == 0 and bool(out[3].all())
    assert not bool(G.pool_valid(*out, bmin, bmax).any()) and not bool(pool_valid_rows(*out, bmin, bmax).any())


# ------------------------------------------------------------------------------------------------ CPU: wrapper columns, controls
def test_wrapper_columns_follow_python_indexing():
    from vid2player3d_b200 import ball_gen as G
    import torch
    for rng, scale in (((0, 30, 0.5), 2), ((0, 3, 0.1), 10), ((-0.5, 30, 0.5), 2), ((-0.25, 30, 0.25), 2), ((-0.3, 3, 0.1), 10)):
        v, c, w = G._grid(rng, scale)
        rv, rc, rw = _raw((v, c, w), scale)
        assert w == P.grid(rng, scale)[2] and np.array_equal(v.numpy(), torch.arange(*rng).numpy()) and np.array_equal(c.numpy(), wrap(rc, w))
    v, c, w = G._grid((-0.5, 30, 0.5), 2)
    assert int(c[0]) == w - 1                                        # x = -0.5 -> column -1 -> the last one
    for rng in ((0.5, 30, 0.5), (-31, -29, 0.5)):                    # column 59 of a 59-wide row; column -62 of a 4-wide row
        with pytest.raises(IndexError):
            G._grid(rng, 2)


def test_oracle_explicit_grids_reproduce_golden():
    """the extended oracle on the shipped grids, passed explicitly and stored in float64, still reproduces v2p_ballgen.npz"""
    import os
    Z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "v2p_ballgen.npz"))
    vh, vv, vs = Z["out_vel"][:, 1], Z["out_vel"][:, 2], Z["out_vspin"]
    m = len(vs)
    lp, lv = np.zeros((m, 3), f32), np.stack([np.zeros(m), vh, vv], 1).astype(f32)
    dx, dy = P.simulate_without_bounce(lp, lv, vs)
    walk = {}
    tx, ty = P.simulate_without_bounce(lp, lv, vs, grid_x=P.grid((0, 30, 0.5), 2), grid_y=P.grid((0, 3, 0.1), 10), table_dtype=f64,
                                       walk=walk)
    assert tx.dtype == f64 and np.array_equal(tx.astype(f32), dx) and np.array_equal(ty.astype(f32), dy)
    assert np.abs(tx - Z["out_x"]).max() < 1e-5
    assert (np.abs(ty - Z["out_y"]) <= 1e-5 + 1e-4 * np.abs(Z["out_y"])).all()
    assert walk["samples"].shape == (m, 122, 2) and (walk["t_x"][:, 0] == 0).all() and (np.diff(walk["t_x"], axis=1) >= 0).all()
    # Python index semantics: column -1 is the last one, -61 / 60 of a 60-wide row raise
    one = P.simulate_without_bounce(lp[:4], lv[:4], vs[:4], grid_x=explicit([5.0], [-1], 60), grid_y=EMPTY_Y)[0]
    assert (one[:, :59] == 0).all() and (one[:, 59] != 0).all()
    for c in (-61, 60):
        with pytest.raises(IndexError):
            P.simulate_without_bounce(lp[:4], lv[:4], vs[:4], grid_x=explicit([5.0], [c], 60), grid_y=EMPTY_Y)


def _sim_ref(n=40, F=17, sub=3):
    inp = sim_inputs(n, seed=3)
    return P.simulate(*(a.astype(f64) for a in inp), num_frames=F, substeps=sub, state32=False, world_kw=P.f32_physics())


def test_simulate_comparators_reject_mutations():
    ref = _sim_ref()
    got = tuple(a.copy() for a in ref[:3]) + (ref[3].astype(np.uint8),)
    check_sim_double(got, ref, 0, "unmutated")
    check_sim_double((got[0][:, :, 1:],) + got[1:], ref, 1, "unmutated first_comp 1")
    shifted = got[0].copy()
    shifted[:, 8:16] = got[0][:, 0:8]                                 # a chunk's frames written one chunk late
    with pytest.raises(AssertionError, match="traj"):
        check_sim_double((shifted,) + got[1:], ref, 0, "chunk shift")
    bidx = got[2].copy()
    k = int(np.nonzero(bidx < 16)[0][0])
    bidx[k] += 1
    with pytest.raises(AssertionError, match="bounce_idx"):
        check_sim_double(got[:2] + (bidx, got[3]), ref, 0, "bounce index")
    for frac, fails in ((1.01, True), (0.99, False)):
        t = got[0].copy()
        t[5, 9, 1] += frac * TOL64                                    # one element just outside / inside the bound
        if fails:
            with pytest.raises(AssertionError, match="traj"):
                check_sim_double((t,) + got[1:], ref, 0, "one element")
        else:
            check_sim_double((t,) + got[1:], ref, 0, "one element")
    # the float comparator: 1 % of 40 rows is none, one row over its bound fails
    f = (got[0].astype(f32), got[1].astype(f32), got[2], got[3])
    check_sim_float(f, ref, 17 * 2 * 3, "unmutated float")
    t = f[0].copy()
    t[30, 4, 0] += 0.1
    with pytest.raises(AssertionError, match="rows off"):
        check_sim_float((t,) + f[1:], ref, 17 * 2 * 3, "one row off")


def test_table_comparator_rejects_mutations():
    inp = out_inputs(40, seed=4)
    grids = GRIDS["dup"]()
    tx, ty, bx, by = out_oracle(inp, 40, grids, 17, 2)
    cov = (covered(grids[0][1], grids[0][2]), covered(grids[1][1], grids[1][2]))
    ref = (tx, ty, bx, by) + cov

    def as_got(x, y):
        x, y = x.copy(), y.copy()
        x[:, ~cov[0]], y[:, ~cov[1]] = SENT, SENT
        return x, y
    check_tables_double(as_got(tx, ty), ref, "unmutated")
    # the sample-0 entries x = -0.25 and y = -0.05 rewritten after the later values of their columns (what the kernel did)
    gx, cx, nx = grids[0]
    gy, cy, ny = grids[1]
    late_x, late_y = P.simulate_without_bounce(np.zeros((40, 3)), np.stack([np.zeros(40), inp[0], inp[1]], 1).astype(f64),
                                               inp[2].astype(f64), control_freq_inv=2, num_frames=17, state32=False,
                                               world_kw=P.f32_physics(), grid_x=(gx[:1], cx[:1], nx), grid_y=(gy[:1], cy[:1], ny),
                                               table_dtype=f64)
    assert cx[0] == cx[1] == cx[2] == 0 and cy[0] == cy[1] == cy[2] == 0
    mx = tx.copy()
    mx[:, 0] = late_x[:, 0]
    with pytest.raises(AssertionError, match="out_x"):
        check_tables_double(as_got(mx, ty), ref, "sample-0 x rewritten last")
    my = ty.copy()
    my[:, 0] = late_y[:, 0]
    with pytest.raises(AssertionError, match="out_y"):
        check_tables_double(as_got(tx, my), ref, "sample-0 y rewritten last")
    # one element just outside / inside its own bound, in each table
    for frac, fails in ((1.01, True), (0.99, False)):
        mx, my = tx.copy(), ty.copy()
        mx[7, 11] += frac * bx[7, 11]
        my[9, 5, 1] -= frac * by[9, 5, 1]
        for a, b in ((mx, ty), (tx, my)):
            if fails:
                with pytest.raises(AssertionError, match="bound"):
                    check_tables_double(as_got(a, b), ref, "one element")
            else:
                check_tables_double(as_got(a, b), ref, "one element")
    # an uncovered column written, and non-finite in one only
    x, y = as_got(tx, ty)
    x[2, -1] = 0.0
    with pytest.raises(AssertionError, match="uncovered out_x"):
        check_tables_double((x, y), ref, "uncovered")
    x, y = as_got(tx, ty)
    x[2, 3] = np.inf
    with pytest.raises(AssertionError, match="finite in one only"):
        check_tables_double((x, y), ref, "non-finite")
