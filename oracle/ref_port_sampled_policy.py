"""Float64 restatement of the sampled action's noise (include/b200nn.h noise fields, csrc/counter_rng.cuh counter_normal): the N(0, 1)
draw of output element (row, col) of a layer at launch `step` under `seed` is Box-Muller on the 24-bit fields of
counter_hash(seed, step, row * ldo + out_col0 + col).  The uniforms are rounded to float32 as the kernel forms them; log, sqrt and cos
are taken in float64, so the restatement differs from the kernel by the float32 rounding of those three functions only."""
import numpy as np

from oracle.ref_port_v2p import counter_hash


def element_index(row, col, ldo, out_col0=0):
    """the draw index of output (row, col) of a layer writing out[:, out_col0:] with leading dimension ldo: the flat index of the
    element in the output buffer (env * actions + col for both the single policy and each network of the dual one)"""
    return np.asarray(row, np.uint64) * np.uint64(ldo) + np.uint64(out_col0) + np.asarray(col, np.uint64)


def counter_normal(seed, step, row, col, ldo, out_col0=0):
    """eps [len(row) x len(col)] (broadcast of row[:, None], col[None, :]) in float64"""
    f = np.float32
    idx = element_index(np.asarray(row)[:, None], np.asarray(col)[None, :], ldo, out_col0)
    h = counter_hash(int(seed) & 0xFFFFFFFFFFFFFFFF, step, idx)
    u1 = ((h >> np.uint64(40)).astype(np.uint32) + np.uint32(1)).astype(f) * f(1.0 / 16777217.0)     # (0, 1): finite log
    u2 = ((h >> np.uint64(8)) & np.uint64(0xFFFFFF)).astype(f) * f(1.0 / 16777216.0)
    ang = (f(6.283185307179586) * u2).astype(np.float64)
    return np.sqrt(-2.0 * np.log(u1.astype(np.float64))) * np.cos(ang)


def log_amplification(seed, step, row, col, ldo, out_col0=0):
    """1 / sqrt(-2 ln u1) of each draw: the factor by which an error in log(u1) reaches eps.  Near u1 = 1 (|eps| ~ 1e-4) the float32
    logf's last-bit error becomes ~1e-3 in eps; a comparison with the kernel allows a few float32 ulps times this factor."""
    f = np.float32
    idx = element_index(np.asarray(row)[:, None], np.asarray(col)[None, :], ldo, out_col0)
    h = counter_hash(int(seed) & 0xFFFFFFFFFFFFFFFF, step, idx)
    u1 = ((h >> np.uint64(40)).astype(np.uint32) + np.uint32(1)).astype(f) * f(1.0 / 16777217.0)
    return 1.0 / np.sqrt(-2.0 * np.log(u1.astype(np.float64)))


def sample(mu, sigma, seed, step, ldo=None, out_col0=0, clip=None):
    """clamp(mu + sigma * eps, -clip, clip) of a float64 mu [rows, n] (the reference's Normal(mu, sigma).sample() then the wrapper's
    clamp), eps keyed like the kernel; ldo defaults to n"""
    rows, n = mu.shape
    eps = counter_normal(seed, step, np.arange(rows), np.arange(n), n if ldo is None else ldo, out_col0)
    a = mu + np.asarray(sigma, np.float64)[None, :] * eps
    return np.clip(a, -clip, clip) if clip else a
