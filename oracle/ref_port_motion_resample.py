"""Integer / float64 restatement of the training resample of HumanoidSMPLIM (cfg.env.b200_resample_motions; include/b200env.h:
b200env_resample_motions and b200env_motion_weights).  Before a reset, every masked env that played a step (progress_buf > 0):
  - with h = cfg.env.b200_hard_motion_share > 0, adds one try to the motion it finished, and one fail when terminate_buf is set;
  - draws u = (counter_bits(seed', c, e) >> 11) 2^-53 at the launch counter c, seed' = splitmix64(seed ^ "motionid"), and takes the
    smallest motion m with cdf[m] > u cdf[M - 1], clamped to M - 1;
and the launch counter advances by one.  The rebuild (pre_epoch) sets r_m = fails / tries for the motions tried since the last one, zeroes
the counts and writes the CDF of p_m = (1 - h) b_m / sum b + h b_m r_m / sum b r (b_m / sum b when sum b r = 0 or h = 0), with b_m the base
weights of _sample_motion_ids (motion_lengths under motion_weights_from_length, else 1).  Test infrastructure: the device launches and
the task are held to it."""
import numpy as np

from .ref_port_v2p import M64, splitmix64

RESAMPLE_KEY = 0x6D6F74696F6E6964          # "motionid" in ASCII


def counter_bits(seed, counter, idx):
    """splitmix64(splitmix64(seed ^ counter * 0xD1B54A32D192ED03) + idx), all mod 2^64 (csrc/counter_rng.cuh)"""
    with np.errstate(over="ignore"):
        h0 = splitmix64(np.uint64(int(seed) & M64) ^ np.uint64((int(counter) * 0xD1B54A32D192ED03) & M64))
        return splitmix64(h0 + np.asarray(idx, np.uint64))


def resample_seed(seed):
    """seed' of the motion draws: the cfg seed re-keyed, so no draw shares a key with the masked reset's or the transforms'"""
    with np.errstate(over="ignore"):
        return int(splitmix64(np.uint64((int(seed) ^ RESAMPLE_KEY) & M64)))


def uniforms(seed, counter, n):
    """u_e in [0, 1) of envs e < n at launch counter `counter`, in 53 bits"""
    bits = counter_bits(resample_seed(seed), counter, np.arange(n, dtype=np.uint64))
    return (bits >> np.uint64(11)).astype(np.float64) * 2.0 ** -53


def draw(cdf, u):
    """the smallest m with cdf[m] > u cdf[M - 1], clamped to M - 1"""
    cdf = np.asarray(cdf, np.float64)
    return np.minimum(np.searchsorted(cdf, np.asarray(u, np.float64) * cdf[-1], side="right"), len(cdf) - 1).astype(np.int64)


def base_weights(motion_lengths, from_length):
    """b_m of _sample_motion_ids: the motion lengths (float32 widened) under motion_weights_from_length, else 1"""
    lengths = np.asarray(motion_lengths, np.float32)
    return lengths.astype(np.float64) if from_length else np.ones(len(lengths))


def motion_cdf(base, rate, h):
    """the running sum in extended precision: a float64 running sum over 10^5 motions drifts by ~1e-11, far more than the launch's
    blocked scan"""
    b = np.asarray(base, np.float64)
    s_br = (b * rate).sum() if h > 0 else 0.0
    p = (1.0 - h) * b / b.sum() + h * b * rate / s_br if s_br > 0 else b / b.sum()
    return np.cumsum(p.astype(np.longdouble)).astype(np.float64)


class Resampler:
    """the resample's state: cdf, rate (1 at the start), tries, fails and the launch counter"""

    def __init__(self, base, h, seed):
        self.base, self.h, self.seed = np.asarray(base, np.float64), float(h), int(seed)
        M = len(self.base)
        self.rate = np.ones(M)
        self.tries, self.fails = np.zeros(M, np.int64), np.zeros(M, np.int64)
        self.counter = 0
        self.cdf = motion_cdf(self.base, self.rate, 0.0)

    def resample(self, motion_ids, mask, progress, terminate):
        """one launch: (new motion ids, the envs that drew)"""
        motion_ids = np.asarray(motion_ids, np.int64)
        drew = np.asarray(mask, bool) & (np.asarray(progress) > 0)
        if self.h > 0:
            np.add.at(self.tries, motion_ids[drew], 1)
            np.add.at(self.fails, motion_ids[drew & (np.asarray(terminate) != 0)], 1)
        out = motion_ids.copy()
        out[drew] = draw(self.cdf, uniforms(self.seed, self.counter, len(out))[drew])
        self.counter += 1
        return out, drew

    def rebuild(self):
        """pre_epoch: nothing when h = 0"""
        if self.h == 0:
            return
        seen = self.tries > 0
        self.rate[seen] = self.fails[seen] / self.tries[seen]
        self.tries[:] = 0
        self.fails[:] = 0
        self.cdf = motion_cdf(self.base, self.rate, self.h)
