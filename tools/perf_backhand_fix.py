"""Time of the two-hand backhand fix (b200v2p_backhand_fix, one launch for all exported episodes) against the reference's method, the
torch-autograd restatement oracle/ref_port_backhand.py run on the GPU in float32 (500 Adam steps over the SMPL FK, one episode after
the other), for num_eg in {1, 10} episodes of 300 (single) and 1800 (dual capacity) frames, two backhand segments each (about 40 % of
the frames selected).  Device events around each; the launch is timed over --reps calls after a warm-up, the restatement once per
configuration after a warm-up episode.  Prints one JSON line per configuration and the card name and power limit read in the same run.

    python tools/perf_backhand_fix.py [--reps 20]
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import ref_port_backhand as B  # noqa: E402
from tools.perf_eval import card  # noqa: E402
from vid2player3d_b200 import native_v2p  # noqa: E402

DEV = "cuda:0"


def episodes(n, T, seed):
    g = torch.Generator().manual_seed(seed)
    rest = torch.randn(24, 3, generator=g) * 0.1
    out = []
    for _ in range(n):
        jr = 0.35 * torch.randn(1, 24, 3, generator=g) + 0.03 * torch.randn(T, 24, 3, generator=g).cumsum(0)
        phase, swing = torch.rand(T, generator=g) * 2.0, torch.zeros(T, dtype=torch.long)
        for a, b in ((T // 10, T // 10 + T // 5), (T // 2, T // 2 + T // 5)):
            phase[a:b], swing[a:b] = 2.05 + 2.9 * torch.rand(b - a, generator=g), 2
        out.append(dict(joint_rot=jr.to(DEV), phase=phase.to(DEV), swing_type=swing.to(DEV), rest=rest.to(DEV), righthand=True))
    return out


def timed(fn, reps):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(reps):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    name, power, clock = card()
    for T in (300, 1800):
        for n in (1, 10):
            probs = episodes(n, T, seed=T + n)
            native_v2p.backhand_fix(probs)
            launch_ms = timed(lambda: native_v2p.backhand_fix(probs), a.reps)
            B.fix_episode(probs[0]["joint_rot"], probs[0]["phase"], probs[0]["swing_type"], probs[0]["rest"], True, 5)   # warm-up
            ref_ms = timed(lambda: [B.fix_episode(p["joint_rot"], p["phase"], p["swing_type"], p["rest"], True) for p in probs], 1)
            M = int(sum(B.select(p["swing_type"], p["phase"]).sum() for p in probs))
            print(json.dumps(dict(frames=T, num_eg=n, selected_frames=M, iters=native_v2p.BACKHAND_ITERS, launch_ms=round(launch_ms, 3),
                                  autograd_ms=round(ref_ms, 1), speedup=round(ref_ms / launch_ms, 1), gpu=name, power_limit=power,
                                  max_sm_clock=clock)), flush=True)


if __name__ == "__main__":
    main()
