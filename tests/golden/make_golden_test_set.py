"""Golden fixture for the fixed test set of incoming balls, produced by EXECUTING the reference's own code on CPU:

  - TennisBallGeneratorOffline(file, sample_random=False, num_envs) and its generate(n, need_init_state=True, start_pos, env_ids)
    (vid2player/utils/tennis_ball.py:422-456) over a sequence of env id lists per case: envs repeated across calls, cursors wrapping
    at P, a pool of one row, a pool larger than the env count, and start positions with y > 0 that the sequential branch ignores;
  - the test_mode rule of vid2player/env/utils/player_builder.py:154-156 (its three lines, executed as they stand) on a few file names.

Run in the build container only:

    python tests/golden/make_golden_test_set.py      ->  tests/golden/v2p_ball_test_set.npz
"""
import os
import sys
import tempfile
import textwrap

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import _refenv  # noqa: E402

_refenv.setup("vid2player")

from utils import tennis_ball as TB  # noqa: E402

# (name, N, P, env id lists)
CASES = [
    ("wrap", 5, 3, [[0, 1, 2, 3, 4], [1, 3], [0, 1, 2, 3, 4], [3], [3], [4, 2, 0], [1, 3, 4], [0, 1, 2, 3, 4]]),
    ("one_row", 4, 1, [[0, 1, 2, 3], [1, 2], [2], [3, 0]]),
    ("pool_larger", 3, 7, [[0, 1, 2], [2, 0], [1], [0, 1, 2], [2], [2], [2], [2], [0, 2]]),
]
FILE_NAMES = ["data/ball_traj/ball_traj_in_test_single.npy", "data/ball_traj/ball_traj_in_test.npy", "single.npy", "SINGLE.npy",
              "singles/test.npy", "multiple_single_cycle.npy"]


def player_builder_rule():
    """the three lines of player_builder.py:154-156, dedented, as a function of cfg"""
    path = os.path.join(_refenv.REF, "vid2player", "env", "utils", "player_builder.py")
    lines = open(path).read().splitlines()[153:156]
    assert "ball_traj_file_test" in lines[0] and "test_mode" in lines[2], lines
    code = compile(textwrap.dedent("\n".join(lines)), path, "exec")

    def run(cfg):
        exec(code, {}, {"cfg": cfg})
        return cfg
    return run


def main():
    rng = np.random.default_rng(31)
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        for name, N, P, calls in CASES:
            pool = rng.uniform(-20, 20, (P, 307)).astype(np.float32)
            f = os.path.join(tmp, f"{name}.npy")
            np.save(f, pool)
            gen = TB.TennisBallGeneratorOffline(f, sample_random=False, num_envs=N)
            ids, idx, traj, pos, vel, spin, start, lens = [], [], [], [], [], [], [], []
            for c in calls:
                sp = rng.uniform(-5, 5, (len(c), 3)).astype(np.float32)
                sp[::2, 1] = rng.uniform(0.5, 12, len(sp[::2]))             # the far side: the random branch would remap these
                env_ids = torch.tensor(c, dtype=torch.long)
                before = gen.sample_idx.clone()
                t, lp, lv, ls = gen.generate(len(c), need_init_state=True, start_pos=torch.from_numpy(sp), env_ids=env_ids)
                ids.append(c)
                idx.append(before[env_ids].numpy())
                traj.append(t.numpy()), pos.append(lp.numpy()), vel.append(lv.numpy()), spin.append(ls.numpy())
                start.append(sp)
                lens.append(len(c))
            cat = np.concatenate
            out.update({f"{name}_pool": pool, f"{name}_num_envs": np.int64(N), f"{name}_lens": np.array(lens, np.int64),
                        f"{name}_env_ids": cat(ids).astype(np.int64), f"{name}_index": cat(idx).astype(np.int64),
                        f"{name}_start_pos": cat(start), f"{name}_traj": cat(traj), f"{name}_launch_pos": cat(pos),
                        f"{name}_launch_vel": cat(vel), f"{name}_launch_vspin": cat(spin),
                        f"{name}_cursor": gen.sample_idx.numpy().astype(np.int64)})
    out["cases"] = np.array([c[0] for c in CASES])
    rule = player_builder_rule()
    modes = [rule(dict(env=dict(ball_traj_file_test=n, vid2player={})))["env"]["vid2player"]["test_mode"] for n in FILE_NAMES]
    unset = rule(dict(env=dict(ball_traj_file_test=None, vid2player={})))["env"]["vid2player"]
    assert unset == {}, unset
    out.update(file_names=np.array(FILE_NAMES), test_modes=np.array(modes))
    np.savez_compressed(os.path.join(HERE, "v2p_ball_test_set.npz"), **out)
    print({k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()
