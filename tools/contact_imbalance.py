"""How unevenly is the ground-contact work of the step kernel spread?  (CPU only: float64 restatement + numpy.)

Rolls N humanoids forward with a random policy until they lie on the ground (the state the bench workload is in: 92 % of the envs),
then counts, per env and body, the hull vertices below the ground plane - the per-vertex loop of contact_hull is the part of the
body pass whose cost differs between lanes.  Reports, for the packed kernel's lane mapping (body b of env g is handled by lane
(g, b % 8) in round b / 8; a warp = 4 consecutive envs; a CTA batch = 8 warps, the split form's step_kernel_packed):
  * penetrating vertices per env (mean, p90, max),
  * executed vs useful iterations of the vertex loop: a warp runs max-over-lanes iterations per round,
  * the spread of the per-warp totals inside a CTA batch (what the batch barrier waits for)."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
from scipy.spatial.transform import Rotation

from oracle import physics_ref
from vid2player3d_b200 import abi, model_compiler


def main(n=224, steps=45, seed=0):
    mod = model_compiler.load_compiled("smpl_mesh_humanoid_amass_v1")
    ms, verts = abi.pack_model(mod, float(mod["mass"].sum()) / 90.0)
    cfg = abi.make_cfg(mod)
    rng = np.random.default_rng(seed)
    root = np.zeros((n, 13)); root[:, 2] = 0.9; root[:, 3:7] = [0.5, 0.5, 0.5, 0.5]
    root[:, 0:2] = rng.uniform(-2, 2, (n, 2))
    q, qd = rng.normal(0, 0.1, (n, 69)), np.zeros((n, 69))
    for s in range(steps):
        a = rng.uniform(-1, 1, (n, 69))
        tar = np.clip(a, q - 0.5 * np.pi, q + 0.5 * np.pi)               # _action_to_pd_targets with a random policy
        rb, _ = physics_ref.control_step(ms, verts, cfg, root, q, qd, tar, None)
    nb = ms.nb
    V = np.asarray(verts, np.float64).reshape(nb, -1, 3)
    nv = np.asarray(mod["nverts"])
    pen = np.zeros((n, nb), int)
    for b in range(nb):
        R = Rotation.from_quat(rb[:, b, 3:7]).as_matrix()                # [n,3,3]
        z = rb[:, b, 2:3] + np.einsum("nk,vk->nv", R[:, 2, :], V[b, :nv[b]])
        pen[:, b] = (z < 0).sum(1)
    fallen = rb[:, 0, 2] < 0.5
    per_env = pen.sum(1)
    print(f"{n} envs after {steps} random-policy steps: {fallen.mean() * 100:.0f} % lying (root z < 0.5 m)")
    print(f"penetrating hull vertices per env: mean {per_env.mean():.1f}, p90 {np.percentile(per_env, 90):.0f}, max {per_env.max()}"
          f"; bodies in contact per env: mean {(pen > 0).sum(1).mean():.1f}")
    # packed mapping: warp = 4 envs, lane (g, s) handles bodies s, 8+s, 16+s in rounds 0..2
    useful = executed = 0
    warp_tot = []
    for w0 in range(0, n - 3, 4):
        tot = 0
        for r in range(3):
            lanes = pen[w0:w0 + 4, r * 8:(r + 1) * 8]                    # [4 envs, 8 slots]
            useful += lanes.sum()
            executed += lanes.max() * lanes.size                          # every lane waits for the slowest one of the round
            tot += lanes.max()
        warp_tot.append(tot)
    warp_tot = np.array(warp_tot)
    print(f"vertex-loop iterations per control-step substep: useful {useful}, executed in lock step {executed} -> lanes busy {useful / executed * 100:.0f} %")
    print(f"serial vertex iterations per warp and substep (sum over the 3 rounds of the max over lanes): mean {warp_tot.mean():.1f}, max {warp_tot.max()}")
    nbatch = len(warp_tot) // 8
    b = warp_tot[:nbatch * 8].reshape(nbatch, 8)
    print(f"inside a CTA batch of 8 warps: mean of max {b.max(1).mean():.1f} vs mean {b.mean():.1f} -> the slowest warp has "
          f"{(b.max(1).mean() / b.mean() - 1) * 100:.0f} % more vertex iterations than the average one (~70 instructions each)")
    def layout(order):
        """serial vertex iterations per warp / per batch when the envs are handed out in `order`"""
        P = pen[order]
        wt = np.array([sum(P[w0:w0 + 4, r * 8:(r + 1) * 8].max() for r in range(3)) for w0 in range(0, n - 3, 4)])
        bt = wt[:len(wt) // 8 * 8].reshape(-1, 8)
        return wt.mean(), bt.max(1).mean()
    env_serial = np.array([sum(pen[e, r * 8:(r + 1) * 8].max() for r in range(3)) for e in range(n)])
    print("hand-out order of the envs -> (mean serial iterations per warp, mean over batches of the slowest warp):")
    for name, key in (("as they are (today)", None), ("sorted by the env's own serial count (exact)", env_serial), ("sorted by total penetrating vertices", per_env),
                      ("sorted by bodies in contact", (pen > 0).sum(1)), ("8 bins of the serial count", np.minimum(env_serial // 4, 7))):
        order = np.arange(n) if key is None else np.argsort(-key, kind="stable")
        w, b = layout(order)
        print(f"  {name:48s} warp {w:5.1f}   batch max {b:5.1f}")


if __name__ == "__main__":
    main(*(int(x) for x in sys.argv[1:]))
