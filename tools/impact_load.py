"""Ground-contact load of a falling humanoid, step by step (CPU only: float64 restatement): bodies in contact per env and penetrating hull
vertices per body - the length of the serial vertex loop that decides when the LAST warp of the one-wave physics launch finishes.   python tools/impact_load.py"""
import sys
import os
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'tests'))
import numpy as np
from scipy.spatial.transform import Rotation
from oracle import physics_ref
from vid2player3d_b200 import abi, model_compiler
mod = model_compiler.load_compiled("smpl_mesh_humanoid_amass_v1")
ms, verts = abi.pack_model(mod, float(mod["mass"].sum()) / 90.0)
cfg = abi.make_cfg(mod)
rng = np.random.default_rng(0)
n=512
root = np.zeros((n, 13)); root[:, 2] = 0.9; root[:, 3:7] = [0.5, 0.5, 0.5, 0.5]
root[:, 0:2] = rng.uniform(-2, 2, (n, 2))
q, qd = rng.normal(0, 0.1, (n, 69)), np.zeros((n, 69))
nb = ms.nb
V = np.asarray(verts, np.float64).reshape(nb, -1, 3); nv = np.asarray(mod["nverts"])
for s in range(70):
    a = rng.uniform(-1, 1, (n, 69))
    tar = np.clip(a, q - 0.5 * np.pi, q + 0.5 * np.pi)
    rb, _ = physics_ref.control_step(ms, verts, cfg, root, q, qd, tar, None)
    if s % 5 == 4:
        pen = np.zeros((n, nb), int)
        for b in range(nb):
            R = Rotation.from_quat(rb[:, b, 3:7]).as_matrix()
            z = rb[:, b, 2:3] + np.einsum("nk,vk->nv", R[:, 2, :], V[b, :nv[b]])
            pen[:, b] = (z < 0).sum(1)
        nbod = (pen > 0).sum(1); mx = pen.max(1); tot = pen.sum(1)
        # serial cost model per substep with 8 lanes per env: chunks of 8 bodies, each chunk costs its max vertex count
        cost8 = np.array([sum(sorted(p[p > 0], reverse=True)[i] for i in range(0, (p > 0).sum(), 8)) if (p > 0).any() else 0 for p in pen])
        print(f"step {s+1:2d}: fallen {np.mean(rb[:,0,2]<0.5):.2f}  bodies in contact mean {nbod.mean():.1f} p99 {np.percentile(nbod,99):.0f} max {nbod.max()}  "
              f"max verts/body mean {mx.mean():.1f} p99 {np.percentile(mx,99):.0f} max {mx.max()}  total verts mean {tot.mean():.1f} max {tot.max()}  serial-8 cost mean {cost8.mean():.1f} p99 {np.percentile(cost8,99):.0f} max {cost8.max()}")
