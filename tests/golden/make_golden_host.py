"""Generates the fixtures of the host tests that compare with the reference (tests/test_host.py); needs the reference checkout
(V2P_REFERENCE).  Run from the repository root: python tests/golden/make_golden_host.py
  poselib_quat.npz        poselib's rotation3d quat_mul / quat_conjugate / quat_from_angle_axis / quat_rotate on seeded inputs
  mjcf_amass_v1.npz       the reference's smpl_mesh_humanoid_amass_v1 MJCF and the STL meshes it names (relative paths kept), the input
                          of model_compiler.compile_mjcf
  ref_motion_lib.pth      a reference `torch.save(motion_lib)` pickle (utils.motion_lib.MotionLib built from make_golden.small_lib())
  ref_motion_lib_flat.npz the FlatMotionLib arrays that pickle was built from"""
import os
import sys
import xml.etree.ElementTree as ET

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)
import _refenv  # noqa: E402

REF = _refenv.REF


def poselib_quat():
    sys.path.insert(0, os.path.join(REF, "poselib"))
    from poselib.core import rotation3d as P
    g = torch.Generator().manual_seed(0)
    a = torch.nn.functional.normalize(torch.randn(64, 4, generator=g), dim=-1)
    b = torch.nn.functional.normalize(torch.randn(64, 4, generator=g), dim=-1)
    v = torch.randn(64, 3, generator=g)
    ang = torch.rand(64, generator=g) * 6 - 3
    out = dict(a=a, b=b, v=v, ang=ang, quat_mul=P.quat_mul(a, b), quat_conjugate=P.quat_conjugate(a),
               quat_from_angle_axis=P.quat_from_angle_axis(ang, v), quat_rotate=P.quat_rotate(a, v))
    np.savez_compressed(os.path.join(HERE, "poselib_quat.npz"), **{k: t.numpy() for k, t in out.items()})


def mjcf():
    xml = os.path.join(REF, "embodied_pose", "data", "assets", "mjcf", "smpl_mesh_humanoid_amass_v1.xml")
    names, blobs = ["mjcf/smpl_mesh_humanoid_amass_v1.xml"], [open(xml, "rb").read()]
    for m in ET.parse(xml).getroot().findall("asset/mesh"):
        rel = os.path.normpath(os.path.join("mjcf", m.get("file")))
        names.append(rel)
        blobs.append(open(os.path.join(os.path.dirname(os.path.dirname(xml)), rel), "rb").read())
    np.savez_compressed(os.path.join(HERE, "mjcf_amass_v1.npz"), names=np.array(names),
                        **{f"blob{i}": np.frombuffer(b, np.uint8) for i, b in enumerate(blobs)})


def motion_lib_pickle():
    import make_golden as G
    from vid2player3d_b200.motion_lib import FlatMotionLib
    model, flat, key = G.small_lib()
    ml = G.make_ref_motion_lib(flat, key, model["dof_body_ids"])
    torch.save(ml, os.path.join(HERE, "ref_motion_lib.pth"))
    np.savez_compressed(os.path.join(HERE, "ref_motion_lib_flat.npz"), **{k: np.asarray(getattr(flat, k)) for k in FlatMotionLib.FIELDS})


if __name__ == "__main__":
    poselib_quat()
    mjcf()
    motion_lib_pickle()
