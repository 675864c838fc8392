"""CPU-side checks: C ABI exports, struct layouts, shim cross-checks, model compiler, host logic."""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import golden

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    from vid2player3d_b200 import build, native
    lib = build.build()
    from vid2player3d_b200 import native_v2p
    from vid2player3d_b200 import ball_gen
    hdr = "".join(open(os.path.join(ROOT, "include", h)).read() for h in ("b200env.h", "b200env_v2p.h", "b200ball.h"))
    declared = sorted(set(re.findall(r"\b(b200(?:env|v2p|ball)_[a-z_0-9]+)\s*\(", hdr)))
    assert declared == sorted(native.SYMBOLS + native_v2p.SYMBOLS + ball_gen.SYMBOLS)
    L = C.CDLL(lib)  # loads without a GPU; no compute call is made here
    for name in declared:
        assert hasattr(L, name), name
    from vid2player3d_b200 import abi
    assert L.b200env_abi_version() == abi.ABI_VERSION


def test_struct_layouts_match_header(tmp_path):
    from vid2player3d_b200 import abi
    src = tmp_path / "sz.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "%s/include/b200env.h"\n'
                   'int main(){printf("%%zu %%zu %%zu %%zu %%zu %%zu\\n",sizeof(b200_model_t),sizeof(b200_cfg_t),'
                   'sizeof(b200_motion_lib_t),sizeof(b200_buffers_t),offsetof(b200_model_t,kp),offsetof(b200_cfg_t,key_body));}' % ROOT)
    exe = tmp_path / "sz"
    subprocess.check_call(["gcc", str(src), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    want = [C.sizeof(abi.Model), C.sizeof(abi.Cfg), C.sizeof(abi.MotionLibView), C.sizeof(abi.Buffers), abi.Model.kp.offset,
            abi.Cfg.key_body.offset]
    assert got == want
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "%s/include/b200env_v2p.h"\n'
                   'int main(){printf("%%zu %%zu %%zu %%zu %%zu %%zu %%zu %%zu\\n",sizeof(b200v2p_state_t),sizeof(b200v2p_ctrl_t),'
                   'offsetof(b200v2p_state_t,root_pos),offsetof(b200v2p_ctrl_t,est_x),sizeof(b200v2p_treset_t),sizeof(b200v2p_areset_t),'
                   'offsetof(b200v2p_treset_t,swing_type_cycle),offsetof(b200v2p_areset_t,terminate_buf));}' % ROOT)
    subprocess.check_call(["gcc", str(src), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert got == [C.sizeof(abi.V2PState), C.sizeof(abi.V2PCtrl), abi.V2PState.root_pos.offset, abi.V2PCtrl.est_x.offset,
                   C.sizeof(abi.V2PTaskReset), C.sizeof(abi.V2PActorReset), abi.V2PTaskReset.swing_type_cycle.offset,
                   abi.V2PActorReset.terminate_buf.offset]


def test_no_gpu_means_loud_failure():
    """the product path has no CPU fallback: creating an env without a CUDA device raises"""
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from vid2player3d_b200 import abi, model_compiler, native
    mod = model_compiler.load_compiled("smpl_mesh_humanoid_amass_v1")
    m, v = abi.pack_model(mod, 1.0)
    with pytest.raises(RuntimeError, match="no CUDA device|CUDA error"):
        native.Env(m, v, abi.make_cfg(mod), 4, 0)
    from vid2player3d_b200.tasks import BaseTask
    with pytest.raises(RuntimeError, match="CUDA device only"):
        BaseTask({"device_type": "cpu", "headless": True, "env": {"numEnvs": 1}})


def test_shim_quaternion_helpers_match_poselib_conventions():
    """the only foreign arithmetic of the oracle (isaacgym.torch_utils) is cross-checked against the reference's own poselib
    definitions (their outputs on seeded inputs, tests/golden/poselib_quat.npz from make_golden_host.py) and against closed forms"""
    import sys
    sys.path.insert(0, os.path.join(ROOT, "vid2player3d_b200", "shim"))
    from isaacgym import torch_utils as IG
    g = torch.Generator().manual_seed(0)
    a = torch.nn.functional.normalize(torch.randn(64, 4, generator=g), dim=-1)
    b = torch.nn.functional.normalize(torch.randn(64, 4, generator=g), dim=-1)
    v = torch.randn(64, 3, generator=g)
    P = {k: torch.from_numpy(x) for k, x in golden("poselib_quat.npz").items()}
    assert torch.equal(P["a"], a) and torch.equal(P["b"], b) and torch.equal(P["v"], v)
    assert torch.allclose(IG.quat_mul(a, b), P["quat_mul"], atol=1e-6)
    assert torch.allclose(IG.quat_conjugate(a), P["quat_conjugate"])
    ang = P["ang"]
    assert torch.allclose(IG.quat_from_angle_axis(ang, v), P["quat_from_angle_axis"], atol=1e-6)
    assert torch.allclose(IG.quat_rotate(a, v), P["quat_rotate"], atol=1e-5)
    # closed forms
    ident = torch.tensor([[0.0, 0, 0, 1]]).repeat(64, 1)
    assert torch.allclose(IG.quat_mul(a, IG.quat_conjugate(a)), ident, atol=1e-6)
    assert torch.allclose(IG.quat_rotate(a, v).norm(dim=-1), v.norm(dim=-1), atol=1e-5)
    assert torch.allclose(IG.normalize_angle(torch.tensor([3.5, -3.5, 0.1])), torch.tensor([3.5 - 2 * np.pi, 2 * np.pi - 3.5, 0.1]), atol=1e-6)


def test_compiled_models():
    from vid2player3d_b200 import abi, model_compiler
    m = model_compiler.load_compiled("smpl_mesh_humanoid_amass_v1")
    assert len(m["parent"]) == 24 and len(m["kp"]) == 69
    assert m["parent"].tolist() == [-1, 0, 1, 2, 3, 0, 5, 6, 7, 0, 9, 10, 11, 12, 11, 14, 15, 16, 17, 11, 19, 20, 21, 22]
    assert abs(m["mass"].sum() - 102.418) < 0.01  # SURVEY.md 7 sanity value
    f = model_compiler.load_compiled("smpl_mesh_humanoid_federer")
    assert len(f["parent"]) == 25 and f["fixed"][-1] == 1 and str(f["body_names"][-1]) == "Racket"
    assert abs(f["dyn_mass"].sum() - f["mass"].sum()) < 1e-9 and f["dyn_mass"][-1] == 0
    ms, verts = abi.pack_model(f, 1.0)
    assert ms.nb == 25 and ms.vmax % 4 == 0 and verts.shape == (25, ms.vmax, 3)
    # principal inertias positive, triangle inequality
    for I in m["inertia"]:
        w = np.linalg.eigvalsh(I)
        assert w.min() > 0 and w[0] + w[1] >= w[2] * (1 - 1e-9)


def test_hull_faces_of_compiled_models_are_closed_outward_meshes():
    """abi.pack_faces (b200env_set_hull_faces): every body's faces form a closed triangle mesh (Euler: F = 2V' - 4 over the vertices
    used), every hull vertex satisfies every plane, normals point away from the centroid; the body permutation of a left-handed
    asset carries the faces with it"""
    from vid2player3d_b200 import abi, model_compiler
    for name in ("smpl_mesh_humanoid_amass_v1", "smpl_mesh_humanoid_nadal"):
        mod = model_compiler.canonical_racket_last(model_compiler.load_compiled(name))
        ms, verts = abi.pack_model(mod, 1.0)
        planes, tris, ntris, tmax = abi.pack_faces(mod, verts)
        assert planes.shape == (ms.nb, tmax, 4) and tris.shape == (ms.nb, tmax, 4) and tmax <= 255
        for b in range(ms.nb):
            nv, nt = int(ms.nverts[b]), int(ntris[b])
            if nv == 0:
                assert nt == 0                                                   # the welded racket has no hull (prims instead)
                continue
            assert nt >= 4
            T = tris[b, :nt, :3].astype(int)
            assert T.max() < nv
            used = np.unique(T)
            edges = {}
            for t in T:
                for i in range(3):
                    e = (t[i], t[(i + 1) % 3])
                    edges[e] = edges.get(e, 0) + 1
            assert all(c == 1 for c in edges.values()) and all((e[1], e[0]) in edges for e in edges)   # oriented, closed, manifold
            assert nt == 2 * len(used) - 4
            V = verts[b, :nv].astype(np.float64)
            sd = V @ planes[b, :nt, :3].T.astype(np.float64) - planes[b, :nt, 3]
            assert sd.max() < 1e-6
            cen = V[used].mean(0)
            assert ((cen @ planes[b, :nt, :3].T - planes[b, :nt, 3]) < 0).all()
            np.testing.assert_allclose(np.linalg.norm(planes[b, :nt, :3], axis=1), 1.0, atol=1e-6)


def test_left_handed_asset_in_canonical_order():
    """nadal (Racket welded to L_Wrist, body 19) -> right-handed body order; head slab normal = the semi_western grip normal"""
    from vid2player3d_b200 import abi, model_compiler, native_v2p
    raw = model_compiler.load_compiled("smpl_mesh_humanoid_nadal")
    fed = model_compiler.load_compiled("smpl_mesh_humanoid_federer")
    m = model_compiler.canonical_racket_last(raw)
    assert [str(x) for x in m["body_names"]] == [str(x) for x in fed["body_names"]]
    assert int(m["parent"][24]) == 17 and int(fed["parent"][24]) == 22 and int(m["fixed"][24]) == 1
    assert np.isclose(m["mass"].sum(), raw["mass"].sum()) and np.isclose(m["dyn_mass"].sum(), raw["dyn_mass"].sum())
    assert np.array_equal(m["dof_of_body"][:24], fed["dof_of_body"][:24])          # DOF order untouched
    assert model_compiler.canonical_racket_last(fed) is fed
    h = abi.racket_head_from_prims(m)
    x, y, z, w = h["racket_head_quat"]
    normal = np.array([2 * (x * y - z * w), 1 - 2 * (x * x + z * z), 2 * (y * z + x * w)])   # R(q) e_y
    np.testing.assert_allclose(normal, native_v2p.GRIP_NORMAL['semi_western'], atol=1e-12)
    np.testing.assert_allclose(abi.racket_head_from_prims(fed)["racket_head_quat"], (0, 0, 0, 1), atol=1e-12)
    cfg = abi.make_cfg(m, ball={}, task_mode=1, pd_mode=1)
    assert cfg.racket_body == 24 and abs(cfg.racket_head_halfthick - 0.015 * 2 ** 0.5) < 1e-6


def test_model_compiler_reproduces_committed_blob(tmp_path):
    """the reference's MJCF + STL meshes (tests/golden/mjcf_amass_v1.npz) compile to the committed model blob"""
    from vid2player3d_b200 import model_compiler
    z = golden("mjcf_amass_v1.npz")
    for i, name in enumerate(z["names"]):
        f = tmp_path / str(name)
        f.parent.mkdir(parents=True, exist_ok=True)
        f.write_bytes(z[f"blob{i}"].tobytes())
    ref = str(tmp_path / str(z["names"][0]))
    a = model_compiler.compile_mjcf(ref)
    b = model_compiler.load_compiled("smpl_mesh_humanoid_amass_v1")
    for k in ("mass", "com", "inertia", "verts", "kp", "limits", "offset"):
        np.testing.assert_allclose(a[k], b[k], atol=1e-12)


def test_synthetic_motion_lib_is_consistent():
    """FK consistency of the synthetic MoCap buffer: grs/gts follow from lrs and the skeleton"""
    from vid2player3d_b200 import model_compiler, motion_lib
    from oracle import ref_port as R
    m = model_compiler.load_compiled("smpl_mesh_humanoid_amass_v1")
    flat = motion_lib.synthetic(m, num_motions=3, num_frames=20, seed=1, ragged=True)
    assert flat.length_starts.tolist() == [0] + np.cumsum(flat.num_frames)[:-1].tolist()
    assert flat.gts.shape[0] == flat.num_frames.sum()
    np.testing.assert_allclose(np.linalg.norm(flat.grs, axis=-1), 1, atol=1e-6)
    f = 7
    for b in range(1, 24):
        p = m["parent"][b]
        want = R.quat_mul(flat.grs[f, p].astype(np.float64), flat.lrs[f, b].astype(np.float64))
        np.testing.assert_allclose(want, flat.grs[f, b], atol=1e-5)
        np.testing.assert_allclose(flat.gts[f, p] + R.my_quat_rotate(flat.grs[f, p].astype(np.float64), m["offset"][b]),
                                   flat.gts[f, b], atol=1e-5)


def test_physics_oracle_invariants():
    """float64 restatement: momentum drift is O(h) (refining the step shrinks it), weight is carried at rest"""
    from vid2player3d_b200 import abi, model_compiler
    from oracle import physics_ref as P
    mod = model_compiler.load_compiled("smpl_mesh_humanoid_amass_v1")
    rng = np.random.default_rng(0)
    drift = []
    for substeps in (2, 20):
        md = dict(mod); md["armature"] = np.zeros(69)
        m0, verts = abi.pack_model(md, 0.0)
        cfg0 = abi.make_cfg(mod, gravity_z=0.0, ang_damping=0.0, substeps=substeps)
        root = np.zeros((1, 13)); root[:, 2] = 5; root[:, 6] = 1; root[:, 7:10] = [1, 0.5, 0.2]; root[:, 10:13] = [0.5, -1, 2]
        rs = np.random.default_rng(1)
        q = rs.normal(0, 0.3, (1, 69)); qd = rs.normal(0, 2, (1, 69)); tar = np.zeros((1, 69))
        d0 = P.diagnostics(m0, cfg0, root[0], q[0], qd[0])
        P.control_step(m0, verts, cfg0, root, q, qd, tar, n_steps=15)
        d1 = P.diagnostics(m0, cfg0, root[0], q[0], qd[0])
        drift.append(max(np.abs(d1["P"] - d0["P"]).max(), np.abs(d1["L"] - d0["L"]).max()))
    assert drift[1] < 0.2 * drift[0]
    # lying drop (config 1) comes to rest carrying its weight
    m, verts = abi.pack_model(mod, mod["mass"].sum() / 90.0)
    cfg = abi.make_cfg(mod)
    root = np.zeros((1, 13)); root[0, 2] = 0.89; root[0, 6] = 1
    q = np.zeros((1, 69)); qd = np.zeros((1, 69)); tar = np.zeros((1, 69))
    rb, cf = P.control_step(m, verts, cfg, root, q, qd, tar, n_steps=60)
    assert abs(cf[0, :, 2].sum() - mod["mass"].sum() * 9.81) < 2.0
    assert np.abs(qd).max() < 0.05 and abs(root[0, 9]) < 1e-3


def test_vec_task_and_parse_task_surface():
    from vid2player3d_b200.tasks import parse_task as pt
    with pytest.raises(Exception, match="Unrecognized task"):
        class A:  # noqa: D401
            task = "Nope"; device_id = 0; rl_device = "cpu"; physics_engine = 1; device = "cuda"; headless = True
        pt(A, {"env": {}}, {}, None)


def test_flat_motion_library_file_roundtrip(tmp_path):
    """SURVEY.md 8f-3: the mmap-able on-disk MoCap format holds exactly the arrays the sampler reads"""
    from vid2player3d_b200 import model_compiler, motion_lib
    model = model_compiler.load_compiled("smpl_mesh_humanoid_amass_v1")
    flat = motion_lib.synthetic(model, num_motions=5, num_frames=40, seed=3, ragged=True)
    path = str(tmp_path / "lib.b200ml")
    flat.save_flat(path)
    for mm in (True, False):
        back = motion_lib.FlatMotionLib.load_flat(path, mmap=mm)
        for k in motion_lib.FlatMotionLib.FIELDS:
            a, b = getattr(flat, k), getattr(back, k)
            assert a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a, b), k
    assert isinstance(back.gts, np.ndarray) and motion_lib.FlatMotionLib.load_any(path).num_motions() == 5
    assert os.path.getsize(path) % 64 == 0
    flat.save(str(tmp_path / "lib.npz"))
    assert np.array_equal(motion_lib.FlatMotionLib.load_any(str(tmp_path / "lib.npz")).dvs, flat.dvs)
    (tmp_path / "bad.b200ml").write_bytes(b"not a library" * 4)
    with pytest.raises(ValueError, match="not a B200ML01"):
        motion_lib.FlatMotionLib.load_flat(str(tmp_path / "bad.b200ml"))


def test_quaternion_to_angle_axis_matches_scipy():
    """torch_ops.quaternion_wxyz_to_angle_axis (the ceres formula of konia_transform.py:558-628, test-time `_joint_rot` export)"""
    from scipy.spatial.transform import Rotation
    from vid2player3d_b200.torch_ops import quaternion_wxyz_to_angle_axis
    rng = np.random.default_rng(0)
    q = rng.normal(size=(256, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    q[0] = [1, 0, 0, 0]
    got = quaternion_wxyz_to_angle_axis(torch.tensor(q)).numpy()
    want = Rotation.from_quat(q[:, [1, 2, 3, 0]]).as_rotvec()
    # q and -q are the same rotation: the formula keeps the angle in (-pi, pi] like the reference
    assert np.abs(got - want).max() < 1e-9
    assert np.all(got[0] == 0)


def test_nn_library_exports_and_layout(tmp_path):
    """libb200nn.so (include/b200nn.h): loads without a GPU, exports every declared symbol, descriptor layout == ctypes mirror,
    and refuses to build a layer without a CUDA device (no fallback)."""
    from vid2player3d_b200 import build, nn
    build.build()
    hdr = open(os.path.join(ROOT, "include", "b200nn.h")).read()
    declared = sorted(set(re.findall(r"\b(b200nn_[a-z_0-9]+)\s*\(", hdr)))
    assert declared == sorted(nn.SYMBOLS)
    L = nn.lib()
    for name in declared:
        assert hasattr(L, name), name
    src = tmp_path / "sz.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "%s/include/b200nn.h"\n'
                   'int main(){printf("%%zu %%zu %%zu\\n",sizeof(b200nn_linear_desc_t),offsetof(b200nn_linear_desc_t,out),'
                   'offsetof(b200nn_linear_desc_t,k_padded));}' % ROOT)
    exe = tmp_path / "sz"
    subprocess.check_call(["gcc", str(src), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert got == [C.sizeof(nn.LinearDesc), nn.LinearDesc.out.offset, nn.LinearDesc.k_padded.offset]
    if not torch.cuda.is_available():
        with pytest.raises(RuntimeError, match="CUDA device only"):
            nn.Linear(torch.zeros(128, 64, dtype=torch.bfloat16), torch.zeros(8, 64), torch.zeros(8), torch.zeros(128, 64, dtype=torch.bfloat16), 4)


def test_nn_linear_create_rejects_bad_descriptors():
    """b200nn_linear_create validates the descriptor before it looks up the driver, so fake (aligned, non-null, never dereferenced)
    pointers reach every rule on a machine without a GPU: each malformed descriptor returns -2 with its own message; a valid one
    gets past validation (-3 without a CUDA driver, 0 with one)."""
    from vid2player3d_b200 import build, nn
    build.build()
    L = nn.lib()

    def desc(**kw):
        d = dict(a=0x10000, lda=128, w=0x20000, ldw=128, bias=0x30000, coef=0x40000, out=0x50000, ldo=256, out_col0=0, rows=200, n=100,
                 n_padded=128, k_padded=128, num_experts=1, act=1, out_bf16=1, out_min=0.0, out_max=0.0)
        d.update(kw)
        return nn.LinearDesc(**d)

    def create(d):
        h = C.c_void_p()
        rc = L.b200nn_linear_create(C.byref(d), C.c_int32(0), C.byref(h))
        if h:
            L.b200nn_linear_destroy(h)
        return rc, L.b200nn_last_error().decode()

    bad = [
        (dict(num_experts=0), "num_experts must be 1..6"),
        (dict(num_experts=7), "num_experts must be 1..6"),
        (dict(k_padded=96), "padded to multiples of 64"),
        (dict(k_padded=0), "padded to multiples of 64"),
        (dict(lda=96), "padded to multiples of 64"),
        (dict(ldw=64), "padded to multiples of 64"),              # ldw < k_padded
        (dict(n_padded=96), "n_padded must be a multiple"),
        (dict(n=0), "n_padded must be a multiple"),
        (dict(n=129), "n_padded must be a multiple"),
        (dict(num_experts=2, n_padded=48, n=40), "n_padded must be a multiple"),
        (dict(rows=0), "rows < 1"),
        (dict(ldo=252), "multiples of 8"),
        (dict(out_col0=4), "multiples of 8"),
        (dict(a=0x10008), "16-byte aligned"),
        (dict(w=0x20004), "16-byte aligned"),
        (dict(out=0x50002), "16-byte aligned"),
        (dict(out_col0=-8), "out_col0 < 0"),
        (dict(out_bf16=0, out_col0=-1), "out_col0 < 0"),
        (dict(ldo=96), "ldo < out_col0 \\+ n"),
        (dict(out_col0=160), "ldo < out_col0 \\+ n"),
        (dict(out_bf16=0, ldo=103, out_col0=5, n=99), "ldo < out_col0 \\+ n"),
        (dict(act=3), "unknown activation"),
        (dict(act=-1), "unknown activation"),
    ]
    for kw, msg in bad:
        rc, err = create(desc(**kw))
        assert rc == -2 and re.search(msg, err), (kw, rc, err)
    rc, err = create(desc(num_experts=2, n_padded=32, n=32, coef=None))
    assert rc == -1 and "coefficient" in err                      # a mixture layer without its coefficients
    want = 0 if torch.cuda.is_available() else -3
    for kw in (dict(), dict(num_experts=6, n_padded=64, n=33, act=2), dict(out_bf16=0, ldo=103, out_col0=3, n=100, act=0),
               dict(out_col0=32, ldo=136, n=100, out_min=-1.0, out_max=1.0)):
        rc, err = create(desc(**kw))
        assert rc == want, (kw, rc, err)


def test_v2p_glue_struct_layouts(tmp_path):
    from vid2player3d_b200 import abi
    src = tmp_path / "sz.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "%s/include/b200env_v2p.h"\n'
                   'int main(){printf("%%zu %%zu %%zu %%zu %%zu %%zu %%zu\\n",sizeof(b200v2p_prestep_t),offsetof(b200v2p_prestep_t,actions),'
                   'sizeof(b200v2p_stream_t),offsetof(b200v2p_stream_t,ring_phase),offsetof(b200v2p_ctrl_t,advance),offsetof(b200v2p_ctrl_t,touch_mask),offsetof(b200v2p_state_t,only_mask));}' % ROOT)
    exe = tmp_path / "sz"
    subprocess.check_call(["gcc", str(src), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert got == [C.sizeof(abi.V2PPreStep), abi.V2PPreStep.actions.offset, C.sizeof(abi.V2PStream), abi.V2PStream.ring_phase.offset,
                   abi.V2PCtrl.advance.offset, abi.V2PCtrl.touch_mask.offset, abi.V2PState.only_mask.offset]


def test_motion_lib_formats_directory_and_merge(tmp_path):
    """motion_file handling of HumanoidSMPLIM._load_motion (reference humanoid_smpl_im.py:420-440): .npz / .b200ml files, a directory
    of them with motion_file_range, merge = concatenation with rebuilt frame offsets; unknown formats fail loudly"""
    from vid2player3d_b200 import model_compiler, motion_lib as ML
    model = model_compiler.load_compiled("smpl_mesh_humanoid_amass_v1")
    libs = [ML.synthetic(model, num_motions=m, num_frames=20, seed=s, ragged=True) for m, s in ((2, 1), (3, 2), (1, 3))]
    d = tmp_path / "libs"
    d.mkdir()
    for i, l in enumerate(libs):
        l.save_flat(str(d / f"part{i}.b200ml"))
    libs[0].save(str(tmp_path / "one.npz"))
    a = ML.FlatMotionLib.load_any(str(tmp_path / "one.npz"))
    assert np.array_equal(a.gts, libs[0].gts)
    merged = ML.FlatMotionLib.load_any(str(d))
    assert merged.num_motions() == 6 and merged.gts.shape[0] == sum(l.gts.shape[0] for l in libs)
    assert np.array_equal(merged.length_starts, np.concatenate([[0], np.cumsum(merged.num_frames)[:-1]]))
    assert np.array_equal(merged.gts[libs[0].gts.shape[0]:libs[0].gts.shape[0] + libs[1].gts.shape[0]], libs[1].gts)
    part = ML.FlatMotionLib.load_any(str(d), motion_file_range=[1, 3])
    assert part.num_motions() == 4 and np.array_equal(part.motion_lengths, np.concatenate([libs[1].motion_lengths, libs[2].motion_lengths]))
    bad = tmp_path / "x.bin"
    bad.write_bytes(b"not a motion library")
    with pytest.raises(ValueError, match="unknown motion library format"):
        ML.FlatMotionLib.load_any(str(bad))
    with pytest.raises(FileNotFoundError):
        ML.FlatMotionLib.load_any(str(tmp_path / "missing.pth"))
    empty = tmp_path / "empty"
    empty.mkdir()
    with pytest.raises(FileNotFoundError):
        ML.FlatMotionLib.load_any(str(empty))


def test_from_reference_motion_lib_pickle():
    """a reference `torch.save(motion_lib)` pickle (what every reference yaml's motion_file names; tests/golden/ref_motion_lib.pth from
    make_golden_host.py) loads through FlatMotionLib.load_any / from_reference to the arrays it was built from.  Run in a subprocess:
    the pickle names the reference's class utils.motion_lib.MotionLib, which torch.load must import; a stand-in module provides it."""
    code = r'''
import os, sys, types
sys.path.insert(0, %(root)r)
import numpy as np
from vid2player3d_b200.motion_lib import FlatMotionLib
utils, mlmod = types.ModuleType("utils"), types.ModuleType("utils.motion_lib")
class MotionLib:
    pass
mlmod.MotionLib, utils.motion_lib = MotionLib, mlmod
sys.modules["utils"], sys.modules["utils.motion_lib"] = utils, mlmod
back = FlatMotionLib.load_any(os.path.join(%(root)r, "tests", "golden", "ref_motion_lib.pth"))
want = np.load(os.path.join(%(root)r, "tests", "golden", "ref_motion_lib_flat.npz"))
for k in FlatMotionLib.FIELDS:
    assert np.array_equal(np.asarray(getattr(back, k)), want[k]), k
print("ok")
''' % {"root": ROOT}
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout[-1500:] + r.stderr[-2500:]
