"""The packed articulated step executed on the CPU, lane by lane (tests/emu: 32 host threads per warp, __syncwarp = barrier,
the very device code of csrc/packed*.cuh compiled as host C++, float64) vs the float64 restatement oracle/physics_ref.c.
Same check as tests/test_gpu_parity.py::test_physics_f64_matches_oracle, but it needs no GPU: a change to the lane mapping of the
kernel is debugged here first."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "emu"))
from helpers import rand_quat  # noqa: E402

from oracle import physics_ref  # noqa: E402
from vid2player3d_b200 import abi, model_compiler  # noqa: E402


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def emu_step(variant, ms, verts, cfg, root, q, qd, tar, ext, n_steps=1, ball=None, hits=None, faces=None):
    import build as emu_build
    lib = C.CDLL(emu_build.build(variant))
    if faces is not None:                                        # abi.pack_faces: exact ball / hull query
        planes, tris, ntris, tmax = faces
        lib.emu_set_hull_faces(_p(planes), _p(tris), _p(ntris), C.c_int(tmax))
    else:
        lib.emu_set_hull_faces(None, None, None, C.c_int(0))
    n = root.shape[0]
    rb = np.zeros((n, ms.nb, 13))
    cf = np.zeros((n, ms.nb, 3))
    rc = lib.emu_packed_physics(C.byref(ms), _p(np.ascontiguousarray(verts, np.float32)), C.byref(cfg), C.c_int(n), C.c_int(n_steps),
                                _p(root), _p(q), _p(qd), _p(tar), _p(ext), _p(rb), _p(cf), _p(ball), _p(hits))
    assert rc == 0
    return rb, cf


def states(n, seed, contact):
    rng = np.random.default_rng(seed)
    root = np.zeros((n, 13))
    root[:, 0:2] = rng.uniform(-3, 3, (n, 2))
    root[:, 2] = rng.uniform(0.7, 1.1, n) if contact else rng.uniform(3, 5, n)
    root[:, 3:7] = rand_quat(rng, n)
    root[: n // 2, 3:7] = [0.5, 0.5, 0.5, 0.5]
    root[:, 7:10] = rng.normal(0, 0.5, (n, 3))
    root[:, 10:13] = rng.normal(0, 1.0, (n, 3))
    q = rng.normal(0, 0.3, (n, 69))
    qd = rng.normal(0, 1.5, (n, 69))
    return root, q, qd, q + rng.normal(0, 0.2, (n, 69)), rng.normal(0, 30, (n, 6))


VARIANTS = ["packed", "packedt"] + (["packed3"] if os.path.exists(os.path.join(HERE, "..", "tools", "variants", "packed3.cuh")) else [])


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("contact", [False, True])
def test_emulated_packed_step_matches_oracle(variant, contact):
    mod = model_compiler.load_compiled("smpl_mesh_humanoid_amass_v1")
    ms, verts = abi.pack_model(mod, float(mod["mass"].sum()) / 90.0)
    cfg = abi.make_cfg(mod)
    n = 6                                                        # one full warp of envs + a ragged one
    root, q, qd, tar, ext = states(n, 11, contact)
    for steps, tol in ((1, 1e-9), (4, 1e-7)):
        r1, q1, v1 = root.copy(), q.copy(), qd.copy()
        rb1, cf1 = emu_step(variant, ms, verts, cfg, r1, q1, v1, tar.copy(), ext.copy(), steps)
        r2, q2, v2 = root.copy(), q.copy(), qd.copy()
        rb2, cf2 = physics_ref.control_step(ms, verts, cfg, r2, q2, v2, tar.copy(), ext.copy(), n_steps=steps)
        for a, b, name, sc in ((r1, r2, "root", 1), (q1, q2, "dof_pos", 1), (v1, v2, "dof_vel", 1), (rb1, rb2, "rb", 1), (cf1, cf2, "contact", 1e3)):
            np.testing.assert_allclose(a, b, rtol=0, atol=tol * sc, err_msg=f"{variant} {name} steps={steps}")
    if contact:
        assert np.abs(cf2).max() > 10.0


@pytest.mark.parametrize("variant", VARIANTS)
def test_emulated_packed_step_with_racket_and_ball(variant):
    mod = model_compiler.canonical_racket_last(model_compiler.load_compiled("smpl_mesh_humanoid_federer"))
    ms, verts = abi.pack_model(mod, float(mod["mass"].sum()) / 90.0)
    cfg = abi.make_cfg(mod, substeps=6, ball={}, task_mode=1, pd_mode=1)
    n = 5
    root, q, qd, tar, ext = states(n, 5, True)
    rng = np.random.default_rng(2)
    ball = np.zeros((n, 13))
    ball[:, 0:3] = root[:, 0:3] + rng.normal(0, 0.6, (n, 3)) + [0, 0.5, 0.3]
    ball[:, 2] = np.abs(ball[:, 2]) + 0.04
    ball[:, 7:10] = rng.normal(0, 8, (n, 3))
    ball[:, 10:13] = rng.normal(0, 40, (n, 3))
    b1, b2 = ball.copy(), ball.copy()
    h1, h2 = np.zeros(n, np.int32), np.zeros(n, np.int32)
    r1, q1, v1 = root.copy(), q.copy(), qd.copy()
    rb1, _ = emu_step(variant, ms, verts, cfg, r1, q1, v1, tar.copy(), ext.copy(), 2, b1, h1)
    r2, q2, v2 = root.copy(), q.copy(), qd.copy()
    rb2, _ = physics_ref.control_step(ms, verts, cfg, r2, q2, v2, tar.copy(), ext.copy(), n_steps=2, ball=b2, hits=h2)
    np.testing.assert_allclose(b1, b2, rtol=0, atol=1e-7)
    np.testing.assert_allclose(q1, q2, rtol=0, atol=1e-7)
    np.testing.assert_allclose(rb1, rb2, rtol=0, atol=1e-5)


@pytest.mark.parametrize("variant", VARIANTS)
def test_emulated_float32_path_config1_drop(variant):
    """BASELINE config 1 on the CPU: one humanoid in the default pose (identity root at z = 0.89), zero action, 60 control steps incl.
    the ground impact - the kernel's float32 arithmetic (128-bit record accesses, float device functions) vs the float64 restatement.
    The GPU twin (tests/test_gpu_parity.py::test_physics_f32_config1_drop) runs the same 60 steps with the MUFU reciprocals."""
    import build as emu_build
    mod = model_compiler.load_compiled("smpl_mesh_humanoid_amass_v1")
    ms, verts = abi.pack_model(mod, float(mod["mass"].sum()) / 90.0)
    cfg = abi.make_cfg(mod)
    n, steps = 3, 60
    root = np.zeros((n, 13))
    root[:, 2], root[:, 6] = 0.89, 1.0
    root[1, 0:2] = [0.4, -0.3]
    root[2, 2] = 0.95
    q, qd = np.zeros((n, 69)), np.zeros((n, 69))
    tar, ext = np.zeros((n, 69)), np.zeros((n, 6))
    r64, q64, v64 = root.copy(), q.copy(), qd.copy()
    physics_ref.control_step(ms, verts, cfg, r64, q64, v64, tar.copy(), ext.copy(), n_steps=steps)
    f = lambda a: np.ascontiguousarray(a, np.float32)  # noqa: E731
    r32, q32, v32, t32, e32 = f(root), f(q), f(qd), f(tar), f(ext)
    rb, cf = np.zeros((n, ms.nb, 13), np.float32), np.zeros((n, ms.nb, 3), np.float32)
    lib = C.CDLL(emu_build.build(variant))
    rc = lib.emu_packed_physics_f32(C.byref(ms), _p(np.ascontiguousarray(verts, np.float32)), C.byref(cfg), C.c_int(n), C.c_int(steps), _p(r32),
                                    _p(q32), _p(v32), _p(t32), _p(e32), _p(rb), _p(cf), None, None)
    assert rc == 0
    assert np.abs(q32 - q64).max() < 1e-4 and np.abs(v32 - v64).max() < 1e-3          # north_star: joint q within 1e-4
    assert np.abs(r32[:, :7] - r64[:, :7]).max() < 1e-4
    assert r64[0, 2] < 0.885 and np.abs(cf).max() > 1.0                               # it fell and touched the ground



@pytest.mark.parametrize("variant", VARIANTS)
def test_emulated_ball_body_and_handle_contacts(variant):
    """optional ball contacts (b200_cfg_t::ball_body_contact): balls thrown at the torso, at a forearm and at the racket handle of
    flying humanoids - lane emulation of the kernel code vs the float64 restatement, and the contacts really happen"""
    mod = model_compiler.canonical_racket_last(model_compiler.load_compiled("smpl_mesh_humanoid_federer"))
    ms, verts = abi.pack_model(mod, float(mod["mass"].sum()) / 90.0)
    cfg_on = abi.make_cfg(mod, substeps=6, ball={"ball_body_contact": 1}, task_mode=1, pd_mode=1)
    cfg_off = abi.make_cfg(mod, substeps=6, ball={}, task_mode=1, pd_mode=1)
    assert cfg_on.racket_handle[6] > 0 and cfg_off.ball_body_contact == 0
    names = [str(x) for x in mod["body_names"]]
    n = 6
    root, q, qd, tar, ext = states(n, 21, False)
    root[:, 2] = 2.0
    qd *= 0.2
    # body poses at the start (a control step of ~0 length through the oracle)
    tiny = abi.Cfg.from_buffer_copy(cfg_off)
    tiny.sim_dt = 1e-12
    rb, _ = physics_ref.control_step(ms, verts, tiny, root.copy(), q.copy(), qd.copy(), tar.copy(), None)
    from scipy.spatial.transform import Rotation
    rng = np.random.default_rng(3)
    ball = np.zeros((n, 13))
    targets = ["Torso", "Chest", "L_Elbow", "R_Knee", "HANDLE", "HANDLE"]
    for e, tname in enumerate(targets):
        if tname == "HANDLE":
            b = names.index("Racket")
            Rr = Rotation.from_quat(rb[e, b, 3:7]).as_matrix()
            hd = np.array(list(cfg_on.racket_handle))
            tgt = rb[e, b, 0:3] + Rr @ (0.5 * (hd[0:3] + hd[3:6]))
            direction = Rr @ np.array([0.0, 0.0, 1.0])                   # across the handle, in the plane of the string bed
        else:
            b = names.index(tname)
            Rb = Rotation.from_quat(rb[e, b, 3:7]).as_matrix()
            tgt = rb[e, b, 0:3] + Rb @ np.asarray(mod["com"][b])
            direction = rng.normal(size=3)
            direction /= np.linalg.norm(direction)
        ball[e, 0:3] = tgt + 0.12 * direction
        ball[e, 7:10] = rb[e, b, 7:10] - 12.0 * direction                  # 12 m/s towards the target: 3.3 cm per substep
        ball[e, 10:13] = rng.normal(0, 20, 3)
    outs = {}
    faces = abi.pack_faces(mod, verts)
    assert faces[2][names.index("Chest")] > 8 and faces[2][names.index("Racket")] == 0
    # "on": exact sphere / convex-hull query (hull faces installed on both sides); "approx": no faces - spheres on the hull vertices
    for name, cfg, fc in (("on", cfg_on, faces), ("approx", cfg_on, None), ("off", cfg_off, None)):
        b1, b2 = ball.copy(), ball.copy()
        h1, h2 = np.zeros(n, np.int32), np.zeros(n, np.int32)
        r1, q1, v1 = root.copy(), q.copy(), qd.copy()
        emu_step(variant, ms, verts, cfg, r1, q1, v1, tar.copy(), ext.copy(), 1, b1, h1, faces=fc)
        r2, q2, v2 = root.copy(), q.copy(), qd.copy()
        if fc is not None:
            physics_ref.set_hull_faces(*fc)
        try:
            physics_ref.control_step(ms, verts, cfg, r2, q2, v2, tar.copy(), ext.copy(), n_steps=1, ball=b2, hits=h2)
        finally:
            physics_ref.clear_hull_faces()
        np.testing.assert_allclose(b1, b2, rtol=0, atol=1e-8, err_msg=name)
        np.testing.assert_allclose(q1, q2, rtol=0, atol=1e-9, err_msg=name)
        outs[name] = b2
    dv = np.linalg.norm(outs["on"][:, 7:10] - outs["off"][:, 7:10], axis=1)
    assert (dv > 3.0).sum() >= 5, dv                                        # the ball bounced off the bodies / the handle
    assert np.isfinite(outs["on"]).all()
    # the exact surface and the vertex-sphere approximation differ (the approximation bulges by up to the vertex radius)
    assert np.abs(outs["on"][:4] - outs["approx"][:4]).max() > 1e-4


def test_compacted_contact_phase_is_bit_identical():
    """-DPK_CONTACT_COMPACT=1 (pk_contact_phase: bodies in contact compacted per env group, one lane per body) must reproduce the
    in-place form bit for bit - float64 and float32 - on humanoids in natural ground contact over several control steps"""
    import build as emu_build
    mod = model_compiler.load_compiled("smpl_mesh_humanoid_amass_v1")
    ms, verts = abi.pack_model(mod, float(mod["mass"].sum()) / 90.0)
    cfg = abi.make_cfg(mod)
    n = 9
    root, q, qd, tar, ext = states(n, 31, True)
    ext[:] = 0
    root[:, 3:7] = [0.5, 0.5, 0.5, 0.5]
    rng = np.random.default_rng(2)
    for _ in range(35):                                           # let them fall: the restatement brings them to the ground
        tar = np.clip(rng.uniform(-1, 1, (n, 69)), q - 0.5 * np.pi, q + 0.5 * np.pi)
        physics_ref.control_step(ms, verts, cfg, root, q, qd, tar, None)
    assert (root[:, 2] < 0.5).sum() >= 6                          # lying humanoids: many bodies in contact, uneven vertex counts
    res = {}
    for tag, flags in (("plain", ()), ("compact", ("-DPK_CONTACT_COMPACT=1",))):
        lib = C.CDLL(emu_build.build("packed", flags))
        r, qq, vv = root.copy(), q.copy(), qd.copy()
        rb, cf = np.zeros((n, ms.nb, 13)), np.zeros((n, ms.nb, 3))
        assert lib.emu_packed_physics(C.byref(ms), _p(np.ascontiguousarray(verts, np.float32)), C.byref(cfg), C.c_int(n), C.c_int(3), _p(r), _p(qq),
                                      _p(vv), _p(tar.copy()), _p(ext.copy()), _p(rb), _p(cf), None, None) == 0
        f = lambda a: np.ascontiguousarray(a, np.float32)  # noqa: E731
        r32, q32, v32 = f(root), f(q), f(qd)
        rb32, cf32 = np.zeros((n, ms.nb, 13), np.float32), np.zeros((n, ms.nb, 3), np.float32)
        assert lib.emu_packed_physics_f32(C.byref(ms), _p(np.ascontiguousarray(verts, np.float32)), C.byref(cfg), C.c_int(n), C.c_int(3), _p(r32),
                                          _p(q32), _p(v32), _p(f(tar)), _p(f(ext)), _p(rb32), _p(cf32), None, None) == 0
        res[tag] = (r, qq, vv, rb, cf, r32, q32, v32, rb32, cf32)
    for a, b in zip(res["plain"], res["compact"]):
        assert np.array_equal(a, b)
    assert (np.abs(res["plain"][4]).sum(-1) > 0).sum() >= 8       # bodies really were in contact (the last substep's contact forces)
    r2, q2, v2 = root.copy(), q.copy(), qd.copy()
    physics_ref.control_step(ms, verts, cfg, r2, q2, v2, tar.copy(), ext.copy(), n_steps=3)
    np.testing.assert_allclose(res["compact"][1], q2, rtol=0, atol=1e-7)


def _emu_f32(variant, flags, ms, verts, cfg, root, q, qd, tar, ext, steps):
    import build as emu_build
    lib = C.CDLL(emu_build.build(variant, flags))
    lib.emu_set_hull_faces(None, None, None, C.c_int(0))
    n = root.shape[0]
    rb = np.zeros((n, ms.nb, 13), np.float32)
    cf = np.zeros((n, ms.nb, 3), np.float32)
    rc = lib.emu_packed_physics_f32(C.byref(ms), _p(np.ascontiguousarray(verts, np.float32)), C.byref(cfg), C.c_int(n), C.c_int(steps),
                                    _p(root), _p(q), _p(qd), _p(tar), _p(ext), _p(rb), _p(cf), None, None)
    assert rc == 0
    return root, q, qd, rb, cf


@pytest.mark.parametrize("flags", [(), ("-DPT_CX=1",), ("-DPT_CONTACT_COMPACT=0",)], ids=["compact", "overflow", "inplace"])
@pytest.mark.parametrize("asset", ["smpl_mesh_humanoid_amass_v1", "smpl_mesh_humanoid_federer"])
def test_one_wave_form_is_bit_identical_to_packed_in_float32(asset, flags):
    """csrc/packed_t.cuh (owner lanes, private store, mailbox hand-over, compacted contact through the mailbox entries - also with one entry
    only, so that the in-place overflow path runs, and with the in-place contact) runs the operations of csrc/packed.cuh in the same
    order: in float32 emulation (no FMA contraction on the host) every output is bit-identical, 3 control steps with ground contact."""
    mod = model_compiler.canonical_racket_last(model_compiler.load_compiled(asset))
    ms, verts = abi.pack_model(mod, float(mod["mass"].sum()) / 90.0)
    cfg = abi.make_cfg(mod)
    st = [a.astype(np.float32) for a in states(10, 5, True)]
    ref = _emu_f32("packed", (), ms, verts, cfg, *[a.copy() for a in st], 3)
    got = _emu_f32("packedt", flags, ms, verts, cfg, *[a.copy() for a in st], 3)
    for a, b, name in zip(ref, got, ("root", "dof_pos", "dof_vel", "rigid bodies", "contact forces")):
        assert np.array_equal(a, b), name
    assert np.abs(ref[4]).max() > 10.0


def _pt_tables(ms):
    import build as emu_build
    lib = C.CDLL(emu_build.build("packedt"))
    MB, LV, SL = 32, 16, 8
    blk, slot, mbox = (np.zeros(MB, np.int8) for _ in range(3))
    body, lvl, lblk = np.zeros((3, SL), np.int8), np.zeros((LV, SL), np.int8), np.zeros(LV, np.int8)
    nm = C.c_int32(0)
    ok = lib.emu_pt_tables(C.byref(ms), _p(blk), _p(slot), _p(body), _p(lvl), _p(lblk), _p(mbox), C.byref(nm))
    return ok, blk, slot, body, lvl, lblk, mbox, nm.value


@pytest.mark.parametrize("asset", ["smpl_mesh_humanoid_amass_v1", "smpl_mesh_humanoid_federer", "smpl_mesh_humanoid_djokovic", "smpl_mesh_humanoid_nadal"])
def test_owner_slot_tables_of_the_one_wave_form(asset):
    """csrc/dyn_common.cuh::build_pt_tables: every dynamic body has one (block, slot) of its own; the bodies of a tree depth share a block
    (one warp-uniform private-store column block per level pass) and sit in different slots; a welded body has a lane at its depth but no block; the
    mailbox rank of a body is its rank among the dynamic bodies of its depth"""
    mod = model_compiler.canonical_racket_last(model_compiler.load_compiled(asset))
    ms, _ = abi.pack_model(mod, float(mod["mass"].sum()) / 90.0)
    ok, blk, slot, body, lvl, lblk, mbox, nm = _pt_tables(ms)
    assert ok == 1
    nb, depth, fixed = ms.nb, list(ms.depth)[:ms.nb], list(ms.fixed)[:ms.nb]
    seen = set()
    for b in range(nb):
        d = depth[b]
        assert 0 <= slot[b] < 8 and lvl[d][slot[b]] == b
        if fixed[b]:
            assert blk[b] == -1
            continue
        assert 0 <= blk[b] < 3 and blk[b] == lblk[d] and body[blk[b]][slot[b]] == b
        assert (blk[b], slot[b]) not in seen
        seen.add((blk[b], slot[b]))
        assert mbox[b] == sum(1 for c in range(b) if depth[c] == d and not fixed[c])
    assert len(seen) == sum(1 for b in range(nb) if not fixed[b])
    for d in range(16):
        on = [lvl[d][s] for s in range(8) if lvl[d][s] >= 0]
        assert sorted(on) == [b for b in range(nb) if depth[b] == d]
    assert nm == max(sum(1 for b in range(nb) if depth[b] == d and not fixed[b]) for d in range(1, 16))


def test_owner_slot_tables_reject_a_tree_that_does_not_fit():
    """a tree with 11 jointed bodies at one depth: more than the 8 lane slots of an env's group -> pt_ok = 0 (b200env_create then keeps
    the two-round packed kernel)"""
    mod = model_compiler.load_compiled("smpl_mesh_humanoid_amass_v1")
    ms, _ = abi.pack_model(mod, float(mod["mass"].sum()) / 90.0)
    import copy
    m2 = copy.deepcopy(ms)
    m2.nb = 26
    for b in range(26):
        m2.parent[b] = b - 1
        m2.depth[b] = b if b < 16 else 15          # 16 depths are what the tables hold; bodies 15.. share the last one
        m2.fixed[b] = 0
    ok = _pt_tables(m2)[0]
    assert ok == 0


@pytest.mark.parametrize("form", [0, 1], ids=["one_lane", "eight_lanes"])
def test_hull_query_of_the_kernels_matches_the_restatement(form):
    """csrc/dyn_common.cuh::hull_sphere (one lane walks the hull, four faces per iteration, nearest-face shortcut) and hull_sphere_coop (the
    hull's faces over the 8 lanes of an env's group: ballot for the separating plane, shuffle reductions with the serial tie rule) in
    float64 on the lane emulator against oracle/physics_ref.c::hull_sphere_ref, which walks every face: hit / miss identical, depth and
    normal to 1e-12, on points inside the hull, just outside faces, near edges and vertices, and far away"""
    import build as emu_build
    from oracle import physics_ref as P
    mod = model_compiler.load_compiled("smpl_mesh_humanoid_amass_v1")
    ms, verts = abi.pack_model(mod, 1.0)
    planes, tris, ntris, tmax = abi.pack_faces(mod, verts)
    lib = C.CDLL(emu_build.build("packedt"))
    lib.emu_set_hull_faces(_p(planes), _p(tris), _p(ntris), C.c_int(tmax))
    P.set_hull_faces(planes, tris, ntris, tmax)
    rng = np.random.default_rng(4)
    R = 0.032
    try:
        seen = {"inside": 0, "contact": 0, "miss": 0}
        for b in (0, 4, 9, 13, 18, 23):
            nv = int(mod["nverts"][b])
            V = verts[b, :nv].astype(np.float64)
            ctr, ext = V.mean(0), np.ptp(V, axis=0).max()
            pts = [ctr + rng.normal(size=3) * ext * sc for sc in (0.1, 0.3, 0.45, 0.6) for _ in range(10)]
            pts += [V[i] + rng.normal(size=3) * 0.01 for i in rng.integers(0, nv, 12)]                       # near vertices
            pts += [0.5 * (V[i] + V[j]) + rng.normal(size=3) * 0.01 for i, j in rng.integers(0, nv, (12, 2))]   # near edges / through the hull
            pts = np.ascontiguousarray(np.array(pts))
            n = len(pts)
            hit, pen, nl = np.zeros(n, np.int32), np.zeros(n), np.zeros((n, 3))
            rc = lib.emu_hull_sphere(C.byref(ms), _p(np.ascontiguousarray(verts, np.float32)), C.c_int(b), C.c_int(form), C.c_int(n), _p(pts),
                                     C.c_double(R), _p(hit), _p(pen), _p(nl))
            assert rc == 0
            for i in range(n):
                h0, p0, n0 = P.hull_sphere(ms, verts, b, pts[i], R)
                assert hit[i] == h0, (b, i)
                if h0:
                    assert abs(pen[i] - p0) < 1e-12 and np.abs(nl[i] - n0).max() < 1e-9, (b, i, pen[i], p0)
                    seen["inside" if p0 >= R else "contact"] += 1
                else:
                    seen["miss"] += 1
        assert min(seen.values()) > 20, seen
    finally:
        P.clear_hull_faces()
        lib.emu_set_hull_faces(None, None, None, C.c_int(0))
