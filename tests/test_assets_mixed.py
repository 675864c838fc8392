"""The mixed plan of a handle of several assets (include/b200env.h: b200env_plan_assets_mixed, b200env_choose_asset_plan), the parts that
need no GPU:

1. the mixed planner's invariants: every env exactly once, in ascending order, batches of at most B consecutive envs;
2. the rule that picks the plan, at S = 1, 8, 64, 256 and N distinct assets for N = 8192 envs on a grid of 132 CTAs;
3. the grouped planner b200env_plan_assets keeps its output;
4. the lane emulator (tests/emu) running warps whose envs have different assets, as step_kernel_packed<true, false, true> does: in
   float64 against oracle/physics_ref.c run with each env's own model, in float32 bit for bit against the one-asset emulation."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "emu"))
from test_emu_packed import states  # noqa: E402

from oracle import physics_ref  # noqa: E402
from vid2player3d_b200 import abi, model_compiler, native  # noqa: E402

B = native.ENVS_PER_BATCH
AMASS = "smpl_mesh_humanoid_amass_v1"


def check_mixed_plan(env_asset, B, rows, batches):
    env_asset = np.asarray(env_asset)
    n = len(env_asset)
    assert rows.tolist() == list(range(n)), "the mixed plan keeps the env order"
    assert len(batches) == -(-n // B)
    assert batches[:, 1].tolist() == list(range(0, n, B)), "batches are consecutive runs of B envs"
    assert (batches[:, 2] >= 1).all() and (batches[:, 2] <= B).all() and batches[:, 2].sum() == n
    for a, first, cnt in batches.tolist():
        own = env_asset[first:first + cnt]
        assert a == (int(own[0]) if (own == own[0]).all() else -1)


@pytest.mark.parametrize("n,num_assets,Bp,seed", [(1, 1, 32, 0), (31, 2, 32, 1), (32, 2, 32, 2), (33, 3, 32, 3), (97, 4, 32, 4),
                                                   (8453, 3, 32, 5), (8192, 256, 32, 6), (8192, 8192, 32, 7), (50, 7, 8, 8)])
def test_mixed_plan_covers_every_env_once_in_order(n, num_assets, Bp, seed):
    ea = np.random.default_rng(seed).integers(0, num_assets, n)
    rows, batches = native.plan_assets(ea, num_assets, Bp, mixed=True)
    check_mixed_plan(ea, Bp, rows, batches)
    rows2, batches2 = native.plan_assets(ea.copy(), num_assets, Bp, mixed=True)
    assert np.array_equal(rows, rows2) and np.array_equal(batches, batches2)


def test_mixed_plan_names_the_asset_of_a_one_asset_batch():
    ea = np.concatenate([np.zeros(B, int), np.arange(B) % 3, np.full(5, 2)])
    _, batches = native.plan_assets(ea, 3, B, mixed=True)
    assert batches.tolist() == [[0, 0, B], [-1, B, B], [2, 2 * B, 5]]


def grouped_plan(env_asset, num_assets, Bp):
    """the documented grouped plan: envs stably sorted by asset, ceil(n_a / B) batches per asset in ascending asset order"""
    ea = np.asarray(env_asset)
    rows = np.argsort(ea, kind="stable")
    batches, pos = [], 0
    for a in range(num_assets):
        n_a = int((ea == a).sum())
        for p in range(pos, pos + n_a, Bp):
            batches.append([a, p, min(Bp, pos + n_a - p)])
        pos += n_a
    return rows, np.array(batches, np.int64).reshape(-1, 3)


@pytest.mark.parametrize("n,num_assets,seed", [(1, 1, 0), (33, 3, 1), (97, 4, 2), (8453, 3, 3), (8192, 256, 4), (8192, 8192, 5)])
def test_grouped_plan_is_unchanged(n, num_assets, seed):
    ea = np.random.default_rng(seed).integers(0, num_assets, n)
    rows, batches = native.plan_assets(ea, num_assets, B)
    r2, b2 = grouped_plan(ea, num_assets, B)
    assert np.array_equal(rows, r2) and np.array_equal(batches, b2)


def rounds(batches, G):
    return -(-batches // G)


@pytest.mark.parametrize("S,assign,mixed", [(1, "interleaved", False), (8, "interleaved", False), (64, "random", True),
                                            (256, "random", True), (8192, "interleaved", True)])
def test_rule_picks_the_plan_of_fewer_rounds(S, assign, mixed):
    """8192 envs, G = 132 (an H100 SXM): one asset, or 8 in equal shares, fill their batches (256 of them: 2 rounds either way) and
    keep the grouped plan; 64 or 256 assets at random need a third round grouped and take the mixed plan's two; a body per env
    (S = N) needs 8192 grouped batches, 63 rounds"""
    N, G = 8192, 132
    ea = np.arange(N) % S if assign == "interleaved" else np.random.default_rng(S).integers(0, S, N)
    grouped = int(sum(-(-c // B) for c in np.bincount(ea, minlength=S)))
    assert native.choose_asset_plan(ea, S, G) == (rounds(-(-N // B), G) < rounds(grouped, G)) == mixed
    if mixed:
        assert rounds(-(-N // B), G) == 2


def test_rule_at_the_edges():
    G = 132
    assert not native.choose_asset_plan([0], 1, G)
    assert not native.choose_asset_plan(np.arange(G) % G, G, G)                  # G batches of one env: one round either way
    assert native.choose_asset_plan(np.arange(G + 1) % (G + 1), G + 1, G)        # G + 1 batches grouped, 5 mixed
    assert not native.choose_asset_plan(np.arange(G + 1) % (G + 1), G + 1, 200)  # a grid of 200: one round either way


def test_mixed_planner_and_rule_reject_bad_arguments():
    for fn in (lambda ea, na, b: native.plan_assets(ea, na, b, mixed=True), lambda ea, na, b: native.choose_asset_plan(ea, na, b)):
        for ea, na, b, what in (([0, 4], 4, 32, "out of range"), ([-1], 2, 32, "out of range"), ([0], 0, 32, "num_assets"),
                                ([], 1, 32, "num_envs")):
            with pytest.raises(RuntimeError, match=what):
                fn(ea, na, b)
    with pytest.raises(RuntimeError, match="envs_per_batch"):
        native.plan_assets([0], 1, 0, mixed=True)
    with pytest.raises(RuntimeError, match="grid"):
        native.choose_asset_plan([0], 1, 0)


# ---- lane emulator

def _emu():
    """tests/emu/emu_mixed.cpp with the flags of tests/emu/build.py"""
    import build as emu_build
    out = os.path.join(emu_build.HERE, "build", "libemu_mixed.so")
    src = os.path.join(emu_build.HERE, "emu_mixed.cpp")
    deps = [src, os.path.join(emu_build.HERE, "emu_packed.cpp"), os.path.join(emu_build.HERE, "cuda_compat.h")] + \
        [os.path.join(emu_build.CSRC, f) for f in os.listdir(emu_build.CSRC) if f.endswith(".cuh")]
    if not (os.path.exists(out) and all(os.path.getmtime(s) <= os.path.getmtime(out) for s in deps)):
        os.makedirs(os.path.dirname(out), exist_ok=True)
        cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        subprocess.check_call([cxx, "-O1", "-std=c++17", "-pthread", "-shared", "-fPIC", "-x", "c++", "-Wno-unknown-pragmas",
                               "-ffp-contract=off", "-DEMU_PACKED=1", "-o", out, src])
    return C.CDLL(out)


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def scaled(model, s):
    """the asset scaled by s (as tests/test_gpu_assets.py): lengths, COMs, vertices, radii x s, mass x s^3, inertia x s^5"""
    m = dict(model)
    for k in ("offset", "com", "dyn_com", "verts", "radius"):
        m[k] = model[k] * s
    for k in ("mass", "dyn_mass"):
        m[k] = model[k] * s ** 3
    for k in ("inertia", "dyn_inertia"):
        m[k] = model[k] * s ** 5
    if len(model["prims"]):
        m["prims"] = model["prims"].copy()
        m["prims"][:, 1:8] *= s
    return m


def _assets():
    base = model_compiler.load_compiled(AMASS)
    mods = [base, scaled(base, 0.9), scaled(base, 1.1)]
    packed = [abi.pack_model(m, float(m["mass"].sum()) / 90.0) for m in mods]
    return base, [m for m, _ in packed], [np.ascontiguousarray(v, np.float32) for _, v in packed]


def emu_mixed(models, verts, env_asset, cfg, root, q, qd, tar, ext, n_steps, f32=False):
    lib = _emu()
    n = root.shape[0]
    dt = np.float32 if f32 else np.float64
    rb, cf = np.zeros((n, models[0].nb, 13), dt), np.zeros((n, models[0].nb, 3), dt)
    marr = (abi.Model * len(models))(*models)
    varr = (C.c_void_p * len(verts))(*[v.ctypes.data for v in verts])
    ea = np.ascontiguousarray(env_asset, np.int32)
    fn = lib.emu_mixed_physics_f32 if f32 else lib.emu_mixed_physics
    rc = fn(marr, varr, C.c_int(len(models)), _p(ea), C.byref(cfg), C.c_int(n), C.c_int(n_steps), _p(root), _p(q), _p(qd), _p(tar), _p(ext),
            _p(rb), _p(cf))
    assert rc == 0
    return rb, cf


# 4 envs per warp: warp 0 holds assets 0, 1, 2, 0 - warp 1 (ragged) 2, 1, 1
ENV_ASSET = np.array([0, 1, 2, 0, 2, 1, 1])


@pytest.mark.parametrize("contact", [False, True])
def test_emulated_mixed_warps_match_oracle_per_env_model(contact):
    base, models, verts = _assets()
    cfg = abi.make_cfg(base)
    n = len(ENV_ASSET)
    root, q, qd, tar, ext = states(n, 13, contact)
    for steps, tol in ((1, 1e-9), (4, 1e-7)):
        r1, q1, v1 = root.copy(), q.copy(), qd.copy()
        rb1, cf1 = emu_mixed(models, verts, ENV_ASSET, cfg, r1, q1, v1, tar.copy(), ext.copy(), steps)
        r2, q2, v2 = root.copy(), q.copy(), qd.copy()
        rb2, cf2 = np.zeros_like(rb1), np.zeros_like(cf1)
        for a in range(len(models)):
            idx = np.flatnonzero(ENV_ASSET == a)
            r, qq, vv = r2[idx].copy(), q2[idx].copy(), v2[idx].copy()
            rb2[idx], cf2[idx] = physics_ref.control_step(models[a], verts[a], cfg, r, qq, vv, tar[idx].copy(), ext[idx].copy(), n_steps=steps)
            r2[idx], q2[idx], v2[idx] = r, qq, vv
        for x, y, name, sc in ((r1, r2, "root", 1), (q1, q2, "dof_pos", 1), (v1, v2, "dof_vel", 1), (rb1, rb2, "rb", 1), (cf1, cf2, "contact", 1e3)):
            np.testing.assert_allclose(x, y, rtol=0, atol=tol * sc, err_msg=f"{name} steps={steps}")
    if contact:
        assert np.abs(cf2).max() > 10.0
    # the assets really differ: asset 0's model for every env misses the others
    r3, q3, v3 = root.copy(), q.copy(), qd.copy()
    physics_ref.control_step(models[0], verts[0], cfg, r3, q3, v3, tar.copy(), ext.copy(), n_steps=4)
    assert np.abs(q3 - q2)[ENV_ASSET != 0].max() > 1e-4


def test_emulated_mixed_warps_float32_bit_identical_to_one_asset_runs():
    import build as emu_build
    base, models, verts = _assets()
    cfg = abi.make_cfg(base)
    n = len(ENV_ASSET)
    f = lambda a: np.ascontiguousarray(a, np.float32)  # noqa: E731
    root, q, qd, tar, ext = (f(x) for x in states(n, 17, True))
    r1, q1, v1 = root.copy(), q.copy(), qd.copy()
    rb1, cf1 = emu_mixed(models, verts, ENV_ASSET, cfg, r1, q1, v1, tar, ext, 3, f32=True)
    one = C.CDLL(emu_build.build("packed"))
    one.emu_set_hull_faces(None, None, None, C.c_int(0))
    for a in range(len(models)):
        idx = np.flatnonzero(ENV_ASSET == a)
        r, qq, vv, t, e = f(root[idx]), f(q[idx]), f(qd[idx]), f(tar[idx]), f(ext[idx])
        rb, cf = np.zeros((len(idx), models[a].nb, 13), np.float32), np.zeros((len(idx), models[a].nb, 3), np.float32)
        assert one.emu_packed_physics_f32(C.byref(models[a]), _p(verts[a]), C.byref(cfg), C.c_int(len(idx)), C.c_int(3), _p(r), _p(qq), _p(vv),
                                          _p(t), _p(e), _p(rb), _p(cf), None, None) == 0
        for x, y, name in ((r, r1[idx], "root"), (qq, q1[idx], "dof_pos"), (vv, v1[idx], "dof_vel"), (rb, rb1[idx], "rb"), (cf, cf1[idx], "contact")):
            assert np.array_equal(x.view(np.uint32), y.view(np.uint32)), f"asset {a}: {name} differs from the one-asset emulation"
