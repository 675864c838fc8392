"""GPU checks of the two-hand backhand fix launch (include/b200env_v2p.h b200v2p_backhand_fix) against the torch restatement
oracle/ref_port_backhand.py, and of the test-time tasks' export with vid2player.fix_two_hand_backhand_post.

Float32 bound.  The double instantiation follows the float64 restatement to rounding.  The float32 one may take an L1 sign the other
way where a term sits within rounding of zero (after the first step every fitted component is about +-lr and neighbours differ by
far less).  One flip changes that component's step by at most about 2 lr, effects through the Adam moments included, so after k
steps a fitted angle-axis differs by at most 2 lr k per component, sqrt(3) 2 lr k in norm, and a rotation matrix entry by no more
than that angle.  The other joints see only the float32 round trip (1e-4 allows for it near theta = pi)."""
import ctypes as C

import numpy as np
import pytest
import torch

from conftest import golden
from helpers import SIM_PARAMS, v2p_cfg, v2p_dual_cfg
from oracle import ref_port_backhand as B

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
Z = golden("v2p_backhand.npz")


def fixture_case(c, dtype):
    t = lambda k: torch.tensor(Z[f"c{c}_{k}"])  # noqa: E731
    return dict(joint_rot=t("joint_rot").to(dtype), phase=t("phase").to(dtype), swing_type=t("swing_type"), rest=t("rest").to(dtype),
                righthand=bool(Z[f"c{c}_righthand"]))


def episode(g, T, segments, righthand=True, dtype=torch.float64):
    jr = 0.35 * torch.randn(1, 24, 3, generator=g) + 0.03 * torch.randn(T, 24, 3, generator=g).cumsum(0)
    phase, swing = torch.rand(T, generator=g) * 2.0, torch.randint(0, 2, (T,), generator=g)
    for a, b in segments:
        phase[a:b] = 2.05 + 2.9 * torch.rand(b - a, generator=g)
        swing[a:b] = 2
    rest = torch.tensor(Z["c0_rest" if righthand else "c3_rest"])
    return dict(joint_rot=jr.to(dtype), phase=phase.to(dtype), swing_type=swing, rest=rest.to(dtype), righthand=righthand)


def on_device(p):
    return {k: v.to(DEV).contiguous() if torch.is_tensor(v) else v for k, v in p.items()}


def launch(problems, iters, dtype=None):
    from vid2player3d_b200 import native_v2p as V
    ps = [on_device({k: v.to(dtype) if dtype and torch.is_tensor(v) and v.is_floating_point() else v for k, v in p.items()}) for p in problems]
    outs, losses = V.backhand_fix(ps, iters=iters)
    torch.cuda.synchronize()
    return [o.cpu() for o in outs], losses.cpu().numpy()


def restated(p, iters):
    torch.set_num_threads(4)
    return B.fix_episode(p["joint_rot"].double(), p["phase"], p["swing_type"], p["rest"].double(), p["righthand"], iters)


def rotmats(jr):
    return B.angle_axis_to_rotation_matrix(jr.double()).view(-1, 24, 3, 3)


@pytest.mark.parametrize("iters", [1, 2, 10, 500])
def test_double_matches_float64_restatement(iters):
    """the fixture's four episodes (M = 1, 2, 60, 60 left-handed; identical neighbours, near-pi and at-rest joints) in one launch"""
    probs = [fixture_case(c, torch.float64) for c in range(int(Z["num_cases"]))]
    outs, losses = launch(probs, iters)
    for p, o, lo in zip(probs, outs, losses):
        want, wl = restated(p, iters)
        np.testing.assert_allclose(o.numpy(), want.numpy(), atol=1e-9, rtol=0)
        np.testing.assert_allclose(lo, wl, atol=1e-9, rtol=0)     # NaN smoothness where M = 1


@pytest.mark.parametrize("iters", [1, 10, 500])
def test_float_within_bound_of_float64(iters):
    probs = [fixture_case(c, torch.float32) for c in range(int(Z["num_cases"]))]
    outs, losses = launch(probs, iters)
    for p, o in zip(probs, outs):
        want, _ = restated(p, iters)
        need = B.select(p["swing_type"], p["phase"])
        np.testing.assert_array_equal(o[~need].numpy(), p["joint_rot"][~need].numpy())
        ik = B.arm_joints(p["righthand"])[0]
        other = [j for j in range(24) if j not in ik]
        d = (rotmats(o[need]) - rotmats(want[need])).abs()
        assert float(d[:, other].max()) <= 1e-4
        assert float(d[:, ik].max()) <= 2 * 3 ** 0.5 * B.LR * iters + 1e-4


def test_no_frame_selected_is_the_input_bit_for_bit():
    g = torch.Generator().manual_seed(1)
    p = episode(g, 50, [], dtype=torch.float32)
    outs, losses = launch([p], 500)
    assert torch.equal(outs[0], p["joint_rot"]) and np.isnan(losses).all()


def test_single_frame_and_every_frame_selected():
    g = torch.Generator().manual_seed(2)
    probs = [episode(g, 9, [(4, 5)]), episode(g, 40, [(0, 40)], righthand=False)]
    outs, losses = launch(probs, 10)
    for p, o, lo in zip(probs, outs, losses):
        want, wl = restated(p, 10)
        np.testing.assert_allclose(o.numpy(), want.numpy(), atol=1e-9, rtol=0)
        np.testing.assert_allclose(lo, wl, atol=1e-9, rtol=0)
    assert np.isnan(losses[0, 2]) and not np.isnan(losses[1]).any()


def test_more_frames_than_threads_at_the_dual_capacity():
    """1800 frames (the dual recording capacity), three segments: M = 1300 rows over the CTA's 256 threads"""
    g = torch.Generator().manual_seed(3)
    p = episode(g, 1800, [(0, 500), (700, 1200), (1400, 1700)])
    outs, losses = launch([p], 10)
    want, wl = restated(p, 10)
    np.testing.assert_allclose(outs[0].numpy(), want.numpy(), atol=1e-9, rtol=0)
    np.testing.assert_allclose(losses[0], wl, atol=1e-9, rtol=0)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_problems_of_different_length_in_one_launch_equal_their_own_launch(dtype):
    g = torch.Generator().manual_seed(4)
    probs = [episode(g, 300, [(20, 90), (150, 200)], dtype=dtype), episode(g, 7, [(2, 5)], False, dtype),
             episode(g, 0, [], dtype=dtype), episode(g, 1800, [(100, 400)], dtype=dtype), episode(g, 33, [(0, 33)], False, dtype)]
    outs, losses = launch(probs, 20)
    for i, p in enumerate(probs):
        o, lo = launch([p], 20)
        assert torch.equal(outs[i], o[0])
        np.testing.assert_array_equal(losses[i], lo[0])


def test_nan_frame_gives_what_the_restatement_gives():
    g = torch.Generator().manual_seed(5)
    p = episode(g, 60, [(10, 40)])
    p["joint_rot"][25] = float("nan")
    outs, losses = launch([p], 10)
    want, wl = restated(p, 10)
    np.testing.assert_allclose(outs[0].numpy(), want.numpy(), atol=1e-9, rtol=0, equal_nan=True)
    np.testing.assert_allclose(losses[0], wl, atol=1e-9, rtol=0, equal_nan=True)
    assert torch.isnan(outs[0][25]).all() and torch.isfinite(outs[0][torch.arange(60) != 25]).all()


def test_malformed_input_is_refused():
    from vid2player3d_b200 import abi
    from vid2player3d_b200.native import lib
    T = 8
    jr, out = torch.zeros(T, 24, 3, device=DEV), torch.zeros(T, 24, 3, device=DEV)
    ph, rest, sw = torch.zeros(T, device=DEV), torch.zeros(24, 3, device=DEV), torch.zeros(T, dtype=torch.long, device=DEV)
    scratch = torch.zeros(abi.bhfix_scratch_bytes([T], 4), dtype=torch.uint8, device=DEV)

    def call(iters=5, precision=0, scratch_bytes=None, **over):
        q = (abi.V2PBhProb * 1)()
        q[0].joint_rot, q[0].phase, q[0].swing_type, q[0].rest, q[0].out = (x.data_ptr() for x in (jr, ph, sw, rest, out))
        q[0].T, q[0].swing_type_len, q[0].righthand = T, T, 1
        for k, v in over.items():
            setattr(q[0], k, v)
        f = abi.V2PBhFix(num_problems=1, iters=iters, problems=C.addressof(q), scratch=scratch.data_ptr(),
                         scratch_bytes=scratch.numel() if scratch_bytes is None else scratch_bytes, precision=precision)
        rc = lib().b200v2p_backhand_fix(C.byref(f), None)
        return rc, lib().b200v2p_last_error().decode()

    assert call()[0] == 0
    for over, msg in ((dict(T=-1), "T must"), (dict(joint_rot=None), "null"), (dict(out=None), "null"), (dict(swing_type=None), "null"),
                      (dict(swing_type_len=T - 1), "shorter than T"), (dict(iters=-1), "negative"), (dict(precision=2), "precision"),
                      (dict(scratch_bytes=16), "scratch too small")):
        kw = {k: over.pop(k) for k in ("iters", "precision", "scratch_bytes") if k in over}
        rc, err = call(**kw, **over)
        assert rc != 0 and msg in err, (over, kw, rc, err)
    torch.cuda.synchronize()


def fill_swings(phase, swing, g):
    """two backhand segments in each recorded row: swing_type 2, phase inside (2, 5)"""
    T = phase.shape[-1]
    phase.copy_(torch.rand(phase.shape, generator=g) * 2.0)
    swing.zero_()
    for a, b in ((T // 6, T // 3), (T // 2, 5 * T // 6)):
        phase[..., a:b] = 2.05 + 2.9 * torch.rand(phase[..., a:b].shape, generator=g)
        swing[..., a:b] = 2
    return phase, swing


def check_export(z_fixed, z_rot, z_phase, z_swing, rest, rh, iters, losses):
    need = B.select(torch.tensor(z_swing), torch.tensor(z_phase))
    np.testing.assert_array_equal(z_fixed[~need.numpy()], z_rot[~need.numpy()])     # frames not selected: bit-identical
    if iters == 1:
        want, wl = B.fix_episode(torch.tensor(z_rot).double(), torch.tensor(z_phase), torch.tensor(z_swing), rest.double(), rh, 1)
        d = (rotmats(torch.tensor(z_fixed)) - rotmats(want)).abs()
        assert float(d.max()) <= 2 * 3 ** 0.5 * B.LR + 1e-4
        np.testing.assert_allclose(losses, wl, rtol=1e-4)
    else:
        before = B.free_hand_distance(torch.tensor(z_rot).double()[need], rest, rh)
        after = B.free_hand_distance(torch.tensor(z_fixed).double()[need], rest, rh)
        assert float(after.mean()) < float(before.mean())


def test_single_export_writes_the_fixed_rows(tmp_path, monkeypatch):
    """djokovic-style cfg (flag set, semi-western grip, right hand): joint_rot as recorded, joint_rot_fixed the fix of the rows"""
    from vid2player3d_b200 import native_v2p
    from vid2player3d_b200.tasks import MVAEControllerVis
    monkeypatch.chdir(tmp_path)
    cfg = v2p_cfg(64, player="djokovic", grip="semi_western", fix_two_hand_backhand_post=True)
    cfg["env"]["physics"]["assetFileName"] = "smpl_mesh_humanoid_djokovic.xml"
    cfg["env"].update(record=True, num_rec_frames=120, num_eg=2)
    cfg["args"] = type("Args", (), {"cfg": "djokovic"})
    env = MVAEControllerVis(cfg, SIM_PARAMS, 1, "cuda", 0, True)
    env.reset()
    env.render_vis(init=True)
    for _ in range(10):
        env.reset_done()
        env.step(torch.randn(env.num_envs, env.num_actions, device=DEV))
        env.render_vis()
    g = torch.Generator().manual_seed(6)
    ph, sw = fill_swings(torch.empty(64, 120), torch.empty(64, 120, dtype=torch.long), g)
    env._rec["phase"].copy_(ph)
    env._rec["swing_type"].copy_(sw)
    rec = {k: v.cpu().numpy() for k, v in env._rec.items()}
    rest = env._physics_player.task._rest_t[0].cpu()
    for iters in (1, native_v2p.BACKHAND_ITERS):
        monkeypatch.setattr(native_v2p, "BACKHAND_ITERS", iters)
        env.exported.clear()
        env.export_episodes()
        assert len(env.exported) == 2
        for i, p in enumerate(env.exported):
            z = np.load(p)
            e = int(z["env_id"])
            np.testing.assert_array_equal(z["joint_rot"], rec["joint_rot"][e])
            check_export(z["joint_rot_fixed"], z["joint_rot"], z["phase"], z["swing_type"], rest, True, iters, env.backhand_losses[i + 1])


def test_dual_export_fixes_the_player_not_named_federer(tmp_path, monkeypatch):
    from vid2player3d_b200 import native_v2p
    from vid2player3d_b200.tasks import MVAEControllerVisDual
    monkeypatch.chdir(tmp_path)
    cfg = v2p_dual_cfg(64, fix_two_hand_backhand_post=True)
    cfg["env"].update(record=True, num_rec_frames=1000, num_eg=2, rec_fname=None)
    env = MVAEControllerVisDual(cfg, SIM_PARAMS, 1, "cuda", 0, True, capacity=150)
    env.reset()
    env.render_vis(init=True)
    for _ in range(10):
        env.reset_done()
        env.step(torch.randn(env.num_envs, env.num_actions, device=DEV))
        env.render_vis()
    # two list entries by hand: rallies of 150 and 97 frames, poses from the recording, backhand segments in every row
    g = torch.Generator().manual_seed(7)
    best = env._best
    src = env._rec["joint_rot"][:4, :11]
    best["joint_rot"][:, :, :] = src.reshape(2, 2, 11, 24, 3).repeat(1, 1, 14, 1, 1)[:, :, :150]
    best["joint_rot"] += 0.01 * torch.randn(best["joint_rot"].shape, generator=g).to(DEV)
    ph, sw = fill_swings(torch.empty(2, 2, 150), torch.empty(2, 2, 150, dtype=torch.long), g)
    best["phase"].copy_(ph)
    best["swing_type"].copy_(sw)
    env._list["list_len"].fill_(2)
    env._list["order"].copy_(torch.tensor([1, 0], device=DEV))
    env._list["best_nframes"].copy_(torch.tensor([150, 97], device=DEV))
    env._list["best_distance"].copy_(torch.tensor([1.0, 2.0], device=DEV))
    rests = env._physics_player.task._rest_t.cpu()
    for iters in (1, native_v2p.BACKHAND_ITERS):
        monkeypatch.setattr(native_v2p, "BACKHAND_ITERS", iters)
        env.exported.clear()
        env.export_episodes()
        assert len(env.exported) == 2
        for i, p in enumerate(env.exported):
            z = np.load(p)
            assert z["joint_rot_fixed"].shape == z["joint_rot"].shape == (2, (97, 150)[i], 24, 3)
            np.testing.assert_array_equal(z["joint_rot_fixed"][0], z["joint_rot"][0])          # federer: left alone
            assert np.isnan(env.backhand_losses[i + 1][0]).all()
            check_export(z["joint_rot_fixed"][1], z["joint_rot"][1], z["phase"][1], z["swing_type"][1], rests[1], True, iters,
                         env.backhand_losses[i + 1][1])
