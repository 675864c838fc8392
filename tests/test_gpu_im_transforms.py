"""The context window's transforms on the device (cfg.env.b200_device_transforms; include/b200env.h: b200_motion_context_t), on the GPU.

1. The window launch with a program equals the float64 restatement fed the restated counter draws, for the specs of every golden
   case, at N = 1, 131 (ragged, listed in a permuted order) and 8192 (a sample of rows): body_pos and joint_conf within 1e-5, the
   occlusion decisions equal except within 1e-6 of min_conf; every other column and the mask bitwise equal to the launch without one.
2. Under the opt-in, reset_masked equals the id-list reset bitwise at the same counter (the twin tasks of test_gpu_im_reset_masked).
3. Statistics over 8192 x 48 x 24 joints: the Bernoulli rates within 4 sigma, the noise's mean and variance, the root never dropped.
4. Successive windows draw anew; the same seed and counter draw the same.
5. A random-policy rollout with the step graph and the reset_done graph equals the eager rollout bitwise, and the graphed reset makes
   no host synchronisation.
6. HumanoidSMPLIMVis.run_test with transforms is identical graphed and eager.
7. The refusals: the task's cfg (ValueError) and the C side's, before any launch."""
import ctypes as C
import json

import numpy as np
import pytest
import torch

from conftest import golden
from oracle import ref_port_transforms as X
from test_gpu_im_reset_masked import N as N_RAGGED, _graphed_and_eager, differing, id_list_reset, prefill, reset_mask_of
from test_gpu_task import make_task

pytestmark = pytest.mark.gpu

G = golden("im_transforms.npz")
CASES = [str(c) for c in G["case_names"]]
SPECS = {c: json.loads(str(G[f"{c}_specs"])) for c in CASES}
ALL = {"noisy_joints": {"prob": 0.5, "noise_std": 0.05, "conf_std": 0.04, "min_conf": 0.3},
       "mask_joints": {"joints": ["L_Knee", "R_Wrist", "Head"]}, "mask_random_joints": {"prob": 0.3}}


def opt_in(specs=ALL, **over):
    return dict(over, transform_specs=specs, b200_device_transforms=True)


_tasks = {}


def plain_task(n):
    if n not in _tasks:
        _tasks[n] = make_task(n, 0.3, stateInit="Random")
    return _tasks[n]


def windows(t, specs, rows, seed=10, counter=5):
    """(plain [n, P, W], transformed [n, P, W + nb], masks) of the windows of rows (a permutation of the task's envs) at random times"""
    from vid2player3d_b200 import abi
    N, P, dev = t.num_envs, t.context_length + 2 * t.context_padding, t.device
    nb = t._num_lib_bodies
    W = 2 * (3 * nb + t.num_dof) + 4 * nb
    g = torch.Generator(device=dev).manual_seed(len(rows))
    ids = torch.from_numpy(rows).to(dev)
    mids = t._reset_ref_motion_ids[ids].contiguous()
    times = (torch.rand(len(rows), device=dev, generator=g) * t._ml_t["motion_lengths"][mids]).contiguous()
    plain, feat = torch.full((N, P, W), 7.0, device=dev), torch.full((N, P, W + nb), 7.0, device=dev)
    m0, m1 = torch.zeros(N, P, dtype=torch.bool, device=dev), torch.zeros(N, P, dtype=torch.bool, device=dev)
    ctr = torch.full((1,), counter, dtype=torch.long, device=dev)
    t._env.motion_context(ids, mids, times, P, -t.context_padding, t.dt, plain, m0)
    t._env.motion_context(ids, mids, times, P, -t.context_padding, t.dt, feat, m1,
                          transforms=abi.transform_program(specs, t.body_names, nb), seed=seed, counter=ctr)
    torch.cuda.synchronize()
    assert int(ctr.item()) == counter, "the window launch advanced the counter"
    return plain, feat, m0, m1


@pytest.mark.parametrize("N", [1, N_RAGGED, 8192])
def test_window_equals_the_restatement(N):
    t = plain_task(N)
    nb, P = t._num_lib_bodies, t.context_length + 2 * t.context_padding
    W = 2 * (3 * nb + t.num_dof) + 4 * nb
    rows = np.random.default_rng(N).permutation(N) if N == N_RAGGED else np.arange(N)
    check = np.unique(np.r_[0, N - 1, np.random.default_rng(1).integers(0, N, 253)]) if N == 8192 else np.arange(N)
    seed, counter = 10, 5
    noisy_u = X.draws(seed, counter, N, check, P, nb, {"noisy_joints": {"prob": 2.0}, "mask_random_joints": {"prob": 2.0}})[1]
    base = X.draw_index(N, check, P, nb)
    from oracle.ref_port_v2p import counter_hash
    u = lambda k: (counter_hash(seed, counter, base + np.uint64(k)) >> np.uint64(40)).astype(np.float32) * np.float32(2.0 ** -24)  # noqa: E731
    u0, u4 = u(0), u(4)
    for name in CASES:
        specs = SPECS[name]
        plain, feat, m0, m1 = windows(t, specs, rows, seed, counter)
        assert torch.equal(m0, m1), name
        assert torch.equal(feat[..., 3 * nb:W].view(torch.int32), plain[..., 3 * nb:].view(torch.int32)), f"{name}: other columns"
        pos = plain[check, :, :3 * nb].reshape(len(check), P, nb, 3).double().cpu().numpy()
        noisy = u0 < np.float32(specs.get("noisy_joints", {}).get("prob", 0.0))
        drop = u4 < np.float32(specs.get("mask_random_joints", {}).get("prob", 0.0))
        want_pos, want_conf = X.transform_target(pos, specs, t.body_names, noisy=noisy, noise=noisy_u, drop=drop)
        got_pos = feat[check, :, :3 * nb].reshape(len(check), P, nb, 3).double().cpu().numpy()
        got_conf = feat[check, :, W:].double().cpu().numpy()
        keep = np.ones(noisy.shape, bool)
        if "noisy_joints" in specs:
            keep = np.abs(X.pre_occlusion_conf(specs, noisy, noisy_u) - specs["noisy_joints"]["min_conf"]) >= 1e-6
        assert np.abs(got_pos - want_pos)[keep].max() <= 1e-5, f"{name}: body_pos"
        assert np.abs(got_conf - want_conf)[keep].max() <= 1e-5, f"{name}: joint_conf"
        assert np.array_equal(got_conf[keep] == 0, want_conf[keep] == 0), f"{name}: occlusion decisions"


def test_masked_reset_equals_id_list_at_the_same_counter():
    over = opt_in(stateInit="Hybrid", hybridInitProb=0.7)
    a, b = make_task(N_RAGGED, 0.3, **over), make_task(N_RAGGED, 0.3, **over)
    prefill([a, b])
    mask = reset_mask_of(N_RAGGED)
    for t in (a, b):
        t._reset_rng.fill_(3)
    from test_gpu_im_reset_masked import expected
    times, ref = expected(a, 3)
    a.reset_masked(torch.from_numpy(mask).to(a.device))
    id_list_reset(b, mask, times, ref)
    assert int(a._reset_rng.item()) == int(b._reset_rng.item()) == 4
    assert differing(a, b) == [], "the masked reset with transforms differs from the id-list reset"
    nb = a._num_lib_bodies
    conf = a.context_feat[torch.from_numpy(mask & ref).to(a.device), :, -nb:]
    assert (conf == 0).any() and (conf == 1).any() and ((conf > 0) & (conf < 1)).any()


def test_draw_statistics():
    t = plain_task(8192)
    nb, P = t._num_lib_bodies, t.context_length + 2 * t.context_padding
    W = 2 * (3 * nb + t.num_dof) + 4 * nb
    pn, pr, sd = 0.3, 0.2, 0.5
    specs = {"noisy_joints": {"prob": pn, "noise_std": sd, "conf_std": 1.0, "min_conf": 0.0}, "mask_random_joints": {"prob": pr}}
    plain, feat, _, _ = windows(t, specs, np.arange(8192), seed=123, counter=9)
    conf = feat[..., W:]
    d = (feat[..., :3 * nb] - plain[..., :3 * nb]).view(8192, P, nb, 3).double()
    dropped = conf == 0
    assert not dropped[..., 0].any(), "the root was dropped"
    n = dropped[..., 1:].numel()
    rate = dropped[..., 1:].double().mean().item()
    assert abs(rate - pr) <= 4 * (pr * (1 - pr) / n) ** 0.5, rate
    kept = ~dropped
    noised = kept & (d != 0).any(-1)
    m = kept.sum().item()
    nrate = noised.sum().item() / m
    assert abs(nrate - pn) <= 4 * (pn * (1 - pn) / m) ** 0.5, nrate
    z = d[noised]
    k = z.numel()
    assert abs(z.mean().item()) <= 4 * sd / k ** 0.5
    assert abs(z.var().item() - sd * sd) <= 4 * sd * sd * (2.0 / k) ** 0.5 + 1e-6
    assert (conf[noised] < 1).all() and (conf[kept & ~noised] == 1).all()


def test_successive_windows_draw_anew_and_replay():
    t = make_task(N_RAGGED, 0.3, **opt_in(stateInit="Start"))
    t2 = make_task(N_RAGGED, 0.3, **opt_in(stateInit="Start"))
    ids = torch.arange(N_RAGGED, device=t.device)
    times = torch.zeros(N_RAGGED, device=t.device)
    t._init_context(ids, t._reset_ref_motion_ids, times)
    f1 = t.context_feat.clone()
    t._init_context(ids, t._reset_ref_motion_ids, times)
    f2 = t.context_feat.clone()
    assert int(t._reset_rng.item()) == 2
    nb = t._num_lib_bodies
    assert (f1[..., -nb:] != f2[..., -nb:]).float().mean() > 0.3, "two windows drew the same transforms"
    t._reset_rng.fill_(0)
    t._init_context(ids, t._reset_ref_motion_ids, times)
    assert torch.equal(t.context_feat, f1)
    t2._init_context(ids, t2._reset_ref_motion_ids, times)
    assert torch.equal(t2.context_feat, f1)


def test_graphed_rollout_equals_eager_reset_masked():
    n, steps = N_RAGGED, 48
    w, a, b = _graphed_and_eager(n, opt_in(stateInit="Hybrid", hybridInitProb=0.5))
    assert a._reset_graph is not None
    g = torch.Generator(device=a.device).manual_seed(11)
    acts = [torch.rand(n, a.num_actions, device=a.device, generator=g) * 2 - 1 for _ in range(steps)]
    mask_b = torch.zeros(n, dtype=torch.bool, device=b.device)
    resets = torch.zeros((), dtype=torch.long, device=a.device)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for i in range(steps):
            w.step(acts[i])
            resets += a.reset_buf.sum()
            obs = w.reset_done()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    for i in range(steps):
        b.step(torch.clamp(acts[i], -1.0, 1.0))
        torch.ne(b.reset_buf, 0, out=mask_b)
        b.reset_masked(mask_b)
    torch.cuda.synchronize()
    assert int(resets) > 0, "no env finished: the rollout did not exercise the reset"
    assert differing(a, b) == [], "graphed step + reset_done differs from the eager rollout"
    assert torch.equal(obs, torch.clamp(b.obs_buf, -5.0, 5.0))
    assert int(a._reset_rng.item()) == int(b._reset_rng.item()) == steps + 2


def test_run_test_graphed_equals_eager():
    from test_gpu_im_policy import make_task as vis_task, network
    torch.manual_seed(0)
    t = vis_task(1024, **opt_in())
    net, _ = network(9, "running")
    outs = []
    for graph in (False, True):
        t._reset_rng.zero_()
        hist = []
        r = t.run_test(net, games_num=1500, max_steps=70, graph=graph, print_stats=False, history=hist, clip_obs=5.0, clip_actions=1.0)
        outs.append((r, t._im_policy.out.clone(), t.obs_buf.clone(), t.context_feat.clone(), int(t._reset_rng.item()),
                     [torch.stack([x for x, _ in g]) for g in hist]))
    (r0, a0, o0, c0, k0, h0), (r1, a1, o1, c1, k1, h1) = outs
    assert r0 == r1 and k0 == k1 and k0 > 1
    assert torch.equal(a0, a1) and torch.equal(o0, o1) and torch.equal(c0, c1)
    assert all(torch.equal(x, y) for x, y in zip(h0, h1))


def test_refusals():
    from vid2player3d_b200 import abi, native
    with pytest.raises(ValueError, match="not a body"):
        make_task(4, 0.3, **opt_in({"mask_joints": {"joints": ["Tail"]}}))
    with pytest.raises(ValueError, match="unknown transform"):
        make_task(4, 0.3, **opt_in({"blur": {}}))
    with pytest.raises(ValueError, match=r"outside \[0, 1\]"):
        make_task(4, 0.3, **opt_in({"mask_random_joints": {"prob": 2.0}}))
    t = plain_task(N_RAGGED)
    nb, P, dev = t._num_lib_bodies, 4, t.device
    W = 2 * (3 * nb + t.num_dof) + 4 * nb
    ids = torch.arange(2, device=dev)
    mids, times = t._reset_ref_motion_ids[:2].contiguous(), torch.zeros(2, device=dev)
    feat, mask = torch.zeros(N_RAGGED, P, W + nb, device=dev), torch.zeros(N_RAGGED, P, dtype=torch.bool, device=dev)
    ctr = torch.zeros(1, dtype=torch.long, device=dev)
    good = abi.transform_program(ALL, t.body_names, nb)

    def call(feat=feat, counter=ctr, **over):
        scalars = dict(good, n=2, num_frames=P, first_frame=0, dt=t.dt, feat_width=feat.shape[-1], seed=1)
        scalars.update(over)
        d = native.fill(abi.MotionContext, scalars,
                        dict(env_ids=ids, motion_ids=mids, motion_times=times, context_feat=feat, context_mask=mask, counter=counter))
        return native.lib().b200env_motion_context(t._env._h, C.byref(d), native._stream())

    before = feat.clone()
    for over, msg in ((dict(xf_ops=[1, 2, 1]), b"repeated"), (dict(xf_ops=[1, 0, 2]), b"after the program's end"),
                      (dict(xf_ops=[4, 0, 0]), b"unknown"), (dict(xf_noisy_prob=1.5), b"prob outside"),
                      (dict(xf_random_prob=-0.5), b"prob outside"), (dict(xf_conf_std=0.0), b"conf_std"),
                      (dict(xf_noise_std=-1.0), b"noise_std"), (dict(feat_width=W), b"row width"),
                      (dict(feat_width=W + nb + 1), b"row width")):
        assert call(**over) == -2, over
        assert msg in native.lib().b200env_last_error(), (over, native.lib().b200env_last_error())
    assert call(counter=None) == -2 and b"draw counter" in native.lib().b200env_last_error()
    assert call(xf_ops=[1, 0, 0], counter=None) == 0                # mask_joints alone draws nothing
    torch.cuda.synchronize()
    assert not torch.equal(feat, before)
    assert call(xf_ops=[0, 0, 0], feat=torch.zeros(N_RAGGED, P, W + nb + 2, device=dev)) == -2
