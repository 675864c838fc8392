"""GPU checks of the embodied_pose imitation policy at test time (HumanoidSMPLIMVis): the operand launch b200env_im_policy_rows, the
residual epilogue of the GEMM layer, the actions against the float64 restatement oracle/ref_port_im_policy.py, the device bookkeeping
b200env_play_stats against the restatement fed the device's own (rew_buf, reset_buf) history, and the graphed loop against the eager one.

Tolerance of the actions: as tests/test_gpu_v2p_policy.py states, bf16 operands and fp32 accumulation keep the three hidden layers'
action within ~1 % of max|mu|; LOOSE = 2.5e-2 of max|mu| per output.  The operand row and the residual layer have no tolerance: they are
bit for bit the unfused launches on the same inputs."""
import numpy as np
import pytest
import torch

from helpers import SIM_PARAMS, im_cfg
from oracle import ref_port_im_policy as R

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
LOOSE = 2.5e-2
UNITS = (1024, 1024, 512)


def make_task(N, **over):
    from vid2player3d_b200 import model_compiler, motion_lib
    from vid2player3d_b200.tasks import HumanoidSMPLIMVis
    model = model_compiler.load_compiled("smpl_mesh_humanoid_amass_v1")
    flat = motion_lib.synthetic(model, num_motions=4, num_frames=60, seed=1)
    cfg = im_cfg(N, flat, stateInit="Start", **over)
    return HumanoidSMPLIMVis(cfg, SIM_PARAMS, 1, "cuda", 0, True)


@pytest.fixture(scope="module")
def task():
    torch.manual_seed(0)
    return make_task(8192)


def network(seed, norm="running", out=75, inp=734, units=UNITS):
    """random actor of the shipped shape, as im_networks_from_checkpoint returns it; norm: running (RunningNorm statistics), rms
    (rl_games), None (n == 0)"""
    g = torch.Generator().manual_seed(seed)
    dims = (inp,) + units + (out,)
    layers = [((torch.rand(dims[i + 1], dims[i], generator=g) * 2 - 1) / dims[i] ** 0.5,
               (torch.rand(dims[i + 1], generator=g) * 2 - 1) / dims[i] ** 0.5) for i in range(4)]
    if norm is None:
        return dict(layers=layers, mean=None, rstd=None, clip=float("inf")), dict(layers=[(w.double(), b.double()) for w, b in layers], norm=None)
    mean = torch.randn(inp, generator=g) * 0.5
    if norm == "running":
        std = torch.rand(inp, generator=g) * 2 + 0.05
        net = dict(layers=layers, mean=mean, rstd=1.0 / (std + 1e-8), clip=5.0)
        ref = dict(layers=layers, norm="running", n=1, mean=mean.double().numpy(), std=(1.0 / net["rstd"].double() - 1e-8).numpy())
    else:
        var = torch.rand(inp, generator=g) * 2 + 0.05
        net = dict(layers=layers, mean=mean, rstd=1.0 / torch.sqrt(var + 1e-5), clip=5.0)
        ref = dict(layers=layers, norm="rms", mean=mean.double().numpy(), var=var.double().numpy())
    ref["layers"] = [(w.double().numpy(), b.double().numpy()) for w, b in layers]
    return net, ref


def scramble(task, steps=3, seed=1):
    """a full reset and a few steps of random actions, so obs_buf holds moving bodies"""
    task.reset()
    g = torch.Generator(device=DEV).manual_seed(seed)
    for _ in range(steps):
        task.step(torch.rand(task.num_envs, task.num_actions, device=DEV, generator=g) * 2 - 1)
    torch.cuda.synchronize()


def expected_row(task, clip_obs, t, mean, rstd, clip):
    """nn.cast_rows(task.compute_imitation_obs(clamped obs_buf chunks, context slot t)) and the slot's target dof_pos"""
    from vid2player3d_b200 import nn
    N, nb, nd = task.num_envs, task._num_lib_bodies, task.num_dof
    obs = torch.clamp(task.obs_buf, -clip_obs, clip_obs)
    ch = {}
    o = 0
    for name, d, s in zip(task.obs_names, task.obs_dims, task.obs_shapes):
        ch[name] = obs[:, o:o + d].reshape((N,) + tuple(s))
        o += d
    f = task.context_feat[:, task.context_padding + t]
    tp, tr, td = f[:, :3 * nb].reshape(N, nb, 3), f[:, 3 * nb:7 * nb].reshape(N, nb, 4), f[:, 7 * nb:7 * nb + nd]
    h = task.compute_imitation_obs(ch["body_pos"], ch["body_rot"], tp, tr, ch["dof_pos"], ch["dof_vel"], td, ch["body_vel"],
                                   ch["body_ang_vel"], ch["motion_bodies"], True, True)
    x = nn.padded_bf16(N, h.shape[1], DEV)
    if mean is None:
        nn.cast_rows(h, x, h.shape[1])
    else:
        nn.cast_rows(h, x, h.shape[1], mean, rstd, -clip, clip)
    return x, td.contiguous()


@pytest.mark.parametrize("norm", ["running", "rms", None])
@pytest.mark.parametrize("clip_obs", [float("inf"), 5.0])
def test_operand_row_is_the_unfused_cast(task, norm, clip_obs):
    net, _ = network(3, norm)
    task.set_policy(net, clip_obs=clip_obs, clip_actions=1.0)
    p = task._im_policy
    for rebuild in (False, True):
        scramble(task, steps=4)
        if rebuild:     # the host-decided rebuild of every env's window at the current motion times
            task._init_context(torch.arange(task.num_envs, device=DEV), task._reset_ref_motion_ids, task._cur_ref_motion_times)
        for t in (0, 1, task.context_length - 1):
            task._im_step.fill_(t + 5 * task.context_length)    # the slot is step % context_length
            p.x.fill_(-7.75)
            task.policy_rows()
            x, td = expected_row(task, clip_obs, t, p.mean, p.rstd, task._im_clip)
            got, want = p.x[:task.num_envs, :734].view(torch.int16), x[:task.num_envs, :734].view(torch.int16)
            assert torch.equal(got, want), f"t={t}, rebuild={rebuild}: {(got != want).sum().item()} operand entries differ"
            assert torch.equal(task._im_resid, td), f"t={t}: the residual is not the slot's target dof_pos"


@pytest.mark.parametrize("clamp", [None, (-1.0, 1.0)])
def test_residual_layer_is_the_plain_layer_plus_resid(clamp):
    from vid2player3d_b200 import nn
    g = torch.Generator().manual_seed(4)
    rows, K, N, cols = 300, 512, 75, 69
    a = nn.padded_bf16(rows, K, DEV)
    a[:rows, :K] = (torch.randn(rows, K, generator=g) * 0.5).to(DEV, torch.bfloat16)
    w, b = torch.randn(N, K, generator=g) / K ** 0.5, torch.randn(N, generator=g) * 0.1
    resid = (torch.randn(rows, 80, generator=g) * 0.7).to(DEV)
    o1, o2 = torch.zeros(rows, N, device=DEV), torch.zeros(rows, N, device=DEV)
    l1 = nn.Linear(a, w, b, o1, rows, out_clamp=clamp, residual=(resid, cols))
    l2 = nn.Linear(a, w, b, o2, rows)
    l1.run()
    l2.run()
    want = o2.clone()
    want[:, :cols] = want[:, :cols] + resid[:, :cols]
    if clamp:
        want = want.clamp(*clamp)
    torch.cuda.synchronize()
    assert torch.equal(o1, want)


@pytest.mark.parametrize("N", [1, 127, 128, 129, 8192])
@pytest.mark.parametrize("clip_actions", [None, 1.0])
def test_actions_match_the_float64_restatement(task, N, clip_actions):
    from vid2player3d_b200 import nn
    net, ref = network(5, "running")
    scramble(task, steps=3, seed=N)
    # a few rows far outside the clamps
    for e in (0, N // 2, N - 1):
        task.obs_buf[e, ::7] = 40.0 * (1 if e % 2 else -1)
    nd, t = task.num_dof, 3
    step = torch.full((1,), t, device=DEV, dtype=torch.long)
    resid = torch.zeros(N, nd, device=DEV)
    pol = nn.PolicyMLP(net["layers"], N, DEV, obs_mean=net["mean"], obs_rstd=net["rstd"], clamp_obs=5.0, clamp_actions=clip_actions,
                       residual=(resid, nd))
    task._env.im_policy_rows(
        dict(n=N, num_obs=task.num_obs, num_frames=task.context_feat.shape[1], feat_width=task.context_feat.shape[2],
             context_padding=task.context_padding, context_length=task.context_length, ld=pol.x.shape[1], clip_obs=5.0, clip=5.0),
        dict(obs_buf=task.obs_buf, context_feat=task.context_feat, step=step, mean=pol.mean, rstd=pol.rstd, x=pol.x, resid=resid))
    mu = pol.forward_prepared()
    torch.cuda.synchronize()
    want = R.act(task.obs_buf[:N].cpu().numpy(), task.context_feat[:N].cpu().numpy(), ref, task._num_lib_bodies, nd, task.context_padding,
                 t, clip_obs=5.0, clip_actions=clip_actions)
    got = mu.cpu().numpy().astype(np.float64)
    scale = max(np.abs(want).max(), 1e-6)
    assert np.abs(got - want).max() <= LOOSE * scale, np.abs(got - want).max() / scale


def run(task, net, history=None, **kw):
    return task.run_test(net, print_stats=False, history=history, clip_obs=5.0, clip_actions=1.0, **kw)


@pytest.mark.parametrize("sync_every", [1, None])
def test_statistics_match_the_restatement_on_the_device_history(sync_every):
    torch.manual_seed(0)
    task = make_task(512)
    net, _ = network(7, None)
    hist = []
    games_num, max_steps = 700, 90                      # 700 of 512 envs: the second game ends mid-step
    out = run(task, net, history=hist, games_num=games_num, max_steps=max_steps, sync_every=sync_every)
    games = [[(r.cpu().numpy(), d.cpu().numpy()) for r, d in g] for g in hist]
    lines, sr, ss, gp = R.run_stats(games, games_num, max_steps)
    assert out["games_played"] == gp
    assert abs(out["sum_steps"] - ss) <= 1e-6 * max(1.0, abs(ss))
    assert abs(out["sum_rewards"] - sr) <= 1e-5 * max(1.0, abs(sr))
    assert gp >= games_num


def test_printed_lines_match_the_restatement(capsys):
    torch.manual_seed(0)
    task = make_task(256)
    net, _ = network(7, None)
    hist = []
    task.run_test(net, games_num=300, max_steps=70, history=hist, clip_obs=5.0, clip_actions=1.0)
    printed = capsys.readouterr().out.splitlines()
    games = [[(r.cpu().numpy(), d.cpu().numpy()) for r, d in g] for g in hist]
    lines, sr, ss, gp = R.run_stats(games, 300, 70)
    body = [l for l in printed if l.startswith("reward:")]
    assert len(body) == len(lines)
    for l, (c, r, s) in zip(body, lines):
        parts = l.split()
        assert abs(float(parts[1]) - r / c) <= 1e-5 * max(1.0, abs(r / c)) and float(parts[3]) == s / c
    assert printed[-1].startswith("av reward:")


def test_graph_replays_the_eager_loop():
    torch.manual_seed(0)
    task = make_task(1024)
    net, _ = network(9, "running")
    outs = []
    for graph in (False, True):
        r = run(task, net, games_num=1500, max_steps=40, graph=graph)
        outs.append((r, task._im_policy.out.clone(), task.obs_buf.clone()))
    (r0, a0, o0), (r1, a1, o1) = outs
    assert r0 == r1
    assert torch.equal(a0, a1) and torch.equal(o0, o1)


def test_refusals(task):
    from vid2player3d_b200 import nn
    net, _ = network(3, "running")
    task.set_policy(net, clip_obs=5.0)
    p = task._im_policy
    base = dict(n=task.num_envs, num_obs=task.num_obs, num_frames=task.context_feat.shape[1], feat_width=task.context_feat.shape[2],
                context_padding=task.context_padding, context_length=task.context_length, ld=p.x.shape[1], clip_obs=5.0, clip=5.0)
    tens = dict(obs_buf=task.obs_buf, context_feat=task.context_feat, step=task._im_step, mean=p.mean, rstd=p.rstd, x=p.x, resid=task._im_resid)
    for over, msg in ((dict(ld=733), "ld is smaller"), (dict(ld=767), "ld must be even"), (dict(context_length=41), "outside the window"),
                      (dict(context_padding=-1), "outside the window"), (dict(num_obs=400), "num_obs"), (dict(feat_width=100), "feat_width"),
                      (dict(clip=0.0), "positive clip")):
        with pytest.raises(RuntimeError, match=msg):
            task._env.im_policy_rows(dict(base, **over), tens)
    with pytest.raises(RuntimeError, match="4-byte aligned"):
        task._env.im_policy_rows(base, dict(tens, x=p.x.view(-1)[1:]))
    with pytest.raises(RuntimeError, match="mean and rstd"):
        task._env.im_policy_rows(base, dict(tens, rstd=None))
    a = nn.padded_bf16(128, 64, DEV)
    r = torch.zeros(128, 64, device=DEV)
    for kw, msg in ((dict(weight=torch.zeros(2, 32, 64), bias=torch.zeros(2, 32), coef=torch.zeros(128, 2, device=DEV),
                          out=torch.zeros(128, 32, device=DEV), residual=(r, 8)), "single-expert"),
                    (dict(out=nn.padded_bf16(128, 64, DEV), residual=(r, 8)), "float output"),
                    (dict(residual=(r, 65)), "resid_cols")):
        args = dict(weight=torch.zeros(64, 64), bias=torch.zeros(64), out=torch.zeros(128, 64, device=DEV))
        args.update(kw)
        with pytest.raises(RuntimeError, match=msg):
            nn.Linear(a, args.pop("weight"), args.pop("bias"), args.pop("out"), 128, **args)
    with pytest.raises(ValueError, match="MuJoCo viewer"):
        from vid2player3d_b200.tasks import HumanoidSMPLIMVis
        HumanoidSMPLIMVis(im_cfg(4, None), SIM_PARAMS, 1, "cuda", 0, False)
