"""GPU checks of the tennis controller's trained low-level imitation policy: the dual layout of the observation launch's bf16 operand rows
(b200env_obs_imitation_rows_dual), nn.V2PPolicy's wgmma layers on those rows against the float64 restatement (oracle/ref_port_v2p_policy.act), and
PhysicsMVAEController(Dual) / MVAEControllerVis(Dual) driven by physics.pretrained_model_cp / dual_model_cp.

The operand rows have no tolerance: they are bit for bit the cast launch of libb200nn.so (nn.cast_rows) on the launch's own float row,
player block by player block.  The actions have the bf16 tolerance of tests/test_gpu_v2p_policy.py: LOOSE = 2.5e-2 of max|mu|."""
import numpy as np
import pytest
import torch

from helpers import SIM_PARAMS, v2p_cfg, v2p_dual_cfg
from oracle import ref_port_v2p_policy as R
from test_gpu_obs_imitation import dev_inputs, make_inputs

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
LOOSE = 2.5e-2
OBS, ACT, UNITS = 734, 75, (1024, 1024, 512)
LD = 768
SLACK = 3
INF = float("inf")


def networks(P, seed, identity_second=False, units=UNITS):
    """random actors of the shipped shape with RunningNorm statistics (float32, CPU), as low_level_networks_from_cfg returns them"""
    g = torch.Generator().manual_seed(seed)
    nets = []
    for p in range(P):
        dims = (OBS,) + units + (ACT,)
        layers = [((torch.rand(dims[i + 1], dims[i], generator=g) * 2 - 1) / dims[i] ** 0.5,
                   (torch.rand(dims[i + 1], generator=g) * 2 - 1) / dims[i] ** 0.5) for i in range(4)]
        if identity_second and p == 1:
            nets.append(dict(layers=layers, mean=None, rstd=None, clip=INF))
        else:
            std = torch.rand(OBS, generator=g) * 2 + 0.05
            nets.append(dict(layers=layers, mean=torch.randn(OBS, generator=g), rstd=1.0 / (std + 1e-8), clip=5.0))
    return nets


def oracle_nets(nets):
    out = []
    for n in nets:
        layers = [(w.double().to(DEV), b.double().to(DEV)) for w, b in n["layers"]]
        if n["mean"] is None:
            out.append(dict(layers=layers, norm=None))
        else:
            out.append(dict(layers=layers, norm="running", n=1, mean=n["mean"].double().to(DEV), std=(1.0 / n["rstd"].double() - 1e-8).to(DEV)))
    return out


def policy(nets, N):
    from vid2player3d_b200 import nn
    return nn.V2PPolicy(nets, N, DEV, clip_obs=INF, clip_actions=None)


@pytest.fixture(scope="module")
def handle():
    from vid2player3d_b200.tasks import PhysicsMVAEController
    ctl = PhysicsMVAEController(v2p_cfg(8), SIM_PARAMS, 1, "cuda", 0, True)
    yield ctl._physics_player.task._env
    del ctl


@pytest.fixture(scope="module")
def inputs():
    return dev_inputs(make_inputs(8192, 21)[0], 26)


def launch(env, d, n, pol, op):
    """the observation launch with pol's operand fields into op; returns the float rows"""
    obs = torch.full((n, OBS), 12345.0, device=DEV)
    env.obs_imitation_rows(n, d["rbs"], d["bpe"], d["dofs"], d["target_pos"], d["target_rot"], d["target_dof_pos"], d["motion_bodies"],
                           True, True, obs, obs_bf16=op, mean=pol.mean, rstd=pol.rstd, clamp=pol.clip[0], dual=pol.dual, clamp1=pol.clip[-1])
    torch.cuda.synchronize()
    return obs


def cast_blocks(obs, pol, buf):
    """nn.cast_rows of obs into buf, player block by player block (env e -> row (e & 1) * N/2 + (e >> 1) in dual mode)"""
    from vid2player3d_b200 import nn
    P = 2 if pol.dual else 1
    H = obs.shape[0] // P
    for p in range(P):
        nn.cast_rows(obs[p::P].contiguous(), buf[p * H:], OBS, pol.mean[p] if pol.mean is not None else None,
                     pol.rstd[p] if pol.rstd is not None else None, -pol.clip[p], pol.clip[p])
    torch.cuda.synchronize()
    return buf


def nan_buffer(n):
    return torch.full((n + SLACK, LD), float("nan"), device=DEV, dtype=torch.bfloat16)


@pytest.mark.parametrize("N", [2, 4, 130, 258, 8192])
def test_dual_operand_rows_are_the_cast_of_each_players_block(handle, inputs, N):
    """player 0 normalised (clamp 5), player 1 at n == 0 (identity, clamp inf); NaN sentinels in columns [734, 768) and in the rows
    past N stay untouched; the float rows are those of the single launch"""
    pol = policy(networks(2, seed=N, identity_second=True), N)
    assert pol.dual and pol.clip == [5.0, INF]
    op = nan_buffer(N)
    obs = launch(handle, inputs, N, pol, op)
    want = cast_blocks(obs, pol, nan_buffer(N))
    assert torch.equal(op.view(torch.int16), want.view(torch.int16))
    assert bool(op[:, OBS:].isnan().all()) and bool(op[N:].isnan().all())
    single = policy(networks(1, seed=N), N)
    assert torch.equal(launch(handle, inputs, N, single, nan_buffer(N)).view(torch.int32), obs.view(torch.int32))


@pytest.mark.parametrize("N", [130, 8192])
def test_single_operand_rows_unchanged(handle, inputs, N):
    pol = policy(networks(1, seed=N), N)
    op = nan_buffer(N)
    obs = launch(handle, inputs, N, pol, op)
    assert torch.equal(op.view(torch.int16), cast_blocks(obs, pol, nan_buffer(N)).view(torch.int16))


@pytest.mark.parametrize("n, clamp, clamp1, msg", [(3, 5.0, 5.0, "even n"), (129, 5.0, INF, "even n"), (4, 5.0, 0.0, "positive clamps"),
                                                   (4, -1.0, 5.0, "positive clamp"), (4, 5.0, float("nan"), "positive clamps")])
def test_dual_refusals_before_any_launch(handle, inputs, n, clamp, clamp1, msg):
    pol = policy(networks(2, seed=1), 4)
    op = nan_buffer(n)
    obs = torch.full((n, OBS), 12345.0, device=DEV)
    with pytest.raises(RuntimeError, match=rf"error -2: .*{msg}"):
        handle.obs_imitation_rows(n, inputs["rbs"], 26, inputs["dofs"], inputs["target_pos"], inputs["target_rot"], inputs["target_dof_pos"],
                                  inputs["motion_bodies"], True, True, obs, obs_bf16=op, mean=pol.mean, rstd=pol.rstd, clamp=clamp, dual=True,
                                  clamp1=clamp1)
    torch.cuda.synchronize()
    assert bool(op.isnan().all()) and bool((obs == 12345.0).all())


SINGLE_N = (1, 2, 127, 128, 130, 258, 8192)
DUAL_N = (2, 128, 130, 258, 8192)


@pytest.mark.parametrize("mode,N", [("single", n) for n in SINGLE_N] + [("dual", n) for n in DUAL_N])
def test_actions_match_restatement(handle, inputs, mode, N):
    """operand launch + forward_prepared (the step's path) within LOOSE of max|mu| of the float64 restatement on the same obs rows"""
    P = 2 if mode == "dual" else 1
    nets = networks(P, seed=N, identity_second=(N % 4 == 2))
    pol = policy(nets, N)
    obs = launch(handle, inputs, N, pol, pol.x)
    mu = pol.forward_prepared().clone()
    want = R.act(obs.double(), oracle_nets(nets))
    assert mu.shape == (N, ACT) and bool(torch.isfinite(mu).all())
    assert float((mu.double() - want).abs().max()) <= LOOSE * float(want.abs().max())


@pytest.mark.parametrize("N", [2, 130, 258, 8192])
def test_dual_equals_two_single_runs(handle, inputs, N):
    nets = networks(2, seed=7)
    dual = policy(nets, N)
    obs = launch(handle, inputs, N, dual, dual.x)
    got = dual.forward_prepared().clone()
    for p in range(2):
        single = policy([nets[p]], N // 2)
        assert torch.equal(got[p::2], single(obs[p::2].contiguous()))


# ------------------------------------------------------------------------------------------------ the controllers, from checkpoints
def save_checkpoints(tmp_path, P, units=(64, 64, 32), seed=3):
    """embodied_pose-style checkpoints (a2c_network.* + RunningNorm buffers; the second of a pair as rl_games running_mean_std)"""
    paths, nets = [], []
    for p, net in enumerate(networks(P, seed, units=units)):
        model = {}
        for k, (w, b) in zip(("actor_mlp.0", "actor_mlp.2", "actor_mlp.4", "mu"), net["layers"]):
            model[f"a2c_network.{k}.weight"], model[f"a2c_network.{k}.bias"] = w * 4, b
        std = 1.0 / net["rstd"] - 1e-8
        ck = {"model": model}
        if p == 0:
            model["a2c_network.running_obs.n"] = torch.tensor(1000)
            model["a2c_network.running_obs.mean"], model["a2c_network.running_obs.std"] = net["mean"], std
            model["a2c_network.running_obs.var"] = std ** 2
        else:
            ck["running_mean_std"] = {"running_mean": net["mean"].double(), "running_var": (std ** 2).double(), "count": torch.tensor(64.0)}
        paths.append(str(tmp_path / f"im_{p}.pth"))
        torch.save(ck, paths[-1])
    return paths


def controller_cfg(mode, N, tmp_path, **over):
    cfg = v2p_dual_cfg(N, **over) if mode == "dual" else v2p_cfg(N, **over)
    paths = save_checkpoints(tmp_path, 2 if mode == "dual" else 1)
    cfg["env"]["physics"].update(dual_model_cp=paths) if mode == "dual" else cfg["env"]["physics"].update(pretrained_model_cp=paths[0])
    return cfg


def loaded(cfg, mode):
    from vid2player3d_b200 import nn
    phys = cfg["env"]["physics"]
    return nn.low_level_networks_from_cfg(phys, OBS, ACT, mode == "dual")


@pytest.mark.parametrize("mode", ["single", "dual"])
def test_step_acts_with_the_trained_policy(mode, tmp_path, monkeypatch):
    """the actions each step hands to task.step are the restatement on that step's obs_buf; the operand needs no cast launch"""
    from vid2player3d_b200 import nn
    from vid2player3d_b200.tasks import PhysicsMVAEController, PhysicsMVAEControllerDual
    N = 258
    cfg = controller_cfg(mode, N, tmp_path)
    monkeypatch.setattr(nn, "cast_rows", None)                   # the step must not fall back to the cast launch
    env = (PhysicsMVAEControllerDual if mode == "dual" else PhysicsMVAEController)(cfg, SIM_PARAMS, 1, "cuda", 0, True)
    task = env._physics_player.task
    assert isinstance(env._low_level_policy, nn.V2PPolicy) and env._low_level_policy.dual == (mode == "dual")
    assert task._obs_operand[0] is env._low_level_policy.x
    seen, step = [], task.step
    monkeypatch.setattr(task, "step", lambda a: (seen.append((task.obs_buf.clone(), a.clone())), step(a)))
    ref = oracle_nets(loaded(cfg, mode))
    env.reset()
    g = torch.Generator(device=DEV).manual_seed(2)
    for _ in range(4):
        env.step(torch.clamp(torch.randn(N, env.num_actions, device=DEV, generator=g), -5, 5))
    torch.cuda.synchronize()
    assert len(seen) == 4
    for obs, act in seen:
        want = R.act(obs.double(), ref)
        assert float((act.double() - want).abs().max()) <= LOOSE * float(want.abs().max())
        if float(want.abs().max()) > 1.5:
            assert float(act.abs().max()) > 1.0                    # no action clamp (clip_actions_val is inf)


@pytest.mark.parametrize("mode", ["single", "dual"])
def test_graphed_step_loop_equals_eager_loop(mode, tmp_path):
    from vid2player3d_b200.tasks import PhysicsMVAEController, PhysicsMVAEControllerDual

    def tensors(obj):
        return {k: v for k, v in vars(obj).items() if isinstance(v, torch.Tensor)}
    outs = []
    for use_graph in (False, True):
        torch.manual_seed(5)
        N = 128
        cfg = controller_cfg(mode, N, tmp_path)
        cfg["env"]["motion_player"] = "stream+decoder"
        env = (PhysicsMVAEControllerDual if mode == "dual" else PhysicsMVAEController)(cfg, SIM_PARAMS, 1, "cuda", 0, True)
        env.reset()
        task, player = env._physics_player.task, env._mvae_player
        objs = [env, task, player, player.decoder]
        if use_graph:
            snaps = [{k: v.clone() for k, v in tensors(o).items()} for o in objs]
            env.enable_cuda_graph()                      # warm-up + capture advance the state: restore it
            for snap, o in zip(snaps, objs):
                for k, v in snap.items():
                    getattr(o, k).copy_(v)
        g = torch.Generator(device=DEV).manual_seed(3)
        for i in range(6):
            env.step(torch.clamp(torch.randn(N, env.num_actions, device=DEV, generator=g), -5, 5))
        torch.cuda.synchronize()
        outs.append({n: t.clone() for o in (env, task) for n, t in tensors(o).items()})
        outs[-1]["policy_out"] = env._low_level_policy.out.clone()
        outs[-1]["policy_x"] = env._low_level_policy.x.clone()
    for k in ("_dof_state", "_root_states", "_rigid_body_state", "obs_buf", "_target_dof_pos", "_pd_target_dof_pos", "rew_buf", "reset_buf",
              "progress_buf", "policy_out", "policy_x"):
        assert torch.equal(outs[0][k].view(torch.uint8), outs[1][k].view(torch.uint8)), k


@pytest.mark.parametrize("mode", ["single", "dual"])
def test_run_test_with_both_trained_policies_graphed_equals_eager(mode, tmp_path, monkeypatch):
    """MVAEControllerVis(Dual).run_test with a trained high-level policy and the trained low-level policy: the graphed loop exports
    the same arrays as the eager loop"""
    from vid2player3d_b200 import nn
    from vid2player3d_b200.tasks import MVAEControllerVis, MVAEControllerVisDual
    N, frames = 256, 60
    results = []
    for graph in (False, True):
        d = tmp_path / ("graph" if graph else "eager")
        d.mkdir()
        monkeypatch.chdir(d)
        torch.manual_seed(0)
        np.random.seed(0)
        cfg = controller_cfg(mode, N, tmp_path)
        cfg["env"].update(record=True, num_rec_frames=frames, num_eg=3, episodeLength=25)
        env = (MVAEControllerVisDual if mode == "dual" else MVAEControllerVis)(cfg, SIM_PARAMS, 1, "cuda", 0, True)
        assert isinstance(env._low_level_policy, nn.V2PPolicy)
        g = torch.Generator().manual_seed(9)
        P, obs_dim = (2 if mode == "dual" else 1), env.num_obs
        high = []
        for _ in range(P):
            dims = (obs_dim, 64, 64, 32, env.num_actions)
            high.append(dict(layers=[((torch.rand(dims[i + 1], dims[i], generator=g) * 2 - 1) / dims[i] ** 0.5,
                                      (torch.rand(dims[i + 1], generator=g) * 2 - 1) / dims[i] ** 0.5) for i in range(4)],
                             mean=None, rstd=None, clip=INF))
        pol = nn.V2PPolicy(high, N, DEV, clip_obs=5.0, clip_actions=1.0)
        torch.manual_seed(1)
        with pytest.raises(SystemExit):
            env.run_test(pol, frames + 5, graph=graph)
        assert graph == (env._test_graphs is not None)
        results.append(([dict(np.load(p)) for p in env.exported], [p.split("/")[-1] for p in env.exported]))
    (f0, p0), (f1, p1) = results
    assert p0 == p1 and len(f0) > 0
    for a, b in zip(f0, f1):
        assert a.keys() == b.keys()
        for k in a:
            np.testing.assert_array_equal(a[k], b[k], k)


def test_no_key_steps_with_zero_actions():
    """neither key: the default zero-residual policy, as before"""
    from vid2player3d_b200.tasks import PhysicsMVAEController
    N = 64
    env = PhysicsMVAEController(v2p_cfg(N), SIM_PARAMS, 1, "cuda", 0, True)
    task = env._physics_player.task
    assert task._obs_operand is None and not hasattr(env._low_level_policy, "forward_prepared")
    seen, step = [], task.step
    task.step = lambda a: (seen.append(a.clone()), step(a))
    env.reset()
    env.step(torch.zeros(N, env.num_actions, device=DEV))
    torch.cuda.synchronize()
    assert len(seen) == 1 and not bool(seen[0].any())
