"""Several assets of one topology in one handle (include/b200env.h: b200env_create_assets), the parts that need no GPU: the batch
planner b200env_plan_assets, the de-duplication of HumanoidSMPLIM's cfg.env.motion_assets, and the validation of the assets and of
env_asset, which b200env_create_assets does before it touches a device."""
import numpy as np
import pytest

from vid2player3d_b200 import abi, model_compiler, native


def check_plan(env_asset, num_assets, B, rows, batches):
    """every env in exactly one batch, no batch mixes assets, counts <= B, sum ceil(n_a / B) batches, none for an empty asset,
    rows grouped by asset in ascending env order"""
    env_asset = np.asarray(env_asset)
    n = len(env_asset)
    assert sorted(rows.tolist()) == list(range(n))
    counts = np.bincount(env_asset, minlength=num_assets)
    assert len(batches) == int(sum(-(-c // B) for c in counts))
    seen = np.zeros(n, int)
    for a, first, cnt in batches.tolist():
        assert 1 <= cnt <= B
        envs = rows[first:first + cnt]
        assert (env_asset[envs] == a).all(), "a batch mixes assets"
        seen[envs] += 1
    assert (seen == 1).all(), "an env is in no batch or in two"
    for a in range(num_assets):
        mine = rows[np.flatnonzero(env_asset[rows] == a)]
        assert (np.diff(mine) > 0).all(), "envs of an asset are not in ascending order"
        assert (batches[:, 0] == a).sum() == -(-counts[a] // B)
    assert (np.diff(batches[:, 0]) >= 0).all()


@pytest.mark.parametrize("n,num_assets,B,seed", [(1, 1, 32, 0), (31, 1, 32, 1), (32, 2, 32, 2), (33, 3, 32, 3), (97, 4, 32, 4),
                                                  (8453, 3, 32, 5), (8192, 256, 32, 6), (50, 7, 8, 7), (5, 9, 32, 8)])
def test_plan_covers_every_env_once(n, num_assets, B, seed):
    rng = np.random.default_rng(seed)
    ea = rng.integers(0, num_assets, n)
    if num_assets > 2:
        ea[ea == 1] = 0                      # asset 1 without envs: it gets no batch
    rows, batches = native.plan_assets(ea, num_assets, B)
    check_plan(ea, num_assets, B, rows, batches)
    if num_assets > 2:
        assert not (batches[:, 0] == 1).any()
    rows2, batches2 = native.plan_assets(ea.copy(), num_assets, B)
    assert np.array_equal(rows, rows2) and np.array_equal(batches, batches2), "the plan is not deterministic"


def test_plan_of_counts_around_the_batch():
    """per-asset counts 1, B-1, B, B+1, interleaved: 1 + 1 + 1 + 2 batches, the last one of asset 3 holding 1 env"""
    B = 32
    ea = np.repeat(np.arange(4), [1, B - 1, B, B + 1])
    ea = ea[np.random.default_rng(0).permutation(len(ea))]
    rows, batches = native.plan_assets(ea, 4, B)
    check_plan(ea, 4, B, rows, batches)
    assert batches.tolist() == [[0, 0, 1], [1, 1, B - 1], [2, B, B], [3, 2 * B, B], [3, 3 * B, 1]]


def test_plan_rejects_bad_arguments():
    for ea, na, B, what in (([0, 4], 4, 32, "out of range"), ([-1], 2, 32, "out of range"), ([0], 0, 32, "num_assets"),
                            ([0], 1, 0, "envs_per_batch")):
        with pytest.raises(RuntimeError, match=what):
            native.plan_assets(ea, na, B)


def _packed(*names):
    ms = [abi.pack_model(model_compiler.load_compiled(n)) for n in names]
    return [m for m, _ in ms], [v for _, v in ms]


def test_create_assets_refuses_another_topology():
    """nadal's Racket hangs from another body than federer's: the pair is refused (before any device is needed)"""
    f, n = (model_compiler.load_compiled(x) for x in ("smpl_mesh_humanoid_federer", "smpl_mesh_humanoid_nadal"))
    assert list(f["parent"]) != list(n["parent"])
    models, verts = _packed("smpl_mesh_humanoid_federer", "smpl_mesh_humanoid_nadal")
    cfg = abi.make_cfg(f)
    with pytest.raises(RuntimeError, match="topology of asset 0"):
        native.Env(models, verts, cfg, 4, 0, env_asset=[0, 1, 0, 1])
    amass, _ = _packed("smpl_mesh_humanoid_amass_v1")
    with pytest.raises(RuntimeError, match="topology of asset 0"):       # 24 bodies against 25
        native.Env([models[0], amass[0]], [verts[0], _packed("smpl_mesh_humanoid_amass_v1")[1][0]], cfg, 2, 0, env_asset=[0, 1])


def test_create_assets_refuses_out_of_range_env_asset():
    models, verts = _packed("smpl_mesh_humanoid_federer", "smpl_mesh_humanoid_djokovic")
    cfg = abi.make_cfg(model_compiler.load_compiled("smpl_mesh_humanoid_federer"))
    for ea in ([0, 1, 2, 0], [0, -1, 0, 1]):
        with pytest.raises(RuntimeError, match="env_asset out of range"):
            native.Env(models, verts, cfg, 4, 0, env_asset=ea)
    with pytest.raises(RuntimeError, match="num_assets must be at least 1"):
        native.Env([], [], cfg, 0, 0, env_asset=[])


def test_motion_assets_are_deduplicated():
    """identical compiled assets (a file name and the dict it compiles to, or the same dict twice) are one asset; motions of one
    subject share it; another scale is another asset"""
    from vid2player3d_b200.tasks import HumanoidSMPLIM
    base = model_compiler.load_compiled("smpl_mesh_humanoid_amass_v1")
    big = dict(base)
    big["mass"] = base["mass"] * 1.2
    big["dyn_mass"] = base["dyn_mass"] * 1.2

    class Lib:
        def num_motions(self):
            return 6

    t = object.__new__(HumanoidSMPLIM)
    t.cfg = {"env": {"motion_assets": ["mjcf/smpl_mesh_humanoid_amass_v1.xml", dict(base), big, "smpl_mesh_humanoid_amass_v1.xml",
                                       dict(big), "smpl_mesh_humanoid_federer.xml"]}}
    t._motion_lib, t.kp_scale, t.kd_scale = Lib(), 1.0, 1.0
    models, of_motion = t._motion_asset_models()
    assert of_motion.tolist() == [0, 0, 1, 0, 1, 2] and len(models) == 3
    t.cfg["env"]["motion_assets"] = t.cfg["env"]["motion_assets"][:5]
    with pytest.raises(ValueError, match="5 entries for 6 motions"):
        t._motion_asset_models()
