"""The physics launch of b200env_step (step_kernel_packed<true> by default: configs 2, 3 and 5) at every batch position.

The float64 / float32 physics parity tests of test_gpu_parity.py run b200env_physics_only, a separate test launch: a non-persistent
grid, the whole DevBlob staged in shared memory, caller arrays and its own prologue and epilogue.  It shares only the control step
(control_step_packed) with the step.  The tests here drive the real step through the task classes - HumanoidSMPLIM on amass_v1
(task_mode 0, residual wrench on) and HumanoidSMPLIMMVAE on federer (racket, ball, ball-body contact against the hull faces,
residual wrench on) - from chosen states written into the task's state rows, and read back every row the physics launch writes.

1. Position invariance, exact.  An env's rows must not depend on where it runs: its round (batch b of the hand-out order runs in
   round b // G), its CTA batch, its warp, its env slot g in the warp, or whether it is in the ragged last batch.  B (envs per CTA
   batch) and G (the persistent grid) come from b200env_physics_launch_shape.  Sizes around B and B G, natural order and seeded
   permutations, B200ENV_SORT=1, two env slices over one asset, and the fused (B200ENV_SPLIT=0) and tmem forms.
2. Parity of the launch at N = 2 B G + 5 with the float64 restatement (oracle/physics_ref.c), every env held to the bounds
   test_gpu_parity.py holds the test kernel to.
3. Negative controls (CPU): both comparators reject the mistakes a batch-indexing bug makes."""
import contextlib
import os

import numpy as np
import pytest
import torch

EPW = 4              # envs per warp of the packed physics kernels (csrc/packed.cuh): env slot g = position % EPW
RES = 31.85          # residual_force_scale of both workloads
SENTINEL = 12345.0   # rigid-body rows are filled with it, contact forces with -SENTINEL: the launch must overwrite every one
WORKLOADS = ("humanoid", "ball")
FORMS = {"default": {}, "sort": {"B200ENV_SORT": "1"}, "fused": {"B200ENV_SPLIT": "0"}, "tmem": {"B200ENV_KERNEL": "tmem"}}
HUMANOID_KINDS = ("free flight", "settled contact", "deep contact")
BALL_KINDS = ("ball at the racket, front", "ball at the racket, back", "ball onto the ground", "ball far away", "ball at the body",
              "deep contact, ball far away")


# ------------------------------------------------------------------------------------------------ layouts and comparators (CPU)
def position(p, B, G):
    """(round, CTA batch, warp, g) of launch position p"""
    b = p // B
    return int(b // G), int(b), int((p % B) // EPW), int(p % EPW)


class Layout:
    """where each pool env ran: pos[e] = launch position of pool env e (-1 = not in this launch)"""

    def __init__(self, label, B, G, pos):
        self.label, self.B, self.G, self.pos = label, B, G, np.asarray(pos)

    @classmethod
    def of_perm(cls, label, B, G, perm, n_pool):
        pos = np.full(n_pool, -1)
        pos[perm] = np.arange(len(perm))
        return cls(label, B, G, pos)

    def where(self, e):
        return position(int(self.pos[e]), self.B, self.G)


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint8).reshape(a.shape[0], -1)


def assert_identical(ref, got, envs, ref_layout, got_layout):
    """ref, got: name -> array [pool envs, ...]; the rows of `envs` must agree bit for bit"""
    envs = np.asarray(envs)
    diff = {k: (_bits(ref[k][envs]) != _bits(got[k][envs])).any(1) for k in ref}
    bad = np.logical_or.reduce(list(diff.values()))
    if not bad.any():
        return
    lines = []
    for i in np.flatnonzero(bad)[:6]:
        e = int(envs[i])
        names = [k for k in ref if diff[k][i]]
        d = max(float(np.abs(ref[k][e].astype(np.float64) - got[k][e].astype(np.float64)).max()) for k in names)
        lines.append(f"  env {e}: {', '.join(names)} differ (max |diff| {d:.3e}); (round, batch, warp, g) {ref_layout.where(e)} in "
                     f"{ref_layout.label}, {got_layout.where(e)} in {got_layout.label}")
    raise AssertionError(f"{int(bad.sum())} of {len(envs)} envs differ between {ref_layout.label} and {got_layout.label}:\n" + "\n".join(lines))


def _layout_cost(perm, kinds, i, n, B, G, tail_lo, full_hi):
    """rule violations charged to launch position i of the permuted layout (a round kept costs 100: see permuted_layout)"""
    e = perm[i]
    v = ((i % B) // EPW == (e % B) // EPW) + (i % EPW == e % EPW) + (i // B == e // B)
    if e >= tail_lo and (i >= full_hi or i % B in (0, B - 1)):
        v += 1
    k = kinds[e]
    if i > 0 and kinds[perm[i - 1]] == k:
        v += 1
    if i >= B * G and kinds[perm[i - B * G]] == k:
        v += 1
    if (i // B) // G == (e // B) // G:
        v += 100
    return v


def layout_problems(perm, kinds, B, G):
    """the rules a permuted layout of pool envs 0..n-1 (perm[p] = env at launch position p) must meet, as a list of violations:
    every env runs in another CTA batch, warp and env slot g; in another round too, except the fewest envs the round sizes force
    to stay (a partial last round: 2 max(round size) - n); the envs of the natural ragged tail run mid-batch in full batches; the
    envs at p - 1 (neighbour) and p - B G (same slot of the batch the CTA ran in the round before) are of another kind."""
    n = len(perm)
    p, e = np.arange(n), np.asarray(perm)
    assert np.array_equal(np.sort(e), p), "not a permutation"
    out = []
    for name, same in (("CTA batch", p // B == e // B), ("warp", (p % B) // EPW == (e % B) // EPW), ("slot g", p % EPW == e % EPW)):
        if same.any():
            out.append(f"{int(same.sum())} envs keep their {name}")
    rounds = (p // B) // G
    forced = max(0, 2 * int(np.bincount(rounds).max()) - n)
    kept = int((rounds == (e // B) // G).sum())
    if kept > forced:
        out.append(f"{kept} envs keep their round, {forced} must")
    tail_lo = (n // B) * B if n % B else n
    t = e >= tail_lo
    if (t & ((p >= (n // B) * B) | (p % B == 0) | (p % B == B - 1))).any():
        out.append("a tail env is not mid-batch in a full batch")
    k = np.asarray(kinds)[e]
    if (k[1:] == k[:-1]).any():
        out.append(f"{int((k[1:] == k[:-1]).sum())} neighbours of the same kind")
    if n > B * G and (k[B * G:] == k[:-B * G]).any():
        out.append(f"{int((k[B * G:] == k[:-B * G]).sum())} envs of the same kind as the env of their slot one round before")
    return out


def _broken(perm, kinds, B, G):
    """per launch position: does it break one of layout_problems' rules other than the round (vectorised _layout_cost)"""
    n = len(perm)
    p, e = np.arange(n), perm
    bad = ((p % B) // EPW == (e % B) // EPW) | (p % EPW == e % EPW) | (p // B == e // B)
    bad |= (e >= ((n // B) * B if n % B else n)) & ((p >= (n // B) * B) | (p % B == 0) | (p % B == B - 1))
    k = kinds[e]
    same = np.zeros(n, bool)
    same[1:] = k[1:] == k[:-1]
    bad |= same | np.roll(same, -1)
    if n > B * G:
        bg = np.zeros(n, bool)
        bg[B * G:] = k[B * G:] == k[:-B * G]
        bad |= bg | np.roll(bg, -B * G)
    return bad


def permuted_layout(n, B, G, kinds, seed):
    """a seeded layout of pool envs 0..n-1 that meets layout_problems' rules: rounds exchanged by a rotation of the round-sorted
    order (the fewest envs keep their round), then random swaps of two envs, kept when they do not raise the count of broken rules
    around the two positions (a round kept weighs 100, so no swap adds one), until none is left"""
    rng = np.random.default_rng(seed)
    rounds = (np.arange(n) // B) // G
    envs = np.concatenate([rng.permutation(np.flatnonzero(rounds == r)) for r in range(rounds.max() + 1)])
    slots = np.concatenate([rng.permutation(np.flatnonzero(rounds == r)) for r in range(rounds.max() + 1)])
    m = int(np.bincount(rounds).max())
    perm = np.empty(n, np.int64)
    perm[slots] = np.roll(envs, -m)
    kinds = np.asarray(kinds)
    pl, kl = perm.tolist(), kinds.tolist()
    tail_lo, full_hi = ((n // B) * B if n % B else n), (n // B) * B
    cost = lambda i: _layout_cost(pl, kl, i, n, B, G, tail_lo, full_hi)  # noqa: E731
    for _ in range(2000):
        bad = np.flatnonzero(_broken(np.array(pl), kinds, B, G))
        if not len(bad):
            break
        for i in rng.permutation(bad).tolist():
            for j in rng.integers(0, n, 16).tolist():
                s = {x for x in (i - 1, i, i + 1, i - B * G, i + B * G, j - 1, j, j + 1, j - B * G, j + B * G) if 0 <= x < n}
                before = sum(cost(x) for x in s)
                pl[i], pl[j] = pl[j], pl[i]
                after = sum(cost(x) for x in s)
                if after < before or (after == before and rng.random() < 0.3):
                    break
                pl[i], pl[j] = pl[j], pl[i]
    perm = np.array(pl)
    assert int((rounds == (perm // B) // G).sum()) == max(0, 2 * m - n)
    return perm


def parity_failures(k, o, cls, excused=None):
    """k, o: the launch's and the float64 restatement's root [n,13], q [n,nd], qd [n,nd] (and ball [n,13], hit [n] bool for the ball
    workload); cls [n]: 'free' | 'settled' | 'ball' | anything else (not held to a bound).  The bounds of test_gpu_parity.py:
    free flight q and root within 1e-5, qd 1e-3; settled contact q and root within 1e-4 for every env, qd 5e-4 at the 95th
    percentile and 2e-3 at most; ball workload: the same racket hit on >= 95 % of the envs, on those ball position 1e-4, ball
    velocity 2e-3, q 1e-4.  excused [n] bool: settled envs held to neither per-env bound, at most 0.5 % of the settled envs (the GPU test
    excuses an env only where b200env_physics_only, the launch test_gpu_parity.py validates, gives the same rows bit for bit: the
    excess is then the float32 arithmetic of the control step at that contact state, not the launch's).  Returns (failure messages,
    per-env errors)."""
    eq = np.abs(k["q"] - o["q"]).max(1)
    er = np.abs(k["root"] - o["root"]).max(1)
    ev = np.abs(k["qd"] - o["qd"]).max(1)
    err = dict(q=eq, root=er, qd=ev)
    fails = []

    def every(mask, name, e, tol, what):
        bad = np.flatnonzero(mask & ~(e < tol))      # NaN fails too
        if len(bad):
            fails.append(f"{what}: {name} error {np.nanmax(e[bad]):.3e} > {tol:g} on {len(bad)} envs, first {bad[:5].tolist()}")

    free, settled, ball = cls == "free", cls == "settled", cls == "ball"
    if excused is not None and excused.any():
        if (excused & ~settled).any() or excused.sum() > 0.005 * settled.sum():
            fails.append(f"{int(excused.sum())} excused envs: only settled ones, at most 0.5 % of {int(settled.sum())}")
        settled_all, settled = settled, settled & ~excused
    else:
        settled_all = settled
    every(free, "q", eq, 1e-5, "free flight")
    every(free, "root", er, 1e-5, "free flight")
    every(free, "qd", ev, 1e-3, "free flight")
    every(settled, "q and root", np.maximum(eq, er), 1e-4, "settled contact")
    if settled.any():
        p95 = float(np.quantile(ev[settled_all], 0.95))
        if not p95 < 5e-4:
            fails.append(f"settled contact: qd error {p95:.3e} at the 95th percentile > 5e-4")
        every(settled, "qd", ev, 2e-3, "settled contact")
    if ball.any():
        same = ball & (k["hit"] == o["hit"])
        frac = same.sum() / ball.sum()
        if frac < 0.95:
            fails.append(f"ball workload: the racket hit agrees on {frac:.3f} of the envs < 0.95")
        err["ball_p"] = np.abs(k["ball"][:, 0:3] - o["ball"][:, 0:3]).max(1)
        err["ball_v"] = np.abs(k["ball"][:, 7:10] - o["ball"][:, 7:10]).max(1)
        every(same, "ball position", err["ball_p"], 1e-4, "ball workload")
        every(same, "ball velocity", err["ball_v"], 2e-3, "ball workload")
        every(same, "q", eq, 1e-4, "ball workload")
    return fails, err


# ------------------------------------------------------------------------------------------------ negative controls (CPU)
def _toy_step(x):
    return dict(root=(x["root"] * np.float32(0.999) + np.float32(0.01)).astype(np.float32), dof=(x["dof"] * np.float32(1.001)).astype(np.float32),
                flag=(x["root"][:, 0] > 0).astype(np.uint8))


def _toy(n, seed=0):
    rng = np.random.default_rng(seed)
    x = dict(root=rng.normal(size=(n, 13)).astype(np.float32), dof=rng.normal(size=(n, 12)).astype(np.float32))
    return x, _toy_step(x)


def test_exact_comparator_rejects_misplaced_envs():
    """each row of the toy launch result is what a plausible batch-indexing bug would leave; assert_identical must name the env"""
    B, G = 16, 3
    n = 2 * B * G + 5
    x, ref = _toy(n)
    lay = Layout("natural order", B, G, np.arange(n))
    assert_identical(ref, {k: v.copy() for k, v in ref.items()}, np.arange(n), lay, lay)

    def bad(mutate, env):
        got = {k: v.copy() for k, v in ref.items()}
        mutate(got)
        with pytest.raises(AssertionError, match=rf"env {env}: "):
            assert_identical(ref, got, np.arange(n), lay, lay)

    def swap(got):                       # two envs of one warp (batch 0, warp 1) swapped
        for v in got.values():
            v[[4, 5]] = v[[5, 4]]
    bad(swap, 4)
    tail = n - 2                         # ragged last batch (round 2), left at its input state
    bad(lambda got: [got[k].__setitem__(tail, x[k][tail]) for k in x], tail)
    r2 = B * G + 3                       # an env of the second round ...
    assert position(r2, B, G)[0] == 1
    twice = _toy_step({k: v[r2:r2 + 1] for k, v in ref.items() if k != "flag"})
    bad(lambda got: [got[k].__setitem__(r2, twice[k][0]) for k in twice], r2)                      # ... stepped twice
    bad(lambda got: got["root"].__setitem__((r2, 5), np.nextafter(got["root"][r2, 5], np.float32(np.inf))), r2)   # ... 1 ulp off
    bad(lambda got: got["flag"].__setitem__(r2, 1 - got["flag"][r2]), r2)                        # ... one ball flag flipped
    # the permuted layout: a correct result is accepted, a result stored at the natural positions is not
    kinds = np.arange(n) % 3
    perm = permuted_layout(n, B, G, kinds, seed=1)
    assert layout_problems(perm, kinds, B, G) == []
    launched = _toy_step({k: v[perm] for k, v in x.items()})
    by_env = {k: np.empty_like(v) for k, v in launched.items()}
    for k, v in launched.items():
        by_env[k][perm] = v
    pl = Layout.of_perm("permuted", B, G, perm, n)
    assert_identical(ref, by_env, np.arange(n), lay, pl)
    with pytest.raises(AssertionError, match=r"in natural order, \(\d+, \d+, \d+, \d+\) in permuted"):
        assert_identical(ref, launched, np.arange(n), lay, pl)


@pytest.mark.parametrize("B,G,n", [(32, 132, 2 * 32 * 132 + 5), (32, 132, 8195), (28, 132, 2 * 28 * 132 + 5), (16, 3, 51)])
def test_permuted_layout_meets_its_rules(B, G, n):
    """the permutations the GPU tests use: every rule of layout_problems holds (with a partial last round, exactly the envs the
    round sizes force stay in their round); a layout that breaks a rule is reported"""
    kinds = np.arange(n) % 3
    perm = permuted_layout(n, B, G, kinds, seed=7)
    assert layout_problems(perm, kinds, B, G) == []
    assert layout_problems(np.arange(n), kinds, B, G) != []
    same_slot = perm.copy()
    j = int(np.flatnonzero(perm % EPW == 0)[0])                  # an env of slot g = 0 moved to position 0
    same_slot[[0, j]] = same_slot[[j, 0]]
    assert any("slot g" in s for s in layout_problems(same_slot, kinds, B, G))


def _toy_parity(n=800, seed=3):
    rng = np.random.default_rng(seed)
    o = dict(root=rng.normal(size=(n, 13)), q=rng.normal(size=(n, 69)), qd=rng.normal(size=(n, 69)), ball=rng.normal(size=(n, 13)),
             hit=rng.random(n) < 0.4)
    k = {key: (v + rng.uniform(-1, 1, v.shape) * 1e-7 if v.dtype != bool else v.copy()) for key, v in o.items()}
    cls = np.array(["free", "settled", "ball", "deep"])[np.arange(n) % 4]
    return k, o, cls


def test_parity_comparator_rejects_one_env_just_outside_a_bound():
    k, o, cls = _toy_parity()
    assert parity_failures(k, o, cls)[0] == []
    cases = [("free", "q", 0, 1e-5), ("free", "root", 2, 1e-5), ("free", "qd", 1, 1e-3), ("settled", "q", 3, 1e-4),
             ("settled", "root", 5, 1e-4), ("settled", "qd", 7, 2e-3), ("ball", "ball", 0, 1e-4), ("ball", "ball", 8, 2e-3),
             ("ball", "q", 4, 1e-4)]
    for c, key, col, tol in cases:
        e = int(np.flatnonzero((cls == c) & (c != "ball" or k["hit"] == o["hit"]))[3])
        for f, ok in ((0.99, True), (1.01, False)):
            kk = {x: v.copy() for x, v in k.items()}
            kk[key][e, col] = o[key][e, col] + f * tol
            fails = parity_failures(kk, o, cls)[0]
            assert (fails == []) == ok, (c, key, col, f, fails)
            if not ok:
                assert any(f"first [{e}" in s for s in fails), fails
    # an excused settled env is not held to the per-env bounds; excusing more than 0.5 % of them, or another kind, fails
    s_env = np.flatnonzero(cls == "settled")
    kk = {x: v.copy() for x, v in k.items()}
    kk["q"][s_env[0], 0] += 1e-3
    assert parity_failures(kk, o, cls)[0] != []
    assert parity_failures(kk, o, cls, excused=np.isin(np.arange(len(cls)), s_env[:1]))[0] == []
    assert parity_failures(kk, o, cls, excused=np.isin(np.arange(len(cls)), s_env[:2]))[0] != []
    assert parity_failures(k, o, cls, excused=np.isin(np.arange(len(cls)), np.flatnonzero(cls == "free")[:1]))[0] != []
    # deep-contact envs are reported, not bounded
    kk = {x: v.copy() for x, v in k.items()}
    kk["q"][np.flatnonzero(cls == "deep")[0], 0] += 1.0
    assert parity_failures(kk, o, cls)[0] == []
    # settled: the 95th percentile of qd, and the racket hit on 95 % of the ball envs
    kk = {x: v.copy() for x, v in k.items()}
    s = np.flatnonzero(cls == "settled")
    kk["qd"][s[: len(s) // 10], 0] += 6e-4
    assert any("95th percentile" in f for f in parity_failures(kk, o, cls)[0])
    kk = {x: v.copy() for x, v in k.items()}
    b = np.flatnonzero(cls == "ball")
    kk["hit"][b[: len(b) // 15]] ^= True
    assert any("racket hit agrees" in f for f in parity_failures(kk, o, cls)[0])


# ------------------------------------------------------------------------------------------------ GPU: tasks, pools, launches
@contextlib.contextmanager
def _form(form):
    """the environment variables b200env_create reads, for the handles created inside the block"""
    names = ("B200ENV_SORT", "B200ENV_SPLIT", "B200ENV_KERNEL")
    old = {k: os.environ.pop(k, None) for k in names}
    os.environ.update(FORMS[form])
    try:
        yield
    finally:
        for k in names:
            os.environ.pop(k, None)
            if old[k] is not None:
                os.environ[k] = old[k]


_cache = {}


def _memo(key, fn):
    if key not in _cache:
        _cache[key] = fn()
    return _cache[key]


def _flat():
    from vid2player3d_b200 import model_compiler, motion_lib
    return _memo("flat", lambda: motion_lib.synthetic(model_compiler.load_compiled("smpl_mesh_humanoid_amass_v1"), num_motions=4,
                                                      num_frames=60, seed=1))


def _ball_cfg(n, handles):
    from helpers import v2p_cfg
    from vid2player3d_b200 import ball as ball_data
    pool = _memo("ball_pool", lambda: ball_data.synthetic_pool(2048, seed=10, spin_scale=5))
    v2p = dict(v2p_cfg(n)["env"]["vid2player"], ball_pool=pool)
    asset = "smpl_mesh_humanoid_federer.xml"
    return {"env": dict(numEnvs=n, episodeLength=300, residual_force_scale=RES, is_train=True,
                        asset=dict(assetFileName=asset if handles == 1 else [asset] * handles),
                        plane=dict(staticFriction=1.0, dynamicFriction=1.0, restitution=0.5), vid2player=v2p, keyBodies=[], contactBodies=[]),
            "sim": {"substeps": 6}}


def _task(wl, n, form="default", handles=1):
    from helpers import SIM_PARAMS, im_cfg
    from vid2player3d_b200.tasks import HumanoidSMPLIM, HumanoidSMPLIMMVAE
    with _form(form):
        torch.manual_seed(0)
        if wl == "humanoid":
            t = HumanoidSMPLIM(im_cfg(n, _flat()), SIM_PARAMS, 1, "cuda", 0, True)
        else:
            t = HumanoidSMPLIMMVAE(_ball_cfg(n, handles), SIM_PARAMS, 1, "cuda", 0, True)
    assert t._env.kernel_form == ("tmem" if form == "tmem" else "packed")
    return t


def _probe(wl, form):
    return _memo(("probe", wl, form), lambda: _task(wl, 1, form))


def shape(wl, form):
    """(B, G) of the physics launch, from the library"""
    return _probe(wl, form)._env.physics_launch_shape


def _pool_size(wl):
    return max([8195] + [2 * b * g + 5 for b, g in (shape(wl, f) for f in FORMS)])


def _pool(wl):
    return _memo(("pool", wl), lambda: _make_pool(wl, _pool_size(wl)))


def _make_pool(wl, P):
    """seeded input states of P envs, float32 as they are written into the rows; kind = the state builder of each env"""
    from test_gpu_parity import ball_scene, phys_states, settled_contact_states
    rng = np.random.default_rng(2024)
    if wl == "humanoid":
        kind = np.arange(P) % 3
        parts = [phys_states(None, int((kind == 0).sum()), 101, False), settled_contact_states(_probe(wl, "default"), None, int((kind == 1).sum()), 102),
                 phys_states(None, int((kind == 2).sum()), 103, True)]
        root, q, qd, tar, ext = (np.empty((P,) + p.shape[1:]) for p in parts[0])
        for kk, part in enumerate(parts):
            for dst, src in zip((root, q, qd, tar, ext), part):
                dst[kind == kk] = src
        act = np.concatenate([tar, ext / RES], 1)
        pool = dict(root=root, q=q, qd=qd, act=act)
    else:
        t = _probe(wl, "default")
        root, q, qd, tar, ext, ball = ball_scene(t._model, t._model_struct, t._verts, t._cfg_struct, P, 31)
        kind = np.arange(P) % 4
        at_body = np.arange(P) % 5 == 4          # thrown at the body, as in test_tmem_ball_physics_bit_identical_to_packed
        kind[at_body] = 4
        ball[at_body, 0:3] = root[at_body, 0:3] + rng.normal(0, 0.15, (at_body.sum(), 3)) + np.array([0.0, 0.5, 0.0])
        ball[at_body, 7:10] = np.stack([rng.normal(0, 1, at_body.sum()), -rng.uniform(5, 15, at_body.sum()), rng.normal(0, 1, at_body.sum())], 1)
        deep = np.arange(P) % 7 == 6             # a humanoid in deep ground contact, the ball far away
        kind[deep] = 5
        d = phys_states(None, int(deep.sum()), 104, True)
        root[deep], q[deep], qd[deep], tar[deep], ext[deep] = d
        nd_ = int(deep.sum())
        ball[deep, 0:3] = np.stack([rng.uniform(-3, 3, nd_), rng.uniform(5, 9, nd_), rng.uniform(1, 2, nd_)], 1)
        ball[deep, 7:10] = np.stack([rng.normal(0, 2, nd_), -rng.uniform(20, 30, nd_), rng.normal(2, 2, nd_)], 1)
        a_dof = rng.normal(0, 0.1, q.shape)
        pool = dict(root=root, q=q, qd=qd, act=np.concatenate([a_dof, ext / RES], 1), ball=ball,
                    t_dof=(tar - a_dof), has_bounce=rng.random(P) < 0.5, hit_in=rng.random(P) < 0.5,
                    bounce_in=rng.uniform(-5, 5, (P, 3)))
    pool = {k: (v.astype(np.float32) if v.dtype == np.float64 else v) for k, v in pool.items()}
    pool["kind"] = kind
    return pool


def _load(t, wl, pool, perm):
    """write the pool envs perm[0..n-1] into launch positions 0..n-1 of the task's rows; returns the action rows"""
    n = len(perm)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a[perm])).to(t.device)  # noqa: E731
    if wl == "humanoid":
        t._root_states.copy_(T(pool["root"]))
        t.reset_buf.zero_()                      # the step zeroes the actions of envs flagged for reset
    else:
        rs = t._root_states.view(n, 2, 13)
        rs[:, 0] = T(pool["root"])
        rs[:, 1] = T(pool["ball"])
        t._target_dof_pos.copy_(T(pool["t_dof"]))
        t._has_bounce.copy_(T(pool["has_bounce"]))
        t._has_bounce_now.fill_(True)
        t._racket_hit_now.copy_(T(pool["hit_in"]))
        t._bounce_pos.copy_(T(pool["bounce_in"]))
    dof = t._dof_state.view(n, -1, 2)
    dof[..., 0] = T(pool["q"])
    dof[..., 1] = T(pool["qd"])
    rb = t._rigid_body_state.view(n, -1, 13)
    rb.fill_(SENTINEL)
    rb[:, 0, 3:7] = T(pool["root"][:, 3:7])      # the residual wrench is turned by the heading of rigid body 0
    t._contact_force_tensor.fill_(-SENTINEL)
    return T(pool["act"])


def _read(t, wl, n):
    g = lambda x: x.detach().cpu().numpy().reshape(n, -1).copy()  # noqa: E731
    out = dict(root=g(t._root_states), dof=g(t._dof_state), rb=g(t._rigid_body_state), cf=g(t._contact_force_tensor))
    if wl == "ball":
        for k in ("has_bounce", "has_bounce_now", "bounce_pos", "racket_hit_now"):
            out[k] = g(getattr(t, "_" + k))
    return out


def _by_env(rows, perm, P):
    out = {}
    for k, v in rows.items():
        out[k] = np.zeros((P,) + v.shape[1:], v.dtype)
        out[k][perm] = v
    return out


def _run(wl, form, perm):
    """one step of a fresh task of len(perm) envs with pool env perm[p] at position p; rows in pool order"""
    pool, n = _pool(wl), len(perm)
    t = _task(wl, n, form)
    a = _load(t, wl, pool, perm)
    l0 = t._env.launch_count
    t.step(a)
    torch.cuda.synchronize()
    per_step = (3 if wl == "humanoid" else 2) + (2 if form == "sort" else 0) if form != "fused" else 1
    assert t._env.launch_count - l0 == per_step
    rows = _read(t, wl, n)
    nb = t.num_bodies
    rb, cf = rows["rb"].reshape(n, -1, 13), rows["cf"].reshape(n, -1, 3)
    assert not (rb[:, :nb] == SENTINEL).any() and not (cf[:, :nb] == -SENTINEL).any(), "a body row was not written"
    pd = t._pd_target_dof_pos.cpu().numpy()
    P = len(pool["kind"])
    return _by_env(rows, perm, P), _by_env(dict(pd=pd), perm, P)["pd"]


def _reference(wl, form):
    """the natural-order launch at 2 B G + 5 envs: what every other layout of the form is compared with"""
    def run():
        B, G = shape(wl, form)
        n = 2 * B * G + 5
        rows, pd = _run(wl, form, np.arange(n))
        return dict(rows=rows, pd=pd, n=n, layout=Layout(f"natural order at N={n}", B, G, np.arange(len(_pool(wl)["kind"]))))
    return _memo(("ref", wl, form), run)


def _rounds(n, B, G):
    return -(-(-(-n // B)) // G)


@pytest.mark.gpu
@pytest.mark.parametrize("form", ["default", "sort", "fused", "tmem"])
@pytest.mark.parametrize("wl", WORKLOADS)
def test_rows_do_not_depend_on_the_launch_position(wl, form):
    """bit-identical rows for every env in every layout: sizes around the batch and the grid, and seeded permutations that move
    every env to another round, warp and slot.  B200ENV_SORT=1 hands the envs out by contact load and must match the default
    form; the fused and tmem forms are compared with themselves"""
    B, G = shape(wl, form)
    ref_form = "default" if form == "sort" else form
    ref = _reference(wl, ref_form)
    pool = _pool(wl)
    BG = B * G
    if form == "default":
        sizes = [1, 3, 4, 5, B - 1, B + 1, 2 * B + 3, BG - 1, BG + 1, BG + 3, 2 * BG + 5, 8195]
        permuted = [2 * BG + 5, 8195]
        assert 8195 > BG and 8195 % B, "8195 envs should take two rounds with a ragged last batch"
    elif form == "sort":
        sizes, permuted = [5, B + 1, BG + 1, 2 * BG + 5, 8195], [2 * BG + 5]
    else:
        sizes, permuted = [1, 5, B + 1, 2 * B + 3, BG - 1, BG + 1, 2 * BG + 5], [2 * BG + 5]
    print(f"\n{wl} / {form}: B = {B} envs per CTA batch, G = {G} CTAs; reference: {ref['layout'].label}")
    for n in sorted(set(sizes)):
        r = _rounds(n, B, G)
        print(f"  N = {n:5d}: {-(-n // B)} batches, {r} round(s), last batch {n - (n - 1) // B * B} of {B}")
        if n in (BG + 1, BG + 3, 2 * BG + 5):
            assert n > BG and r >= 2
        if form != "sort" and n == ref["n"]:
            continue
        rows, _ = _run(wl, form, np.arange(n))
        label = f"natural order at N={n}" + (" (position before the sort)" if form == "sort" else "")
        assert_identical(ref["rows"], rows, np.arange(n), ref["layout"], Layout(label, B, G, np.arange(len(pool["kind"]))))
    for seed, n in enumerate(permuted):
        perm = permuted_layout(n, B, G, pool["kind"][:n], seed=11 + seed)
        assert layout_problems(perm, pool["kind"][:n], B, G) == []
        rows, _ = _run(wl, form, perm)
        assert_identical(ref["rows"], rows, np.arange(n), ref["layout"], Layout.of_perm(f"permuted layout at N={n}", B, G, perm, len(pool["kind"])))
        print(f"  N = {n:5d}, permuted: bit-identical")


@pytest.mark.gpu
def test_env_slices_match_one_handle():
    """two handles over the even / odd rows with the same asset (b200env_set_env_slice, stride 2), B G + 2 envs each: two rounds
    per handle.  Stepping one handle gives its rows what the single-handle launch gave them and leaves every bit of the other
    slice's rows as it was."""
    wl = "ball"
    B, G = shape(wl, "default")
    ref = _reference(wl, "default")
    pool = _pool(wl)
    P = len(pool["kind"])
    n = 2 * (B * G + 2)
    assert n // 2 > B * G and n <= ref["n"]
    t = _task(wl, n, "default", handles=2)
    assert len(t._envs) == 2 and all(h.num_envs == n // 2 for h in t._envs)
    a = _load(t, wl, pool, np.arange(n))
    torch.cuda.synchronize()
    rows = [_by_env(_read(t, wl, n), np.arange(n), P)]
    for h in t._envs:
        h.step(a)
        torch.cuda.synchronize()
        rows.append(_by_env(_read(t, wl, n), np.arange(n), P))
    for k in range(2):
        mine, other = np.arange(k, n, 2), np.arange(1 - k, n, 2)
        local = np.full(P, -1)
        local[mine] = np.arange(len(mine))
        assert_identical(ref["rows"], rows[k + 1], mine, ref["layout"], Layout(f"env slice {k} of 2", B, G, local))
        assert_identical(rows[k], rows[k + 1], other, Layout(f"before slice {k}'s step", B, G, np.arange(P)),
                         Layout(f"after slice {k}'s step", B, G, np.arange(P)))
    print(f"\nenv slices: 2 x {n // 2} envs (B = {B}, G = {G}: {_rounds(n // 2, B, G)} rounds per handle), bit-identical")


@pytest.mark.gpu
@pytest.mark.parametrize("wl", WORKLOADS)
def test_launch_matches_float64_restatement(wl):
    """one control step at N = 2 B G + 5 against oracle/physics_ref.c, fed the PD targets the launch consumed (read back from
    _pd_target_dof_pos, and checked bit for bit against the clamp of step_prologue) and the residual wrench of the reference's
    pre_physics_step (ref_port.pre_physics).  Every env of a bounded kind is held to its bound."""
    from oracle import physics_ref, ref_port as R
    from vid2player3d_b200 import abi
    B, G = shape(wl, "default")
    ref = _reference(wl, "default")
    n = ref["n"]
    pool = {k: v[:n] for k, v in _pool(wl).items()}
    t = _probe(wl, "default")
    cfg = t._cfg_struct
    rows = {k: v[:n] for k, v in ref["rows"].items()}
    pd = ref["pd"][:n]
    lim = np.float32(cfg.pd_tar_lim)
    a = pool["act"][:, :69]
    base = a if wl == "humanoid" else pool["t_dof"] + a        # pd_mode 0: the action; 1: target dof + action
    assert np.array_equal(pd, np.maximum(np.minimum(base, pool["q"] + lim), pool["q"] - lim)), "PD targets differ from the clamp"
    f64 = lambda x: np.ascontiguousarray(x, np.float64)  # noqa: E731
    _, _, force, torque = R.pre_physics(f64(pool["act"]), np.zeros(n), f64(pool["q"]), f64(pool["root"][:, 3:7]), 69, float(lim),
                                        float(cfg.res_force_scale), float(cfg.res_torque_scale))
    o = dict(root=f64(pool["root"]), q=f64(pool["q"]), qd=f64(pool["qd"]))
    ext = f64(np.concatenate([force, torque], 1))
    if wl == "humanoid":
        physics_ref.control_step(t._model_struct, t._verts, cfg, o["root"], o["q"], o["qd"], f64(pd), ext)
        cls = np.array(["free", "settled", "deep"])[pool["kind"]]
        k = dict(root=rows["root"].astype(np.float64))
    else:
        o["ball"], hits = f64(pool["ball"]), np.zeros(n, np.int32)
        physics_ref.set_hull_faces(*abi.pack_faces(t._model, t._verts))
        try:
            physics_ref.control_step(t._model_struct, t._verts, cfg, o["root"], o["q"], o["qd"], f64(pd), ext, ball=o["ball"], hits=hits)
        finally:
            physics_ref.clear_hull_faces()
        o["hit"] = hits > 0
        cls = np.where(pool["kind"] == 5, "deep", "ball")
        k = dict(root=rows["root"][:, :13].astype(np.float64), ball=rows["root"][:, 13:26].astype(np.float64), hit=rows["racket_hit_now"][:, 0] != 0)
        assert o["hit"].sum() >= n // 8, "the workload must have racket impacts"
    dof = rows["dof"].reshape(n, 69, 2).astype(np.float64)
    k["q"], k["qd"] = dof[..., 0], dof[..., 1]
    excused = None
    if wl == "humanoid":
        # settled envs outside the bound: run b200env_physics_only (the launch test_gpu_parity.py validates) on their inputs; an env
        # is excused when it gives the same rows bit for bit.  Their residual wrench is zero, so both launches see the same inputs.
        out = (cls == "settled") & ~((np.maximum(np.abs(k["q"] - o["q"]).max(1), np.abs(k["root"] - o["root"]).max(1)) < 1e-4) &
                                      (np.abs(k["qd"] - o["qd"]).max(1) < 2e-3))
        idx = np.flatnonzero(out)
        if len(idx):
            assert not pool["act"][idx, 69:].any()
            T = lambda a: torch.tensor(np.ascontiguousarray(a), dtype=torch.float32, device="cuda:0")  # noqa: E731
            r, q, qd = T(pool["root"][idx]), T(pool["q"][idx]), T(pool["qd"][idx])
            rb = torch.zeros(len(idx), 24, 13, device="cuda:0")
            cf = torch.zeros(len(idx), 24, 3, device="cuda:0")
            t._env.physics_only(r, q, qd, T(pd[idx]), T(np.zeros((len(idx), 6))), rb, cf)
            torch.cuda.synchronize()
            same = (np.array_equal(r.cpu().numpy(), rows["root"][idx]) and
                    np.array_equal(np.stack([q.cpu().numpy(), qd.cpu().numpy()], -1).reshape(len(idx), -1), rows["dof"][idx]))
            print(f"\n{len(idx)} settled envs outside the bound {idx.tolist()}: b200env_physics_only gives the same rows bit for bit: {same}")
            if same:
                excused = out
    fails, err = parity_failures(k, o, cls, excused)
    e = np.arange(n)
    rnd, g = (e // B) // G, e % EPW
    kinds = HUMANOID_KINDS if wl == "humanoid" else BALL_KINDS
    print(f"\n{wl}: N = {n}, B = {B}, G = {G}; worst |error| against the float64 restatement")
    for kk in np.unique(pool["kind"]):
        m = pool["kind"] == kk
        cols = [c for c in ("q", "root", "qd", "ball_p", "ball_v") if c in err]
        for name, grp in (("round", rnd), ("g", g)):
            cells = "  ".join(f"{name} {v}: " + " ".join(f"{c} {err[c][m & (grp == v)].max():.1e}" for c in cols)
                              for v in np.unique(grp[m]))
            print(f"  {kinds[kk]:28s} by {name:5s} {cells}")
    if wl == "ball":
        print(f"  racket hits: {int(o['hit'].sum())} of {n}; the launch agrees on {float((k['hit'] == o['hit']).mean()):.4f}")
    assert not fails, "\n".join(fails)
