"""ctypes binding of the vid2player entry points (include/b200env_v2p.h) - same library, no CPU fallback."""
import ctypes as C

import torch

from . import abi
from .native import _ptr, _stream, fill, lib

GRIP_NORMAL = {'eastern': (0.0, 1.0, 0.0), 'semi_western': (0.0, 2.0 ** -0.5, 2.0 ** -0.5)}
REWARD_TYPES = {'reach': 0, 'return': 1, 'return_w_estimate': 2}


def _check(rc):
    if rc != 0:
        raise RuntimeError(f"b200v2p error {rc}: {lib().b200v2p_last_error().decode()}")


def _c(t):
    assert t is None or (t.is_cuda and t.is_contiguous()), "tensors must be contiguous CUDA tensors"
    return _ptr(t)


def smpl_to_sim(root_pos, joint_rotmat, rest, parents, smpl_2_mujoco, dt, out, prev_root_pos=None, prev_rb_rot=None, prev_root_pos_update=None,
                target_root_pos_out=None, only_mask=None):
    """out: dict with root_rot[n,4] dof_pos[n,69] root_vel[n,3] root_ang_vel[n,3] dof_vel[n,69] rb_pos[n,24,3] rb_rot[n,24,4];
    prev_root_pos_update / target_root_pos_out: the root position of this call is also stored there (may alias prev_root_pos)"""
    num_rest = 1 if rest.dim() == 2 else int(rest.shape[0])      # rest [24,3] or [S,24,3]: env e uses shape e % S
    assert rest.shape[-2:] == (24, 3)
    d = fill(abi.V2PSmpl, dict(n=root_pos.shape[0], num_rest=num_rest, dt=dt),
             dict(out, root_pos=root_pos, joint_rotmat=joint_rotmat, rest=rest, parents=parents, smpl_2_mujoco=smpl_2_mujoco,
                  prev_root_pos=prev_root_pos, prev_rb_rot=prev_rb_rot, prev_root_pos_update=prev_root_pos_update,
                  target_root_pos_out=target_root_pos_out, only_mask=only_mask))
    _check(lib().b200v2p_smpl_to_sim(C.byref(d), _stream()))


def fix_head(rb_pos, rb_rot, ball_pos, root_pos, joint_rotmat, head_body=13):
    d = fill(abi.V2PHead, dict(n=rb_pos.shape[0], head_body=head_body),
             dict(rb_pos=rb_pos, rb_rot=rb_rot, ball_pos=ball_pos, root_pos=root_pos, joint_rotmat=joint_rotmat))
    _check(lib().b200v2p_fix_head(C.byref(d), _stream()))


def ball_aero(ball_states, has_bounce, has_bounce_now, bounce_pos, force, substeps, spin_scale, stride=None):
    d = fill(abi.V2PAero, dict(n=has_bounce.shape[0], stride=stride or ball_states.stride(0), substeps=substeps, spin_scale=spin_scale),
             dict(ball_states=ball_states, has_bounce=has_bounce, has_bounce_now=has_bounce_now, bounce_pos=bounce_pos, force=force))
    _check(lib().b200v2p_ball_aero(C.byref(d), _stream()))


def ball_reset(env_ids, pool_index, pool, ball_states, ball_pos, ball_vel, has_bounce, bounce_pos, has_contact, traj, stride=None):
    """ball_states: first ball row; `stride` floats between consecutive envs' ball rows (26 when the ball is actor 1 of 2)"""
    d = fill(abi.V2PBallReset, dict(n=env_ids.shape[0], stride=stride or ball_states.stride(0)),
             dict(env_ids=env_ids, pool_index=pool_index, pool=pool, ball_states=ball_states, ball_pos=ball_pos, ball_vel=ball_vel,
                  has_bounce=has_bounce, bounce_pos=bounce_pos, has_contact=has_contact, traj=traj))
    _check(lib().b200v2p_ball_reset(C.byref(d), _stream()))


def update_state(n, bodies_per_env, rigid_body_state, root_states, root_stride, ball_states, ball_stride, t, grip='eastern',
                 racket_body=24, wrist_body=22, only_mask=None):
    """grip / racket_body / wrist_body may be 2-sequences (dual_mode 'different': even envs, odd envs)"""
    pair = lambda v: (v[0], v[1], 1) if isinstance(v, (list, tuple)) else (v, v, 0)  # noqa: E731
    g0, g1, d0 = pair(grip)
    r0, r1, d1 = pair(racket_body)
    w0, w1, d2 = pair(wrist_body)
    s = fill(abi.V2PState, dict(n=n, bodies_per_env=bodies_per_env, ball_stride=ball_stride, root_stride=root_stride, racket_body=r0,
                                wrist_body=w0, grip_normal=GRIP_NORMAL[g0], dual=int(bool(d0 or d1 or d2)), racket_body2=r1, wrist_body2=w1,
                                grip_normal2=GRIP_NORMAL[g1]),
             dict(t, rigid_body_state=rigid_body_state, root_states=root_states, ball_states=ball_states, only_mask=only_mask))
    _check(lib().b200v2p_update_state(C.byref(s), _stream()))


def ball_in_estimate(contact_ids, ball_states, stride, table, params, traj, states_in, states_out):
    """TennisBallInEstimator.estimate for the balls of envs `contact_ids`; params [4,3] float64 (HEIGHT, VEL_X, VEL_Y, VSPIN)"""
    n = int(contact_ids.shape[0])
    assert table.shape[1:] == (50, 2) and traj.shape == (n, 50, 3) and states_in.shape == (n, 13) and states_out.shape == (n, 13)
    d = fill(abi.V2PInEst, dict(n=n, stride=stride, table_rows=table.shape[0],
                                params=torch.as_tensor(params, dtype=torch.float64).reshape(12).tolist()),
             dict(contact_ids=contact_ids, ball_states=ball_states, table=table, traj=traj, states_in=states_in, states_out=states_out))
    _check(lib().b200v2p_ball_in_estimate(C.byref(d), _stream()))


def controller_post(cfg, t):
    """cfg: dict of scalars (see abi.V2PCtrl); t: dict of tensors keyed like the struct's pointer fields (est_x/est_y may be None).
    The high-level policy's operand row is written when t holds `policy_x` (bf16 [rows, policy_ld]); its scalars policy_dual,
    policy_clip_obs and policy_clip (one float, or one per player with policy_dual) come in cfg."""
    px = t.get("policy_x")
    if px is not None:
        assert px.dtype == torch.bfloat16 and px.dim() == 2, "policy_x: bf16 [rows, policy_ld]"
        assert px.shape[0] >= cfg["n"], "policy_x has fewer rows than there are envs"
        clip = cfg.get("policy_clip", float("inf"))
        cfg = dict(cfg, policy_ld=int(px.shape[1]), policy_clip_obs=cfg.get("policy_clip_obs", float("inf")),
                   policy_clip=clip if isinstance(clip, (list, tuple)) else (clip, clip))
    _check(lib().b200v2p_controller_post(C.byref(fill(abi.V2PCtrl, cfg, t)), _stream()))


def task_reset(cfg, t):
    """cfg: scalars of abi.V2PTaskReset (n, pool_size, ball_stride, bodies_per_env, reaction_nframes, target_mode, target_min/max);
    t: tensors keyed like the struct's pointer fields"""
    _check(lib().b200v2p_task_reset(C.byref(fill(abi.V2PTaskReset, cfg, t)), _stream()))


def eval_ball_stats(cfg, t):
    """cfg: n, pool_size; t: pool_cursor and either the draws form - the task reset's reset_reaction, row_served (int64 [pool_size]) -
    or the events form - the post launch's reset_recovery / has_contact / swing_type_cycle / est_bounce_in / est_bounce_pos /
    target_bounce_pos and buckets (int64 [pool_size, abi.BSTATS_COLS]); see include/b200env_v2p.h b200v2p_bstats_t"""
    _check(lib().b200v2p_eval_ball_stats(C.byref(fill(abi.V2PBallStats, cfg, t)), _stream()))


def eval_rally_stats(cfg, t):
    """cfg: n (even); t: the dual post launch's tar_action / has_contact / has_bounce / bounce_in / ball_pos / root_pos /
    swing_type_cycle / progress_buf, the pair state pair_open (bool [n/2]) / pair_hits (int64 [n/2, 2]) and the int64 accumulators
    totals [3], ends [2, 3], player [2, 3], shots_hist [abi.RSTATS_HIST]; see include/b200env_v2p.h b200v2p_rstats_t"""
    _check(lib().b200v2p_eval_rally_stats(C.byref(fill(abi.V2PRallyStats, cfg, t)), _stream()))


def actor_reset(cfg, t):
    """cfg: scalars of abi.V2PActorReset; racket_offset2 (with racket_parent2, default racket_parent) sets dual"""
    two = cfg.get("racket_offset2") is not None
    cfg = dict(cfg, dual=int(two), racket_parent2=cfg.get("racket_parent2", cfg["racket_parent"]) if two else None)
    _check(lib().b200v2p_actor_reset(C.byref(fill(abi.V2PActorReset, cfg, t)), _stream()))


def pre_step(cfg, t):
    """cfg: n, num_actions, num_latent, num_res_dof, random_walk_in_recovery, vae_action_scale, residual_dof_scale, seed;
    t: actions, tar_action, step_counter (int64 [1]), done_counter (int32 [1]), mvae_actions, res_dof_actions (or None)"""
    _check(lib().b200v2p_pre_step(C.byref(fill(abi.V2PPreStep, cfg, t)), _stream()))


def stream_gather(n, frames, advance, t, reseed_mask=None, seed=0):
    """t: clock (int64 [1]), done_counter (int32 [1]), offset [n] int64, ring_* / live buffers of include/b200env_v2p.h b200v2p_stream_t;
    reseed_mask (bool [n]): the masked envs draw a new offset and re-read their frame, the others are left alone"""
    s = fill(abi.V2PStream, dict(n=n, frames=frames, advance=advance, seed=seed), dict(t, reseed_mask=reseed_mask))
    _check(lib().b200v2p_stream_gather(C.byref(s), _stream()))


def eval_record(n, cap, t):
    """t: the source fields (joint_rot, root_pos, ball_pos, target_pos, phase, swing_type, tar_action), the rec_* buffers [n, cap, ...]
    and the row source: row_counter + done_counter (single) or progress_buf (dual); see include/b200env_v2p.h b200v2p_rec_t"""
    _check(lib().b200v2p_eval_record(C.byref(fill(abi.V2PRec, dict(n=n, cap=cap), t)), _stream()))


def eval_best(n, cap, num_eg, t):
    """t: tensors keyed like the pointer fields of b200v2p_best_t (include/b200env_v2p.h)"""
    _check(lib().b200v2p_eval_best(C.byref(fill(abi.V2PBest, dict(n=n, cap=cap, num_eg=num_eg), t)), _stream()))


BACKHAND_ITERS = 500    # optimize_two_hand_backhand(single=True): 500 Adam steps


def backhand_fix(problems, iters=BACKHAND_ITERS):
    """the two-hand backhand fix of include/b200env_v2p.h b200v2p_backhand_fix, every problem in one launch.  problems: dicts with
    joint_rot [T,24,3], phase [T], swing_type [>= T] int64, rest [24,3], righthand (bool) and optionally out [T,24,3] (joint_rot itself
    fixes in place); float tensors all float32 or all float64 on the device.  Returns (outs, losses): the fixed rows per problem and
    the [P,3] target / reg / smooth loss terms of the last evaluated step (NaN where none was)."""
    P = len(problems)
    assert P > 0
    dtype, dev = problems[0]["joint_rot"].dtype, problems[0]["joint_rot"].device
    assert dtype in (torch.float32, torch.float64)
    table, outs = (abi.V2PBhProb * P)(), []
    for q, pr in zip(table, problems):
        jr = pr["joint_rot"]
        out = pr.get("out")
        out = torch.empty_like(jr) if out is None else out
        T = int(jr.shape[0])
        for k, x in (("joint_rot", jr), ("phase", pr["phase"]), ("rest", pr["rest"]), ("out", out)):
            assert x.dtype == dtype and x.device == dev, k
        assert jr.shape[1:] == (24, 3) and out.shape == jr.shape and pr["rest"].shape == (24, 3) and pr["phase"].numel() >= T
        assert pr["swing_type"].dtype == torch.int64 and pr["swing_type"].device == dev
        q.joint_rot, q.phase, q.swing_type, q.rest, q.out = (_c(x) for x in (jr, pr["phase"], pr["swing_type"], pr["rest"], out))
        q.T, q.swing_type_len, q.righthand = T, pr["swing_type"].numel(), int(bool(pr["righthand"]))
        outs.append(out)
    S = 8 if dtype == torch.float64 else 4
    nbytes = abi.bhfix_scratch_bytes([q.T for q in table], S)
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    losses = torch.empty(P, 3, dtype=dtype, device=dev)
    f = abi.V2PBhFix(num_problems=P, iters=int(iters), problems=C.addressof(table), scratch=scratch.data_ptr(), scratch_bytes=nbytes,
                     losses=losses.data_ptr(), precision=int(S == 8))
    _check(lib().b200v2p_backhand_fix(C.byref(f), _stream()))
    return outs, losses


def ctrl_reset(mask, progress_buf, reset_buf, terminate_buf, num_reset_reaction, distance, num_reset):
    d = fill(abi.V2PCtrlReset, dict(n=mask.shape[0]),
             dict(mask=mask, progress_buf=progress_buf, reset_buf=reset_buf, terminate_buf=terminate_buf, num_reset_reaction=num_reset_reaction,
                  distance=distance, num_reset=num_reset))
    _check(lib().b200v2p_ctrl_reset(C.byref(d), _stream()))
