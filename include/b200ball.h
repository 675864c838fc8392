/* b200ball.h - C ABI of the offline tennis-ball data generators (SURVEY.md 8f-2), same library (libb200env.so).
 *
 * The reference builds three data products offline by stepping N free balls in Isaac Gym from Python:
 *   pool        [P,307]       launch pos/vel/spin + 100-frame trajectory   vid2player/utils/tennis_ball.py:221-394
 *   in-table    [rows,50,2]   incoming-ball table of dual mode             vid2player/utils/tennis_ball_in_estimator.py:82-140
 *   out-tables  [rows,60] + [rows,30,2]  outgoing-ball estimator           vid2player/utils/tennis_ball_out_estimator.py:21-121,208-258
 * Both loops (`simulate`, tennis_ball.py:113-218; `simulate_without_bounce`, tennis_ball_out_estimator.py:21-121) are one
 * launch each here: a thread per ball integrates the same ball model the env step kernel uses (csrc/b200env.cu: ball_substep)
 * and emits the samples / the grid-resampled rows directly in the reference's .npy layouts.
 * All pointers are device pointers; `stream` is a cudaStream_t; return 0 = ok, else b200env_last_error().
 * prec: 0 = float arrays (product), 1 = double arrays (parity instantiation of the same code, tests only).
 */
#ifndef B200BALL_H
#define B200BALL_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

typedef struct b200ball_sim {
  int32_t num_frames;       /* samples per trajectory (30 Hz frames for `simulate`) */
  int32_t control_freq_inv; /* sim steps per frame (2) */
  int32_t substeps;         /* substeps per sim step; > 2 also selects the 6R (else 4R) bounce-flag threshold (:185-188) */
  int32_t first_comp;       /* first position component written to traj (0: xyz, 1: yz like the in-table, 2: z) */
  float sim_dt;             /* 1/60 */
  float spin_scale;
  float gravity_z;
  float ball_mass, ball_inertia, ball_radius;
  float e_ground, mu_ground, bounce_threshold_velocity;
} b200ball_sim_t;

/* replaces simulate() (tennis_ball.py:113-218) for n balls:
 * traj [n, num_frames, 3 - first_comp], bounce_pos [n,3], bounce_idx [n] (int64, num_frames-1 when no bounce),
 * pass_net [n] (uint8).  launch_pos/vel [n,3], launch_vspin [n] (revolutions/s, sign = top(+)/back(-) spin). */
int b200ball_simulate(const b200ball_sim_t* cfg, int64_t n, int32_t prec, const void* launch_pos, const void* launch_vel,
                      const void* launch_vspin, void* traj, void* bounce_pos, int64_t* bounce_idx, uint8_t* pass_net, void* stream);

/* replaces simulate_without_bounce() (tennis_ball_out_estimator.py:21-121) for n rows launched straight out
 * (vel = (0, vel_h, vel_v)) over a world without ground; heights are relative to the launch height.
 * grid_x [ngx] / col_x [ngx]: the values of torch.arange(*TRAJ_X_RANGE) and the column each one is written to (int(x*2));
 * grid_y / col_y likewise (int(y*10)).  The grids may be unsorted and may map several values to one column: the columns are
 * written in grid order, so the last of them wins.  A column outside [0, nx) (resp. [0, ny)) is skipped, never stored: the
 * caller wraps the reference's negative Python indices first.  ngx, ngy in [0, 4096].
 * out_x [n, nx] and out_y [n, ny, 2] must be zero-initialised by the caller (columns no grid value maps to stay 0, like the
 * reference's torch.zeros); any base address works, 16-byte aligned ones take the vector stores.
 * cfg->num_frames = 60 -> (num_frames + 1) * control_freq_inv samples at 60 Hz (:55-57). */
int b200ball_out_rows(const b200ball_sim_t* cfg, int64_t n, int32_t prec, const void* vel_h, const void* vel_v, const void* vspin,
                      const float* grid_x, const int32_t* col_x, int32_t ngx, int32_t nx, const float* grid_y, const int32_t* col_y,
                      int32_t ngy, int32_t ny, void* out_x, void* out_y, void* stream);

#ifdef __cplusplus
}
#endif
#endif
