/* b200nn.h - C ABI of libb200nn.so: the two network forwards that sit on either side of the physics in the vid2player
 * rollout step (SURVEY.md 8f-1), as hand-written sm_90a GEMMs (wgmma.mma_async, register accumulators, TMA operand loads).
 *
 * What it replaces in the reference (Python / PyTorch, no C ABI there):
 *   - the low-level policy forward of ImitatorPlayer.run_one_step (vid2player/players/im_player.py:187-202 ->
 *     embodied_pose/models/im_network_builder.py:191-230: running-mean-std normalisation, actor MLP
 *     734 -> 1024 -> 1024 -> 512 with ReLU (cfg/amass_im.yaml:87-88), linear `mu` head -> 75);
 *   - the MVAE mixture-of-experts decoder MixedDecoder.forward (vid2player/motion_vae/model.py:237-252), called once per
 *     env step by MVAEPlayer.step (players/mvae_player.py:184-199) under autocast (motion_vae/base.py:390-406):
 *     y = sum_e c_e (x W_e + b_e) per layer, c = softmax(gate(z, c)).  The reference materialises a blended weight matrix
 *     PER ENV (2.7 GB per layer at 8192 envs); here the E expert products of an output tile are E register accumulators and the
 *     blend is the epilogue.
 *
 * One `linear` object = one launch: out[:, col0 : col0 + N] = act( sum_e coef[:, e] * (A W_e^T + bias_e) ).
 * All pointers are DEVICE pointers; operands are bf16 (K contiguous), accumulation fp32, bias / coef fp32.
 * Shapes are padded by the caller (the Python binding does it): rows of A / out to a multiple of 128, K and the leading
 * dimensions to a multiple of 64 elements with zero padding, rows of W_e to a multiple of the output tile (128, or 32 when E > 1).
 * Functions return 0 on success; b200nn_last_error() describes the last failure.  No allocation and no host sync in `run`.
 *
 * Non-finite values propagate as in torch: ReLU, the output clamp and the cast clamp keep a NaN a NaN (torch.relu / torch.clamp
 * semantics), so an env whose observation blew up yields NaN actions instead of plausible clamped ones.
 */
#ifndef B200NN_H
#define B200NN_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define B200NN_ABI_VERSION 1

enum { B200NN_ACT_NONE = 0, B200NN_ACT_RELU = 1, B200NN_ACT_ELU = 2 };

typedef struct b200nn_linear* b200nn_linear_handle;

typedef struct b200nn_linear_desc {
  const void* a;      /* [rows_padded, lda] bf16 activations, K contiguous */
  int32_t lda;        /* elements, multiple of 64 */
  const void* w;      /* [num_experts, n_padded, ldw] bf16 weights (torch nn.Linear layout: out x in, per expert) */
  int32_t ldw;        /* elements, multiple of 64, >= k_padded */
  const float* bias;  /* [num_experts, n_padded] */
  const float* coef;  /* [rows, num_experts] blend coefficients (softmax of the gate), NULL when num_experts == 1 */
  void* out;          /* [rows_padded, ldo] bf16 (out_bf16 = 1) or float */
  int32_t ldo;        /* elements; bf16 output: multiple of 8 */
  int32_t out_col0;   /* first output column (the MVAE layers write behind the latent: col0 = 32); bf16 output: multiple of 8 */
  int32_t rows;       /* M: envs */
  int32_t n;          /* N: output features actually stored (<= n_padded) */
  int32_t n_padded;   /* rows of W per expert, multiple of the tile (128, or 32 when num_experts > 1) */
  int32_t k_padded;   /* K: multiple of 64; A[:, K:k_padded] and W[:, K:k_padded] must be zero */
  int32_t num_experts;/* 1 (plain linear layer) or 2..6 (mixture of experts) */
  int32_t act;        /* B200NN_ACT_* */
  int32_t out_bf16;   /* 1: bf16 output (feeds the next layer), 0: float output */
  float out_min, out_max; /* clamp applied after the activation (im_player.py:198 clamps the action to +-1); out_min >= out_max: none */
} b200nn_linear_desc_t;

int b200nn_abi_version(void);
const char* b200nn_last_error(void);

/* builds the TMA tensor maps of the operands (host side, once); the device buffers must stay where they are.  Returns -2 (before any
 * driver call) for a descriptor the kernel cannot run: num_experts outside 1..6, K / lda / ldw not padded to 64, n_padded not a
 * multiple of the tile or n outside 1..n_padded, rows < 1, bf16 ldo / out_col0 not multiples of 8, operands not 16-byte aligned,
 * out_col0 < 0, ldo < out_col0 + n, an unknown act. */
int b200nn_linear_create(const b200nn_linear_desc_t* desc, int32_t device, b200nn_linear_handle* out);
int b200nn_linear_destroy(b200nn_linear_handle h);
/* one launch on `stream` (CUDA-graph capturable) */
int b200nn_linear_run(b200nn_linear_handle h, void* stream);

/* dst[r, c] = bf16( clamp((src[r, c] - mean[c]) * rstd[c], lo, hi) ) for c < cols (mean / rstd may be NULL = identity);
 * the policy's input normalisation + clamp (im_player.py:187-190, RunningMeanStd) and the cast of a float buffer into a padded
 * bf16 operand.  Columns [cols, ld_dst) of dst are left untouched (zero from the allocation). */
int b200nn_cast_rows(const float* src, int32_t ld_src, void* dst_bf16, int32_t ld_dst, int32_t rows, int32_t cols, const float* mean,
                     const float* rstd, float lo, float hi, void* stream);

/* the cast for the rows whose mask entry (bool [rows]) is set only: the condition of the envs being reset <- their initial frame
 * (MVAEPlayer.reset, players/mvae_player.py:162-166) inside the mask-driven reset graph */
int b200nn_cast_rows_masked(const float* src, int32_t ld_src, void* dst_bf16, int32_t ld_dst, int32_t rows, int32_t cols, const uint8_t* row_mask,
                            float lo, float hi, void* stream);

/* the same cast of one float block into up to three bf16 buffers of the same leading dimension (dst2 / dst3 may be NULL): the latent z
 * is the first block of all three MixedDecoder layer inputs (`torch.cat((z, layer_out), dim=1)`, model.py:247) */
int b200nn_cast_rows3(const float* src, int32_t ld_src, void* dst_bf16, void* dst2_bf16, void* dst3_bf16, int32_t ld_dst, int32_t rows,
                      int32_t cols, void* stream);

/* coef[r, :] = softmax( h[r, :k] W^T + b ) over num_experts outputs: last layer of the MixedDecoder gate (model.py:226-235) */
int b200nn_gate_softmax(const void* h_bf16, int32_t ldh, int32_t k, const float* w, const float* b, int32_t num_experts, float* coef,
                        int32_t rows, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200NN_H */
