// b200nn.cu - libb200nn.so (C ABI: include/b200nn.h): the policy MLP and the MVAE mixture-of-experts decoder layers as
// hand-written sm_90a GEMMs.  One launch per layer:
//
//     out[:, col0 : col0 + N] = act( sum_e coef[:, e] * (A W_e^T + bias_e) )        bf16 operands, fp32 accumulate
//
// Structure of `linear_kernel` (persistent: the grid is the resident CTA slots, CTA c takes output tiles c, c + grid, ...; 2 consumer
// warpgroups + 1 producer warp per CTA; tiles of 128 rows x BN columns, column tiles fastest):
//   warp 8       TMA producer: cp.async.bulk.tensor tiles of A [128 x 64] and W [E x BN x 64] (128-byte swizzle) into a ring of
//                STAGES shared-memory stages, completion on mbarriers (expect_tx).  The ring runs across tile boundaries, so the next
//                tile's first k blocks load while the consumers run the current tile's epilogue.
//   warpgroups 0, 1  rows 0-63 / 64-127 of the tile: per 64-wide k block 4 wgmma.mma_async m64nNk16 (N = E * BN: one MMA covers every
//                expert, so the A slice leaves shared memory once per k16 step), operands straight from the swizzled stages, fp32
//                accumulators in registers.  One wgmma group stays in flight: after committing k block kb the warpgroup waits for kb - 1
//                and releases that stage on its `empty` mbarrier.  Epilogue from the registers: bias, expert blend, activation, clamp;
//                bf16 outputs leave as 16-byte stores (a quad shuffle gathers 8 consecutive columns of a row per thread).  The sampled
//                action (NOISE, last policy layer) adds sigma[col] * N(0, 1) from the counter-based generator (counter_rng.cuh) before
//                the clamp; the last CTA advances the device step counter, so a graph replay draws fresh noise.
// E = 1: BN = 128 columns, or 64 when the layer has n <= 64.  E > 1 (mixture of experts, vid2player/motion_vae/model.py:237-252): the
// tile is MOE_BN output columns x E experts = E * MOE_BN accumulator columns; the per-row softmax coefficients are applied in the
// epilogue in fp32, so the per-env blended weight matrices of the reference never exist.
// Every output element is the same sequence of k16 MMAs in ascending k, fp32 accumulation, then the same epilogue arithmetic, whatever
// the tile width, the MMA width or the tile-to-CTA mapping: the result of a row does not depend on the launch it is part of.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include "../../include/b200nn.h"
#include "counter_rng.cuh"

static thread_local char g_err[512] = "";
static int fail(int code, const char* msg) {
  snprintf(g_err, sizeof(g_err), "%s", msg);
  return code;
}
#define CUDA_OK(x)                                                                                   \
  do {                                                                                               \
    cudaError_t e_ = (x);                                                                            \
    if (e_ != cudaSuccess) {                                                                         \
      snprintf(g_err, sizeof(g_err), "%s failed: %s (%s:%d)", #x, cudaGetErrorString(e_), __FILE__, __LINE__); \
      return -100;                                                                                   \
    }                                                                                                \
  } while (0)

// ------------------------------------------------------------------------------------------ device helpers (PTX)
namespace {

// mixture-of-experts layers: output tile = MOE_BN columns x E experts (32 x 6 experts = 192 accumulator columns, 40 KB per stage)
constexpr int MOE_BN = 32;
constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;                        // 64 bf16 = 128 bytes = one swizzle-128B row
constexpr int MMA_K = 16;
constexpr int A_STAGE_BYTES = BLOCK_M * BLOCK_K * 2;
constexpr int NUM_THREADS = 288;                   // warpgroups 0, 1: MMA + epilogue; warp 8: TMA producer

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// bounded wait: a broken pipeline traps after ~2 s instead of hanging the GPU
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  const uint32_t addr = smem_u32(bar);
  const long long t0 = clock64();
  for (;;) {
    uint32_t done;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(addr), "r"(parity)
        : "memory");
    if (done) return;
    if (clock64() - t0 > 4000000000LL) __trap();   // surfaces as a launch failure on the host
  }
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(smem_u32(dst)),
               "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* map, int c0, int c1, int c2, uint64_t* bar) {
  asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(smem_u32(dst)),
               "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
// shared-memory matrix descriptor of a K-major bf16 tile written by TMA with CU_TENSOR_MAP_SWIZZLE_128B: rows of 128 bytes,
// 8-row swizzle atoms of 1024 bytes (stride byte offset), start address in 16-byte units, layout type 1 = SWIZZLE_128B (sm_90 wgmma
// descriptor; the leading byte offset is unused for swizzled K-major tiles).  A K step of 16 elements inside the 128-byte row advances
// the start address by 32 bytes: the hardware applies the swizzle to the computed address.
__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFF) >> 4);   // start address            bits [0,14)
  d |= (uint64_t)1 << 16;                    // leading byte offset      bits [16,30)
  d |= (uint64_t)(1024 >> 4) << 32;          // stride byte offset       bits [32,46)
  d |= (uint64_t)1 << 62;                    // layout type SWIZZLE_128B bits [62,64)
  return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// D[64 x N] (+)= A[64 x 16] B[N x 16]^T, bf16 operands K-major in shared memory, fp32 accumulators: N / 2 registers per thread
// (N = 64, 96, 128, 160, 192: the E = 1 tiles of 64 and 128 columns and E = 2..6 experts x MOE_BN).
// Register i of thread t of the warpgroup holds row 16 (t / 32) + (t % 32) / 4 + 8 ((i / 2) % 2), column 8 (i / 4) + 2 (t % 4) + i % 2.
template <int N> __device__ __forceinline__ void wgmma_bf16(float* d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate);
template <> __device__ __forceinline__ void wgmma_bf16<64>(float* d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
      "%24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
        "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]),
        "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]),
        "+f"(d[30]), "+f"(d[31])
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
template <> __device__ __forceinline__ void wgmma_bf16<96>(float* d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %50, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n96k16.f32.bf16.bf16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
      "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47}, %48, %49, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
        "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]),
        "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]),
        "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47])
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
template <> __device__ __forceinline__ void wgmma_bf16<128>(float* d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
      "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
        "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]),
        "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]),
        "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]),
        "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]),
        "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
template <> __device__ __forceinline__ void wgmma_bf16<160>(float* d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %82, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n160k16.f32.bf16.bf16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
      "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, "
      "%72, %73, %74, %75, %76, %77, %78, %79}, %80, %81, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
        "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]),
        "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]),
        "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]),
        "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]),
        "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]),
        "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79])
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
template <> __device__ __forceinline__ void wgmma_bf16<192>(float* d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %98, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n192k16.f32.bf16.bf16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
      "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, "
      "%72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95}, %96, %97, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
        "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]),
        "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]),
        "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]),
        "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]),
        "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]),
        "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
        "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]),
        "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95])
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}

// min / max that return NaN when an input is NaN (torch.relu / torch.clamp semantics; fminf / fmaxf would turn a NaN into the other
// operand and hide a blown-up env behind a plausible value).  One instruction each, like fminf / fmaxf; equal to them otherwise.
__device__ __forceinline__ float fmax_nan(float a, float b) { float r; asm("max.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b)); return r; }
__device__ __forceinline__ float fmin_nan(float a, float b) { float r; asm("min.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b)); return r; }
__device__ __forceinline__ float clamp_nan(float x, float lo, float hi) { return fmin_nan(fmax_nan(x, lo), hi); }

__device__ __forceinline__ float apply_act(float x, int act) {
  if (act == B200NN_ACT_RELU) return fmax_nan(x, 0.f);
  if (act == B200NN_ACT_ELU) return x > 0.f ? x : expm1f(x);   // F.elu, alpha = 1
  return x;
}


struct LinearParams {
  const float* bias;
  const float* coef;
  void* out;
  int ldo, out_col0, rows, n, n_padded, k_padded, act, out_bf16;
  float out_min, out_max;
  int n_tiles, tiles;                              // output tiles across the columns, in all
  const float* resid;                              // RES: x += resid[row * ld_resid + col] for col < resid_cols, before act and clamp
  int ld_resid, resid_cols;
  const float* noise_sigma;                        // NOISE: x += noise_sigma[col] * eps(seed, *noise_step, row * ldo + out_col0 + col),
  uint64_t noise_seed;                             // after the residual, before act and clamp
  int64_t* noise_step;
  unsigned int* noise_done;
};

__device__ __forceinline__ float finish(float x, const LinearParams& p) {
  x = apply_act(x, p.act);
  return p.out_min < p.out_max ? clamp_nan(x, p.out_min, p.out_max) : x;
}

__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

// two consecutive outputs (col, col + 1) of one row -> global memory; col is even
__device__ __forceinline__ void store2(const LinearParams& p, int row, int col, float a, float b) {
  if (row >= p.rows || col >= p.n) return;
  float* o = reinterpret_cast<float*>(p.out) + (size_t)row * p.ldo + p.out_col0 + col;
  if (col + 1 < p.n && ((uintptr_t)o & 7) == 0) {
    *reinterpret_cast<float2*>(o) = make_float2(a, b);
  } else {
    o[0] = a;
    if (col + 1 < p.n) o[1] = b;
  }
}

__device__ __forceinline__ uint32_t pick4(uint32_t a, uint32_t b, uint32_t c, uint32_t d, int i) {
  const uint32_t lo = (i & 1) ? b : a, hi = (i & 1) ? d : c;
  return (i & 2) ? hi : lo;
}
// v[j] = this lane's bf16 pair of 8-column group j (columns 8 j + 2 q, + 1, q = lane % 4) of one row, held by the 4 lanes of a quad.
// w = the 16 bytes of group q: word i is lane i's pair.  Round s swaps with lane q ^ s the pair that lane wants.
__device__ __forceinline__ void quad_transpose(const uint32_t (&v)[4], int q, uint32_t (&w)[4]) {
  uint32_t r[4];
#pragma unroll
  for (int s = 0; s < 4; s++) r[s] = __shfl_xor_sync(0xffffffffu, pick4(v[0], v[1], v[2], v[3], q ^ s), s);
#pragma unroll
  for (int i = 0; i < 4; i++) w[i] = pick4(r[0], r[1], r[2], r[3], q ^ i);
}

// Accumulator register i (of E * BN / 2) of this thread: expert i / (BN / 2), row row0 + 8 ((i / 2) % 2), column
// 8 ((i % (BN / 2)) / 4) + 2 (lane % 4) + i % 2 of the tile (columns n0 ..).  Taken 32 columns at a time.
template <int E, int BN, bool RES, bool NOISE>
__device__ __forceinline__ void epilogue(const float* acc, const float (&coef)[2][E], const float* sbias, const LinearParams& p, int row0,
                                         int n0, int lane, uint64_t step) {
  const int q = lane & 3;
#pragma unroll
  for (int h = 0; h < 2; h++) {
    const int row = row0 + 8 * h;
#pragma unroll
    for (int g = 0; g < BN / 32; g++) {
      float y[8];                                  // y[2 t + u]: column n0 + 8 (4 g + t) + 2 q + u
#pragma unroll
      for (int t = 0; t < 4; t++)
#pragma unroll
        for (int u = 0; u < 2; u++) {
          const int i = 4 * (4 * g + t) + 2 * h + u, col = n0 + 8 * (4 * g + t) + 2 * q + u;
          float x;
          if (E == 1) {
            x = acc[i] + sbias[col];
            if constexpr (RES) {
              if (col < p.resid_cols && row < p.rows) x += __ldg(p.resid + (size_t)row * p.ld_resid + col);
            }
            if constexpr (NOISE) {                 // sigma 0: no add at all, so the column keeps mu bit for bit (even -0)
              const float s = (row < p.rows && col < p.n) ? __ldg(p.noise_sigma + col) : 0.f;
              if (s != 0.f) x = fmaf(s, counter_normal(p.noise_seed, step, (uint64_t)row * p.ldo + p.out_col0 + col), x);
            }
          } else {
            x = 0.f;
#pragma unroll
            for (int e = 0; e < E; e++) x = fmaf(coef[h][e], acc[e * (BN / 2) + i] + sbias[e * p.n_padded + col], x);
          }
          y[2 * t + u] = finish(x, p);
        }
      if (p.out_bf16) {
        uint32_t v[4], w[4];
#pragma unroll
        for (int t = 0; t < 4; t++) {
          const __nv_bfloat162 b2 = __floats2bfloat162_rn(y[2 * t], y[2 * t + 1]);
          v[t] = *reinterpret_cast<const uint32_t*>(&b2);
        }
        quad_transpose(v, q, w);
        const int col = n0 + 32 * g + 8 * q;
        if (row < p.rows && col < p.n) {
          __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(p.out) + (size_t)row * p.ldo + p.out_col0 + col;   // 16-byte aligned
          if (col + 8 <= p.n) {
            *reinterpret_cast<uint4*>(o) = make_uint4(w[0], w[1], w[2], w[3]);
          } else {
#pragma unroll
            for (int c = 0; c < 8; c++)
              if (col + c < p.n) o[c] = __ushort_as_bfloat16((unsigned short)(w[c / 2] >> (16 * (c % 2))));
          }
        }
      } else {
#pragma unroll
        for (int t = 0; t < 4; t++) store2(p, row, n0 + 8 * (4 * g + t) + 2 * q, y[2 * t], y[2 * t + 1]);
      }
    }
  }
}

// E = 1: two CTAs per SM (64 accumulator registers per thread); E > 1: one CTA per SM, deeper ring (5 k blocks make a tile at K = 320)
template <int E, int BN> __host__ __device__ constexpr int stages() { return E == 1 ? (BN == 128 ? 3 : 4) : 5; }
template <int E> __host__ __device__ constexpr int ctas_per_sm() { return E == 1 ? 2 : 1; }
template <int E, int BN> __host__ __device__ constexpr int stage_bytes() { return A_STAGE_BYTES + E * BN * BLOCK_K * 2; }
// the stages, 1 KB for their alignment, the mbarriers, then every column's bias [E][n_padded]
template <int E, int BN> __host__ __device__ constexpr int bias_offset() { return stages<E, BN>() * stage_bytes<E, BN>() + 16 * stages<E, BN>(); }
template <int E, int BN> int smem_bytes(int n_padded) { return 1024 + bias_offset<E, BN>() + E * n_padded * 4; }

// RES (residual epilogue, the policy's last layer): launch bounds of one CTA per SM, a register budget that holds the residual's addressing
// without spilling; a layer with more tiles than CTA slots walks several tiles per CTA like any other.  NOISE (sampled action, also only on the last layer): the
// same budget for the counter-based normal; the last CTA to finish advances the step counter (producer and consumers both take part).
template <int E, int BN, bool RES = false, bool NOISE = false>
__global__ void __launch_bounds__(NUM_THREADS, (RES || NOISE) ? 1 : ctas_per_sm<E>())
linear_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmW, const LinearParams p) {
  constexpr int ACC = E * BN;                          // accumulator columns = the N of every wgmma
  constexpr int STAGES = stages<E, BN>();
  constexpr int STAGE_BYTES = stage_bytes<E, BN>();
  static_assert(ACC % 32 == 0 && ACC <= 256, "wgmma N");

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);   // swizzle-128B atoms: 1024-byte aligned
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES);
  uint64_t* empty = full + STAGES;
  float* sbias = reinterpret_cast<float*>(smem + bias_offset<E, BN>());

  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;
  const int nkb = p.k_padded / BLOCK_K;

  if (warp == 8 && lane == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmW) : "memory");
    for (int i = 0; i < STAGES; i++) { mbar_init(&full[i], 1); mbar_init(&empty[i], 2); }   // empty: one arrival per consumer warpgroup
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  for (int i = threadIdx.x; i < E * p.n_padded; i += NUM_THREADS) sbias[i] = __ldg(p.bias + i);
  __syncthreads();
  // Programmatic dependent launch: everything above ran while the previous layer was still finishing.  Every read of data a previous
  // kernel produced (the A operand, the blend coefficients) comes after griddepcontrol.wait = previous grid complete and visible.
  // A thread signals launch_dependents when it has no work left, so the next layer's CTAs take the slots this grid gives up.

  if (warp == 8) {
    if (lane == 0) {   // ---------------- TMA producer: (stage, phase) runs on across tiles
      asm volatile("griddepcontrol.wait;" ::: "memory");
      int s = 0;
      uint32_t ph = 0;
      for (int tile = blockIdx.x; tile < p.tiles; tile += gridDim.x) {
        const int m0 = tile / p.n_tiles * BLOCK_M, n0 = tile % p.n_tiles * BN;
        for (int kb = 0; kb < nkb; kb++) {
          mbar_wait(&empty[s], ph ^ 1);
          uint8_t* sa = smem + s * STAGE_BYTES;
          mbar_expect_tx(&full[s], STAGE_BYTES);
          tma_load_2d(sa, &tmA, kb * BLOCK_K, m0, &full[s]);
          tma_load_3d(sa + A_STAGE_BYTES, &tmW, kb * BLOCK_K, n0, 0, &full[s]);
          if (++s == STAGES) { s = 0; ph ^= 1; }
        }
      }
    }
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    if constexpr (NOISE) last_block_advance(p.noise_step, p.noise_done, 1);
    return;
  }
  // ---------------- consumers: warpgroup wg owns rows 64 wg .. + 63 of each tile
  const int wg = warp >> 2;
  const int t = threadIdx.x & 127;
  if (E > 1) asm volatile("griddepcontrol.wait;" ::: "memory");    // the coefficients come from the gate kernel before us
  uint64_t step = 0;
  if constexpr (NOISE) {                          // every launch before us is complete: the counter holds its final value
    asm volatile("griddepcontrol.wait;" ::: "memory");
    step = (uint64_t)__ldcg(p.noise_step);
  }
  int s = 0;
  uint32_t ph = 0;
  for (int tile = blockIdx.x; tile < p.tiles; tile += gridDim.x) {
    const int m0 = tile / p.n_tiles * BLOCK_M, n0 = tile % p.n_tiles * BN;
    float acc[ACC / 2];                            // the first wgmma of a tile ignores it (scale-d 0); zeroed per tile, the previous
#pragma unroll                                     // tile's values are dead once the epilogue has read them
    for (int i = 0; i < ACC / 2; i++) acc[i] = 0.f;
    const int row0 = m0 + 64 * wg + 16 * (t >> 5) + (lane >> 2);   // this thread's rows: row0 and row0 + 8
    float coef[2][E];
#pragma unroll
    for (int h = 0; h < 2; h++)
#pragma unroll
      for (int e = 0; e < E; e++) coef[h][e] = (E == 1) ? 1.f : (row0 + 8 * h < p.rows ? p.coef[(size_t)(row0 + 8 * h) * E + e] : 0.f);
    int prev = 0;
    for (int kb = 0; kb < nkb; kb++) {
      mbar_wait(&full[s], ph);
      const uint32_t a_addr = smem_u32(smem + s * STAGE_BYTES) + wg * (64 * 128), b_addr = smem_u32(smem + s * STAGE_BYTES) + A_STAGE_BYTES;
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BLOCK_K / MMA_K; k++)    // B row r <-> accumulator column r (expert-major)
        wgmma_bf16<ACC>(acc, wgmma_desc_sw128(a_addr + k * MMA_K * 2), wgmma_desc_sw128(b_addr + k * MMA_K * 2), (uint32_t)((kb | k) != 0));
      wgmma_commit();
      wgmma_wait<1>();                               // k block kb - 1 is done: its stage goes back to the producer
      if (kb > 0 && t == 0) mbar_arrive(&empty[prev]);
      prev = s;
      if (++s == STAGES) { s = 0; ph ^= 1; }
    }
    wgmma_wait<0>();
    if (t == 0) mbar_arrive(&empty[prev]);
    epilogue<E, BN, RES, NOISE>(acc, coef, sbias, p, row0, n0, lane, step);
  }
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  if constexpr (NOISE) last_block_advance(p.noise_step, p.noise_done, 1);
}

// ------------------------------------------------------------------------------------------ small SIMT kernels
// rows strided by the grid, columns by the block: coalesced, no integer division; up to three destinations of the same leading
// dimension get the same values (the latent block of the three MixedDecoder layer inputs)
__global__ void cast_rows_kernel(const float* __restrict__ src, int ld_src, __nv_bfloat16* __restrict__ dst, __nv_bfloat16* __restrict__ dst2,
                                 __nv_bfloat16* __restrict__ dst3, int ld_dst, int rows, int cols, const float* __restrict__ mean,
                                 const float* __restrict__ rstd, float lo, float hi, const uint8_t* __restrict__ row_mask) {
  for (int r = blockIdx.x * blockDim.y + threadIdx.y; r < rows; r += gridDim.x * blockDim.y) {
    if (row_mask && !row_mask[r]) continue;
    const float* s = src + (size_t)r * ld_src;
    const size_t o = (size_t)r * ld_dst;
    for (int c = threadIdx.x; c < cols; c += blockDim.x) {
      float x = s[c];
      if (mean) x = (x - __ldg(mean + c)) * __ldg(rstd + c);
      const __nv_bfloat16 v = __float2bfloat16_rn(clamp_nan(x, lo, hi));
      dst[o + c] = v;
      if (dst2) dst2[o + c] = v;
      if (dst3) dst3[o + c] = v;
    }
  }
}

// one warp per row: logits_e = h . w_e + b_e (k <= 256), softmax over E <= 8
__global__ void gate_softmax_kernel(const __nv_bfloat16* __restrict__ h, int ldh, int k, const float* __restrict__ w, const float* __restrict__ b,
                                    int E, float* __restrict__ coef, int rows) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= rows) return;
  float acc[8];
#pragma unroll
  for (int e = 0; e < 8; e++) acc[e] = 0.f;
  for (int j = lane; j < k; j += 32) {
    const float x = __bfloat162float(h[(size_t)row * ldh + j]);
#pragma unroll
    for (int e = 0; e < 8; e++)
      if (e < E) acc[e] = fmaf(x, w[e * k + j], acc[e]);
  }
#pragma unroll
  for (int e = 0; e < 8; e++)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc[e] += __shfl_xor_sync(0xffffffffu, acc[e], o);
  if (lane == 0) {
    float m = -1e30f, s = 0.f;
    for (int e = 0; e < E; e++) { acc[e] += b[e]; m = fmaxf(m, acc[e]); }
    for (int e = 0; e < E; e++) { acc[e] = expf(acc[e] - m); s += acc[e]; }
    for (int e = 0; e < E; e++) coef[(size_t)row * E + e] = acc[e] / s;
  }
}

// ------------------------------------------------------------------------------------------ host side
typedef CUresult (*encode_tiled_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                    const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

encode_tiled_fn get_encode() {
  static encode_tiled_fn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<encode_tiled_fn>(p);
  }
  return fn;
}

}  // namespace

// A/B switch (B200NN_CARVEOUT=1): every kernel of this library asks for the same L1 / shared-memory split (all shared), so that
// neighbouring launches never re-partition the SMs' L1.  Off by default: the small cast / gate kernels use their L1.
template <class K> static void prefer_max_shared(K kernel) {
  static const bool on = getenv("B200NN_CARVEOUT") && getenv("B200NN_CARVEOUT")[0] == '1';
  if (on) cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, (int)cudaSharedmemCarveoutMaxShared);
}

struct b200nn_linear {
  b200nn_linear_desc_t d;
  CUtensorMap tmA, tmW;
  LinearParams p;
  int device, bn, pdl, grid;
};

// prepare (at create, on the handle's device): the kernel's shared-memory size, and the grid = the CTA slots resident on the device
// at once, at most one per tile.  Otherwise launch.
template <int E, int BN, bool RES = false, bool NOISE = false> static int prepare_or_launch(b200nn_linear* h, cudaStream_t st, bool prepare) {
  if (prepare) {
    // the attribute is per kernel, not per handle: allow the device's limit, so that handles of other widths launch too
    int sms = 0, per_sm = 0, limit = 0;
    CUDA_OK(cudaDeviceGetAttribute(&limit, cudaDevAttrMaxSharedMemoryPerBlockOptin, h->device));
    cudaFuncAttributes fa;                         // the static shared memory (NOISE: the done flag) comes off the dynamic limit
    CUDA_OK(cudaFuncGetAttributes(&fa, linear_kernel<E, BN, RES, NOISE>));
    limit -= (int)fa.sharedSizeBytes;
    if (smem_bytes<E, BN>(h->d.n_padded) > limit) return fail(-2, "b200nn_linear_create: n_padded too large for the bias in shared memory");
    CUDA_OK(cudaFuncSetAttribute(linear_kernel<E, BN, RES, NOISE>, cudaFuncAttributeMaxDynamicSharedMemorySize, limit));
    prefer_max_shared(linear_kernel<E, BN, RES, NOISE>);
    CUDA_OK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, h->device));
    CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, linear_kernel<E, BN, RES, NOISE>, NUM_THREADS, smem_bytes<E, BN>(h->d.n_padded)));
    if (per_sm < 1) return fail(-3, "b200nn_linear_create: the GEMM kernel does not fit on an SM");
    h->grid = h->p.tiles < sms * per_sm ? h->p.tiles : sms * per_sm;
    return 0;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(h->grid, 1, 1);
  cfg.blockDim = dim3(NUM_THREADS, 1, 1);
  cfg.dynamicSmemBytes = smem_bytes<E, BN>(h->d.n_padded);
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = h->pdl ? 1 : 0;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  CUDA_OK(cudaLaunchKernelEx(&cfg, linear_kernel<E, BN, RES, NOISE>, h->tmA, h->tmW, h->p));
  return 0;
}

static int dispatch(b200nn_linear* h, cudaStream_t st, bool prepare) {
  switch (h->d.num_experts) {
    case 1:
      if (h->d.noise_sigma) {
        if (h->d.resid) return h->bn == 64 ? prepare_or_launch<1, 64, true, true>(h, st, prepare) : prepare_or_launch<1, 128, true, true>(h, st, prepare);
        return h->bn == 64 ? prepare_or_launch<1, 64, false, true>(h, st, prepare) : prepare_or_launch<1, 128, false, true>(h, st, prepare);
      }
      if (h->d.resid) return h->bn == 64 ? prepare_or_launch<1, 64, true>(h, st, prepare) : prepare_or_launch<1, 128, true>(h, st, prepare);
      return h->bn == 64 ? prepare_or_launch<1, 64>(h, st, prepare) : prepare_or_launch<1, 128>(h, st, prepare);
    case 2: return prepare_or_launch<2, MOE_BN>(h, st, prepare);
    case 3: return prepare_or_launch<3, MOE_BN>(h, st, prepare);
    case 4: return prepare_or_launch<4, MOE_BN>(h, st, prepare);
    case 5: return prepare_or_launch<5, MOE_BN>(h, st, prepare);
    case 6: return prepare_or_launch<6, MOE_BN>(h, st, prepare);
  }
  return fail(-2, "b200nn_linear: unsupported expert count");
}

extern "C" {

int b200nn_abi_version(void) { return B200NN_ABI_VERSION; }
int32_t b200nn_linear_desc_size(void) { return (int32_t)sizeof(b200nn_linear_desc_t); }
const char* b200nn_last_error(void) { return g_err; }

int b200nn_linear_create(const b200nn_linear_desc_t* d, int32_t device, b200nn_linear_handle* out) {
  if (!d || !out) return fail(-1, "b200nn_linear_create: null argument");
  if (!d->a || !d->w || !d->bias || !d->out) return fail(-1, "b200nn_linear_create: null operand pointer");
  const int E = d->num_experts;
  if (E < 1 || E > 6) return fail(-2, "b200nn_linear_create: num_experts must be 1..6");
  if (E > 1 && !d->coef) return fail(-1, "b200nn_linear_create: mixture layer needs the coefficient tensor");
  const int n_pad = E == 1 ? 128 : MOE_BN;          // padding contract of n_padded
  if (d->k_padded < BLOCK_K || d->k_padded % BLOCK_K || d->lda % BLOCK_K || d->ldw % BLOCK_K || d->lda < d->k_padded || d->ldw < d->k_padded)
    return fail(-2, "b200nn_linear_create: K and the leading dimensions must be padded to multiples of 64");
  if (d->n_padded < n_pad || d->n_padded % n_pad || d->n < 1 || d->n > d->n_padded) return fail(-2, "b200nn_linear_create: n_padded must be a multiple of the output tile");
  if (d->rows < 1) return fail(-2, "b200nn_linear_create: rows < 1");
  if (d->out_bf16 && (d->ldo % 8 || d->out_col0 % 8)) return fail(-2, "b200nn_linear_create: bf16 output needs ldo and out_col0 multiples of 8");
  if (d->out_col0 < 0) return fail(-2, "b200nn_linear_create: out_col0 < 0");
  if ((int64_t)d->ldo < (int64_t)d->out_col0 + d->n) return fail(-2, "b200nn_linear_create: ldo < out_col0 + n");
  if (d->act != B200NN_ACT_NONE && d->act != B200NN_ACT_RELU && d->act != B200NN_ACT_ELU) return fail(-2, "b200nn_linear_create: unknown activation");
  if (((uintptr_t)d->a | (uintptr_t)d->w | (uintptr_t)d->out) & 15) return fail(-2, "b200nn_linear_create: operands must be 16-byte aligned");
  if (d->resid || d->resid_cols || d->ld_resid) {
    if (!d->resid) return fail(-2, "b200nn_linear_create: resid_cols / ld_resid given without resid");
    if (E > 1) return fail(-2, "b200nn_linear_create: a residual needs a single-expert layer (num_experts == 1)");
    if (d->out_bf16) return fail(-2, "b200nn_linear_create: a residual needs a float output");
    if (d->resid_cols < 1 || d->resid_cols > d->n) return fail(-2, "b200nn_linear_create: resid_cols must be in 1..n");
    if (d->ld_resid < d->resid_cols) return fail(-2, "b200nn_linear_create: ld_resid < resid_cols");
    if ((uintptr_t)d->resid & 3) return fail(-2, "b200nn_linear_create: resid must be 4-byte aligned");
  }
  if (d->noise_sigma || d->noise_step || d->noise_done) {
    if (!d->noise_sigma) return fail(-2, "b200nn_linear_create: noise_step / noise_done given without noise_sigma");
    if (E > 1) return fail(-2, "b200nn_linear_create: noise (the sampled action) needs a single-expert layer (num_experts == 1)");
    if (d->out_bf16) return fail(-2, "b200nn_linear_create: noise (the sampled action) needs a float output");
    if (!d->noise_step) return fail(-2, "b200nn_linear_create: noise_sigma needs the device step counter noise_step");
    if (!d->noise_done) return fail(-2, "b200nn_linear_create: noise_sigma needs the done ticket noise_done");
    if (((uintptr_t)d->noise_sigma & 3) || ((uintptr_t)d->noise_step & 7) || ((uintptr_t)d->noise_done & 3))
      return fail(-2, "b200nn_linear_create: noise_sigma / noise_done must be 4-byte and noise_step 8-byte aligned");
  }
  encode_tiled_fn enc = get_encode();
  if (!enc) return fail(-3, "b200nn_linear_create: cuTensorMapEncodeTiled not available (no CUDA driver)");
  CUDA_OK(cudaSetDevice(device));
  b200nn_linear* h = new b200nn_linear();
  h->d = *d;
  h->device = device;
  h->bn = E > 1 ? MOE_BN : (d->n <= 64 ? 64 : 128);  // output tile width: a 64-column layer (the decoder gate) multiplies no padding
  {
    const char* e = getenv("B200NN_PDL");    // A/B switch: B200NN_PDL=0 launches the layers without programmatic dependent launch
    h->pdl = !(e && e[0] == '0');
  }
  const int rows_padded = (d->rows + BLOCK_M - 1) / BLOCK_M * BLOCK_M;
  {
    cuuint64_t dims[2] = {(cuuint64_t)d->k_padded, (cuuint64_t)rows_padded};
    cuuint64_t strides[1] = {(cuuint64_t)d->lda * 2};
    cuuint32_t box[2] = {BLOCK_K, BLOCK_M}, es[2] = {1, 1};
    CUresult r = enc(&h->tmA, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(d->a), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { delete h; snprintf(g_err, sizeof(g_err), "cuTensorMapEncodeTiled(A) failed: %d", (int)r); return -3; }
  }
  {
    cuuint64_t dims[3] = {(cuuint64_t)d->k_padded, (cuuint64_t)d->n_padded, (cuuint64_t)E};
    cuuint64_t strides[2] = {(cuuint64_t)d->ldw * 2, (cuuint64_t)d->ldw * 2 * (cuuint64_t)d->n_padded};
    cuuint32_t box[3] = {BLOCK_K, (cuuint32_t)h->bn, (cuuint32_t)E}, es[3] = {1, 1, 1};
    CUresult r = enc(&h->tmW, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(d->w), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { delete h; snprintf(g_err, sizeof(g_err), "cuTensorMapEncodeTiled(W) failed: %d", (int)r); return -3; }
  }
  const int n_tiles = (d->n + h->bn - 1) / h->bn;
  h->p = LinearParams{d->bias, d->coef, d->out, d->ldo, d->out_col0, d->rows, d->n, d->n_padded, d->k_padded, d->act, d->out_bf16, d->out_min, d->out_max,
                      n_tiles, rows_padded / BLOCK_M * n_tiles, d->resid, d->ld_resid, d->resid_cols,
                      d->noise_sigma, d->noise_seed, d->noise_step, d->noise_done};
  const int rc = dispatch(h, nullptr, true);
  if (rc) { delete h; return rc; }
  *out = h;
  return 0;
}

int b200nn_linear_destroy(b200nn_linear_handle h) {
  delete h;
  return 0;
}

int b200nn_linear_run(b200nn_linear_handle h, void* stream) {
  if (!h) return fail(-1, "b200nn_linear_run: null handle");
  return dispatch(h, (cudaStream_t)stream, false);
}

static int cast_launch(const float* src, int32_t ld_src, void* dst, void* dst2, void* dst3, int32_t ld_dst, int32_t rows, int32_t cols,
                       const float* mean, const float* rstd, float lo, float hi, void* stream, const uint8_t* row_mask = nullptr) {
  if (!src || !dst || rows < 1 || cols < 1 || cols > ld_src || cols > ld_dst) return fail(-2, "b200nn_cast_rows: bad argument");
  if ((mean == nullptr) != (rstd == nullptr)) return fail(-2, "b200nn_cast_rows: mean and rstd go together");
  const int tx = cols >= 256 ? 256 : (cols >= 128 ? 128 : (cols >= 64 ? 64 : 32));
  const dim3 block(tx, 256 / tx, 1);
  const int want = (rows + (int)block.y - 1) / (int)block.y;
  const int blocks = want < 132 * 16 ? want : 132 * 16;
  static bool once = (prefer_max_shared(cast_rows_kernel), true);
  (void)once;
  cast_rows_kernel<<<blocks, block, 0, (cudaStream_t)stream>>>(src, ld_src, reinterpret_cast<__nv_bfloat16*>(dst), reinterpret_cast<__nv_bfloat16*>(dst2),
                                                             reinterpret_cast<__nv_bfloat16*>(dst3), ld_dst, rows, cols, mean, rstd, lo, hi, row_mask);
  CUDA_OK(cudaGetLastError());
  return 0;
}

int b200nn_cast_rows(const float* src, int32_t ld_src, void* dst, int32_t ld_dst, int32_t rows, int32_t cols, const float* mean, const float* rstd,
                     float lo, float hi, void* stream) {
  return cast_launch(src, ld_src, dst, nullptr, nullptr, ld_dst, rows, cols, mean, rstd, lo, hi, stream);
}

int b200nn_cast_rows_masked(const float* src, int32_t ld_src, void* dst, int32_t ld_dst, int32_t rows, int32_t cols, const uint8_t* row_mask,
                            float lo, float hi, void* stream) {
  if (!row_mask) return fail(-2, "b200nn_cast_rows_masked: null mask");
  return cast_launch(src, ld_src, dst, nullptr, nullptr, ld_dst, rows, cols, nullptr, nullptr, lo, hi, stream, row_mask);
}

int b200nn_cast_rows3(const float* src, int32_t ld_src, void* dst, void* dst2, void* dst3, int32_t ld_dst, int32_t rows, int32_t cols, void* stream) {
  return cast_launch(src, ld_src, dst, dst2, dst3, ld_dst, rows, cols, nullptr, nullptr, -3.0e38f, 3.0e38f, stream);
}

int b200nn_gate_softmax(const void* h, int32_t ldh, int32_t k, const float* w, const float* b, int32_t E, float* coef, int32_t rows, void* stream) {
  if (!h || !w || !b || !coef || E < 1 || E > 8 || rows < 1 || k < 1 || k > ldh) return fail(-2, "b200nn_gate_softmax: bad argument");
  static bool once = (prefer_max_shared(gate_softmax_kernel), true);
  (void)once;
  gate_softmax_kernel<<<(rows + 7) / 8, 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const __nv_bfloat16*>(h), ldh, k, w, b, E, coef, rows);
  CUDA_OK(cudaGetLastError());
  return 0;
}

}  // extern "C"
