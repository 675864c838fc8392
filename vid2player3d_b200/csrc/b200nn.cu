// b200nn.cu - libb200nn.so (C ABI: include/b200nn.h): the policy MLP and the MVAE mixture-of-experts decoder layers as
// hand-written sm_90a GEMMs.  One launch per layer:
//
//     out[:, col0 : col0 + N] = act( sum_e coef[:, e] * (A W_e^T + bias_e) )        bf16 operands, fp32 accumulate
//
// Structure of `linear_kernel` (one 128-row output tile per CTA, 2 consumer warpgroups + 1 producer warp):
//   warp 8       TMA producer: cp.async.bulk.tensor tiles of A [128 x 64] and W [E x BN x 64] (128-byte swizzle) into a ring of
//                STAGES shared-memory stages, completion on mbarriers (expect_tx)
//   warpgroups 0, 1  rows 0-63 / 64-127 of the tile: per 64-wide k block 4 wgmma.mma_async of K = 16 per accumulator chunk, operands
//                straight from the swizzled stages, fp32 accumulators in registers; the stage is released on its `empty` mbarrier once
//                the warpgroup's wgmmas have completed.  Epilogue from the registers: bias, expert blend, activation, bf16 / fp32 stores.
// E = 1: BN = 128 accumulator columns.  E > 1 (mixture of experts, vid2player/motion_vae/model.py:237-252): the tile is MOE_BN
// output columns x E experts = E * MOE_BN accumulator columns; the per-row softmax coefficients are applied in the epilogue in fp32,
// so the per-env blended weight matrices of the reference never exist.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include "../../include/b200nn.h"

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
#ifndef MOE_BN
#define MOE_BN 32
#endif
#ifndef MOE_STAGES
#define MOE_STAGES 2
#endif
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
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

// D[64 x N] (+)= A[64 x 16] B[N x 16]^T, bf16 operands K-major in shared memory, fp32 accumulators: N / 2 registers per thread.
// Register i of thread t of the warpgroup holds row 16 (t / 32) + (t % 32) / 4 + 8 ((i / 2) % 2), column 8 (i / 4) + 2 (t % 4) + i % 2.
template <int N> __device__ __forceinline__ void wgmma_bf16(float* d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate);
template <> __device__ __forceinline__ void wgmma_bf16<32>(float* d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
        "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
template <> __device__ __forceinline__ void wgmma_bf16<64>(float* d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, "
      "%27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
        "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]),
        "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]),
        "+f"(d[30]), "+f"(d[31])
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}

__device__ __forceinline__ float apply_act(float x, int act) {
  if (act == B200NN_ACT_RELU) return fmaxf(x, 0.f);
  if (act == B200NN_ACT_ELU) return x > 0.f ? x : expm1f(x);   // F.elu, alpha = 1
  return x;
}


#ifndef B200NN_PROBE
#define B200NN_PROBE 0
#endif
#if B200NN_PROBE
__device__ unsigned long long g_probe[16];
__device__ __forceinline__ unsigned long long gtime() { unsigned long long t; asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t) :: "memory"); return t; }
#define PROBE(i) do { if (blockIdx.x == 0 && blockIdx.y == 0) g_probe[i] = gtime(); } while (0)
__device__ unsigned long long g_cta[4096][8];
#define PROBE_CTA(k) do { const int c_ = blockIdx.y * gridDim.x + blockIdx.x; if (c_ < 4096) g_cta[c_][k] = gtime(); } while (0)
#else
#define PROBE_CTA(k) do { } while (0)
#define PROBE(i) do { } while (0)
#endif

struct LinearParams {
  const float* bias;
  const float* coef;
  void* out;
  int ldo, out_col0, rows, n, n_padded, k_padded, act, out_bf16;
  float out_min, out_max;
};

__device__ __forceinline__ float finish(float x, const LinearParams& p) {
  x = apply_act(x, p.act);
  return p.out_min < p.out_max ? fminf(fmaxf(x, p.out_min), p.out_max) : x;
}

__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

// two consecutive outputs (col, col + 1) of one row -> global memory; col is even
__device__ __forceinline__ void store2(const LinearParams& p, int row, int col, float a, float b) {
  if (row >= p.rows || col >= p.n) return;
  if (p.out_bf16) {
    __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(p.out) + (size_t)row * p.ldo + p.out_col0 + col;
    if (col + 1 < p.n) *reinterpret_cast<__nv_bfloat162*>(o) = __floats2bfloat162_rn(a, b);   // ldo, out_col0 multiples of 8: aligned
    else o[0] = __float2bfloat16_rn(a);
  } else {
    float* o = reinterpret_cast<float*>(p.out) + (size_t)row * p.ldo + p.out_col0 + col;
    if (col + 1 < p.n && ((uintptr_t)o & 7) == 0) {
      *reinterpret_cast<float2*>(o) = make_float2(a, b);
    } else {
      o[0] = a;
      if (col + 1 < p.n) o[1] = b;
    }
  }
}

template <int E, int BN, int STAGES>
__global__ void __launch_bounds__(NUM_THREADS, E == 1 ? 2 : 1)
linear_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmW, const LinearParams p) {
  constexpr int ACC = E * BN;                          // accumulator columns
  constexpr int CN = BN < 64 ? BN : 64;                // columns per wgmma
  constexpr int NCH = BN / CN;                         // wgmma chunks per expert
  constexpr int B_STAGE_BYTES = ACC * BLOCK_K * 2;
  constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
  static_assert(BN % CN == 0 && (CN == 32 || CN == 64), "tile width must be a multiple of 32 columns");

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);   // swizzle-128B atoms: 1024-byte aligned
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES);
  uint64_t* empty = full + STAGES;
  float* sbias = reinterpret_cast<float*>(empty + STAGES);        // [E][BN] bias of this tile's columns

  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;
  const int m0 = blockIdx.x * BLOCK_M, n0 = blockIdx.y * BN;
  const int nkb = p.k_padded / BLOCK_K;

  if (threadIdx.x == 0) { PROBE(0); PROBE_CTA(0); }
  if (warp == 8 && lane == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmW) : "memory");
    for (int i = 0; i < STAGES; i++) { mbar_init(&full[i], 1); mbar_init(&empty[i], 2); }   // empty: one arrival per consumer warpgroup
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  for (int i = threadIdx.x; i < ACC; i += NUM_THREADS) sbias[i] = __ldg(p.bias + (size_t)(i / BN) * p.n_padded + n0 + (i % BN));
  __syncthreads();
  if (threadIdx.x == 0) PROBE(1);
  // Programmatic dependent launch: the next layer's CTAs may be scheduled as soon as ours have all started (they take the SM
  // slots our last wave leaves free, run their set-up and park at griddepcontrol.wait), and everything ABOVE this line ran
  // while the previous layer was still finishing.  Below it, every read of data a previous kernel produced (the A operand, the
  // blend coefficients) comes after griddepcontrol.wait = previous grid complete and visible.
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");

  if (warp == 8) {
    if (lane == 0) {   // ---------------- TMA producer
      asm volatile("griddepcontrol.wait;" ::: "memory");
      for (int kb = 0; kb < nkb; kb++) {
        const int s = kb % STAGES;
        mbar_wait(&empty[s], ((kb / STAGES) & 1) ^ 1);
        uint8_t* sa = smem + s * STAGE_BYTES;
        mbar_expect_tx(&full[s], STAGE_BYTES);
        tma_load_2d(sa, &tmA, kb * BLOCK_K, m0, &full[s]);
        tma_load_3d(sa + A_STAGE_BYTES, &tmW, kb * BLOCK_K, n0, 0, &full[s]);
        if (kb == 0) PROBE(2);
      }
      PROBE(3);
    }
    return;
  }
  // ---------------- consumers: warpgroup wg owns rows m0 + 64 wg .. + 63 of the tile
  const int wg = warp >> 2;
  const int t = threadIdx.x & 127;
  const int row0 = m0 + 64 * wg + 16 * (t >> 5) + (lane >> 2);   // this thread's rows: row0 and row0 + 8
  float coef[2][E];
  if (E > 1) asm volatile("griddepcontrol.wait;" ::: "memory");    // the coefficients come from the gate kernel before us
#pragma unroll
  for (int h = 0; h < 2; h++)
#pragma unroll
    for (int e = 0; e < E; e++) coef[h][e] = (E == 1) ? 1.f : (row0 + 8 * h < p.rows ? p.coef[(size_t)(row0 + 8 * h) * E + e] : 0.f);
  float acc[E * NCH][CN / 2];
#pragma unroll
  for (int c = 0; c < E * NCH; c++)
#pragma unroll
    for (int i = 0; i < CN / 2; i++) acc[c][i] = 0.f;
  for (int kb = 0; kb < nkb; kb++) {
    const int s = kb % STAGES;
    mbar_wait(&full[s], (kb / STAGES) & 1);
    if (kb == 0 && threadIdx.x == 0) PROBE(4);
    const uint32_t a_addr = smem_u32(smem + s * STAGE_BYTES) + wg * (64 * 128), b_addr = smem_u32(smem + s * STAGE_BYTES) + A_STAGE_BYTES;
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < BLOCK_K / MMA_K; k++) {
      const uint64_t adesc = wgmma_desc_sw128(a_addr + k * MMA_K * 2);
#pragma unroll
      for (int c = 0; c < E * NCH; c++)      // B row r <-> accumulator column r (expert-major)
        wgmma_bf16<CN>(acc[c], adesc, wgmma_desc_sw128(b_addr + c * CN * 128 + k * MMA_K * 2), (uint32_t)((kb | k) != 0));
    }
    wgmma_commit();
    wgmma_wait_all();
    if (t == 0) mbar_arrive(&empty[s]);     // this warpgroup's wgmmas have read the stage
  }
  if (threadIdx.x == 0) PROBE(6);
  // ---------------- epilogue: register i of chunk c = row row0 + 8 ((i / 2) % 2), column c CN + 8 (i / 4) + 2 (lane % 4) + i % 2
#pragma unroll
  for (int c = 0; c < NCH; c++) {
    if (n0 + c * CN >= p.n) break;                     // padding columns of the last tile: nothing to store
#pragma unroll
    for (int j = 0; j < CN / 8; j++) {
      const int col = c * CN + 8 * j + 2 * (lane & 3);
#pragma unroll
      for (int h = 0; h < 2; h++) {
        float y[2];
#pragma unroll
        for (int u = 0; u < 2; u++) {
          const int i = 4 * j + 2 * h + u;
          if (E == 1) {
            y[u] = acc[c][i] + sbias[col + u];
          } else {
            y[u] = 0.f;
#pragma unroll
            for (int e = 0; e < E; e++) y[u] = fmaf(coef[h][e], acc[e * NCH + c][i] + sbias[e * BN + col + u], y[u]);
          }
          y[u] = finish(y[u], p);
        }
        store2(p, row0 + 8 * h, n0 + col, y[0], y[1]);
      }
    }
  }
  if (threadIdx.x == 0) PROBE(7);
  if (lane == 0) PROBE_CTA(1 + (warp & 3) + 4 * wg);
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
      const __nv_bfloat16 v = __float2bfloat16_rn(fminf(fmaxf(x, lo), hi));
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

template <int E, int BN, int STAGES> constexpr int smem_bytes() { return STAGES * (A_STAGE_BYTES + E * BN * BLOCK_K * 2) + 1024 + 16 * STAGES + E * BN * 4; }

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
  int device, bn, pdl;
  dim3 grid;
};

template <int E, int BN, int STAGES> static int launch(const b200nn_linear* h, cudaStream_t st) {
  static bool attr_set[16] = {};
  if (!attr_set[h->device & 15]) {
    CUDA_OK(cudaFuncSetAttribute(linear_kernel<E, BN, STAGES>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes<E, BN, STAGES>()));
    prefer_max_shared(linear_kernel<E, BN, STAGES>);
    attr_set[h->device & 15] = true;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = h->grid;
  cfg.blockDim = dim3(NUM_THREADS, 1, 1);
  cfg.dynamicSmemBytes = smem_bytes<E, BN, STAGES>();
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = h->pdl ? 1 : 0;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  CUDA_OK(cudaLaunchKernelEx(&cfg, linear_kernel<E, BN, STAGES>, h->tmA, h->tmW, h->p));
  return 0;
}

extern "C" {

int b200nn_abi_version(void) { return B200NN_ABI_VERSION; }
const char* b200nn_last_error(void) { return g_err; }

int b200nn_linear_create(const b200nn_linear_desc_t* d, int32_t device, b200nn_linear_handle* out) {
  if (!d || !out) return fail(-1, "b200nn_linear_create: null argument");
  if (!d->a || !d->w || !d->bias || !d->out) return fail(-1, "b200nn_linear_create: null operand pointer");
  const int E = d->num_experts;
  if (E < 1 || E > 6) return fail(-2, "b200nn_linear_create: num_experts must be 1..6");
  if (E > 1 && !d->coef) return fail(-1, "b200nn_linear_create: mixture layer needs the coefficient tensor");
  const int bn = E == 1 ? 128 : MOE_BN;
  if (d->k_padded < BLOCK_K || d->k_padded % BLOCK_K || d->lda % BLOCK_K || d->ldw % BLOCK_K || d->lda < d->k_padded || d->ldw < d->k_padded)
    return fail(-2, "b200nn_linear_create: K and the leading dimensions must be padded to multiples of 64");
  if (d->n_padded < bn || d->n_padded % bn || d->n < 1 || d->n > d->n_padded) return fail(-2, "b200nn_linear_create: n_padded must be a multiple of the output tile");
  if (d->rows < 1) return fail(-2, "b200nn_linear_create: rows < 1");
  if (d->out_bf16 && (d->ldo % 8 || d->out_col0 % 8)) return fail(-2, "b200nn_linear_create: bf16 output needs ldo and out_col0 multiples of 8");
  if (((uintptr_t)d->a | (uintptr_t)d->w | (uintptr_t)d->out) & 15) return fail(-2, "b200nn_linear_create: operands must be 16-byte aligned");
  encode_tiled_fn enc = get_encode();
  if (!enc) return fail(-3, "b200nn_linear_create: cuTensorMapEncodeTiled not available (no CUDA driver)");
  CUDA_OK(cudaSetDevice(device));
  b200nn_linear* h = new b200nn_linear();
  h->d = *d;
  h->device = device;
  h->bn = bn;
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
    cuuint32_t box[3] = {BLOCK_K, (cuuint32_t)bn, (cuuint32_t)E}, es[3] = {1, 1, 1};
    CUresult r = enc(&h->tmW, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(d->w), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { delete h; snprintf(g_err, sizeof(g_err), "cuTensorMapEncodeTiled(W) failed: %d", (int)r); return -3; }
  }
  h->p = LinearParams{d->bias, d->coef, d->out, d->ldo, d->out_col0, d->rows, d->n, d->n_padded, d->k_padded, d->act, d->out_bf16, d->out_min, d->out_max};
  h->grid = dim3(rows_padded / BLOCK_M, (d->n + bn - 1) / bn, 1);
  *out = h;
  return 0;
}

int b200nn_linear_destroy(b200nn_linear_handle h) {
  delete h;
  return 0;
}

int b200nn_linear_run(b200nn_linear_handle h, void* stream) {
  if (!h) return fail(-1, "b200nn_linear_run: null handle");
  cudaStream_t st = (cudaStream_t)stream;
  switch (h->d.num_experts) {
    case 1: return launch<1, 128, 3>(h, st);
    case 2: return launch<2, MOE_BN, 3>(h, st);
    case 3: return launch<3, MOE_BN, 3>(h, st);
    case 4: return launch<4, MOE_BN, 3>(h, st);
    case 5: return launch<5, MOE_BN, MOE_STAGES>(h, st);
    case 6: return launch<6, MOE_BN, MOE_STAGES>(h, st);
  }
  return fail(-2, "b200nn_linear_run: unsupported expert count");
}

#if B200NN_PROBE
int b200nn_probe_read_ctas(unsigned long long* out, int n) { return cudaMemcpyFromSymbol(out, g_cta, sizeof(unsigned long long) * 8 * n) == cudaSuccess ? 0 : -1; }
int b200nn_probe_read(unsigned long long* out16) { return cudaMemcpyFromSymbol(out16, g_probe, sizeof(unsigned long long) * 16) == cudaSuccess ? 0 : -1; }
#endif

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
