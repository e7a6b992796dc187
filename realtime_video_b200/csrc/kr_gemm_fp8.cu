// kr_gemm_fp8.cu — FP8 (e4m3) wgmma GEMM with per-tensor, per-row or per-block scales + the dynamic per-tensor activation
// quantisation kernels (the per-row quantiser lives with the row kernels in kr_dit_elem.cu).
//
//   per tensor: out[M,N] = epilogue( (Aq[M,K] @ Wq[N,K]^T) * scale_a * scale_w + bias[N] )    Aq, Wq e4m3, out bf16
//   per row   : out[M,N] = epilogue( (Aq[M,K] @ Wq[N,K]^T) * scale_a[m] * scale_w[n] + bias[N] )
//   per block : out[M,N] = epilogue( sum_kb (Aq[M,kb] @ Wq[N,kb]^T) * scale_a[kb][m] * scale_w[n/128][kb] + bias[N] )
//
// Replaces, on the reference path, what `quantize_(transformer, Float8DynamicActivationFloat8WeightConfig(
// granularity=PerTensor()))` (release_server.py:179-182, `enable_fp8: true`) turns every nn.Linear into: torchao's
// dynamic per-tensor activation cast (amax over the whole activation -> scale = 448 / amax -> saturating e4m3 cast)
// followed by torch._scaled_mm (cuBLASLt FP8, fp32 accumulation, bf16 output) — here a hand-written
// wgmma e4m3 kernel with the same fused epilogues as the bf16 GEMM (bias, GELU, gate + residual, ...).
// torchao is absent from the image: the algorithm is restated from its published definition (oracle/fp8_oracle.py).
// granularity=PerRow() gives one scale per activation row and one per weight output channel, applied in the epilogue
// (torch._scaled_mm with scale_a [M, 1], scale_b [1, N]); oracle/fp8_rowwise_oracle.py restates it.
// granularity=PerBlock() ([1, 128] activations / [128, 128] weights, the DeepSeek-V3 recipe) multiplies each k-block's
// partial by sa[kb][row] * sw[n_blk][kb] at the promotion; oracle/fp8_blockwise_oracle.py restates it.
//
// One kernel template, gemm_fp8_kernel<kEpi, kScale, kFast>, with the structure of kr_gemm.cu (persistent 1 CTA/SM,
// two consumer warpgroups with register accumulators, a TMA warpgroup) and byte-sized elements: a 128-byte swizzle row
// holds 128 k-elements, one wgmma consumes K = 32 (32 bytes).  kFast selects how it accumulates:
//   promoted (default): each 128-wide k-block is accumulated separately and added to the fp32 registers (the e4m3
//            wgmma adder keeps fewer mantissa bits), on a 128 x 128 tile to leave registers for the partial.  Block
//            scales are applied at this promotion; the tile then spans one weight block in N and one activation
//            group per k-block, so the epilogue applies no scale;
//   fast     (torch._scaled_mm(use_fast_accum=True)): the wgmma accumulates in place across the whole K with one group
//            in flight, like the 16-bit GEMM, on a 128 x 256 tile (m64n256k32, half the shared-memory operand bytes
//            per FLOP) without draining the tensor cores after every k-block.
// gemm_i8_kernel<kEpi> (torchao Int8DynamicActivationInt8WeightConfig, oracle/int8_oracle.py) shares the body: the fast
// structure with s8 operands, exact s32 sums and the row-scaled epilogue.
#include "kr_common.cuh"
#include "kr_gemm_epi.cuh"
#include "kr_ops.h"

#include <cuda_fp8.h>

namespace kr {

namespace {
constexpr int F8_BM = 128, F8_BK = 128 /* elements = bytes */;
constexpr int F8_THREADS = 384, F8_STAGES = 4;
constexpr int F8_A_BYTES = F8_BM * F8_BK;
constexpr int F8_SCR_BYTES = 8 * kEpiScrFloats * 4;
__host__ __device__ constexpr int f8_bn(bool fast) { return fast ? 256 : 128; }
constexpr int f8_smem(bool fast) { return F8_STAGES * (F8_A_BYTES + f8_bn(fast) * F8_BK) + F8_SCR_BYTES + 1024 + 256; }
static_assert(f8_smem(true) <= 227 * 1024, "4 stages of 16 KB A + 32 KB W and the epilogue scratch fit one SM");

enum Fp8Scale { F8_SCALE_TENSOR, F8_SCALE_ROW, F8_SCALE_BLOCK };
constexpr int kI8MaxK = 132104;   // 127 * 128 * K < 2^31

// The I-th scale argument: a mode's scale arguments are separate kernel parameters, as many as the mode needs.
template <int I, typename T, typename... R>
__host__ __device__ __forceinline__ auto f8_arg(T t, R... r) {
  if constexpr (I == 0) return t;
  else return f8_arg<I - 1>(r...);
}
}  // namespace

// The body of both 8-bit GEMM kernels.  kKind 2 = e4m3 (gemm_fp8_kernel); 3 = s8 (gemm_i8_kernel: row scales on the
// fast structure, exact s32 sums converted to fp32 by the row-scaled epilogue).
// The scale arguments by kScale.  tensor: scale_a -> one fp32, float scale_w.  row: scale_a -> [M], scale_w -> [N].
// block: scale_a -> fp32 [K/128, ld_sa] (k-block-major: one k-block's row scales are contiguous), then long ld_sa and
// scale_w -> fp32 [N/128, K/128].
template <int kKind, int kEpi, int kScale, bool kFast, typename... ScaleW>
__device__ __forceinline__ void gemm_8bit_body(const CUtensorMap& tmap_a, const CUtensorMap& tmap_b,
                                               const GemmParams p, const float* __restrict__ scale_a,
                                               ScaleW... scale_w) {
  static_assert(!(kFast && kScale == F8_SCALE_BLOCK), "block scales are applied at the promotion");
  static_assert(kKind == 2 || (kFast && kScale == F8_SCALE_ROW), "s8 sums are exact: in place, row scales only");
  constexpr int BN = f8_bn(kFast), B_BYTES = BN * F8_BK, STAGE_BYTES = F8_A_BYTES + B_BYTES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + F8_STAGES * F8_A_BYTES;
  float* scratch = reinterpret_cast<float*>(smem + F8_STAGES * STAGE_BYTES);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + F8_STAGES * STAGE_BYTES + F8_SCR_BYTES);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + F8_STAGES;

  const int warp = threadIdx.x >> 5;
  const int num_m = (p.M + F8_BM - 1) / F8_BM, num_n = p.N / BN, num_tiles = num_m * num_n;
  const int num_k = (p.K + F8_BK - 1) / F8_BK;

  if (threadIdx.x == 256) {
    prefetch_tmap(&tmap_a);
    prefetch_tmap(&tmap_b);
    for (int i = 0; i < F8_STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 2);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp >= 8) {
    producer_regs();
    if (warp == 8 && elect_one()) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int m_blk = tile % num_m, n_blk = tile / num_m;
        for (int kb = 0; kb < num_k; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          mbar_expect_tx(&full_bar[stage], STAGE_BYTES);
          tma_load_2d(smem_a + stage * F8_A_BYTES, &tmap_a, &full_bar[stage], kb * F8_BK, m_blk * F8_BM);
          tma_load_2d(smem_b + stage * B_BYTES, &tmap_b, &full_bar[stage], kb * F8_BK, n_blk * BN);
          if (++stage == F8_STAGES) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
    return;
  }
  consumer_regs();
  const int wg = warp >> 2;
  const uint32_t a_base = smem_u32(smem_a) + wg * 64 * F8_BK, b_base = smem_u32(smem_b);
  float* scr = scratch + warp * kEpiScrFloats;
  float s = 1.f;
  if constexpr (kScale == F8_SCALE_TENSOR) s = __ldg(scale_a) * f8_arg<0>(scale_w...);   // per-tensor dequantisation
  int stage = 0;
  uint32_t phase = 0;
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    const int m_blk = tile % num_m, n_blk = tile / num_m;
    if constexpr (kScale == F8_SCALE_BLOCK) {
      const int row0 = m_blk * F8_BM + wg * 64 + (warp & 3) * 16;
      const int r = row0 + ((threadIdx.x & 31) >> 2);
      BlockScales bs;
      bs.sa0 = r < p.M ? scale_a + r : nullptr;
      bs.sa1 = r + 8 < p.M ? scale_a + r + 8 : nullptr;
      bs.ld = f8_arg<0>(scale_w...);
      bs.sw = f8_arg<1>(scale_w...) + static_cast<long>(n_blk) * num_k;
      float acc[BN / 2];
      gemm_mainloop<BN, 2, 1, true, true>(acc, a_base, b_base, F8_A_BYTES, B_BYTES, F8_STAGES, full_bar, empty_bar,
                                          stage, phase, 0, num_k, bs);
      gemm_frag_epilogue<BN, true, kEpi>(acc, scr, row0, n_blk * BN, BN, 1.f, p);
    } else {
      float acc[BN / 2];
      gemm_mainloop<BN, kKind, 1, !kFast>(acc, a_base, b_base, F8_A_BYTES, B_BYTES, F8_STAGES, full_bar, empty_bar,
                                          stage, phase, 0, num_k);
      if constexpr (kScale == F8_SCALE_ROW)
        gemm_frag_epilogue<BN, true, kEpi, true, kKind == 3>(acc, scr, m_blk * F8_BM + wg * 64 + (warp & 3) * 16,
                                                             n_blk * BN, BN, s, p, scale_a, f8_arg<0>(scale_w...));
      else
        gemm_frag_epilogue<BN, true, kEpi>(acc, scr, m_blk * F8_BM + wg * 64 + (warp & 3) * 16, n_blk * BN, BN, s, p);
    }
  }
}

template <int kEpi, int kScale, bool kFast, typename... ScaleW>
__global__ void __launch_bounds__(F8_THREADS, 1)
gemm_fp8_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                const GemmParams p, const float* __restrict__ scale_a, ScaleW... scale_w) {
  gemm_8bit_body<2, kEpi, kScale, kFast>(tmap_a, tmap_b, p, scale_a, scale_w...);
}

// INT8 (torchao Int8DynamicActivationInt8WeightConfig): s8 x s8 wgmma (m64n256k32) summing exactly in s32 across the
// whole K, then v = (float(acc) * scale_a[m]) * scale_w[n] and the bf16 epilogue.  |acc| <= 127 * 128 * K < 2^31 for
// K <= 132104, which the host checks.
template <int kEpi>
__global__ void __launch_bounds__(F8_THREADS, 1)
gemm_i8_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
               const GemmParams p, const float* __restrict__ scale_a, const float* __restrict__ scale_w) {
  gemm_8bit_body<3, kEpi, F8_SCALE_ROW, true>(tmap_a, tmap_b, p, scale_a, scale_w);
}

// ---------------------------------------------------------------------------
// dynamic per-tensor activation quantisation: amax -> scale -> saturating e4m3 cast
// ---------------------------------------------------------------------------
__global__ void fp8_amax_kernel(const uint16_t* __restrict__ x, long ld, int rows, int cols, float* amax) {
  float m = 0.f;
  const int vec_per_row = cols >> 3;
  const long total = static_cast<long>(rows) * vec_per_row;
  for (long i = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long>(gridDim.x) * blockDim.x) {
    const long r = i / vec_per_row;
    const int c = static_cast<int>(i - r * vec_per_row);
    const uint4 u = *reinterpret_cast<const uint4*>(x + r * ld + c * 8);
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = unpack_bf16x2(w[j]);
      m = fmaxf(m, fmaxf(fabsf(f.x), fabsf(f.y)));
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) atomicMax(reinterpret_cast<int*>(amax), __float_as_int(m));   // m >= 0: int order = float order
}

__global__ void fp8_quant_kernel(const uint16_t* __restrict__ x, long ld, int rows, int cols, uint8_t* __restrict__ q,
                                 long ldq, float* state) {
  // state[0] = amax (input), state[1] = dequantisation scale amax / 448 (output, read by the GEMM epilogue)
  const float amax = fmaxf(state[0], 1e-12f);
  const float mul = 448.0f / amax;
  if (blockIdx.x == 0 && threadIdx.x == 0) state[1] = amax / 448.0f;
  const int vec_per_row = cols >> 3;
  const long total = static_cast<long>(rows) * vec_per_row;
  for (long i = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long>(gridDim.x) * blockDim.x) {
    const long r = i / vec_per_row;
    const int c = static_cast<int>(i - r * vec_per_row);
    const uint4 u = *reinterpret_cast<const uint4*>(x + r * ld + c * 8);
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
    uint32_t out[2];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = unpack_bf16x2(w[j]);
      const __nv_fp8x2_storage_t h = __nv_cvt_float2_to_fp8x2(make_float2(f.x * mul, f.y * mul), __NV_SATFINITE, __NV_E4M3);
      if (j & 1) out[j >> 1] |= static_cast<uint32_t>(h) << 16;
      else out[j >> 1] = static_cast<uint32_t>(h);
    }
    *reinterpret_cast<uint2*>(q + r * ldq + c * 8) = make_uint2(out[0], out[1]);
  }
}

int fp8_quantize(const void* x, long ld, int rows, int cols, void* q, long ldq, float* state, cudaStream_t stream) {
  if (cols % 8 != 0 || ld % 8 != 0 || ldq % 8 != 0 || rows <= 0) {
    set_last_error("fp8_quantize: unsupported rows=%d cols=%d ld=%ld ldq=%ld", rows, cols, ld, ldq);
    return KR_ERR_UNSUPPORTED_SHAPE;
  }
  cudaError_t e = cudaMemsetAsync(state, 0, 2 * sizeof(float), stream);
  if (e != cudaSuccess) {
    set_last_error("fp8_quantize: memset failed: %s", cudaGetErrorString(e));
    return KR_ERR_CUDA;
  }
  const long total = static_cast<long>(rows) * (cols / 8);
  int grid = static_cast<int>((total + 255) / 256);
  if (grid > 148 * 8) grid = 148 * 8;
  fp8_amax_kernel<<<grid, 256, 0, stream>>>(static_cast<const uint16_t*>(x), ld, rows, cols, state);
  fp8_quant_kernel<<<grid, 256, 0, stream>>>(static_cast<const uint16_t*>(x), ld, rows, cols,
                                            static_cast<uint8_t*>(q), ldq, state);
  e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_last_error("fp8_quantize: launch failed: %s", cudaGetErrorString(e));
    return KR_ERR_CUDA;
  }
  return KR_OK;
}

// ---------------------------------------------------------------------------
// host launcher
// ---------------------------------------------------------------------------
template <int kKind, bool kFast, int kEpi, int kScale, typename... ScaleW>
static int launch_fp8(const void* a, int lda, const void* w, int ldw, const GemmParams& p, cudaStream_t stream,
                      const float* scale_a, ScaleW... scale_w) {
  constexpr int BN = f8_bn(kFast), SMEM = f8_smem(kFast);
  constexpr const char* name = kKind == 3 ? "gemm_i8" : kScale == F8_SCALE_BLOCK ? "gemm_fp8_blockwise" : "gemm_fp8";
  CUtensorMap ta, tb;
  // byte tensors: [rows, K] uint8, box [128 | 256 rows, 128 bytes], SWIZZLE_128B
  const uint64_t da[2] = {static_cast<uint64_t>(p.K), static_cast<uint64_t>(p.M)};
  const uint64_t sa[1] = {static_cast<uint64_t>(lda)};
  const uint32_t ba[2] = {F8_BK, F8_BM};
  int rc = make_tmap_u8(&ta, a, 2, da, sa, ba, 128);
  if (rc != KR_OK) return rc;
  const uint64_t db[2] = {static_cast<uint64_t>(p.K), static_cast<uint64_t>(p.N)};
  const uint64_t sb[1] = {static_cast<uint64_t>(ldw)};
  const uint32_t bb[2] = {F8_BK, BN};
  rc = make_tmap_u8(&tb, w, 2, db, sb, bb, 128);
  if (rc != KR_OK) return rc;
  const auto kern = [] {
    if constexpr (kKind == 3) return gemm_i8_kernel<kEpi>;
    else return gemm_fp8_kernel<kEpi, kScale, kFast, ScaleW...>;
  }();
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM);
    if (e != cudaSuccess) {
      set_last_error("%s: cudaFuncSetAttribute failed: %s", name, cudaGetErrorString(e));
      return KR_ERR_CUDA;
    }
    attr_set = true;
  }
  const int num_tiles = ((p.M + F8_BM - 1) / F8_BM) * (p.N / BN);
  int grid = sm_count();
  if (grid > num_tiles) grid = num_tiles;
  kern<<<grid, F8_THREADS, SMEM, stream>>>(ta, tb, p, scale_a, scale_w...);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_last_error("%s: launch failed: %s", name, cudaGetErrorString(e));
    return KR_ERR_CUDA;
  }
  return KR_OK;
}

// The argument checks of every mode, then the kernel of the epilogue (EPI_F32 only with block scales or s8).
template <bool kFast, int kScale, int kKind = 2, typename... ScaleW>
static int gemm_fp8_any(const char* who, int epi, const void* a, int lda, const void* w, int ldw, const GemmParams& p,
                        cudaStream_t stream, const float* scale_a, ScaleW... scale_w) {
  if (p.M <= 0 || p.N <= 0 || p.K <= 0 || p.N % f8_bn(kFast) != 0 || p.K % 16 != 0 || lda % 16 != 0 ||
      ldw % 16 != 0 || p.ldc % 8 != 0) {
    set_last_error("%s: unsupported shape M=%d N=%d K=%d (need N %% %d == 0, K / ld %% 16 == 0)", who, p.M, p.N, p.K,
                   f8_bn(kFast));
    return KR_ERR_UNSUPPORTED_SHAPE;
  }
  if (kKind == 3 && p.K > kI8MaxK) {
    set_last_error("%s: K=%d > %d could overflow the s32 sums", who, p.K, kI8MaxK);
    return KR_ERR_UNSUPPORTED_SHAPE;
  }
  if ((epi == EPI_BIAS_GATE_RES || epi == EPI_BIAS_RES || epi == EPI_MUL) && p.residual == nullptr) {
    set_last_error("%s: residual epilogue without residual pointer", who);
    return KR_ERR_INVALID_ARG;
  }
  if constexpr (kScale == F8_SCALE_TENSOR) {
    if (scale_a == nullptr) {
      set_last_error("%s: null activation scale", who);
      return KR_ERR_INVALID_ARG;
    }
  } else if constexpr (kScale == F8_SCALE_ROW) {
    const float* sw = f8_arg<0>(scale_w...);
    if (scale_a == nullptr || sw == nullptr) {
      set_last_error("%s: null row or channel scales", who);
      return KR_ERR_INVALID_ARG;
    }
    if (reinterpret_cast<uintptr_t>(sw) % 16 != 0) {
      set_last_error("%s: channel scales must be 16-byte aligned", who);
      return KR_ERR_INVALID_ARG;
    }
  } else {
    // the host-side checks of kr_api.cu (shape, pitches, null scales) have passed; these guard direct callers
    if (p.K % F8_BK != 0) {
      set_last_error("%s: K=%d is not a multiple of the 128-wide scale block", who, p.K);
      return KR_ERR_UNSUPPORTED_SHAPE;
    }
    const long ld_sa = f8_arg<0>(scale_w...);
    if (scale_a == nullptr || f8_arg<1>(scale_w...) == nullptr || ld_sa < p.M) {
      set_last_error("%s: null block scales or activation scale pitch %ld < M=%d", who, ld_sa, p.M);
      return KR_ERR_INVALID_ARG;
    }
  }
  switch (epi) {
    case EPI_BIAS: return launch_fp8<kKind, kFast, EPI_BIAS, kScale>(a, lda, w, ldw, p, stream, scale_a, scale_w...);
    case EPI_BIAS_GELU:
      return launch_fp8<kKind, kFast, EPI_BIAS_GELU, kScale>(a, lda, w, ldw, p, stream, scale_a, scale_w...);
    case EPI_BIAS_GATE_RES:
      return launch_fp8<kKind, kFast, EPI_BIAS_GATE_RES, kScale>(a, lda, w, ldw, p, stream, scale_a, scale_w...);
    case EPI_BIAS_RES:
      return launch_fp8<kKind, kFast, EPI_BIAS_RES, kScale>(a, lda, w, ldw, p, stream, scale_a, scale_w...);
    case EPI_F32:
      if constexpr (kScale == F8_SCALE_BLOCK || kKind == 3)
        return launch_fp8<kKind, kFast, EPI_F32, kScale>(a, lda, w, ldw, p, stream, scale_a, scale_w...);
      [[fallthrough]];
    default: set_last_error("%s: unsupported epilogue %d", who, epi); return KR_ERR_INVALID_ARG;
  }
}

int gemm_fp8_tn(int epi, const void* a, int lda, const void* w, int ldw, const GemmParams& p, const float* scale_a,
                float scale_w, cudaStream_t stream) {
  return gemm_fp8_any<false, F8_SCALE_TENSOR>("gemm_fp8", epi, a, lda, w, ldw, p, stream, scale_a, scale_w);
}

int gemm_fp8_rowwise_tn(int epi, const void* a, int lda, const void* w, int ldw, const GemmParams& p,
                        const float* scale_a, const float* scale_w, cudaStream_t stream) {
  return gemm_fp8_any<false, F8_SCALE_ROW>("gemm_fp8_rowwise", epi, a, lda, w, ldw, p, stream, scale_a, scale_w);
}

int gemm_fp8_fast_tn(int epi, const void* a, int lda, const void* w, int ldw, const GemmParams& p,
                     const float* scale_a, float scale_w, cudaStream_t stream) {
  return gemm_fp8_any<true, F8_SCALE_TENSOR>("gemm_fp8_fast", epi, a, lda, w, ldw, p, stream, scale_a, scale_w);
}

int gemm_fp8_rowwise_fast_tn(int epi, const void* a, int lda, const void* w, int ldw, const GemmParams& p,
                             const float* scale_a, const float* scale_w, cudaStream_t stream) {
  return gemm_fp8_any<true, F8_SCALE_ROW>("gemm_fp8_rowwise_fast", epi, a, lda, w, ldw, p, stream, scale_a, scale_w);
}

int gemm_fp8_blockwise_tn(int epi, const void* a, int lda, const void* w, int ldw, const GemmParams& p,
                          const float* scale_a, int ld_sa, const float* scale_w, cudaStream_t stream) {
  return gemm_fp8_any<false, F8_SCALE_BLOCK>("gemm_fp8_blockwise", epi, a, lda, w, ldw, p, stream, scale_a,
                                             static_cast<long>(ld_sa), scale_w);
}

int gemm_i8_rowwise_tn(int epi, const void* a, int lda, const void* w, int ldw, const GemmParams& p,
                       const float* scale_a, const float* scale_w, cudaStream_t stream) {
  return gemm_fp8_any<true, F8_SCALE_ROW, 3>("gemm_i8_rowwise", epi, a, lda, w, ldw, p, stream, scale_a, scale_w);
}

}  // namespace kr
