// kr_gemm_fp8.cu — FP8 (e4m3) wgmma GEMM with per-tensor scales + the dynamic activation quantisation kernels.
//
//   out[M,N] = epilogue( (Aq[M,K] @ Wq[N,K]^T) * scale_a * scale_w + bias[N] )      Aq, Wq e4m3, out bf16
//
// Replaces, on the reference path, what `quantize_(transformer, Float8DynamicActivationFloat8WeightConfig(
// granularity=PerTensor()))` (release_server.py:179-182, `enable_fp8: true`) turns every nn.Linear into: torchao's
// dynamic per-tensor activation cast (amax over the whole activation -> scale = 448 / amax -> saturating e4m3 cast)
// followed by torch._scaled_mm (cuBLASLt FP8, fp32 accumulation, bf16 output) — here a hand-written
// wgmma e4m3 kernel with the same fused epilogues as the bf16 GEMM (bias, GELU, gate + residual, ...).
// torchao is absent from the image: the algorithm is restated from its published definition (oracle/fp8_oracle.py).
//
// Kernel structure = kr_gemm.cu (persistent 1 CTA/SM, two consumer warpgroups with register accumulators, a TMA
// warpgroup), with byte-sized elements: a 128-byte swizzle row holds 128 k-elements, one wgmma consumes K = 32
// (32 bytes); each 128-wide k-block is accumulated separately and added to the fp32 registers (the e4m3 wgmma
// adder keeps fewer mantissa bits), so the tile is 128 x 128 to leave registers for the partial.
#include "kr_common.cuh"
#include "kr_gemm_epi.cuh"
#include "kr_ops.h"

#include <cuda_fp8.h>

namespace kr {

namespace {
constexpr int F8_BM = 128, F8_BN = 128, F8_BK = 128 /* elements = bytes */;
constexpr int F8_THREADS = 384, F8_STAGES = 4;
constexpr int F8_A_BYTES = F8_BM * F8_BK, F8_B_BYTES = F8_BN * F8_BK, F8_STAGE_BYTES = F8_A_BYTES + F8_B_BYTES;
constexpr int F8_SCR_BYTES = 8 * kEpiScrFloats * 4;
constexpr int F8_SMEM = F8_STAGES * F8_STAGE_BYTES + F8_SCR_BYTES + 1024 + 256;
}  // namespace

template <int kEpi>
__global__ void __launch_bounds__(F8_THREADS, 1)
gemm_fp8_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                const GemmParams p, const float* __restrict__ scale_a, const float scale_w) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + F8_STAGES * F8_A_BYTES;
  float* scratch = reinterpret_cast<float*>(smem + F8_STAGES * F8_STAGE_BYTES);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + F8_STAGES * F8_STAGE_BYTES + F8_SCR_BYTES);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + F8_STAGES;

  const int warp = threadIdx.x >> 5;
  const int num_m = (p.M + F8_BM - 1) / F8_BM, num_n = p.N / F8_BN, num_tiles = num_m * num_n;
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
          mbar_expect_tx(&full_bar[stage], F8_STAGE_BYTES);
          tma_load_2d(smem_a + stage * F8_A_BYTES, &tmap_a, &full_bar[stage], kb * F8_BK, m_blk * F8_BM);
          tma_load_2d(smem_b + stage * F8_B_BYTES, &tmap_b, &full_bar[stage], kb * F8_BK, n_blk * F8_BN);
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
  const float s = __ldg(scale_a) * scale_w;       // dequantisation: per-tensor activation x weight scale
  int stage = 0;
  uint32_t phase = 0;
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    const int m_blk = tile % num_m, n_blk = tile / num_m;
    float acc[F8_BN / 2];
    gemm_mainloop<F8_BN, 2>(acc, a_base, b_base, F8_A_BYTES, F8_B_BYTES, F8_STAGES, full_bar, empty_bar, stage, phase,
                            0, num_k);
    gemm_frag_epilogue<F8_BN, true, kEpi>(acc, scr, m_blk * F8_BM + wg * 64 + (warp & 3) * 16, n_blk * F8_BN, F8_BN,
                                          s, p);
  }
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
template <int kEpi>
static int launch_fp8(const void* a, int lda, const void* w, int ldw, const GemmParams& p, const float* scale_a,
                      float scale_w, cudaStream_t stream) {
  CUtensorMap ta, tb;
  // byte tensors: [rows, K] uint8, box [128 | 256 rows, 128 bytes], SWIZZLE_128B
  const uint64_t da[2] = {static_cast<uint64_t>(p.K), static_cast<uint64_t>(p.M)};
  const uint64_t sa[1] = {static_cast<uint64_t>(lda)};
  const uint32_t ba[2] = {F8_BK, F8_BM};
  int rc = make_tmap_u8(&ta, a, 2, da, sa, ba, 128);
  if (rc != KR_OK) return rc;
  const uint64_t db[2] = {static_cast<uint64_t>(p.K), static_cast<uint64_t>(p.N)};
  const uint64_t sb[1] = {static_cast<uint64_t>(ldw)};
  const uint32_t bb[2] = {F8_BK, F8_BN};
  rc = make_tmap_u8(&tb, w, 2, db, sb, bb, 128);
  if (rc != KR_OK) return rc;
  auto kern = gemm_fp8_kernel<kEpi>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, F8_SMEM);
    if (e != cudaSuccess) {
      set_last_error("gemm_fp8: cudaFuncSetAttribute failed: %s", cudaGetErrorString(e));
      return KR_ERR_CUDA;
    }
    attr_set = true;
  }
  const int num_tiles = ((p.M + F8_BM - 1) / F8_BM) * (p.N / F8_BN);
  int grid = sm_count();
  if (grid > num_tiles) grid = num_tiles;
  kern<<<grid, F8_THREADS, F8_SMEM, stream>>>(ta, tb, p, scale_a, scale_w);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_last_error("gemm_fp8: launch failed: %s", cudaGetErrorString(e));
    return KR_ERR_CUDA;
  }
  return KR_OK;
}

int gemm_fp8_tn(int epi, const void* a, int lda, const void* w, int ldw, const GemmParams& p, const float* scale_a,
                float scale_w, cudaStream_t stream) {
  if (p.M <= 0 || p.N <= 0 || p.K <= 0 || p.N % F8_BN != 0 || p.K % 16 != 0 || lda % 16 != 0 || ldw % 16 != 0 ||
      p.ldc % 8 != 0) {
    set_last_error("gemm_fp8: unsupported shape M=%d N=%d K=%d (need N %% 128 == 0, K / ld %% 16 == 0)", p.M, p.N, p.K);
    return KR_ERR_UNSUPPORTED_SHAPE;
  }
  if ((epi == EPI_BIAS_GATE_RES || epi == EPI_BIAS_RES || epi == EPI_MUL) && p.residual == nullptr) {
    set_last_error("gemm_fp8: residual epilogue without residual pointer");
    return KR_ERR_INVALID_ARG;
  }
  if (scale_a == nullptr) {
    set_last_error("gemm_fp8: null activation scale");
    return KR_ERR_INVALID_ARG;
  }
  switch (epi) {
    case EPI_BIAS: return launch_fp8<EPI_BIAS>(a, lda, w, ldw, p, scale_a, scale_w, stream);
    case EPI_BIAS_GELU: return launch_fp8<EPI_BIAS_GELU>(a, lda, w, ldw, p, scale_a, scale_w, stream);
    case EPI_BIAS_GATE_RES: return launch_fp8<EPI_BIAS_GATE_RES>(a, lda, w, ldw, p, scale_a, scale_w, stream);
    case EPI_BIAS_RES: return launch_fp8<EPI_BIAS_RES>(a, lda, w, ldw, p, scale_a, scale_w, stream);
    default: set_last_error("gemm_fp8: unsupported epilogue %d", epi); return KR_ERR_INVALID_ARG;
  }
}

}  // namespace kr
