// kr_gemm_sk.cu — stream-K variant of the persistent wgmma GEMM (kr_gemm.cu) for shapes whose output-tile
// count does not fill the SMs evenly.
//
//   C[M,N] = epilogue( A[M,K] @ W[N,K]^T + bias[N] )        same operands / epilogues as kr_gemm.cu
//
// Why: the data-parallel kernels give every CTA whole 128x256 output tiles.  A sequence-parallel rank of the
// multi-GPU mode owns M = 4680/N token rows (585 at 8 GPUs): to_qkv is then 5 x 60 = 300 tiles = 2.27 waves of
// 132 CTAs (a third wave for 36 tiles), the o / cross-attention / ffn.2 projections are 100 tiles (0.76 of a wave).
// Here the unit of work is one (tile, 64-wide k-block) MMA iteration: the num_tiles * num_k iterations are cut
// into one equal contiguous range per SM, so every SM runs the same number of k-blocks (+-1) whatever the
// tile count.  A range that starts or ends inside a tile yields a PARTIAL accumulator:
//   * every contributor of a split tile writes its fp32 partial (raw accumulator, 128 x 256) to its own slot of a
//     workspace in HBM/L2 (slot 2*cta + {0 first segment, 1 last segment}), fences, and bumps the tile's counter;
//   * the contributor that arrives last (counter == contributors - 1) re-reads all partials of the tile with
//     L1-bypassing loads, sums them in ascending CTA order (deterministic) and runs the fused epilogue.
// Tiles that one CTA covers completely take the data-parallel path (registers -> epilogue) untouched.
// Roles / pipelines are those of kr_gemm.cu: two consumer warpgroups (wgmma on 64 rows each, then the epilogue),
// warp 8 the TMA producer (warps 8..11 hand their registers to the consumers) (128x64 A + 256x64 W per stage, SWIZZLE_128B, 4-stage ring).
#include "kr_common.cuh"
#include "kr_gemm_epi.cuh"
#include "kr_ops.h"

namespace kr {

namespace {
constexpr int SK_BM = 128, SK_BN = 256, SK_BK = 64;
constexpr int SK_THREADS = 384;
constexpr int SK_STAGES = 4;
constexpr int SK_A_BYTES = SK_BM * SK_BK * 2, SK_B_BYTES = SK_BN * SK_BK * 2;
constexpr int SK_STAGE_BYTES = SK_A_BYTES + SK_B_BYTES;
constexpr int SK_SCR_BYTES = 8 * kEpiScrFloats * 4;
constexpr int SK_SMEM = SK_STAGES * SK_STAGE_BYTES + SK_SCR_BYTES + 1024 + 256;
constexpr size_t SK_SLOT_FLOATS = static_cast<size_t>(SK_BM) * SK_BN;
constexpr size_t SK_COUNTER_BYTES = 64 * 1024;      // 16384 tile counters in front of the partial slots

struct SkPlan {
  int num_m, num_n, num_k, num_tiles;
  long long q;       // iterations per CTA (the first r CTAs run q + 1)
  int r;
  float* slots;      // [2 * grid][128][256] fp32
  int* counters;     // [num_tiles], zero between launches (the last arriver resets its tile)
};

KR_DEVICE long long sk_begin(const SkPlan& s, int cta) {
  return static_cast<long long>(cta) * s.q + (cta < s.r ? cta : s.r);
}
KR_DEVICE int sk_cta_of(const SkPlan& s, long long it) {
  const long long split = static_cast<long long>(s.r) * (s.q + 1);
  return it < split ? static_cast<int>(it / (s.q + 1)) : s.r + static_cast<int>((it - split) / s.q);
}
}  // namespace

template <bool kBf16, int kEpi>
__global__ void __launch_bounds__(SK_THREADS, 1)
gemm_sk_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
               const GemmParams p, const SkPlan s) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + SK_STAGES * SK_A_BYTES;
  float* scratch = reinterpret_cast<float*>(smem + SK_STAGES * SK_STAGE_BYTES);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + SK_STAGES * SK_STAGE_BYTES + SK_SCR_BYTES);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + SK_STAGES;
  volatile int* last_flag = reinterpret_cast<volatile int*>(empty_bar + SK_STAGES);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const long long it_begin = sk_begin(s, blockIdx.x), it_end = sk_begin(s, blockIdx.x + 1);

  if (threadIdx.x == 256) {
    prefetch_tmap(&tmap_a);
    prefetch_tmap(&tmap_b);
    for (int i = 0; i < SK_STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 2);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp >= 8) {
    // ===================== TMA producer (warp 8; warps 9..11 only give their registers back) =====================
    producer_regs();
    if (warp == 8 && elect_one()) {
      int stage = 0;
      uint32_t phase = 0;
      for (long long it = it_begin; it < it_end;) {
        const int tile = static_cast<int>(it / s.num_k);
        const int k0 = static_cast<int>(it - static_cast<long long>(tile) * s.num_k);
        const long long left = it_end - it;
        const int k1 = (s.num_k - k0) < left ? s.num_k : k0 + static_cast<int>(left);
        const int m_blk = tile % s.num_m, n_blk = tile / s.num_m;
        for (int kb = k0; kb < k1; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          mbar_expect_tx(&full_bar[stage], SK_STAGE_BYTES);
          tma_load_2d(smem_a + stage * SK_A_BYTES, &tmap_a, &full_bar[stage], kb * SK_BK, m_blk * SK_BM);
          tma_load_2d(smem_b + stage * SK_B_BYTES, &tmap_b, &full_bar[stage], kb * SK_BK, n_blk * SK_BN);
          if (++stage == SK_STAGES) {
            stage = 0;
            phase ^= 1;
          }
        }
        it += k1 - k0;
      }
    }
  } else {
    // ===================== consumer warpgroups =====================
    consumer_regs();
    const int wg = warp >> 2;
    const int etid = threadIdx.x;                // 0..255 among the consumer threads
    const uint32_t a_base = smem_u32(smem_a) + wg * 64 * 128, b_base = smem_u32(smem_b);
    float* scr = scratch + warp * kEpiScrFloats;
    int stage = 0, seg = 0;
    uint32_t phase = 0;
    for (long long it = it_begin; it < it_end; ++seg) {
      const int tile = static_cast<int>(it / s.num_k);
      const int k0 = static_cast<int>(it - static_cast<long long>(tile) * s.num_k);
      const long long left = it_end - it;
      const int k1 = (s.num_k - k0) < left ? s.num_k : k0 + static_cast<int>(left);
      it += k1 - k0;
      const int m_blk = tile % s.num_m, n_blk = tile / s.num_m;
      float acc[SK_BN / 2];
      gemm_mainloop<SK_BN, kBf16 ? 0 : 1>(acc, a_base, b_base, SK_A_BYTES, SK_B_BYTES, SK_STAGES, full_bar,
                                          empty_bar, stage, phase, k0, k1);
      if (k0 == 0 && k1 == s.num_k) {
        gemm_frag_epilogue<SK_BN, kBf16, kEpi>(acc, scr, m_blk * SK_BM + wg * 64 + (warp & 3) * 16, n_blk * SK_BN,
                                               SK_BN, 1.0f, p);
        continue;
      }
      // ---- partial accumulator -> my workspace slot ([128][256] fp32, fragment by fragment) ----
      float* mine = s.slots + static_cast<size_t>(2 * blockIdx.x + (seg == 0 ? 0 : 1)) * SK_SLOT_FLOATS;
      {
        const int r = wg * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
        for (int j = 0; j < SK_BN / 8; ++j) {
          const int col = j * 8 + 2 * (lane & 3);
          __stcg(reinterpret_cast<float2*>(mine + static_cast<size_t>(r) * SK_BN + col),
                 make_float2(acc[4 * j], acc[4 * j + 1]));
          __stcg(reinterpret_cast<float2*>(mine + static_cast<size_t>(r + 8) * SK_BN + col),
                 make_float2(acc[4 * j + 2], acc[4 * j + 3]));
        }
      }
      __threadfence();
      // contributors of this tile: the CTAs whose ranges intersect [tile*num_k, (tile+1)*num_k)
      const long long t0 = static_cast<long long>(tile) * s.num_k;
      const int c_first = sk_cta_of(s, t0), c_last = sk_cta_of(s, t0 + s.num_k - 1);
      named_bar_sync(1, 256);
      if (etid == 0) {
        const int old = atomicAdd(s.counters + tile, 1);
        const int last = (old == c_last - c_first) ? 1 : 0;
        if (last) s.counters[tile] = 0;            // ready for the next launch
        *last_flag = last;
      }
      named_bar_sync(1, 256);
      const bool is_last = *last_flag != 0;
      named_bar_sync(1, 256);   // flag consumed before the next segment rewrites it
      if (is_last) {
        __threadfence();
        // thread = (row, half of the columns); partials summed in ascending CTA order
        const int lrow = etid >> 1, half = etid & 1;
        const int row = m_blk * SK_BM + lrow;
        if (row < p.M) {
          const uint16_t* gate_row = nullptr;
          if constexpr (kEpi == EPI_BIAS_GATE_RES) {
            const int g = (row + p.row_offset) / p.rows_per_gate;
            gate_row = reinterpret_cast<const uint16_t*>(p.gate) + static_cast<size_t>(g) * p.gate_stride;
          }
#pragma unroll 1
          for (int c = half * 4; c < half * 4 + 4; ++c) {
            float v[32];
#pragma unroll
            for (int j = 0; j < 32; ++j) v[j] = 0.f;
            for (int cc = c_first; cc <= c_last; ++cc) {
              // tile is cc's first segment iff cc's range starts inside (or at the start of) this tile
              const int sl = 2 * cc + (sk_begin(s, cc) >= t0 ? 0 : 1);
              const float4* src = reinterpret_cast<const float4*>(
                  s.slots + static_cast<size_t>(sl) * SK_SLOT_FLOATS + static_cast<size_t>(lrow) * SK_BN + c * 32);
#pragma unroll
              for (int j = 0; j < 8; ++j) {
                const float4 f = __ldcg(src + j);
                v[4 * j] += f.x; v[4 * j + 1] += f.y; v[4 * j + 2] += f.z; v[4 * j + 3] += f.w;
              }
            }
            gemm_epilogue_row<kBf16, kEpi, 32>(v, row, n_blk * SK_BN + c * 32, p, gate_row);
          }
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------
// host
// ---------------------------------------------------------------------------
size_t gemm_sk_workspace_bytes() {
  return SK_COUNTER_BYTES + static_cast<size_t>(2) * sm_count() * SK_SLOT_FLOATS * sizeof(float);
}

// Is stream-K worth it for this shape?  Compared on the data-parallel kernel's wave efficiency.
bool gemm_sk_preferred(int epi, int M, int N, int K) {
  if (epi == EPI_F32 || N % SK_BN != 0 || K < 8 * SK_BK) return false;
  const int sms = sm_count();
  const long tiles = static_cast<long>((M + SK_BM - 1) / SK_BM) * (N / SK_BN);
  if (tiles > SK_COUNTER_BYTES / 4) return false;
  const long waves = (tiles + sms - 1) / sms;
  const double eff = static_cast<double>(tiles) / static_cast<double>(waves * sms);
  return eff < 0.86;
}

template <bool kBf16, int kEpi>
static int launch_sk(const void* a, int lda, const void* w, int ldw, const GemmParams& p, void* ws,
                     cudaStream_t stream) {
  CUtensorMap ta, tb;
  int rc = make_tmap_2d(&ta, a, p.M, p.K, lda, SK_BM, SK_BK, kBf16);
  if (rc != KR_OK) return rc;
  rc = make_tmap_2d(&tb, w, p.N, p.K, ldw, SK_BN, SK_BK, kBf16);
  if (rc != KR_OK) return rc;
  auto kern = gemm_sk_kernel<kBf16, kEpi>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SK_SMEM);
    if (e != cudaSuccess) {
      set_last_error("gemm_sk: cudaFuncSetAttribute failed: %s", cudaGetErrorString(e));
      return KR_ERR_CUDA;
    }
    attr_set = true;
  }
  SkPlan s;
  s.num_m = (p.M + SK_BM - 1) / SK_BM;
  s.num_n = p.N / SK_BN;
  s.num_k = (p.K + SK_BK - 1) / SK_BK;
  s.num_tiles = s.num_m * s.num_n;
  const long long total = static_cast<long long>(s.num_tiles) * s.num_k;
  int grid = sm_count();
  if (grid > total) grid = static_cast<int>(total);
  s.q = total / grid;
  s.r = static_cast<int>(total % grid);
  s.counters = reinterpret_cast<int*>(ws);
  s.slots = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(ws) + SK_COUNTER_BYTES);
  kern<<<grid, SK_THREADS, SK_SMEM, stream>>>(ta, tb, p, s);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_last_error("gemm_sk: launch failed: %s", cudaGetErrorString(e));
    return KR_ERR_CUDA;
  }
  return KR_OK;
}

// workspace: gemm_sk_workspace_bytes() bytes, zero-filled once by the caller, private to one stream
int gemm_sk_tn(int dtype, int epi, const void* a, int lda, const void* w, int ldw, const GemmParams& p,
               void* workspace, size_t workspace_bytes, cudaStream_t stream) {
  if (workspace == nullptr || workspace_bytes < gemm_sk_workspace_bytes()) {
    set_last_error("gemm_sk: workspace of %zu bytes required", gemm_sk_workspace_bytes());
    return KR_ERR_INVALID_ARG;
  }
  const bool bf = dtype == 0;
#define KR_SK(E) (bf ? launch_sk<true, E>(a, lda, w, ldw, p, workspace, stream) \
                     : launch_sk<false, E>(a, lda, w, ldw, p, workspace, stream))
  switch (epi) {
    case EPI_BIAS: return KR_SK(EPI_BIAS);
    case EPI_BIAS_GELU: return KR_SK(EPI_BIAS_GELU);
    case EPI_BIAS_GATE_RES: return KR_SK(EPI_BIAS_GATE_RES);
    case EPI_BIAS_RES: return KR_SK(EPI_BIAS_RES);
    case EPI_MUL: return KR_SK(EPI_MUL);
    default: set_last_error("gemm_sk: unsupported epilogue %d", epi); return KR_ERR_INVALID_ARG;
  }
#undef KR_SK
}

}  // namespace kr
