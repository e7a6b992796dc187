// kr_gemm2.cu — 2-CTA cluster variant of the persistent wgmma GEMM (kr_gemm.cu) for the wide DiT projections.
//
//   C[M,N] = epilogue( A[M,K] @ W[N,K]^T + bias[N] )        same operands / epilogues as kr_gemm.cu
//
// The two CTAs of a cluster compute the vertically adjacent 128 x 256 tiles (m, n) and (m+1, n), which use the
// same 256 x 64 W block per k-block.  Each CTA loads its own A tile and HALF of that W block, multicast into both
// CTAs (TMA .multicast::cluster), so the W operand crosses L2 -> SM once per pair of tiles instead of twice: a
// stage costs each SM 16 KB of A + 16 KB of W instead of 16 + 32 KB.
// Pipeline: a stage's full barrier expects A + the whole W block (both halves signal it); its empty barrier
// collects one arrive from each consumer warpgroup of BOTH CTAs (remote arrives through mapa), because the peer
// overwrites this CTA's W half when it refills the stage.  Roles are those of kr_gemm.cu: consumer warpgroups
// 0, 1 (64 rows each), TMA warpgroup 2.
#include "kr_common.cuh"
#include "kr_gemm_epi.cuh"
#include "kr_ops.h"

#include <cstdlib>

namespace kr {

namespace {
constexpr int G2_BM = 128, G2_BN = 256, G2_BK = 64;
constexpr int G2_THREADS = 384;
constexpr int G2_STAGES = 4;
constexpr int G2_A_BYTES = G2_BM * G2_BK * 2, G2_B_BYTES = G2_BN * G2_BK * 2;
constexpr int G2_STAGE_BYTES = G2_A_BYTES + G2_B_BYTES;
constexpr int G2_SCR_BYTES = 8 * kEpiScrFloats * 4;
constexpr int G2_SMEM = G2_STAGES * G2_STAGE_BYTES + G2_SCR_BYTES + 1024 + 256;
}  // namespace

template <bool kBf16, int kEpi>
__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(G2_THREADS, 1)
gemm2_tn_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                const GemmParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + G2_STAGES * G2_A_BYTES;
  float* scratch = reinterpret_cast<float*>(smem + G2_STAGES * G2_STAGE_BYTES);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + G2_STAGES * G2_STAGE_BYTES + G2_SCR_BYTES);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + G2_STAGES;

  const int warp = threadIdx.x >> 5;
  const uint32_t rank = cluster_ctarank();
  const int num_m = (p.M + G2_BM - 1) / G2_BM;
  const int num_pm = (num_m + 1) / 2;                 // row-block pairs (the last CTA of an odd count computes zeros)
  const int num_n = p.N / G2_BN;
  const int num_pairs = num_pm * num_n;
  const int num_k = (p.K + G2_BK - 1) / G2_BK;
  const int cluster = blockIdx.x >> 1, num_clusters = gridDim.x >> 1;

  if (threadIdx.x == 256) {
    prefetch_tmap(&tmap_a);
    prefetch_tmap(&tmap_b);
    for (int i = 0; i < G2_STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 4);   // 2 consumer warpgroups x 2 CTAs
    }
    fence_barrier_init();
  }
  cluster_sync();

  if (warp >= 8) {
    producer_regs();
    if (warp == 8 && elect_one()) {
      int stage = 0;
      uint32_t phase = 0;
      for (int t = cluster; t < num_pairs; t += num_clusters) {
        const int m_blk = 2 * (t % num_pm) + static_cast<int>(rank), n_blk = t / num_pm;
        for (int kb = 0; kb < num_k; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          mbar_expect_tx(&full_bar[stage], G2_STAGE_BYTES);
          tma_load_2d(smem_a + stage * G2_A_BYTES, &tmap_a, &full_bar[stage], kb * G2_BK, m_blk * G2_BM);
          tma_load_2d_mc(smem_b + stage * G2_B_BYTES + rank * (G2_B_BYTES / 2), &tmap_b, &full_bar[stage],
                         kb * G2_BK, n_blk * G2_BN + static_cast<int>(rank) * (G2_BN / 2), 0x3);
          if (++stage == G2_STAGES) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
  } else {
    consumer_regs();
    const int wg = warp >> 2;
    const uint32_t a_base = smem_u32(smem_a) + wg * 64 * 128, b_base = smem_u32(smem_b);
    float* scr = scratch + warp * kEpiScrFloats;
    int stage = 0;
    uint32_t phase = 0;
    for (int t = cluster; t < num_pairs; t += num_clusters) {
      const int m_blk = 2 * (t % num_pm) + static_cast<int>(rank), n_blk = t / num_pm;
      float acc[G2_BN / 2];
      gemm_mainloop<G2_BN, kBf16 ? 0 : 1, 2>(acc, a_base, b_base, G2_A_BYTES, G2_B_BYTES, G2_STAGES, full_bar,
                                             empty_bar, stage, phase, 0, num_k);
      gemm_frag_epilogue<G2_BN, kBf16, kEpi>(acc, scr, m_blk * G2_BM + wg * 64 + (warp & 3) * 16, n_blk * G2_BN,
                                             G2_BN, 1.0f, p);
    }
  }
  cluster_sync();
}

template <bool kBf16, int kEpi>
static int launch_gemm2(const void* a, int lda, const void* w, int ldw, const GemmParams& p, cudaStream_t stream) {
  CUtensorMap ta, tb;
  int rc = make_tmap_2d(&ta, a, p.M, p.K, lda, G2_BM, G2_BK, kBf16);
  if (rc != KR_OK) return rc;
  rc = make_tmap_2d(&tb, w, p.N, p.K, ldw, G2_BN / 2, G2_BK, kBf16);
  if (rc != KR_OK) return rc;
  auto kern = gemm2_tn_kernel<kBf16, kEpi>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, G2_SMEM);
    if (e != cudaSuccess) {
      set_last_error("gemm2: cudaFuncSetAttribute failed: %s", cudaGetErrorString(e));
      return KR_ERR_CUDA;
    }
    attr_set = true;
  }
  const int pairs = ((p.M + G2_BM - 1) / G2_BM + 1) / 2 * (p.N / G2_BN);
  int clusters = sm_count() / 2;
  if (clusters > pairs) clusters = pairs;
  kern<<<2 * clusters, G2_THREADS, G2_SMEM, stream>>>(ta, tb, p);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_last_error("gemm2: launch failed: %s", cudaGetErrorString(e));
    return KR_ERR_CUDA;
  }
  return KR_OK;
}

// N % 256 == 0 (the planner only sends such shapes here)
int gemm2_tn(int dtype, int epi, const void* a, int lda, const void* w, int ldw, const GemmParams& p,
             cudaStream_t stream) {
  const bool bf = dtype == 0;
#define KR_G2(E) (bf ? launch_gemm2<true, E>(a, lda, w, ldw, p, stream) : launch_gemm2<false, E>(a, lda, w, ldw, p, stream))
  switch (epi) {
    case EPI_BIAS: return KR_G2(EPI_BIAS);
    case EPI_BIAS_GELU: return KR_G2(EPI_BIAS_GELU);
    case EPI_BIAS_GATE_RES: return KR_G2(EPI_BIAS_GATE_RES);
    case EPI_BIAS_RES: return KR_G2(EPI_BIAS_RES);
    default: set_last_error("gemm2: unsupported epilogue %d", epi); return KR_ERR_INVALID_ARG;
  }
#undef KR_G2
}

}  // namespace kr
