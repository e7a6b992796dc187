// kr_gemm.cu — persistent wgmma GEMM for sm_90a.
//
//   C[M,N] = epilogue( A[M,K] @ W[N,K]^T + bias[N] )
//
// A and W are row-major with K contiguous (nn.Linear weight layout), 16-bit
// (bf16 or fp16), accumulation in fp32 registers.
//
// Replaces, on the reference path, every cuBLASLt call issued by nn.Linear in the
// DiT block (wan/modules/causal_model.py:246 to_qkv, :396 o, :433-435 ffn;
// wan/modules/model.py:183-227 cross-attn q/k/v/o; causal_model.py:614-623
// patch/text/time embeddings; :507 head) together with the elementwise kernels
// that follow them (bias add, GELU-tanh, per-frame gate, residual add).
//
// Structure (one CTA per SM, persistent over 128 x BLOCK_N output tiles):
//   warps 0..3  : consumer warpgroup 0 (rows 0..63 of the tile): wgmma, then the fused epilogue
//   warps 4..7  : consumer warpgroup 1 (rows 64..127)
//   warps 8..11 : TMA producer warpgroup (warp 8: A tile 128x64, W tile BLOCK_Nx64, SWIZZLE_128B), smem
//                 full/empty ring; it hands most of its registers to the consumers (setmaxnreg)
// BLOCK_N is a template parameter (the wgmma instruction encodes N); gemm_tn_kernel serves the fixed widths
// 32..256, gemm_flex_kernel the wave-fitted widths 96..256 whose last column tile may be narrower.
#include "kr_common.cuh"
#include "kr_gemm_epi.cuh"
#include "kr_ops.h"

#include <cstdlib>

namespace kr {


static constexpr int BLOCK_M = 128;
static constexpr int BLOCK_K = 64;   // 64 x 16-bit = 128 B = one swizzle row
static constexpr int kNumThreads = 384;
static constexpr int kSmemBudget = 227 * 1024;

template <int BLOCK_N>
struct GemmCfg {
  static constexpr int kABytes = BLOCK_M * BLOCK_K * 2;
  static constexpr int kBBytes = BLOCK_N * BLOCK_K * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kScrBytes = 8 * kEpiScrFloats * 4;
  static constexpr int kFit = (kSmemBudget - kScrBytes - 2048) / kStageBytes;
  static constexpr int kStages = kFit > 8 ? 8 : kFit;
  static constexpr int kSmemBytes = kStages * kStageBytes + kScrBytes + 1024 /*align*/ + 256 /*barriers*/;
  static_assert(kStages >= 2, "pipeline needs >= 2 stages");
};

template <int BLOCK_N, bool kBf16, int kEpi>
KR_DEVICE void gemm_body(const CUtensorMap* tmap_a, const CUtensorMap* tmap_b, const GemmParams& p) {
  using Cfg = GemmCfg<BLOCK_N>;
  extern __shared__ uint8_t smem_raw[];
  // 1024 B alignment for SWIZZLE_128B tiles
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + Cfg::kStages * Cfg::kABytes;
  float* scratch = reinterpret_cast<float*>(smem + Cfg::kStages * Cfg::kStageBytes);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + Cfg::kStages * Cfg::kStageBytes + Cfg::kScrBytes);
  uint64_t* full_bar = bars;                       // [kStages]
  uint64_t* empty_bar = bars + Cfg::kStages;       // [kStages]

  const int warp = threadIdx.x >> 5;

  const int num_m = (p.M + BLOCK_M - 1) / BLOCK_M;
  const int num_n = (p.N + BLOCK_N - 1) / BLOCK_N;   // last column tile may be narrower (TMA zero-fills, epilogue skips)
  const int num_tiles = num_m * num_n;
  const int num_k = (p.K + BLOCK_K - 1) / BLOCK_K;   // K tail: TMA zero-fills both operands

  if (threadIdx.x == 256) {
    prefetch_tmap(tmap_a);
    prefetch_tmap(tmap_b);
    for (int i = 0; i < Cfg::kStages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 2);   // one arrive per consumer warpgroup
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
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int m_blk = tile % num_m;
        const int n_blk = tile / num_m;
        for (int kb = 0; kb < num_k; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          mbar_expect_tx(&full_bar[stage], Cfg::kStageBytes);
          tma_load_2d(smem_a + stage * Cfg::kABytes, tmap_a, &full_bar[stage], kb * BLOCK_K,
                      m_blk * BLOCK_M);
          tma_load_2d(smem_b + stage * Cfg::kBBytes, tmap_b, &full_bar[stage], kb * BLOCK_K,
                      n_blk * BLOCK_N);
          if (++stage == Cfg::kStages) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
  } else {
    // ===================== consumer warpgroups =====================
    consumer_regs();
    const int wg = warp >> 2;
    const uint32_t a_base = smem_u32(smem_a) + wg * 64 * 128, b_base = smem_u32(smem_b);
    float* scr = scratch + warp * kEpiScrFloats;
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int m_blk = tile % num_m;
      const int n_blk = tile / num_m;
      float acc[BLOCK_N / 2];
      gemm_mainloop<BLOCK_N, kBf16 ? 0 : 1>(acc, a_base, b_base, Cfg::kABytes, Cfg::kBBytes, Cfg::kStages,
                                            full_bar, empty_bar, stage, phase, 0, num_k);
      const int n_valid = (p.N - n_blk * BLOCK_N) < BLOCK_N ? (p.N - n_blk * BLOCK_N) : BLOCK_N;
      gemm_frag_epilogue<BLOCK_N, kBf16, kEpi>(acc, scr, m_blk * BLOCK_M + wg * 64 + (warp & 3) * 16,
                                               n_blk * BLOCK_N, n_valid, 1.0f, p);
    }
  }
}

template <int BLOCK_N, bool kBf16, int kEpi>
__global__ void __launch_bounds__(kNumThreads, 1)
gemm_tn_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
               const GemmParams p) {
  gemm_body<BLOCK_N, kBf16, kEpi>(&tmap_a, &tmap_b, p);
}

// Same body with a tile width chosen at run time among 96..256 so that the tile count fills whole waves of SMs
// (the M = 4680/N-row shards of the multi-GPU mode).
template <int BLOCK_N, bool kBf16, int kEpi>
__global__ void __launch_bounds__(kNumThreads, 1)
gemm_flex_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                 const GemmParams p) {
  gemm_body<BLOCK_N, kBf16, kEpi>(&tmap_a, &tmap_b, p);
}

// ---------------------------------------------------------------------------
// host launcher
// ---------------------------------------------------------------------------
template <int BLOCK_N, bool kBf16, int kEpi>
static int launch_gemm(const void* a, int lda, const void* w, int ldw, const GemmParams& p,
                       cudaStream_t stream) {
  using Cfg = GemmCfg<BLOCK_N>;
  CUtensorMap ta, tb;
  int rc = make_tmap_2d(&ta, a, p.M, p.K, lda, BLOCK_M, BLOCK_K, kBf16);
  if (rc != KR_OK) return rc;
  rc = make_tmap_2d(&tb, w, p.N, p.K, ldw, BLOCK_N, BLOCK_K, kBf16);
  if (rc != KR_OK) return rc;
  auto kern = gemm_tn_kernel<BLOCK_N, kBf16, kEpi>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         Cfg::kSmemBytes);
    if (e != cudaSuccess) {
      set_last_error("gemm: cudaFuncSetAttribute failed: %s", cudaGetErrorString(e));
      return KR_ERR_CUDA;
    }
    attr_set = true;
  }
  const int num_tiles = ((p.M + BLOCK_M - 1) / BLOCK_M) * ((p.N + BLOCK_N - 1) / BLOCK_N);
  int grid = sm_count();
  if (grid > num_tiles) grid = num_tiles;
  kern<<<grid, kNumThreads, Cfg::kSmemBytes, stream>>>(ta, tb, p);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_last_error("gemm: launch failed: %s", cudaGetErrorString(e));
    return KR_ERR_CUDA;
  }
  return KR_OK;
}

// ---- runtime-width kernel: launcher + width choice -------------------------------------------------
// Cost model of one 128 x bn tile over one 64-wide k-block, in SM clocks: the MMA takes 4*bn at the H100 SXM
// data-sheet rate (989 TFLOP/s dense bf16 over 132 SMs at 1.83 GHz = 4096 FLOP/clk), the operand fetch
// (128 + bn) * 128 B at an assumed 64 B/clk per SM from L2; a shape costs waves * max of the two.
static double flex_tile_cost(int bn) {
  const double mma = 4.0 * bn, fetch = 2.0 * (128 + bn);
  return mma > fetch ? mma : fetch;
}
// Best runtime tile width for a shape the fixed-width kernels fill badly, or 0 to keep them.
int gemm_flex_bn(int epi, int M, int N, int K) {
  static const int mode = [] { const char* e = getenv("KR_GEMM_FLEX"); return e != nullptr ? atoi(e) : 1; }();
  if (mode <= 0 || N % 32 != 0 || K < 512 || N < 512) return 0;
  const int sms = sm_count();
  const long num_m = (M + BLOCK_M - 1) / BLOCK_M;
  // what the fixed-width dispatch would do
  int bn0 = N % 256 == 0 ? 256 : (N % 128 == 0 ? 128 : 0);
  if (bn0 == 256 && num_m * (N / 256) < sms && N % 128 == 0) bn0 = 128;
  if (bn0 == 0) return 0;
  const long t0 = num_m * (N / bn0);
  const double cost0 = static_cast<double>((t0 + sms - 1) / sms) * flex_tile_cost(bn0);
  int best = 0;
  double best_cost = cost0 * 0.94;                      // must win by a margin
  for (int bn = 256; bn >= 96; bn -= 32) {
    const long t = num_m * ((N + bn - 1) / bn);
    const double c = static_cast<double>((t + sms - 1) / sms) * flex_tile_cost(bn);
    if (c < best_cost) {
      best_cost = c;
      best = bn;
    }
  }
  (void)epi;
  return best;
}

template <int BN, bool kBf16, int kEpi>
static int launch_flex(const void* a, int lda, const void* w, int ldw, const GemmParams& p, cudaStream_t stream) {
  using Cfg = GemmCfg<BN>;
  CUtensorMap ta, tb;
  int rc = make_tmap_2d(&ta, a, p.M, p.K, lda, BLOCK_M, BLOCK_K, kBf16);
  if (rc != KR_OK) return rc;
  rc = make_tmap_2d(&tb, w, p.N, p.K, ldw, BN, BLOCK_K, kBf16);
  if (rc != KR_OK) return rc;
  auto kern = gemm_flex_kernel<BN, kBf16, kEpi>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes);
    if (e != cudaSuccess) {
      set_last_error("gemm_flex: cudaFuncSetAttribute failed: %s", cudaGetErrorString(e));
      return KR_ERR_CUDA;
    }
    attr_set = true;
  }
  const int num_tiles = ((p.M + BLOCK_M - 1) / BLOCK_M) * ((p.N + BN - 1) / BN);
  int grid = sm_count();
  if (grid > num_tiles) grid = num_tiles;
  kern<<<grid, kNumThreads, Cfg::kSmemBytes, stream>>>(ta, tb, p);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_last_error("gemm_flex: launch failed: %s", cudaGetErrorString(e));
    return KR_ERR_CUDA;
  }
  return KR_OK;
}

template <bool kBf16, int kEpi>
static int flex_width(const void* a, int lda, const void* w, int ldw, const GemmParams& p, int bn, cudaStream_t s) {
  switch (bn) {
    case 96: return launch_flex<96, kBf16, kEpi>(a, lda, w, ldw, p, s);
    case 128: return launch_flex<128, kBf16, kEpi>(a, lda, w, ldw, p, s);
    case 160: return launch_flex<160, kBf16, kEpi>(a, lda, w, ldw, p, s);
    case 192: return launch_flex<192, kBf16, kEpi>(a, lda, w, ldw, p, s);
    case 224: return launch_flex<224, kBf16, kEpi>(a, lda, w, ldw, p, s);
    case 256: return launch_flex<256, kBf16, kEpi>(a, lda, w, ldw, p, s);
    default: set_last_error("gemm_flex: unsupported tile width %d", bn); return KR_ERR_INVALID_ARG;
  }
}

static int gemm_flex(int dtype, int epi, const void* a, int lda, const void* w, int ldw, const GemmParams& p, int bn,
                     cudaStream_t s) {
  const bool bf = dtype == 0;
#define KR_FLEX(E) (bf ? flex_width<true, E>(a, lda, w, ldw, p, bn, s) : flex_width<false, E>(a, lda, w, ldw, p, bn, s))
  switch (epi) {
    case EPI_BIAS: return KR_FLEX(EPI_BIAS);
    case EPI_BIAS_GELU: return KR_FLEX(EPI_BIAS_GELU);
    case EPI_BIAS_GATE_RES: return KR_FLEX(EPI_BIAS_GATE_RES);
    case EPI_BIAS_RES: return KR_FLEX(EPI_BIAS_RES);
    case EPI_MUL: return KR_FLEX(EPI_MUL);
    default: set_last_error("gemm_flex: unsupported epilogue %d", epi); return KR_ERR_INVALID_ARG;
  }
#undef KR_FLEX
}

template <int BLOCK_N, bool kBf16>
static int dispatch_epi(int epi, const void* a, int lda, const void* w, int ldw,
                        const GemmParams& p, cudaStream_t s) {
  switch (epi) {
    case EPI_BIAS: return launch_gemm<BLOCK_N, kBf16, EPI_BIAS>(a, lda, w, ldw, p, s);
    case EPI_BIAS_GELU: return launch_gemm<BLOCK_N, kBf16, EPI_BIAS_GELU>(a, lda, w, ldw, p, s);
    case EPI_BIAS_GATE_RES:
      return launch_gemm<BLOCK_N, kBf16, EPI_BIAS_GATE_RES>(a, lda, w, ldw, p, s);
    case EPI_BIAS_RES: return launch_gemm<BLOCK_N, kBf16, EPI_BIAS_RES>(a, lda, w, ldw, p, s);
    case EPI_F32: return launch_gemm<BLOCK_N, kBf16, EPI_F32>(a, lda, w, ldw, p, s);
    case EPI_MUL: return launch_gemm<BLOCK_N, kBf16, EPI_MUL>(a, lda, w, ldw, p, s);
    default: set_last_error("gemm: unknown epilogue %d", epi); return KR_ERR_INVALID_ARG;
  }
}

// dtype: 0 = bf16, 1 = fp16
// Which kernel serves a shape:
//   0  the fixed-width kernel above
//   1  the 2-CTA cluster kernel (kr_gemm2.cu): same work per SM per wave as two 128x256 tiles, half the W traffic.
//      Measured on an H100 SXM (400 W limit, bench shapes M = 4680): 275 TFLOP/s against 446 for the single-CTA
//      kernel (its consumers hold a stage until both CTAs release it), so a pair-tile wave is costed 1.62 single
//      waves and the bench shapes keep the single-CTA kernels
//   2  stream-K (kr_gemm_sk.cu), only with a workspace and KR_GEMM_SK=1, when the data-parallel wave efficiency is poor
//   3  the runtime-width kernel (gemm_flex_bn)
// KR_GEMM2: 0 = never the cluster kernel, 1 = by the wave count (default), 2 = whenever N % 256 == 0 (tests)
int gemm_plan(int epi, int M, int N, int K, bool have_workspace) {
  static const int mode = [] { const char* e = getenv("KR_GEMM2"); return e != nullptr ? atoi(e) : 1; }();
  // KR_GEMM_SK: 0 = never stream-K (default), 1 = when the data-parallel wave efficiency is poor
  static const int sk_mode = [] { const char* e = getenv("KR_GEMM_SK"); return e != nullptr ? atoi(e) : 0; }();
  if (have_workspace && sk_mode > 0 && gemm_sk_preferred(epi, M, N, K)) return 2;
  const int flex = (epi == EPI_F32) ? 0 : gemm_flex_bn(epi, M, N, K);
  if (mode <= 0 || epi == EPI_F32 || epi == EPI_MUL || N % 256 != 0 || K < 256) return flex ? 3 : 0;
  if (mode == 2) return 1;
  const int sms = sm_count(), pairs = sms / 2, nb = N / 256;
  const long tiles1 = static_cast<long>((M + 127) / 128) * nb;
  const long tiles_p = static_cast<long>((M + 255) / 256) * nb;
  if (tiles_p < 4L * pairs) return flex ? 3 : 0;
  constexpr double kPairWaveCost = 1.62;   // measured cluster vs single-CTA tile throughput, see above
  if (static_cast<double>((tiles_p + pairs - 1) / pairs) * kPairWaveCost <= static_cast<double>((tiles1 + sms - 1) / sms))
    return 1;
  return flex ? 3 : 0;
}

namespace {
int gemm_single(int dtype, int epi, const void* a, int lda, const void* w, int ldw, const GemmParams& p,
                cudaStream_t stream) {
  int bn;
  if (p.N % 256 == 0) bn = 256;
  else if (p.N % 128 == 0) bn = 128;
  else if (p.N % 64 == 0) bn = 64;
  else if (p.N % 32 == 0) bn = 32;
  else bn = 0;
  // prefer the tile width that fills the machine: small problems use narrower tiles
  const int num_m = (p.M + BLOCK_M - 1) / BLOCK_M;
  if (bn == 256 && num_m * (p.N / 256) < sm_count() && p.N % 128 == 0) bn = 128;
  if (bn == 128 && num_m * (p.N / 128) < sm_count() && p.N % 64 == 0) bn = 64;
  const bool bf = dtype == 0;
  switch (bn) {
    case 256:
      return bf ? dispatch_epi<256, true>(epi, a, lda, w, ldw, p, stream)
                : dispatch_epi<256, false>(epi, a, lda, w, ldw, p, stream);
    case 128:
      return bf ? dispatch_epi<128, true>(epi, a, lda, w, ldw, p, stream)
                : dispatch_epi<128, false>(epi, a, lda, w, ldw, p, stream);
    case 64:
      return bf ? dispatch_epi<64, true>(epi, a, lda, w, ldw, p, stream)
                : dispatch_epi<64, false>(epi, a, lda, w, ldw, p, stream);
    case 32:
      return bf ? dispatch_epi<32, true>(epi, a, lda, w, ldw, p, stream)
                : dispatch_epi<32, false>(epi, a, lda, w, ldw, p, stream);
    default:
      set_last_error("gemm: N=%d not a multiple of 32", p.N);
      return KR_ERR_UNSUPPORTED_SHAPE;
  }
}
}  // namespace

int gemm_tn(int dtype, int epi, const void* a, int lda, const void* w, int ldw, const GemmParams& p,
            cudaStream_t stream, void* workspace, size_t workspace_bytes) {
  if (p.M <= 0 || p.N <= 0 || p.K <= 0) {
    set_last_error("gemm: non-positive shape M=%d N=%d K=%d", p.M, p.N, p.K);
    return KR_ERR_INVALID_ARG;
  }
  if (p.K % 8 != 0 || p.N % 32 != 0 || lda % 8 != 0 || ldw % 8 != 0 || p.ldc % 8 != 0) {
    set_last_error("gemm: unsupported shape M=%d N=%d K=%d (need K%%8==0, N%%32==0, ld%%8==0)",
                   p.M, p.N, p.K);
    return KR_ERR_UNSUPPORTED_SHAPE;
  }
  if ((epi == EPI_BIAS_GATE_RES || epi == EPI_BIAS_RES || epi == EPI_MUL) && p.residual == nullptr) {
    set_last_error("gemm: residual epilogue without residual pointer");
    return KR_ERR_INVALID_ARG;
  }
  if (p.out2 != nullptr && (p.n_split % 256 != 0 || p.ldc2 % 8 != 0 || epi == EPI_F32)) {
    set_last_error("gemm: split output needs n_split %% 256 == 0, ldc2 %% 8 == 0 and a 16-bit epilogue");
    return KR_ERR_INVALID_ARG;
  }
  if (epi == EPI_BIAS_GATE_RES && (p.gate == nullptr || p.rows_per_gate <= 0)) {
    set_last_error("gemm: gate epilogue without gate pointer / rows_per_gate");
    return KR_ERR_INVALID_ARG;
  }
  const bool have_ws = workspace != nullptr && workspace_bytes >= gemm_sk_workspace_bytes();
  const int plan = gemm_plan(epi, p.M, p.N, p.K, have_ws);
  if (plan == 2) return gemm_sk_tn(dtype, epi, a, lda, w, ldw, p, workspace, workspace_bytes, stream);
  if (plan == 1) return gemm2_tn(dtype, epi, a, lda, w, ldw, p, stream);
  if (plan == 3) {
    if (p.out2 != nullptr && p.n_split % 32 != 0) {
      set_last_error("gemm: split output needs n_split %% 32 == 0");
      return KR_ERR_INVALID_ARG;
    }
    return gemm_flex(dtype, epi, a, lda, w, ldw, p, gemm_flex_bn(epi, p.M, p.N, p.K), stream);
  }
  return gemm_single(dtype, epi, a, lda, w, ldw, p, stream);
}

}  // namespace kr
