// kr_attn.cu — wgmma flash-attention forward for sm_90a, head_dim 128.
//
//   O[q, h, :] = softmax_k( scale * Q[q, h, :] . K[k, h, :] ) V[k, h, :]
//
// Replaces flash_attn_func (FA2 mma.sync) on the reference path:
//   * cached self-attention   wan/modules/causal_model.py:386-390 -> attention.py:65-70
//   * recompute (block-causal) self-attention  causal_model.py:339-348 (FlexAttention)
//     mask rule causal_model.py:134-138: allowed iff kv < ends[q] (| q == kv), optional window
//   * T5 cross-attention      wan/modules/model.py:214-215
// Layout is the reference's [L, heads, 128] (row pitch = heads*128 elements), K/V read in place
// from the rolling cache tensors.
//
// CTA = 128 query rows of one head:
//   warps 0..3    : consumer warpgroup 0 (query rows 0..63):  S = Q.K^T (wgmma, SS), online softmax in
//                   registers, O += P.V (wgmma, P from registers, V MN-major from shared memory)
//   warps 4..7    : consumer warpgroup 1 (query rows 64..127)
//   warps 8..11   : TMA producer warpgroup (warp 8: Q once, K/V ring of 32 KB stages K0 V0 K1 V1 ...)
// The two consumer warpgroups run out of step, so one's softmax overlaps the other's MMAs.
// Online softmax with lazy rescaling (O is only rescaled when the running max grows by > 2^8).
#include "kr_common.cuh"
#include "kr_ops.h"

#include <cmath>
#include <cstdlib>

namespace kr {


static constexpr int kHeadDim = 128;
static constexpr int kTileQ = 128;
static constexpr int kTileKV = 128;
static constexpr int kKvStages = 4;
static constexpr int kTileBytes = kTileKV * kHeadDim * 2;   // 32 KB
static constexpr int kHalfBytes = kTileBytes / 2;           // one 64-column swizzle panel
static constexpr int kAttnThreads = 384;
static constexpr int kAttnSmem = kTileBytes + kKvStages * kTileBytes + 1024 + 256;

template <bool kBf16>
__global__ void __launch_bounds__(kAttnThreads, 1)
attn_fwd_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                const __grid_constant__ CUtensorMap tmap_v, const AttnParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* smem_q = smem;                          // [2 panels][128 rows][128 B]
  uint8_t* smem_kv = smem + kTileBytes;            // kKvStages tiles
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_kv + kKvStages * kTileBytes);
  uint64_t* q_full = bars;                 // [1]
  uint64_t* kv_full = bars + 1;            // [kKvStages]
  uint64_t* kv_empty = kv_full + kKvStages;   // [kKvStages]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int nqb = (p.Lq + kTileQ - 1) / kTileQ;
  const int head = blockIdx.x / nqb;
  const int q0 = (blockIdx.x % nqb) * kTileQ;

  // number of KV tiles this CTA visits
  int kv_limit = p.Lkv;
  if (p.mask_mode == 1) {
    int last_q = q0 + kTileQ - 1;
    if (last_q > p.Lq - 1) last_q = p.Lq - 1;
    const int hi = (last_q / p.block_len + 1) * p.block_len;
    if (hi < kv_limit) kv_limit = hi;
  }
  const int n_tiles = (kv_limit + kTileKV - 1) / kTileKV;

  if (threadIdx.x == 256) {
    prefetch_tmap(&tmap_q);
    prefetch_tmap(&tmap_k);
    prefetch_tmap(&tmap_v);
    mbar_init(q_full, 1);
    for (int i = 0; i < kKvStages; ++i) {
      mbar_init(&kv_full[i], 1);
      mbar_init(&kv_empty[i], 2);   // one arrive per consumer warpgroup
    }
    fence_barrier_init();
  }
  __syncthreads();

  // ring items: K_j = 2j, V_j = 2j + 1
  auto st = [](int item) { return item % kKvStages; };
  auto ph = [](int item) { return static_cast<uint32_t>((item / kKvStages) & 1); };

  if (warp >= 8) {
    // ===================== TMA producer =====================
    producer_regs();
    if (warp == 8 && elect_one()) {
      const int col = head * kHeadDim;
      mbar_expect_tx(q_full, kTileBytes);
      for (int h = 0; h < 2; ++h) tma_load_2d(smem_q + h * kHalfBytes, &tmap_q, q_full, col + h * 64, q0);
      for (int it = 0; it < 2 * n_tiles; ++it) {
        const int j = it >> 1;
        const CUtensorMap* tm = (it & 1) ? &tmap_v : &tmap_k;
        mbar_wait(&kv_empty[st(it)], ph(it) ^ 1);
        mbar_expect_tx(&kv_full[st(it)], kTileBytes);
        for (int h = 0; h < 2; ++h)
          tma_load_2d(smem_kv + st(it) * kTileBytes + h * kHalfBytes, tm, &kv_full[st(it)], col + h * 64,
                      j * kTileKV);
      }
    }
    return;
  }

  // ===================== consumer warpgroups =====================
  consumer_regs();
  const int wg = warp >> 2;
  const bool leader = (threadIdx.x & 127) == 0;
  const uint32_t q_addr = smem_u32(smem_q) + wg * 64 * 128;
  const uint32_t kv_addr = smem_u32(smem_kv);
  // this thread's two query rows (fragment rows lane/4 and lane/4 + 8 of its warp's 16)
  int q_row[2], row_hi[2], row_lo[2], n_phantom[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    q_row[r] = q0 + wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * r;
    row_hi[r] = p.Lkv;
    row_lo[r] = 0;
    n_phantom[r] = 0;
    if (p.mask_mode == 1) {
      const int qq = q_row[r] < p.Lq ? q_row[r] : p.Lq - 1;
      const int hi = (qq / p.block_len + 1) * p.block_len;
      if (p.window > 0) row_lo[r] = hi - p.window > 0 ? hi - p.window : 0;
      if (hi < row_hi[r]) row_hi[r] = hi;
      if (hi > p.Lkv) n_phantom[r] = hi - p.Lkv < p.pad_keys ? hi - p.Lkv : p.pad_keys;
    }
  }
  float m_run[2] = {-INFINITY, -INFINITY};
  float l_run[2] = {0.f, 0.f};     // this thread's partial row sums (its 2 columns of every 8)
  const float sl2 = p.scale_log2;
  float o[kHeadDim / 2];
#pragma unroll
  for (int i = 0; i < kHeadDim / 2; ++i) o[i] = 0.f;

  mbar_wait(q_full, 0);
  for (int j = 0; j < n_tiles; ++j) {
    // ---- S = Q . K_j^T ----
    float s[kTileKV / 2];
    mbar_wait(&kv_full[st(2 * j)], ph(2 * j));
    {
      const uint32_t b = kv_addr + st(2 * j) * kTileBytes;
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kHeadDim / 16; ++k) {
        const uint32_t off = (k >> 2) * kHalfBytes + (k & 3) * 32;
        wgmma_ss<kTileKV, kBf16, 0>(s, make_smem_desc(q_addr + off, 16, 1024), make_smem_desc(b + off, 16, 1024),
                                    k != 0 ? 1 : 0);
      }
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence(s);
    }
    if (leader) mbar_arrive(&kv_empty[st(2 * j)]);

    // ---- mask, running max, lazy rescale ----
    float nms[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int hi = row_hi[r] - j * kTileKV, lo = row_lo[r] - j * kTileKV;
      if (hi < kTileKV || lo > 0) {
#pragma unroll
        for (int nb = 0; nb < kTileKV / 8; ++nb)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int c = nb * 8 + 2 * (lane & 3) + e;
            if (c >= hi || c < lo) s[4 * nb + 2 * r + e] = -INFINITY;
          }
      }
      float mt = -INFINITY;
#pragma unroll
      for (int nb = 0; nb < kTileKV / 8; ++nb) mt = fmaxf(mt, fmaxf(s[4 * nb + 2 * r], s[4 * nb + 2 * r + 1]));
      mt = fmaxf(mt, __shfl_xor_sync(0xffffffffu, mt, 1));
      mt = fmaxf(mt, __shfl_xor_sync(0xffffffffu, mt, 2));
      const float m_new = fmaxf(m_run[r], mt);
      const bool need = (m_new - m_run[r]) * sl2 > 8.0f;   // also true when m_run == -inf
      const float m_used = need ? m_new : m_run[r];
      const float alpha = need ? fast_exp2((m_run[r] - m_new) * sl2) : 1.0f;
      if (need && j > 0) {
#pragma unroll
        for (int nb = 0; nb < kHeadDim / 8; ++nb) {
          o[4 * nb + 2 * r] *= alpha;
          o[4 * nb + 2 * r + 1] *= alpha;
        }
      }
      l_run[r] *= alpha;
      m_run[r] = m_used;
      // a row whose every visible key so far is masked (local window) keeps m = -inf: use 0
      nms[r] = (m_used == -INFINITY) ? 0.f : -m_used * sl2;
    }
    // ---- P = exp2(S * scale_log2 - m), packed as the A operand of P.V ----
    uint32_t pa[kTileKV / 16][4];
#pragma unroll
    for (int kk = 0; kk < kTileKV / 16; ++kk) {
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          const int i = 8 * kk + 4 * h + 2 * r;
          const float a0 = fast_exp2(fmaf(s[i], sl2, nms[r]));
          const float a1 = fast_exp2(fmaf(s[i + 1], sl2, nms[r]));
          l_run[r] += a0 + a1;
          pa[kk][2 * h + r] = kBf16 ? pack_bf16x2(a0, a1) : pack_f16x2(a0, a1);
        }
    }
    // ---- O += P . V_j ----
    mbar_wait(&kv_full[st(2 * j + 1)], ph(2 * j + 1));
    {
      const uint32_t b = kv_addr + st(2 * j + 1) * kTileBytes;
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < kTileKV / 16; ++kk)
        // V: 16 key rows of 128 B per panel, the next 64 head dims one panel (kHalfBytes) further
        wgmma_rs<kHeadDim, kBf16>(o, pa[kk], make_smem_desc(b + kk * 2048, kHalfBytes, 1024), 1);
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence(o);
    }
    if (leader) mbar_arrive(&kv_empty[st(2 * j + 1)]);
  }

  // ---- epilogue: O / l -> global ----
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    float l = l_run[r];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    float o_scale = 1.0f;
    if (n_phantom[r] > 0) {
      // phantom keys: score 0, value 0 -> only the softmax denominator (and max) see them
      const float m_fin = fmaxf(m_run[r], 0.f);
      o_scale = fast_exp2((m_run[r] - m_fin) * sl2);
      l = l * o_scale + static_cast<float>(n_phantom[r]) * fast_exp2(-m_fin * sl2);
    }
    const float inv_l = o_scale / l;
    if (q_row[r] < p.Lq) {
      uint16_t* orow = reinterpret_cast<uint16_t*>(p.out) + static_cast<size_t>(q_row[r]) * p.ldo +
                       head * kHeadDim + 2 * (lane & 3);
#pragma unroll
      for (int nb = 0; nb < kHeadDim / 8; ++nb) {
        const float f0 = o[4 * nb + 2 * r] * inv_l, f1 = o[4 * nb + 2 * r + 1] * inv_l;
        *reinterpret_cast<uint32_t*>(orow + nb * 8) = kBf16 ? pack_bf16x2(f0, f1) : pack_f16x2(f0, f1);
      }
    }
  }
}

// q: [Lq, ldq] (head h at columns h*128..), k/v: [>=Lkv, ldk/ldv]; dtype 0 = bf16, 1 = fp16
int attn_fwd(int dtype, const void* q, int ldq, const void* k, int ldk, const void* v, int ldv,
             const AttnParams& p, cudaStream_t stream) {
  if (p.Lq <= 0 || p.Lkv <= 0 || p.heads <= 0) {
    set_last_error("attn_fwd: non-positive shape Lq=%d Lkv=%d heads=%d", p.Lq, p.Lkv, p.heads);
    return KR_ERR_INVALID_ARG;
  }
  if (ldq % 8 != 0 || ldk % 8 != 0 || ldv % 8 != 0 || p.ldo % 8 != 0) {
    set_last_error("attn_fwd: leading dimensions must be multiples of 8 elements");
    return KR_ERR_UNSUPPORTED_SHAPE;
  }
  if (p.mask_mode == 1 && p.block_len <= 0) {
    set_last_error("attn_fwd: block-causal mask needs block_len > 0");
    return KR_ERR_INVALID_ARG;
  }
  const bool bf = dtype == 0;
  CUtensorMap tq, tk, tv;
  int rc = make_tmap_2d(&tq, q, p.Lq, static_cast<uint64_t>(p.heads) * kHeadDim, ldq, kTileQ, 64, bf);
  if (rc != KR_OK) return rc;
  rc = make_tmap_2d(&tk, k, p.Lkv, static_cast<uint64_t>(p.heads) * kHeadDim, ldk, kTileKV, 64, bf);
  if (rc != KR_OK) return rc;
  rc = make_tmap_2d(&tv, v, p.Lkv, static_cast<uint64_t>(p.heads) * kHeadDim, ldv, kTileKV, 64, bf);
  if (rc != KR_OK) return rc;
  using Kern = void (*)(CUtensorMap, CUtensorMap, CUtensorMap, AttnParams);
  Kern kern = bf ? attn_fwd_kernel<true> : attn_fwd_kernel<false>;
  {
    static bool attr_set[2] = {false, false};
    if (!attr_set[bf ? 0 : 1]) {
      cudaError_t e =
          cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kAttnSmem);
      if (e != cudaSuccess) {
        set_last_error("attn_fwd: cudaFuncSetAttribute failed: %s", cudaGetErrorString(e));
        return KR_ERR_CUDA;
      }
      attr_set[bf ? 0 : 1] = true;
    }
    dim3 grid(((p.Lq + kTileQ - 1) / kTileQ) * p.heads);
    kern<<<grid, kAttnThreads, kAttnSmem, stream>>>(tq, tk, tv, p);
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_last_error("attn_fwd: launch failed: %s", cudaGetErrorString(e));
    return KR_ERR_CUDA;
  }
  return KR_OK;
}

}  // namespace kr
