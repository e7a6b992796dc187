// kr_t5attn.cu — wgmma attention for the UMT5 text encoder: head_dim 64, additive relative-position
// bias, key-padding mask, no 1/sqrt(d) scaling.
//
//   O[q, h, :] = softmax_k( bf16(bf16(Q[q,h,:] . K[k,h,:]) + bias[h, k - q]) ) V[k, h, :]
//
// Replaces, on the reference path, T5Attention.forward (wan/modules/t5.py:86-120): the two einsums, the
// [B, heads, L, L] bias tensor (pos_bias of T5RelativeEmbedding :221-264 + masked_fill with finfo.min) and the
// fp32 softmax.
// The position bias only depends on (head, k - q): the host gathers it once per layer into `bias_delta`
// [heads, 2L-1] (entry d = embedding[bucket(d - (L-1))][head]) and the kernel keeps one head's row in shared memory.
// Rounding points follow the reference's bf16 execution: the einsum output is rounded to bf16, the bias add is a
// bf16 add, the softmax runs in fp32 and P is rounded to bf16 before P.V (here un-normalised, flash style; the
// 1/rowsum is applied to the fp32 output).
//
// CTA = 128 query rows of one head; key tiles of 128 (online softmax across tiles):
//   warps 0..7: two consumer warpgroups (64 query rows each): S = Q.K^T and O += P.V with wgmma, softmax in registers
//   warps 8..11: TMA warpgroup (Q 128x64 once, K/V 128x64 tiles through a 4-stage ring K0 V0 K1 V1 ...)
// The op is 4.3 GFLOP per encoder layer (0.1 % of the encoder): the design goal is "one launch, nothing in HBM but
// q/k/v/o".
#include "kr_common.cuh"
#include "kr_ops.h"

#include <cmath>

namespace kr {

namespace {
constexpr int T5_D = 64, T5_TQ = 128, T5_TK = 128, T5_THREADS = 384, T5_STAGES = 4;
constexpr int T5_Q_BYTES = T5_TQ * T5_D * 2, T5_KV_BYTES = T5_TK * T5_D * 2;
constexpr int T5_MAX_L = 1024;
constexpr int T5_SMEM = T5_Q_BYTES + T5_STAGES * T5_KV_BYTES + (2 * T5_MAX_L) * 2 + T5_MAX_L + 1024 + 256;
}  // namespace

__global__ void __launch_bounds__(T5_THREADS, 1)
t5_attn_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
               const __grid_constant__ CUtensorMap tmap_v, const T5AttnParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* smem_q = smem;
  uint8_t* smem_kv = smem + T5_Q_BYTES;                                          // T5_STAGES tiles
  uint16_t* bias_s = reinterpret_cast<uint16_t*>(smem_kv + T5_STAGES * T5_KV_BYTES);   // [2L-1]
  uint8_t* mask_s = reinterpret_cast<uint8_t*>(bias_s + 2 * T5_MAX_L);           // [L]
  uint64_t* bars = reinterpret_cast<uint64_t*>(mask_s + T5_MAX_L);
  uint64_t* q_full = bars;                     // [1]
  uint64_t* kv_full = bars + 1;                // [T5_STAGES]
  uint64_t* kv_empty = kv_full + T5_STAGES;    // [T5_STAGES]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nqb = (p.L + T5_TQ - 1) / T5_TQ;
  const int head = blockIdx.x / nqb, q0 = (blockIdx.x % nqb) * T5_TQ;
  const int n_tiles = (p.L + T5_TK - 1) / T5_TK;
  const int col = head * T5_D;

  if (threadIdx.x == 256) {
    prefetch_tmap(&tmap_q);
    prefetch_tmap(&tmap_k);
    prefetch_tmap(&tmap_v);
    mbar_init(q_full, 1);
    for (int i = 0; i < T5_STAGES; ++i) {
      mbar_init(&kv_full[i], 1);
      mbar_init(&kv_empty[i], 2);
    }
    fence_barrier_init();
  }
  // this head's bias row and the key mask -> shared memory (all threads)
  {
    const uint16_t* src = reinterpret_cast<const uint16_t*>(p.bias_delta) + static_cast<size_t>(head) * (2 * p.L - 1);
    for (int i = threadIdx.x; i < 2 * p.L - 1; i += T5_THREADS) bias_s[i] = src[i];
    for (int i = threadIdx.x; i < p.L; i += T5_THREADS)
      mask_s[i] = p.key_mask != nullptr ? reinterpret_cast<const uint8_t*>(p.key_mask)[i] : 1;
  }
  __syncthreads();

  auto st = [](int item) { return item % T5_STAGES; };
  auto ph = [](int item) { return static_cast<uint32_t>((item / T5_STAGES) & 1); };

  if (warp >= 8) {
    producer_regs();
    if (warp == 8 && elect_one()) {
      mbar_expect_tx(q_full, T5_Q_BYTES);
      tma_load_2d(smem_q, &tmap_q, q_full, col, q0);
      for (int it = 0; it < 2 * n_tiles; ++it) {
        mbar_wait(&kv_empty[st(it)], ph(it) ^ 1);
        mbar_expect_tx(&kv_full[st(it)], T5_KV_BYTES);
        tma_load_2d(smem_kv + st(it) * T5_KV_BYTES, (it & 1) ? &tmap_v : &tmap_k, &kv_full[st(it)], col,
                    (it >> 1) * T5_TK);
      }
    }
    return;
  }

  consumer_regs();
  const int wg = warp >> 2;
  const bool leader = (threadIdx.x & 127) == 0;
  const uint32_t q_addr = smem_u32(smem_q) + wg * 64 * 128, kv_addr = smem_u32(smem_kv);
  const float kLog2e = 1.4426950408889634f;
  const float kMin = -3.3895313892515355e38f;     // torch.finfo(torch.bfloat16).min
  int q_row[2], qq[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    q_row[r] = q0 + wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * r;
    qq[r] = q_row[r] < p.L ? q_row[r] : p.L - 1;
  }
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  float o[T5_D / 2];
#pragma unroll
  for (int i = 0; i < T5_D / 2; ++i) o[i] = 0.f;

  mbar_wait(q_full, 0);
  for (int j = 0; j < n_tiles; ++j) {
    float s[T5_TK / 2];
    mbar_wait(&kv_full[st(2 * j)], ph(2 * j));
    {
      const uint32_t b = kv_addr + st(2 * j) * T5_KV_BYTES;
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < T5_D / 16; ++k)
        wgmma_ss<T5_TK, true, 0>(s, make_smem_desc(q_addr + k * 32, 16, 1024), make_smem_desc(b + k * 32, 16, 1024),
                                 k != 0 ? 1 : 0);
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence(s);
    }
    if (leader) mbar_arrive(&kv_empty[st(2 * j)]);
    // the reference's bf16(bf16(s) + bias), masked keys = finfo.min, key rows past L (TMA zero fill) = -inf
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      float mt = -INFINITY;
#pragma unroll
      for (int nb = 0; nb < T5_TK / 8; ++nb)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int k = j * T5_TK + nb * 8 + 2 * (lane & 3) + e;
          float v = -INFINITY;
          if (k < p.L) {
            const float b = __bfloat162float(__ushort_as_bfloat16(bias_s[k - qq[r] + p.L - 1]));
            v = mask_s[k] ? bf16_round(bf16_round(s[4 * nb + 2 * r + e]) + b) : kMin;
          }
          s[4 * nb + 2 * r + e] = v;
          mt = fmaxf(mt, v);
        }
      mt = fmaxf(mt, __shfl_xor_sync(0xffffffffu, mt, 1));
      mt = fmaxf(mt, __shfl_xor_sync(0xffffffffu, mt, 2));
      const float m_new = fmaxf(m_run[r], mt);
      const float alpha = fast_exp2((m_run[r] - m_new) * kLog2e);     // 0 on the first tile (m_run = -inf)
#pragma unroll
      for (int nb = 0; nb < T5_D / 8; ++nb) {
        o[4 * nb + 2 * r] *= alpha;
        o[4 * nb + 2 * r + 1] *= alpha;
      }
      l_run[r] *= alpha;
      m_run[r] = m_new;
    }
    // P = exp2((v - m) log2e): v and m are bf16 values, so v - m is exact in fp32, 0 when both are finfo.min (a
    // tile whose keys are all masked: P = 1, as torch.softmax over equal finfo.min scores; a later real key's
    // alpha = 0 drops them).  The fused -m * log2e of the usual form overflows to +inf there and makes P = inf.
    uint32_t pa[T5_TK / 16][4];
#pragma unroll
    for (int kk = 0; kk < T5_TK / 16; ++kk)
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          const int i = 8 * kk + 4 * h + 2 * r;
          const float a0 = fast_exp2((s[i] - m_run[r]) * kLog2e);
          const float a1 = fast_exp2((s[i + 1] - m_run[r]) * kLog2e);
          l_run[r] += a0 + a1;
          pa[kk][2 * h + r] = pack_bf16x2(a0, a1);
        }
    mbar_wait(&kv_full[st(2 * j + 1)], ph(2 * j + 1));
    {
      const uint32_t b = kv_addr + st(2 * j + 1) * T5_KV_BYTES;
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < T5_TK / 16; ++kk)
        // V: 16 key rows of 128 B (all 64 head dims) per k-step
        wgmma_rs<T5_D, true>(o, pa[kk], make_smem_desc(b + kk * 2048, 1024, 1024), 1);
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence(o);
    }
    if (leader) mbar_arrive(&kv_empty[st(2 * j + 1)]);
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    float l = l_run[r];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const float inv_l = 1.0f / l;
    if (q_row[r] < p.L) {
      uint16_t* orow = reinterpret_cast<uint16_t*>(p.out) + static_cast<size_t>(q_row[r]) * p.ldo + col + 2 * (lane & 3);
#pragma unroll
      for (int nb = 0; nb < T5_D / 8; ++nb)
        *reinterpret_cast<uint32_t*>(orow + nb * 8) = pack_bf16x2(o[4 * nb + 2 * r] * inv_l, o[4 * nb + 2 * r + 1] * inv_l);
    }
  }
}

int t5_attn(const void* q, int ldq, const void* k, int ldk, const void* v, int ldv, const T5AttnParams& p,
            cudaStream_t stream) {
  if (p.L <= 0 || p.L > T5_MAX_L || p.heads <= 0 || ldq % 8 != 0 || ldk % 8 != 0 || ldv % 8 != 0 || p.ldo % 8 != 0) {
    set_last_error("t5_attn: unsupported L=%d heads=%d (L <= %d, pitches %% 8 == 0)", p.L, p.heads, T5_MAX_L);
    return KR_ERR_UNSUPPORTED_SHAPE;
  }
  CUtensorMap tq, tk, tv;
  const uint64_t cols = static_cast<uint64_t>(p.heads) * T5_D;
  int rc = make_tmap_2d(&tq, q, p.L, cols, ldq, T5_TQ, T5_D, true);
  if (rc != KR_OK) return rc;
  rc = make_tmap_2d(&tk, k, p.L, cols, ldk, T5_TK, T5_D, true);
  if (rc != KR_OK) return rc;
  rc = make_tmap_2d(&tv, v, p.L, cols, ldv, T5_TK, T5_D, true);
  if (rc != KR_OK) return rc;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(t5_attn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, T5_SMEM);
    if (e != cudaSuccess) {
      set_last_error("t5_attn: cudaFuncSetAttribute failed: %s", cudaGetErrorString(e));
      return KR_ERR_CUDA;
    }
    attr_set = true;
  }
  const int nqb = (p.L + T5_TQ - 1) / T5_TQ;
  t5_attn_kernel<<<p.heads * nqb, T5_THREADS, T5_SMEM, stream>>>(tq, tk, tv, p);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_last_error("t5_attn: launch failed: %s", cudaGetErrorString(e));
    return KR_ERR_CUDA;
  }
  return KR_OK;
}

}  // namespace kr
