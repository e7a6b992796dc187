// kr_sage.cu — INT8 / FP8 quantised attention for sm_90a, head_dim 128: the numerics of SageAttention 2's sm_90 path
// (qk INT8 per thread, smoothed K, P.V in e4m3 with an fp32 accumulator), restated from its published algorithm.
//
// Replaces, on the reference path with the sageattention wheel installed (the README's H100 setup):
//   * cached self-attention  wan/modules/causal_model.py:386-390 -> attention.py:166-180 -> sageattn
//   * T5 cross-attention     wan/modules/model.py:201-213 -> sageattn
// Both dispatch to sageattn_qk_int8_pv_fp8_cuda_sm90(qk_quant_gran="per_thread", smooth_k=True,
// pv_accum_dtype="fp32+fp32").  The block-causal recompute branch stays on kr_attn_fwd (bf16), as in the reference.
//
// Quantisation (three launches, no host sync; every scale group is one thread's share of a wgmma fragment, so each
// dequantisation in the attention kernel is a per-thread scalar):
//   sage_quant_q_kernel  : Q -> int8, one fp32 scale per (head, 16-row block b, t < 8) over rows 16b+t and 16b+8+t
//                          (the two S-fragment rows of one thread); scale = amax/127 + 1e-7,
//                          q = trunc(x/scale + 0.5*sign(x))
//   sage_colstats_kernel : per channel, k_mean = bf16(mean over the Lkv rows) and v_scale = max(amax|v|, 1e-12)/448,
//                          reduced in a fixed order inside one CTA (no atomics: the same inputs give the same bytes)
//   sage_quant_kv_kernel : k_s = bf16(k - k_mean) -> int8, one scale per (head, 128-key block c, t < 4) over keys
//                          128c + 8i + 2t + e (the S-fragment columns of one thread); V -> e4m3(v / v_scale)
//                          transposed to [channel, key] with the keys of every 16 stored as
//                          0 1 8 9 2 3 10 11 4 5 12 13 6 7 14 15, so a thread's fp32 S fragment is already the
//                          register A operand of the k32 e4m3 wgmma.  Padded keys (>= Lkv) are 0.
//
// sage_attn_kernel: the skeleton of attn_fwd_kernel (kr_attn.cu) with byte tiles.  CTA = 128 query rows of one head:
//   warps 0..7  : two consumer warpgroups of 64 rows: S = Q.K^T (wgmma s8, SS, s32 accumulators), dequantise with
//                 q_scale*k_scale, exact running max, P = exp2(S - m), l += sum P (fp32), P~ = e4m3(448 P) packed
//                 from the S fragment, O_tile = P~.V~ (wgmma e4m3, RS, fresh accumulator), O = O*alpha + O_tile in
//                 fp32 registers (the e4m3 wgmma adder keeps fewer bits, as in kr_gemm_fp8.cu)
//   warps 8..11 : TMA producer (Q once, then the K / V^T ring; every tile is one 128-byte swizzle panel of 16 KB)
//   out = bf16(O * v_scale[c] / (448 l))
#include "kr_common.cuh"
#include "kr_ops.h"

#include <cuda_fp8.h>
#include <cmath>

namespace kr {

namespace {
constexpr int kSgD = 128;
constexpr int kSgTileQ = 128;
constexpr int kSgTileKV = 128;
constexpr int kSgStages = 8;
constexpr int kSgTileBytes = 128 * 128;                       // 16 KB: 128 rows of one 128-byte swizzle panel
constexpr int kSgThreads = 384;
constexpr int kSgSmem = kSgTileBytes + kSgStages * kSgTileBytes + 1024 + 256;
constexpr float kSgLog2e = 1.4426950408889634f;

struct SageParams {
  const float* q_scale;   // [heads, ceil(Lq/16), 8]
  const float* k_scale;   // [heads, ceil(Lkv/128), 4]
  const float* v_scale;   // [heads*128]
  void* out;
  int ldo, Lq, Lkv, heads;
  float scale_log2;       // softmax_scale * log2(e)
};

KR_DEVICE uint32_t e4m3x2(float a, float b) {
  return static_cast<uint32_t>(__nv_cvt_float2_to_fp8x2(make_float2(a, b), __NV_SATFINITE, __NV_E4M3));
}
KR_DEVICE uint32_t e4m3x4(float a, float b, float c, float d) { return e4m3x2(a, b) | (e4m3x2(c, d) << 16); }

// trunc(x / scale + 0.5 * sign(x)) as a byte
KR_DEVICE uint32_t quant_i8(float x, float scale) {
  const float h = x > 0.f ? 0.5f : (x < 0.f ? -0.5f : 0.f);
  return static_cast<uint32_t>(static_cast<int>(truncf(x / scale + h))) & 0xFFu;
}

template <int N>
KR_DEVICE void reg_fence_i(int32_t (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+r"(d[i])::"memory");
}
}  // namespace

// ---------------------------------------------------------------------------
// quantisers
// ---------------------------------------------------------------------------
// grid = heads * ceil(Lq/16), 256 threads: warp t handles the scale group (b, t), lane l channels 4l..4l+3
__global__ void __launch_bounds__(256) sage_quant_q_kernel(const uint16_t* __restrict__ q, int ldq, int Lq, int heads,
                                                           int8_t* __restrict__ q_i8, float* __restrict__ q_scale) {
  const int nb = (Lq + 15) / 16;
  const int h = blockIdx.x / nb, b = blockIdx.x % nb;
  const int t = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int col = h * kSgD + 4 * lane;
  float x[2][4];
  float m = 0.f;
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int row = 16 * b + t + 8 * r;
    uint2 u = make_uint2(0u, 0u);
    if (row < Lq) u = *reinterpret_cast<const uint2*>(q + static_cast<size_t>(row) * ldq + col);
    const float2 f0 = unpack_bf16x2(u.x), f1 = unpack_bf16x2(u.y);
    x[r][0] = f0.x; x[r][1] = f0.y; x[r][2] = f1.x; x[r][3] = f1.y;
#pragma unroll
    for (int i = 0; i < 4; ++i) m = fmaxf(m, fabsf(x[r][i]));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  const float scale = m / 127.0f + 1e-7f;
  if (lane == 0) q_scale[static_cast<size_t>(blockIdx.x) * 8 + t] = scale;
  const size_t ldo = static_cast<size_t>(heads) * kSgD;
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int row = 16 * b + t + 8 * r;
    if (row >= Lq) continue;
    const uint32_t w = quant_i8(x[r][0], scale) | (quant_i8(x[r][1], scale) << 8) | (quant_i8(x[r][2], scale) << 16) |
                       (quant_i8(x[r][3], scale) << 24);
    *reinterpret_cast<uint32_t*>(q_i8 + row * ldo + col) = w;
  }
}

// grid = heads*128 / 32, 256 threads: 4 channel groups of 8 x 64 row lanes; partial sums / maxima per row lane, then
// summed over the row lanes in index order
__global__ void __launch_bounds__(256) sage_colstats_kernel(const uint16_t* __restrict__ k, int ldk,
                                                            const uint16_t* __restrict__ v, int ldv, int Lkv,
                                                            uint16_t* __restrict__ k_mean, float* __restrict__ v_scale) {
  __shared__ float part_sum[64][33];
  __shared__ float part_max[64][33];
  const int cg = threadIdx.x & 3, rl = threadIdx.x >> 2;
  const int col = blockIdx.x * 32 + cg * 8;
  float s[8], a[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) s[i] = a[i] = 0.f;
#pragma unroll 4
  for (int r = rl; r < Lkv; r += 64) {
    const uint4 uk = *reinterpret_cast<const uint4*>(k + static_cast<size_t>(r) * ldk + col);
    const uint4 uv = *reinterpret_cast<const uint4*>(v + static_cast<size_t>(r) * ldv + col);
    const uint32_t wk[4] = {uk.x, uk.y, uk.z, uk.w}, wv[4] = {uv.x, uv.y, uv.z, uv.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 fk = unpack_bf16x2(wk[j]), fv = unpack_bf16x2(wv[j]);
      s[2 * j] += fk.x;
      s[2 * j + 1] += fk.y;
      a[2 * j] = fmaxf(a[2 * j], fabsf(fv.x));
      a[2 * j + 1] = fmaxf(a[2 * j + 1], fabsf(fv.y));
    }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    part_sum[rl][cg * 8 + i] = s[i];
    part_max[rl][cg * 8 + i] = a[i];
  }
  __syncthreads();
  if (threadIdx.x < 32) {
    float sum = 0.f, mx = 0.f;
    for (int i = 0; i < 64; ++i) {
      sum += part_sum[i][threadIdx.x];
      mx = fmaxf(mx, part_max[i][threadIdx.x]);
    }
    const int c = blockIdx.x * 32 + threadIdx.x;
    const __nv_bfloat16 km = __float2bfloat16_rn(sum / static_cast<float>(Lkv));
    k_mean[c] = *reinterpret_cast<const uint16_t*>(&km);
    v_scale[c] = fmaxf(mx, 1e-12f) / 448.0f;
  }
}

// grid = heads * ceil(Lkv/128), 256 threads: key = tid/2, channels 64*(tid%2).. of K; then the V tile transposed from
// shared memory, channel = tid/2, stored key positions 64*(tid%2)..
__global__ void __launch_bounds__(256) sage_quant_kv_kernel(const uint16_t* __restrict__ k, int ldk,
                                                            const uint16_t* __restrict__ v, int ldv, int Lkv, int heads,
                                                            const uint16_t* __restrict__ k_mean,
                                                            const float* __restrict__ v_scale,
                                                            int8_t* __restrict__ k_i8, float* __restrict__ k_scale,
                                                            uint8_t* __restrict__ v_t8) {
  __shared__ __align__(16) uint16_t sv[kSgTileKV][kSgD + 8];
  __shared__ unsigned int amax_bits[4];
  const int nkb = (Lkv + kSgTileKV - 1) / kSgTileKV;
  const int h = blockIdx.x / nkb, c = blockIdx.x % nkb;
  const int key = threadIdx.x >> 1, half = threadIdx.x & 1;
  const int g = c * kSgTileKV + key;
  const int col = h * kSgD + half * 64;
  if (threadIdx.x < 4) amax_bits[threadIdx.x] = 0u;

  // V tile -> shared memory (zeros past Lkv)
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    uint4 u = make_uint4(0u, 0u, 0u, 0u);
    if (g < Lkv) u = *reinterpret_cast<const uint4*>(v + static_cast<size_t>(g) * ldv + col + 8 * i);
    *reinterpret_cast<uint4*>(&sv[key][half * 64 + 8 * i]) = u;
  }
  // K row share: smoothed, rounded to bf16 like torch's bf16 subtraction
  float ks[64];
  float m = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    uint4 u = make_uint4(0u, 0u, 0u, 0u);
    if (g < Lkv) u = *reinterpret_cast<const uint4*>(k + static_cast<size_t>(g) * ldk + col + 8 * i);
    const uint4 mu = __ldg(reinterpret_cast<const uint4*>(k_mean + col + 8 * i));
    const uint32_t w[4] = {u.x, u.y, u.z, u.w}, mw[4] = {mu.x, mu.y, mu.z, mu.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = unpack_bf16x2(w[j]), fm = unpack_bf16x2(mw[j]);
      ks[8 * i + 2 * j] = bf16_round(f.x - fm.x);
      ks[8 * i + 2 * j + 1] = bf16_round(f.y - fm.y);
    }
  }
  if (g < Lkv) {
#pragma unroll
    for (int i = 0; i < 64; ++i) m = fmaxf(m, fabsf(ks[i]));
  }
  __syncthreads();   // amax_bits initialised
  if (g < Lkv) atomicMax(&amax_bits[(key >> 1) & 3], __float_as_uint(m));   // m >= 0: integer order = float order
  __syncthreads();
  const int grp = (key >> 1) & 3;
  const float scale = __uint_as_float(amax_bits[grp]) / 127.0f + 1e-7f;
  if (threadIdx.x < 4)
    k_scale[static_cast<size_t>(blockIdx.x) * 4 + threadIdx.x] = __uint_as_float(amax_bits[threadIdx.x]) / 127.0f + 1e-7f;
  if (g < Lkv) {
    int8_t* dst = k_i8 + static_cast<size_t>(g) * heads * kSgD + col;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      uint32_t w[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float* x = &ks[16 * i + 4 * j];
        w[j] = quant_i8(x[0], scale) | (quant_i8(x[1], scale) << 8) | (quant_i8(x[2], scale) << 16) | (quant_i8(x[3], scale) << 24);
      }
      *reinterpret_cast<uint4*>(dst + 16 * i) = make_uint4(w[0], w[1], w[2], w[3]);
    }
  }

  // V^T: row (h*128 + ch), stored positions [c*128 + 64*half, +64), keys permuted within every 16
  const int ch = threadIdx.x >> 1;
  const float vs = __ldg(v_scale + h * kSgD + ch);
  const size_t ldvt = static_cast<size_t>(nkb) * kSgTileKV;
  uint8_t* vdst = v_t8 + static_cast<size_t>(h * kSgD + ch) * ldvt + c * kSgTileKV + half * 64;
#pragma unroll
  for (int gi = 0; gi < 4; ++gi) {
    const int k0 = half * 64 + gi * 16;
    float f[16];
#pragma unroll
    for (int p = 0; p < 16; ++p) {
      // stored position p holds key (p/4)*2 + (p%2) + 8*((p/2)%2): 0 1 8 9 2 3 10 11 4 5 12 13 6 7 14 15
      const int kk = (p >> 2) * 2 + (p & 1) + 8 * ((p >> 1) & 1);
      const uint16_t bits = sv[k0 + kk][ch];
      f[p] = __bfloat162float(*reinterpret_cast<const __nv_bfloat16*>(&bits)) / vs;
    }
    *reinterpret_cast<uint4*>(vdst + gi * 16) =
        make_uint4(e4m3x4(f[0], f[1], f[2], f[3]), e4m3x4(f[4], f[5], f[6], f[7]), e4m3x4(f[8], f[9], f[10], f[11]),
                   e4m3x4(f[12], f[13], f[14], f[15]));
  }
}

// ---------------------------------------------------------------------------
// attention
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(kSgThreads, 1)
sage_attn_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                 const __grid_constant__ CUtensorMap tmap_v, const SageParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* smem_q = smem;                          // [128 rows][128 B]
  uint8_t* smem_kv = smem + kSgTileBytes;          // kSgStages tiles
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_kv + kSgStages * kSgTileBytes);
  uint64_t* q_full = bars;
  uint64_t* kv_full = bars + 1;
  uint64_t* kv_empty = kv_full + kSgStages;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int nqb = (p.Lq + kSgTileQ - 1) / kSgTileQ;
  const int head = blockIdx.x / nqb;
  const int q0 = (blockIdx.x % nqb) * kSgTileQ;
  const int n_tiles = (p.Lkv + kSgTileKV - 1) / kSgTileKV;

  if (threadIdx.x == 256) {
    prefetch_tmap(&tmap_q);
    prefetch_tmap(&tmap_k);
    prefetch_tmap(&tmap_v);
    mbar_init(q_full, 1);
    for (int i = 0; i < kSgStages; ++i) {
      mbar_init(&kv_full[i], 1);
      mbar_init(&kv_empty[i], 2);   // one arrive per consumer warpgroup
    }
    fence_barrier_init();
  }
  __syncthreads();

  // ring items: K_j = 2j, V_j = 2j + 1
  auto st = [](int item) { return item % kSgStages; };
  auto ph = [](int item) { return static_cast<uint32_t>((item / kSgStages) & 1); };

  if (warp >= 8) {
    producer_regs();
    if (warp == 8 && elect_one()) {
      const int col = head * kSgD;
      mbar_expect_tx(q_full, kSgTileBytes);
      tma_load_2d(smem_q, &tmap_q, q_full, col, q0);
      for (int it = 0; it < 2 * n_tiles; ++it) {
        const int j = it >> 1;
        mbar_wait(&kv_empty[st(it)], ph(it) ^ 1);
        mbar_expect_tx(&kv_full[st(it)], kSgTileBytes);
        if (it & 1)   // V^T [channels, keys]: box = 128 keys x this head's 128 channels
          tma_load_2d(smem_kv + st(it) * kSgTileBytes, &tmap_v, &kv_full[st(it)], j * kSgTileKV, col);
        else
          tma_load_2d(smem_kv + st(it) * kSgTileBytes, &tmap_k, &kv_full[st(it)], col, j * kSgTileKV);
      }
    }
    return;
  }

  consumer_regs();
  const int wg = warp >> 2;
  const bool leader = (threadIdx.x & 127) == 0;
  const uint32_t q_addr = smem_u32(smem_q) + wg * 64 * 128;
  const uint32_t kv_addr = smem_u32(smem_kv);
  const int row16 = q0 + wg * 64 + (warp & 3) * 16;     // this warp's 16-row block; the thread's rows +lane/4, +8
  const int q_row = row16 + (lane >> 2);
  const int nqb16 = (p.Lq + 15) / 16, nkb = n_tiles;
  const float qs = row16 < p.Lq
                       ? __ldg(p.q_scale + (static_cast<size_t>(head) * nqb16 + row16 / 16) * 8 + (lane >> 2)) *
                             p.scale_log2
                       : 0.f;
  const float* ks_ptr = p.k_scale + static_cast<size_t>(head) * nkb * 4 + (lane & 3);
  float m_run[2] = {-INFINITY, -INFINITY};
  float l_run[2] = {0.f, 0.f};     // this thread's partial row sums (its 2 columns of every 8)
  float o[kSgD / 2];
#pragma unroll
  for (int i = 0; i < kSgD / 2; ++i) o[i] = 0.f;

  float ks_next = __ldg(ks_ptr);
  mbar_wait(q_full, 0);
  for (int j = 0; j < n_tiles; ++j) {
    const float deq = qs * ks_next;
    if (j + 1 < n_tiles) ks_next = __ldg(ks_ptr + 4 * (j + 1));
    // ---- S = Q . K_j^T (int8, exact in s32) ----
    float s[kSgTileKV / 2];
    {
      int32_t si[kSgTileKV / 2];
      mbar_wait(&kv_full[st(2 * j)], ph(2 * j));
      const uint32_t b = kv_addr + st(2 * j) * kSgTileBytes;
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kSgD / 32; ++k)
        wgmma_ss_s8<kSgTileKV>(si, make_smem_desc(q_addr + k * 32, 16, 1024), make_smem_desc(b + k * 32, 16, 1024),
                               k != 0 ? 1 : 0);
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence_i(si);
      if (leader) mbar_arrive(&kv_empty[st(2 * j)]);
#pragma unroll
      for (int i = 0; i < kSgTileKV / 2; ++i) s[i] = static_cast<float>(si[i]) * deq;
    }
    // ---- Lkv tail, exact running max ----
    const int hi = p.Lkv - j * kSgTileKV;
    if (hi < kSgTileKV) {
#pragma unroll
      for (int nb = 0; nb < kSgTileKV / 8; ++nb)
#pragma unroll
        for (int e = 0; e < 2; ++e)
          if (nb * 8 + 2 * (lane & 3) + e >= hi) {
            s[4 * nb + e] = -INFINITY;
            s[4 * nb + 2 + e] = -INFINITY;
          }
    }
    float alpha[2], nm[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      float mt = -INFINITY;
#pragma unroll
      for (int nb = 0; nb < kSgTileKV / 8; ++nb) mt = fmaxf(mt, fmaxf(s[4 * nb + 2 * r], s[4 * nb + 2 * r + 1]));
      mt = fmaxf(mt, __shfl_xor_sync(0xffffffffu, mt, 1));
      mt = fmaxf(mt, __shfl_xor_sync(0xffffffffu, mt, 2));
      const float m_new = fmaxf(m_run[r], mt);          // finite: every tile holds at least one key < Lkv
      alpha[r] = fast_exp2(m_run[r] - m_new);           // 0 on the first tile
      m_run[r] = m_new;
      nm[r] = -m_new;
      l_run[r] *= alpha[r];
    }
    // ---- P = exp2(S - m); l += P; P~ = e4m3(448 P) in the register A layout of the k32 e4m3 wgmma ----
    uint32_t pa[kSgTileKV / 32][4];
#pragma unroll
    for (int kk = 0; kk < kSgTileKV / 32; ++kk)
#pragma unroll
      for (int hh = 0; hh < 2; ++hh)
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          const int i0 = 4 * (4 * kk + 2 * hh) + 2 * r, i1 = i0 + 4;
          const float a0 = fast_exp2(s[i0] + nm[r]), a1 = fast_exp2(s[i0 + 1] + nm[r]);
          const float a2 = fast_exp2(s[i1] + nm[r]), a3 = fast_exp2(s[i1 + 1] + nm[r]);
          l_run[r] += (a0 + a1) + (a2 + a3);
          pa[kk][2 * hh + r] = e4m3x4(a0 * 448.f, a1 * 448.f, a2 * 448.f, a3 * 448.f);
        }
    // ---- O_tile = P~ . V~_j (fresh accumulator), O = O * alpha + O_tile ----
    float ot[kSgD / 2];
    mbar_wait(&kv_full[st(2 * j + 1)], ph(2 * j + 1));
    {
      const uint32_t b = kv_addr + st(2 * j + 1) * kSgTileBytes;
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < kSgTileKV / 32; ++kk)
        wgmma_rs_e4m3<kSgD>(ot, pa[kk], make_smem_desc(b + kk * 32, 16, 1024), kk != 0 ? 1 : 0);
      wgmma_commit();
#pragma unroll
      for (int nb = 0; nb < kSgD / 8; ++nb)
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          o[4 * nb + 2 * r] *= alpha[r];
          o[4 * nb + 2 * r + 1] *= alpha[r];
        }
      wgmma_wait<0>();
      reg_fence(ot);
    }
    if (leader) mbar_arrive(&kv_empty[st(2 * j + 1)]);
#pragma unroll
    for (int i = 0; i < kSgD / 2; ++i) o[i] += ot[i];
  }

  // ---- epilogue: O * v_scale / (448 l) -> bf16 ----
  const float* vsc = p.v_scale + head * kSgD + 2 * (lane & 3);
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    float l = l_run[r];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const float inv_l = 1.0f / (448.0f * l);
    const int row = q_row + 8 * r;
    if (row < p.Lq) {
      uint16_t* orow = reinterpret_cast<uint16_t*>(p.out) + static_cast<size_t>(row) * p.ldo + head * kSgD +
                       2 * (lane & 3);
#pragma unroll
      for (int nb = 0; nb < kSgD / 8; ++nb) {
        const float2 vs = __ldg(reinterpret_cast<const float2*>(vsc + nb * 8));
        const float f0 = o[4 * nb + 2 * r] * vs.x * inv_l, f1 = o[4 * nb + 2 * r + 1] * vs.y * inv_l;
        *reinterpret_cast<uint32_t*>(orow + nb * 8) = pack_bf16x2(f0, f1);
      }
    }
  }
}

// ---------------------------------------------------------------------------
// host
// ---------------------------------------------------------------------------
static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

static int sage_launch_check(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_last_error("%s: launch failed: %s", what, cudaGetErrorString(e));
    return KR_ERR_CUDA;
  }
  return KR_OK;
}

}  // namespace kr

#define KR_SAGE_REQUIRE(cond, msg)               \
  do {                                           \
    if (!(cond)) {                               \
      kr::set_last_error("%s: %s", __func__, msg); \
      return KR_ERR_INVALID_ARG;                 \
    }                                            \
  } while (0)

extern "C" int kr_sage_quantize(const void* q, int ldq, const void* k, int ldk, const void* v, int ldv, int Lq, int Lkv,
                                int heads, void* q_i8, float* q_scale, void* k_mean, void* k_i8, float* k_scale,
                                void* v_t8, float* v_scale, void* stream) {
  KR_SAGE_REQUIRE(q && k && v, "null q/k/v");
  KR_SAGE_REQUIRE(q_i8 && q_scale && k_mean && k_i8 && k_scale && v_t8 && v_scale, "null output buffer");
  KR_SAGE_REQUIRE(Lq > 0 && Lkv > 0 && heads > 0, "non-positive Lq/Lkv/heads");
  KR_SAGE_REQUIRE(ldq >= heads * 128 && ldk >= heads * 128 && ldv >= heads * 128, "row pitch below heads*128");
  KR_SAGE_REQUIRE(ldq % 8 == 0 && ldk % 8 == 0 && ldv % 8 == 0, "row pitches must be multiples of 8 elements");
  KR_SAGE_REQUIRE(kr::aligned16(q) && kr::aligned16(k) && kr::aligned16(v) && kr::aligned16(k_mean) &&
                      kr::aligned16(k_i8) && kr::aligned16(v_t8) && kr::aligned16(q_i8),
                  "q/k/v, q_i8, k_i8, v_t8 and k_mean must be 16-byte aligned");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int nqb16 = (Lq + 15) / 16, nkb = (Lkv + 127) / 128;
  kr::sage_quant_q_kernel<<<heads * nqb16, 256, 0, s>>>(static_cast<const uint16_t*>(q), ldq, Lq, heads,
                                                        static_cast<int8_t*>(q_i8), q_scale);
  kr::sage_colstats_kernel<<<heads * 4, 256, 0, s>>>(static_cast<const uint16_t*>(k), ldk,
                                                     static_cast<const uint16_t*>(v), ldv, Lkv,
                                                     static_cast<uint16_t*>(k_mean), v_scale);
  kr::sage_quant_kv_kernel<<<heads * nkb, 256, 0, s>>>(static_cast<const uint16_t*>(k), ldk,
                                                       static_cast<const uint16_t*>(v), ldv, Lkv, heads,
                                                       static_cast<const uint16_t*>(k_mean), v_scale,
                                                       static_cast<int8_t*>(k_i8), k_scale,
                                                       static_cast<uint8_t*>(v_t8));
  return kr::sage_launch_check("kr_sage_quantize");
}

extern "C" int kr_sage_attn(const void* q_i8, const float* q_scale, const void* k_i8, const float* k_scale,
                            const void* v_t8, const float* v_scale, void* out, int ldo, int Lq, int Lkv, int heads,
                            float softmax_scale, void* stream) {
  KR_SAGE_REQUIRE(q_i8 && q_scale && k_i8 && k_scale && v_t8 && v_scale && out, "null buffer");
  KR_SAGE_REQUIRE(Lq > 0 && Lkv > 0 && heads > 0, "non-positive Lq/Lkv/heads");
  KR_SAGE_REQUIRE(ldo >= heads * 128 && ldo % 8 == 0, "ldo must be >= heads*128 and a multiple of 8");
  KR_SAGE_REQUIRE(softmax_scale > 0.f && softmax_scale < 1e30f, "softmax_scale must be positive and finite");
  KR_SAGE_REQUIRE(kr::aligned16(q_i8) && kr::aligned16(k_i8) && kr::aligned16(v_t8) && kr::aligned16(out),
                  "q_i8/k_i8/v_t8/out must be 16-byte aligned");
  const uint64_t width = static_cast<uint64_t>(heads) * 128;
  const int nkb = (Lkv + 127) / 128;
  CUtensorMap tq, tk, tv;
  {
    const uint64_t d[2] = {width, static_cast<uint64_t>(Lq)}, sd[1] = {width};
    const uint32_t box[2] = {128, kr::kSgTileQ};
    int rc = kr::make_tmap_u8(&tq, q_i8, 2, d, sd, box, 128);
    if (rc != KR_OK) return rc;
  }
  {
    const uint64_t d[2] = {width, static_cast<uint64_t>(Lkv)}, sd[1] = {width};
    const uint32_t box[2] = {128, kr::kSgTileKV};
    int rc = kr::make_tmap_u8(&tk, k_i8, 2, d, sd, box, 128);
    if (rc != KR_OK) return rc;
  }
  {
    const uint64_t d[2] = {static_cast<uint64_t>(nkb) * 128, width}, sd[1] = {static_cast<uint64_t>(nkb) * 128};
    const uint32_t box[2] = {kr::kSgTileKV, 128};
    int rc = kr::make_tmap_u8(&tv, v_t8, 2, d, sd, box, 128);
    if (rc != KR_OK) return rc;
  }
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kr::sage_attn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kr::kSgSmem);
    if (e != cudaSuccess) {
      kr::set_last_error("kr_sage_attn: cudaFuncSetAttribute failed: %s", cudaGetErrorString(e));
      return KR_ERR_CUDA;
    }
    attr_set = true;
  }
  kr::SageParams p;
  p.q_scale = q_scale; p.k_scale = k_scale; p.v_scale = v_scale; p.out = out;
  p.ldo = ldo; p.Lq = Lq; p.Lkv = Lkv; p.heads = heads;
  p.scale_log2 = softmax_scale * kr::kSgLog2e;
  const dim3 grid(((Lq + kr::kSgTileQ - 1) / kr::kSgTileQ) * heads);
  kr::sage_attn_kernel<<<grid, kr::kSgThreads, kr::kSgSmem, static_cast<cudaStream_t>(stream)>>>(tq, tk, tv, p);
  return kr::sage_launch_check("kr_sage_attn");
}
