// kr_vae.cu — causal 3D VAE decoder kernels for sm_90a (channels-last activations).
//
// conv3d_igemm : CausalConv3d / Conv2d / 1x1x1 conv as an implicit GEMM on wgmma.
//   Reference: wan/modules/vae.py:17-36 (CausalConv3d: cat(cache, x) on T, zero-pad H/W, cuDNN
//   conv), :175-209 (ResidualBlock: RMS_norm -> SiLU -> conv, twice, + shortcut),
//   demo_utils/vae_block3.py:46-91 (Resample), :386-443 (VAEDecoder3d).
//   Layout: activations are [frames, H, W, C] (C contiguous).  The input buffer of a causal
//   conv holds the 2 cached frames in front of the T new ones, so tap kt of output frame t reads
//   buffer frame t + kt IN PLACE (no torch.cat / F.pad copies); spatial zero padding is the TMA
//   out-of-bounds fill.  GEMM view per output tile: M = 128 pixels (a TH x TW patch of one
//   frame), N = Cout, K = taps * Cin; the A tile of tap (kt,kh,kw) is ONE 4-D TMA box
//   {64 ch, TW, TH, 1} at (c0, w0+kw-1, h0+kh-1, t+kt) landing in the canonical K-major
//   SWIZZLE_128B layout; weights are pre-permuted to [Cout, taps*Cin].
//   Two consumer warpgroups hold the fp32 accumulators of 64 pixels x Cout each in registers; a TMA
//   warpgroup feeds the smem ring.  Epilogue (from the accumulator fragment: a pixel's channels are spread over
//   the 4 lanes of a quad): bias, optional residual add,
//   optional raw store, optional fused RMS_norm(channel) * sqrt(C) * gamma -> SiLU store
//   (vae.py:39-54, :184-186) for the NEXT conv's input, or clamp -> fp32 NCHW pixels.
// Small HBM-bound kernels: latent un-scaling + conv2 (vae_block3.py:205-214), RMS_norm+SiLU,
//   nearest 2x upsample (vae.py:57-63), row softmax for the middle attention block.
#include "kr_common.cuh"
#include "kr_ops.h"

#include <cstdlib>

namespace kr {

static constexpr int kConvThreads = 384;   // consumer warpgroups 0, 1 + TMA warpgroup

template <int CIN, int N>
struct ConvCfg {
  static constexpr bool kHas32 = (CIN % 64) == 32;
  static constexpr int kChunks = CIN / 64;                       // full 64-channel chunks per tap
  static constexpr int kStagesPerTap = kHas32 ? 1 : kChunks;    // CIN=96: one stage = 64 + 32 ch
  static constexpr int kA64 = 128 * 128;                          // bytes
  static constexpr int kA32 = kHas32 ? 128 * 64 : 0;
  static constexpr int kB64 = N * 128;
  static constexpr int kB32 = kHas32 ? N * 64 : 0;
  static constexpr int kStageBytes = kA64 + kA32 + kB64 + kB32;
  static constexpr int kStages = (200 * 1024) / kStageBytes > 8 ? 8 : (200 * 1024) / kStageBytes;
  static constexpr int kMmaN = N > 256 ? N / 2 : N;              // wgmma N <= 256
  static constexpr int kMmaSplit = N / kMmaN;
  static constexpr int kSmemBytes = kStages * kStageBytes + 1024 + 256;
  static_assert(kStages >= 2, "pipeline needs >= 2 stages");
  static_assert(kB64 % 1024 == 0 && (kB32 % 512) == 0, "swizzle alignment of B tiles");
};

template <bool kBf16>
KR_DEVICE float rnd16(float x) {
  return kBf16 ? __bfloat162float(__float2bfloat16_rn(x)) : __half2float(__float2half_rn(x));
}
template <bool kBf16>
KR_DEVICE float2 unpack16(uint32_t u) {
  return kBf16 ? unpack_bf16x2(u) : unpack_f16x2(u);
}
template <bool kBf16>
KR_DEVICE uint32_t pack16(float a, float b) {
  return kBf16 ? pack_bf16x2(a, b) : pack_f16x2(a, b);
}
template <bool kBf16>
KR_DEVICE float load16(const uint16_t* p) {
  uint16_t u = *p;
  return kBf16 ? __bfloat162float(*reinterpret_cast<__nv_bfloat16*>(&u))
               : __half2float(*reinterpret_cast<__half*>(&u));
}

// Epilogue of the two output pixels of this thread's accumulator fragment (rows lane/4 and lane/4 + 8 of its
// warp's 16; channel pairs 8*nb + 2*(lane%4)): bias, optional residual, rounding, raw store, fused
// RMS_norm*sqrt(C)*gamma -> SiLU store (the sum of squares is reduced over the quad), or clamp -> fp32 NCHW
// pixels (N == 16 head).
template <int N, bool kBf16>
KR_DEVICE void conv_epilogue_frag(const ConvParams& p, float (&acc)[N / 2], int t, const int (&hh)[2],
                                  const int (&ww)[2], int lane) {
  const uint16_t* bias = reinterpret_cast<const uint16_t*>(p.bias);
  const uint16_t* gamma = reinterpret_cast<const uint16_t*>(p.gamma);
  const int cq = 2 * (lane & 3);
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int h = hh[r], w = ww[r];
    // sub2: stride-2 convolution with right/bottom zero pad (ZeroPad2d((0,1,0,1)) + Conv2d(stride 2),
    // vae.py:84-92) evaluated as the stride-1 conv at the odd positions: out(i,j) = full(2i+1, 2j+1)
    const bool ok = h < p.H && w < p.W && (p.sub2 == 0 || ((h & 1) && (w & 1)));
    const long pix = p.sub2 ? static_cast<long>(h >> 1) * (p.W >> 1) + (w >> 1)
                            : static_cast<long>(h) * p.W + w;
    if constexpr (N == 16) {
      // head conv: bias, round, clamp, fp32 NCHW pixels
      if (ok && p.out_pix != nullptr) {
#pragma unroll
        for (int nb = 0; nb < 2; ++nb)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int c = nb * 8 + cq + e;
            if (c < p.cout) {
              float x = acc[4 * nb + 2 * r + e] + (bias ? load16<kBf16>(bias + c) : 0.f);
              x = fminf(fmaxf(rnd16<kBf16>(x), -1.f), 1.f);
              p.out_pix[(static_cast<long>(t) * p.cout + c) * p.H * p.W + pix] = x;
            }
          }
      }
    } else {
      const uint16_t* res = (p.residual && ok)
          ? reinterpret_cast<const uint16_t*>(p.residual) + t * p.res_frame + pix * p.res_pix : nullptr;
      uint16_t* oraw = (p.out_raw && ok)
          ? reinterpret_cast<uint16_t*>(p.out_raw) + t * p.raw_frame + pix * p.raw_pix : nullptr;
      float sumsq = 0.f;
      // ---- pass 1: bias (+ residual), round, raw store, sum of squares ----
#pragma unroll
      for (int nb = 0; nb < N / 8; ++nb) {
        const int c = nb * 8 + cq;
        float f0 = acc[4 * nb + 2 * r], f1 = acc[4 * nb + 2 * r + 1];
        if (bias != nullptr) {
          const float2 g = unpack16<kBf16>(__ldg(reinterpret_cast<const unsigned int*>(bias + c)));
          f0 += g.x;
          f1 += g.y;
        }
        if (res != nullptr) {
          // reference: y = conv(...) (rounded to 16-bit), out = x + y (rounded)
          const float2 g = unpack16<kBf16>(*reinterpret_cast<const uint32_t*>(res + c));
          f0 = g.x + rnd16<kBf16>(f0);
          f1 = g.y + rnd16<kBf16>(f1);
        }
        f0 = rnd16<kBf16>(f0);
        f1 = rnd16<kBf16>(f1);
        sumsq += f0 * f0 + f1 * f1;
        if (oraw != nullptr) *reinterpret_cast<uint32_t*>(oraw + c) = pack16<kBf16>(f0, f1);
        acc[4 * nb + 2 * r] = f0;
        acc[4 * nb + 2 * r + 1] = f1;
      }
      // ---- pass 2: F.normalize(x, dim=C) * sqrt(C) * gamma -> SiLU ----
      if (p.out_norm != nullptr) {
        sumsq += __shfl_xor_sync(0xffffffffu, sumsq, 1);
        sumsq += __shfl_xor_sync(0xffffffffu, sumsq, 2);
        const float nrm = rnd16<kBf16>(sqrtf(sumsq));
        const float inv = 1.0f / fmaxf(nrm, 1e-30f);
        if (ok) {
          uint16_t* onrm = reinterpret_cast<uint16_t*>(p.out_norm) + t * p.norm_frame + pix * p.norm_pix;
#pragma unroll
          for (int nb = 0; nb < N / 8; ++nb) {
            const int c = nb * 8 + cq;
            const float2 g = unpack16<kBf16>(__ldg(reinterpret_cast<const unsigned int*>(gamma + c)));
            float a = rnd16<kBf16>(acc[4 * nb + 2 * r] * inv);
            float b = rnd16<kBf16>(acc[4 * nb + 2 * r + 1] * inv);
            a = rnd16<kBf16>(rnd16<kBf16>(a * p.norm_scale) * g.x);
            b = rnd16<kBf16>(rnd16<kBf16>(b * p.norm_scale) * g.y);
            *reinterpret_cast<uint32_t*>(onrm + c) =
                pack16<kBf16>(a / (1.0f + __expf(-a)), b / (1.0f + __expf(-b)));
          }
        }
      }
    }
  }
}

template <int CIN, int N, bool kBf16>
__global__ void __launch_bounds__(kConvThreads, 1)
conv_igemm_kernel(const __grid_constant__ CUtensorMap tm_in64, const __grid_constant__ CUtensorMap tm_in32,
                  const __grid_constant__ CUtensorMap tm_w64, const __grid_constant__ CUtensorMap tm_w32,
                  const ConvParams p) {
  using Cfg = ConvCfg<CIN, N>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  // per-stage layout: [A64 | B64 | A32 | B32]; all offsets multiples of 1024 (A32/B32: 512)
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + Cfg::kStages * Cfg::kStageBytes);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + Cfg::kStages;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int tiles_w = (p.W + p.TW - 1) / p.TW;
  const int tiles_h = (p.H + p.TH - 1) / p.TH;
  const int tiles_per_frame = tiles_w * tiles_h;
  const int num_tiles = p.T * tiles_per_frame;
  const int taps = p.KT * p.KH * p.KW;
  const int pad_h = p.KH / 2, pad_w = p.KW / 2;

  if (threadIdx.x == 256) {
    prefetch_tmap(&tm_in64);
    prefetch_tmap(&tm_w64);
    if (Cfg::kHas32) {
      prefetch_tmap(&tm_in32);
      prefetch_tmap(&tm_w32);
    }
    for (int i = 0; i < Cfg::kStages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 2);   // one arrive per consumer warpgroup
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp >= 8) {
    // ===================== TMA producer =====================
    producer_regs();
    if (warp == 8 && elect_one()) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int t = tile / tiles_per_frame;
        const int rem = tile % tiles_per_frame;
        const int h0 = (rem / tiles_w) * p.TH;
        const int w0 = (rem % tiles_w) * p.TW;
        for (int tap = 0; tap < taps; ++tap) {
          const int kt = tap / (p.KH * p.KW);
          const int kh = (tap / p.KW) % p.KH;
          const int kw = tap % p.KW;
          for (int c = 0; c < Cfg::kStagesPerTap; ++c) {
            uint8_t* st = smem + stage * Cfg::kStageBytes;
            mbar_wait(&empty_bar[stage], phase ^ 1);
            mbar_expect_tx(&full_bar[stage], Cfg::kStageBytes);
            tma_load_4d(st, &tm_in64, &full_bar[stage], c * 64, w0 + kw - pad_w, h0 + kh - pad_h,
                        t + kt);
#pragma unroll
            for (int j = 0; j < Cfg::kMmaSplit; ++j)
              tma_load_2d(st + Cfg::kA64 + j * Cfg::kMmaN * 128, &tm_w64, &full_bar[stage],
                          tap * CIN + c * 64, j * Cfg::kMmaN);
            if (Cfg::kHas32) {
              tma_load_4d(st + Cfg::kA64 + Cfg::kB64, &tm_in32, &full_bar[stage], 64,
                          w0 + kw - pad_w, h0 + kh - pad_h, t + kt);
#pragma unroll
              for (int j = 0; j < Cfg::kMmaSplit; ++j)
                tma_load_2d(st + Cfg::kA64 + Cfg::kB64 + Cfg::kA32 + j * Cfg::kMmaN * 64, &tm_w32,
                            &full_bar[stage], tap * CIN + 64, j * Cfg::kMmaN);
            }
            if (++stage == Cfg::kStages) {
              stage = 0;
              phase ^= 1;
            }
          }
        }
      }
    }
    return;
  }

  // ===================== consumer warpgroups: wgmma over 64 pixels each, then the epilogue =====================
  consumer_regs();
  const int wg = warp >> 2;
  const bool leader = (threadIdx.x & 127) == 0;
  const int k_stages = taps * Cfg::kStagesPerTap;
  const uint32_t smem0 = smem_u32(smem);
  int stage = 0;
  uint32_t phase = 0;
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    float acc[N / 2];
    for (int ks = 0; ks < k_stages; ++ks) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t st = smem0 + stage * Cfg::kStageBytes;
      const uint32_t a64 = st + wg * 64 * 128, b64 = st + Cfg::kA64;
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const uint64_t a_desc = make_smem_desc(a64 + k * 32, 16, 1024);
#pragma unroll
        for (int j = 0; j < Cfg::kMmaSplit; ++j) {
          const uint64_t b_desc = make_smem_desc(b64 + j * Cfg::kMmaN * 128 + k * 32, 16, 1024);
          wgmma_ss<Cfg::kMmaN, kBf16, 0>(acc + j * (Cfg::kMmaN / 2), a_desc, b_desc, (ks | k) != 0 ? 1 : 0);
        }
      }
      if (Cfg::kHas32) {
        const uint32_t a32 = st + Cfg::kA64 + Cfg::kB64 + wg * 64 * 64;
        const uint32_t b32 = st + Cfg::kA64 + Cfg::kB64 + Cfg::kA32;
#pragma unroll
        for (int k = 0; k < 2; ++k) {
          // SWIZZLE_64B: 64-byte rows, 8-row groups 512 B apart
          const uint64_t a_desc = make_smem_desc(a32 + k * 32, 16, 512, kSwz64);
#pragma unroll
          for (int j = 0; j < Cfg::kMmaSplit; ++j) {
            const uint64_t b_desc = make_smem_desc(b32 + j * Cfg::kMmaN * 64 + k * 32, 16, 512, kSwz64);
            wgmma_ss<Cfg::kMmaN, kBf16, 0>(acc + j * (Cfg::kMmaN / 2), a_desc, b_desc, 1);
          }
        }
      }
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence(acc);
      if (leader) mbar_arrive(&empty_bar[stage]);
      if (++stage == Cfg::kStages) {
        stage = 0;
        phase ^= 1;
      }
    }
    const int t = tile / tiles_per_frame;
    const int rem = tile % tiles_per_frame;
    int hh[2], ww[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int px = wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * r;   // pixel row of the TH x TW tile
      hh[r] = (rem / tiles_w) * p.TH + px / p.TW;
      ww[r] = (rem % tiles_w) * p.TW + px % p.TW;
    }
    conv_epilogue_frag<N, kBf16>(p, acc, t, hh, ww, lane);
  }
}

// ---------------------------------------------------------------------------------------------
// conv_halo_kernel: the 3x3-spatial convs of the wide stages (N = 96 / 192 output channels).
//
// conv_igemm_kernel fetches a fresh 128-pixel input tile AND a fresh weight tile for every one of the
// kt*9 taps.  Here
//   * one work item = 256 output pixels of one frame: two 16(h) x 8(w) MMA tiles side by side;
//   * per (kt, 64-channel chunk) ONE halo box {64 ch, 24 w, 18 h} (18 x 24 = 432 rows of 128 B, pitch 24
//     rows) is loaded, and the 9 spatial taps are wgmmas over SHIFTED WINDOWS of it: a tile's pixel row
//     (h, w) of tap (kh, kw) is box row (h + kh) * 24 + 8u + w + kw, so a 64-pixel slice is 8 groups of 8
//     consecutive box rows, 24 rows (SBO = 3072 B, a multiple of the 1024 B swizzle atom) apart.  Only the
//     start address is off the atom boundary (by kw rows); wgmma derives the 128-byte swizzle from the absolute
//     shared-memory address bits, as TMA does when it writes the box, so the base-offset field stays 0;
//   * every weight tile {64 k, N} is used by both pixel tiles.
// Input traffic per pixel drops 9x * (128/216) and weight traffic 2x.  Borders are the TMA out-of-bounds
// zero fill as before; a partial last channel chunk (CIN = 96) is loaded 64 wide (zero filled) and only
// its valid k-steps are issued.
// Consumer warpgroup u owns pixel tile u (two m64 halves, accumulators N registers per thread); warpgroup 2 is
// the TMA producer.
template <int CIN, int N>
struct HaloCfg {
  static constexpr int kChunks = (CIN + 63) / 64;
  static constexpr int kLastK = (CIN % 64 == 0) ? 4 : (CIN % 64) / 16;   // k-steps of the last chunk
  static constexpr int kBoxW = 24, kBoxH = 18;
  static constexpr int kABytes = kBoxW * kBoxH * 128;             // 55296 = 54 KB
  static constexpr int kAStages = 2;
  static constexpr int kBBytes = N * 128;
  static constexpr int kBStages = (96 * 1024) / kBBytes > 8 ? 8 : (96 * 1024) / kBBytes;
  static constexpr int kSmemBytes = kAStages * kABytes + kBStages * kBBytes + 1024 + 512;
  static_assert(kABytes % 1024 == 0 && kBBytes % 1024 == 0, "swizzle alignment");
};
static constexpr int kHaloThreads = 384;


template <int CIN, int N, bool kBf16>
__global__ void __launch_bounds__(kHaloThreads, 1)
conv_halo_kernel(const __grid_constant__ CUtensorMap tm_in, const __grid_constant__ CUtensorMap tm_w,
                 const ConvParams p) {
  using Cfg = HaloCfg<CIN, N>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + Cfg::kAStages * Cfg::kABytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_b + Cfg::kBStages * Cfg::kBBytes);
  uint64_t* a_full = bars;                         // [kAStages]
  uint64_t* a_empty = a_full + Cfg::kAStages;      // [kAStages]
  uint64_t* b_full = a_empty + Cfg::kAStages;      // [kBStages]
  uint64_t* b_empty = b_full + Cfg::kBStages;      // [kBStages]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int items_w = (p.W + 15) / 16;
  const int items_h = (p.H + 15) / 16;
  const int items_per_frame = items_w * items_h;
  const int num_items = p.T * items_per_frame;

  if (threadIdx.x == 256) {
    prefetch_tmap(&tm_in);
    prefetch_tmap(&tm_w);
    for (int i = 0; i < Cfg::kAStages; ++i) {
      mbar_init(&a_full[i], 1);
      mbar_init(&a_empty[i], 2);
    }
    for (int i = 0; i < Cfg::kBStages; ++i) {
      mbar_init(&b_full[i], 1);
      mbar_init(&b_empty[i], 2);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp >= 8) {
    // ===================== TMA producer =====================
    producer_regs();
    if (warp == 8 && elect_one()) {
      int sa = 0, sb = 0;
      uint32_t pa = 0, pb = 0;
      for (int item = blockIdx.x; item < num_items; item += gridDim.x) {
        const int t = item / items_per_frame;
        const int rem = item % items_per_frame;
        const int h0 = (rem / items_w) * 16;
        const int w0 = (rem % items_w) * 16;
        for (int kt = 0; kt < p.KT; ++kt) {
          for (int c = 0; c < Cfg::kChunks; ++c) {
            mbar_wait(&a_empty[sa], pa ^ 1);
            mbar_expect_tx(&a_full[sa], Cfg::kABytes);
            tma_load_4d(smem_a + sa * Cfg::kABytes, &tm_in, &a_full[sa], c * 64, w0 - 1, h0 - 1, t + kt);
            if (++sa == Cfg::kAStages) {
              sa = 0;
              pa ^= 1;
            }
            for (int sp = 0; sp < 9; ++sp) {
              mbar_wait(&b_empty[sb], pb ^ 1);
              mbar_expect_tx(&b_full[sb], Cfg::kBBytes);
              tma_load_2d(smem_b + sb * Cfg::kBBytes, &tm_w, &b_full[sb], (kt * 9 + sp) * CIN + c * 64, 0);
              if (++sb == Cfg::kBStages) {
                sb = 0;
                pb ^= 1;
              }
            }
          }
        }
      }
    }
    return;
  }

  // ===================== consumer warpgroup u: pixel tile u of the item =====================
  consumer_regs();
  const int u = warp >> 2;
  const bool leader = (threadIdx.x & 127) == 0;
  const uint32_t a0 = smem_u32(smem_a), b0 = smem_u32(smem_b);
  int sa = 0, sb = 0;
  uint32_t pa = 0, pb = 0;
  for (int item = blockIdx.x; item < num_items; item += gridDim.x) {
    float acc[2][N / 2];      // m64 halves: tile rows h 0..7 and 8..15
    bool first = true;
    for (int kt = 0; kt < p.KT; ++kt) {
      for (int c = 0; c < Cfg::kChunks; ++c) {
        const int ksteps = (c == Cfg::kChunks - 1) ? Cfg::kLastK : 4;
        mbar_wait(&a_full[sa], pa);
        const uint32_t a_st = a0 + sa * Cfg::kABytes;
#pragma unroll 1
        for (int sp = 0; sp < 9; ++sp) {
          const int kh = sp / 3, kw = sp - kh * 3;
          mbar_wait(&b_full[sb], pb);
          const uint32_t b_st = b0 + sb * Cfg::kBBytes;
          const uint32_t a_win = a_st + (kh * Cfg::kBoxW + 8 * u + kw) * 128;
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            if (k < ksteps) {
              const uint64_t bd = make_smem_desc(b_st + k * 32, 16, 1024);
#pragma unroll
              for (int mh = 0; mh < 2; ++mh) {
                const uint64_t ad = make_smem_desc(a_win + mh * 8 * Cfg::kBoxW * 128 + k * 32, 16, Cfg::kBoxW * 128);
                wgmma_ss<N, kBf16, 0>(acc[mh], ad, bd, (first && k == 0) ? 0 : 1);
              }
            }
          }
          wgmma_commit();
          wgmma_wait<0>();
          reg_fence(acc[0]);
          reg_fence(acc[1]);
          first = false;
          if (leader) mbar_arrive(&b_empty[sb]);
          if (++sb == Cfg::kBStages) {
            sb = 0;
            pb ^= 1;
          }
        }
        if (leader) mbar_arrive(&a_empty[sa]);
        if (++sa == Cfg::kAStages) {
          sa = 0;
          pa ^= 1;
        }
      }
    }
    const int t = item / items_per_frame;
    const int rem = item % items_per_frame;
#pragma unroll
    for (int mh = 0; mh < 2; ++mh) {
      int hh[2], ww[2];
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const int px = mh * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * r;   // pixel row of the 16 x 8 tile
        hh[r] = (rem / items_w) * 16 + (px >> 3);
        ww[r] = (rem % items_w) * 16 + u * 8 + (px & 7);
      }
      conv_epilogue_frag<N, kBf16>(p, acc[mh], t, hh, ww, lane);
    }
  }
}

template <int CIN, int N, bool kBf16>
static int launch_conv_halo(const void* in, int t_in, const void* wgt, int w_rows, const ConvParams& p,
                            cudaStream_t stream) {
  using Cfg = HaloCfg<CIN, N>;
  CUtensorMap tin, tw;
  const uint64_t idims[4] = {static_cast<uint64_t>(CIN), static_cast<uint64_t>(p.W),
                             static_cast<uint64_t>(p.H), static_cast<uint64_t>(t_in)};
  const uint64_t istr[3] = {static_cast<uint64_t>(CIN) * 2, static_cast<uint64_t>(p.W) * CIN * 2,
                            static_cast<uint64_t>(p.H) * p.W * CIN * 2};
  const uint32_t ibox[4] = {64, Cfg::kBoxW, Cfg::kBoxH, 1};
  int rc = make_tmap_nd(&tin, in, 4, idims, istr, ibox, kBf16, 128);
  if (rc != KR_OK) return rc;
  const int taps = p.KT * 9;
  const uint64_t wdims[2] = {static_cast<uint64_t>(taps) * CIN, static_cast<uint64_t>(w_rows)};
  const uint64_t wstr[1] = {static_cast<uint64_t>(taps) * CIN * 2};
  const uint32_t wbox[2] = {64, static_cast<uint32_t>(N)};
  rc = make_tmap_nd(&tw, wgt, 2, wdims, wstr, wbox, kBf16, 128);
  if (rc != KR_OK) return rc;
  auto kern = conv_halo_kernel<CIN, N, kBf16>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes);
    if (e != cudaSuccess) {
      set_last_error("vae_conv: cudaFuncSetAttribute failed: %s", cudaGetErrorString(e));
      return KR_ERR_CUDA;
    }
    attr_set = true;
  }
  const int num_items = p.T * ((p.W + 15) / 16) * ((p.H + 15) / 16);
  int grid = sm_count();
  if (grid > num_items) grid = num_items;
  kern<<<grid, kHaloThreads, Cfg::kSmemBytes, stream>>>(tin, tw, p);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_last_error("vae_conv: launch failed: %s", cudaGetErrorString(e));
    return KR_ERR_CUDA;
  }
  return KR_OK;
}

// ---------------------------------------------------------------------------
// host launcher
// ---------------------------------------------------------------------------
template <int CIN, int N, bool kBf16>
static int launch_conv(const void* in, int t_in, const void* wgt, int w_rows, const ConvParams& p,
                       cudaStream_t stream) {
  using Cfg = ConvCfg<CIN, N>;
  CUtensorMap in64, in32, w64, w32;
  const uint64_t idims[4] = {static_cast<uint64_t>(CIN), static_cast<uint64_t>(p.W),
                             static_cast<uint64_t>(p.H), static_cast<uint64_t>(t_in)};
  const uint64_t istr[3] = {static_cast<uint64_t>(CIN) * 2, static_cast<uint64_t>(p.W) * CIN * 2,
                            static_cast<uint64_t>(p.H) * p.W * CIN * 2};
  const uint32_t ibox64[4] = {64, static_cast<uint32_t>(p.TW), static_cast<uint32_t>(p.TH), 1};
  int rc = make_tmap_nd(&in64, in, 4, idims, istr, ibox64, kBf16, 128);
  if (rc != KR_OK) return rc;
  const int taps = p.KT * p.KH * p.KW;
  const uint64_t wdims[2] = {static_cast<uint64_t>(taps) * CIN, static_cast<uint64_t>(w_rows)};
  const uint64_t wstr[1] = {static_cast<uint64_t>(taps) * CIN * 2};
  const uint32_t wbox64[2] = {64, static_cast<uint32_t>(Cfg::kMmaN)};
  rc = make_tmap_nd(&w64, wgt, 2, wdims, wstr, wbox64, kBf16, 128);
  if (rc != KR_OK) return rc;
  in32 = in64;
  w32 = w64;
  if (Cfg::kHas32) {
    const uint32_t ibox32[4] = {32, static_cast<uint32_t>(p.TW), static_cast<uint32_t>(p.TH), 1};
    rc = make_tmap_nd(&in32, in, 4, idims, istr, ibox32, kBf16, 64);
    if (rc != KR_OK) return rc;
    const uint32_t wbox32[2] = {32, static_cast<uint32_t>(Cfg::kMmaN)};
    rc = make_tmap_nd(&w32, wgt, 2, wdims, wstr, wbox32, kBf16, 64);
    if (rc != KR_OK) return rc;
  }
  auto kern = conv_igemm_kernel<CIN, N, kBf16>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         Cfg::kSmemBytes);
    if (e != cudaSuccess) {
      set_last_error("vae_conv: cudaFuncSetAttribute failed: %s", cudaGetErrorString(e));
      return KR_ERR_CUDA;
    }
    attr_set = true;
  }
  const int num_tiles = p.T * ((p.W + p.TW - 1) / p.TW) * ((p.H + p.TH - 1) / p.TH);
  int grid = sm_count();
  if (grid > num_tiles) grid = num_tiles;
  kern<<<grid, kConvThreads, Cfg::kSmemBytes, stream>>>(in64, in32, w64, w32, p);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_last_error("vae_conv: launch failed: %s", cudaGetErrorString(e));
    return KR_ERR_CUDA;
  }
  return KR_OK;
}

template <bool kBf16>
static int dispatch_conv(int cin, int n, const void* in, int t_in, const void* wgt, int w_rows,
                         const ConvParams& p, cudaStream_t s) {
  // 3x3 spatial taps with 96 / 192 output channels: halo-reuse kernel (KR_CONV_HALO=0 -> per-tap kernel)
  static const bool halo = [] { const char* e = getenv("KR_CONV_HALO"); return e == nullptr || e[0] != '0'; }();
  if (halo && p.KH == 3 && p.KW == 3 && (p.KT == 1 || p.KT == 3) && w_rows >= n) {
#define KR_HALO_CASE(CI, NN) \
    if (cin == CI && n == NN) return launch_conv_halo<CI, NN, kBf16>(in, t_in, wgt, w_rows, p, s);
    KR_HALO_CASE(384, 192)
    KR_HALO_CASE(192, 192)
    KR_HALO_CASE(192, 96)
    KR_HALO_CASE(96, 96)
    KR_HALO_CASE(96, 192)
#undef KR_HALO_CASE
  }
#define KR_CONV_CASE(CI, NN) \
  if (cin == CI && n == NN) return launch_conv<CI, NN, kBf16>(in, t_in, wgt, w_rows, p, s);
  KR_CONV_CASE(64, 384)
  KR_CONV_CASE(384, 384)
  KR_CONV_CASE(192, 384)
  KR_CONV_CASE(384, 192)
  KR_CONV_CASE(192, 192)
  KR_CONV_CASE(192, 96)
  KR_CONV_CASE(96, 96)
  KR_CONV_CASE(96, 16)
  KR_CONV_CASE(64, 96)
  KR_CONV_CASE(96, 192)
  KR_CONV_CASE(384, 32)
#undef KR_CONV_CASE
  set_last_error("vae_conv: unsupported channel configuration cin=%d n=%d", cin, n);
  return KR_ERR_UNSUPPORTED_SHAPE;
}

int vae_conv(int dtype, int cin, int n, const void* in, int t_in, const void* wgt, int w_rows,
             const ConvParams& p, cudaStream_t stream) {
  if (p.TW * p.TH != 128 || p.T <= 0 || p.H <= 0 || p.W <= 0) {
    set_last_error("vae_conv: bad geometry T=%d H=%d W=%d tile=%dx%d", p.T, p.H, p.W, p.TH, p.TW);
    return KR_ERR_INVALID_ARG;
  }
  if ((p.KT != 1 && p.KT != 3) || (p.KH != 1 && p.KH != 3) || (p.KW != 1 && p.KW != 3)) {
    set_last_error("vae_conv: taps must be 1 or 3");
    return KR_ERR_INVALID_ARG;
  }
  if (t_in < p.T + p.KT - 1) {
    set_last_error("vae_conv: input holds %d frames, needs %d", t_in, p.T + p.KT - 1);
    return KR_ERR_INVALID_ARG;
  }
  if (p.out_norm != nullptr && p.gamma == nullptr) {
    set_last_error("vae_conv: normalised output needs gamma");
    return KR_ERR_INVALID_ARG;
  }
  return dtype == 0 ? dispatch_conv<true>(cin, n, in, t_in, wgt, w_rows, p, stream)
                    : dispatch_conv<false>(cin, n, in, t_in, wgt, w_rows, p, stream);
}

// ---------------------------------------------------------------------------
// RMS_norm (per pixel over C) * sqrt(C) * gamma -> optional SiLU; channels-last rows.
// One warp per pixel.  (vae.py:39-54; used where the producer is not a conv epilogue.)
// ---------------------------------------------------------------------------
template <bool kBf16>
__global__ void rmsnorm_silu_kernel(const uint16_t* __restrict__ x, uint16_t* __restrict__ y,
                                    const uint16_t* __restrict__ gamma, long pixels, int C,
                                    float scale, int do_silu) {
  const long pix = static_cast<long>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (pix >= pixels) return;
  const int lane = threadIdx.x & 31;
  const uint16_t* xr = x + pix * C;
  float v[12];   // C <= 384 -> 12 values per lane
  float ss = 0.f;
  int n = 0;
  for (int c = lane; c < C; c += 32) {
    v[n] = load16<kBf16>(xr + c);
    ss += v[n] * v[n];
    ++n;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  const float nrm = rnd16<kBf16>(sqrtf(ss));
  const float inv = 1.0f / fmaxf(nrm, 1e-30f);
  uint16_t* yr = y + pix * C;
  n = 0;
  for (int c = lane; c < C; c += 32) {
    float a = rnd16<kBf16>(v[n] * inv);
    a = rnd16<kBf16>(rnd16<kBf16>(a * scale) * load16<kBf16>(gamma + c));
    if (do_silu) a = a / (1.0f + __expf(-a));
    const uint32_t pk = pack16<kBf16>(a, 0.f);
    yr[c] = static_cast<uint16_t>(pk & 0xffff);
    ++n;
  }
}

int vae_rmsnorm_silu(int dtype, const void* x, void* y, const void* gamma, long pixels, int C,
                     int do_silu, cudaStream_t stream) {
  if (C > 384 || C <= 0 || pixels <= 0) {
    set_last_error("vae_rmsnorm_silu: unsupported C=%d", C);
    return KR_ERR_UNSUPPORTED_SHAPE;
  }
  const int wpb = 8;
  const unsigned grid = static_cast<unsigned>((pixels + wpb - 1) / wpb);
  const float scale = sqrtf(static_cast<float>(C));
  if (dtype == 0)
    rmsnorm_silu_kernel<true><<<grid, wpb * 32, 0, stream>>>(
        static_cast<const uint16_t*>(x), static_cast<uint16_t*>(y),
        static_cast<const uint16_t*>(gamma), pixels, C, scale, do_silu);
  else
    rmsnorm_silu_kernel<false><<<grid, wpb * 32, 0, stream>>>(
        static_cast<const uint16_t*>(x), static_cast<uint16_t*>(y),
        static_cast<const uint16_t*>(gamma), pixels, C, scale, do_silu);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_last_error("vae_rmsnorm_silu: launch failed: %s", cudaGetErrorString(e));
    return KR_ERR_CUDA;
  }
  return KR_OK;
}

// ---------------------------------------------------------------------------
// nearest 2x spatial upsample, channels-last: in [T, H, W, C] -> out [T, 2H, 2W, C]
// (vae.py:57-63 casts to fp32 and back: an exact copy)
// ---------------------------------------------------------------------------
__global__ void upsample2x_kernel(const uint4* __restrict__ in, uint4* __restrict__ out, int T, int H,
                                  int W, int C8) {
  const long total = static_cast<long>(T) * 4 * H * W * C8;
  const long idx = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int c = idx % C8;
  long r = idx / C8;
  const int w2 = r % (2 * W);
  r /= (2 * W);
  const int h2 = r % (2 * H);
  const int t = r / (2 * H);
  out[idx] = in[((static_cast<long>(t) * H + (h2 >> 1)) * W + (w2 >> 1)) * C8 + c];
}

int vae_upsample2x(const void* in, void* out, int T, int H, int W, int C, cudaStream_t stream) {
  if (C % 8 != 0) {
    set_last_error("vae_upsample2x: C=%d not a multiple of 8", C);
    return KR_ERR_UNSUPPORTED_SHAPE;
  }
  const long total = static_cast<long>(T) * 4 * H * W * (C / 8);
  upsample2x_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(
      static_cast<const uint4*>(in), static_cast<uint4*>(out), T, H, W, C / 8);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_last_error("vae_upsample2x: launch failed: %s", cudaGetErrorString(e));
    return KR_ERR_CUDA;
  }
  return KR_OK;
}

// ---------------------------------------------------------------------------
// latent un-scaling + conv2 (1x1x1, 16 -> 16) + NCHW -> channels-last padded to 64 channels
//   z [T, 16, H, W] (strided) ; x = z / inv_std + mean ; y = W2 x + b2   (vae_block3.py:205-214)
//   out [T, H, W, 64] (channels >= 16 zero) feeds conv1 whose weights are zero-padded likewise.
// ---------------------------------------------------------------------------
template <bool kBf16>
__global__ void scale_input_kernel(const uint16_t* __restrict__ z, long zt, long zc, long zh, long zw,
                                   const uint16_t* __restrict__ mean, const uint16_t* __restrict__ inv_std,
                                   const uint16_t* __restrict__ w2, const uint16_t* __restrict__ b2,
                                   uint16_t* __restrict__ out, int T, int H, int W) {
  const long total = static_cast<long>(T) * H * W;
  const long pix = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (pix >= total) return;
  const int w = pix % W, h = (pix / W) % H, t = pix / (static_cast<long>(W) * H);
  float x[16];
#pragma unroll
  for (int c = 0; c < 16; ++c) {
    const float zv = load16<kBf16>(z + t * zt + c * zc + h * zh + w * zw);
    // z / scale[1] + scale[0], each op rounded to the 16-bit dtype
    x[c] = rnd16<kBf16>(rnd16<kBf16>(zv / load16<kBf16>(inv_std + c)) + load16<kBf16>(mean + c));
  }
  uint32_t o[32];
#pragma unroll
  for (int n = 0; n < 16; n += 2) {
    float a = 0.f, b = 0.f;
#pragma unroll
    for (int c = 0; c < 16; ++c) {
      a += load16<kBf16>(w2 + n * 16 + c) * x[c];
      b += load16<kBf16>(w2 + (n + 1) * 16 + c) * x[c];
    }
    a += load16<kBf16>(b2 + n);
    b += load16<kBf16>(b2 + n + 1);
    o[n / 2] = pack16<kBf16>(a, b);
  }
#pragma unroll
  for (int i = 8; i < 32; ++i) o[i] = 0u;
  uint4* op = reinterpret_cast<uint4*>(out + pix * 64);
#pragma unroll
  for (int q = 0; q < 8; ++q) op[q] = make_uint4(o[q * 4], o[q * 4 + 1], o[q * 4 + 2], o[q * 4 + 3]);
}

int vae_scale_input(int dtype, const void* z, long zt, long zc, long zh, long zw, const void* mean,
                    const void* inv_std, const void* w2, const void* b2, void* out, int T, int H,
                    int W, cudaStream_t stream) {
  const long total = static_cast<long>(T) * H * W;
  const unsigned grid = static_cast<unsigned>((total + 127) / 128);
  if (dtype == 0)
    scale_input_kernel<true><<<grid, 128, 0, stream>>>(
        static_cast<const uint16_t*>(z), zt, zc, zh, zw, static_cast<const uint16_t*>(mean),
        static_cast<const uint16_t*>(inv_std), static_cast<const uint16_t*>(w2),
        static_cast<const uint16_t*>(b2), static_cast<uint16_t*>(out), T, H, W);
  else
    scale_input_kernel<false><<<grid, 128, 0, stream>>>(
        static_cast<const uint16_t*>(z), zt, zc, zh, zw, static_cast<const uint16_t*>(mean),
        static_cast<const uint16_t*>(inv_std), static_cast<const uint16_t*>(w2),
        static_cast<const uint16_t*>(b2), static_cast<uint16_t*>(out), T, H, W);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_last_error("vae_scale_input: launch failed: %s", cudaGetErrorString(e));
    return KR_ERR_CUDA;
  }
  return KR_OK;
}

// ---------------------------------------------------------------------------
// row softmax: fp32 scores [rows, ld] (first `cols` valid) -> 16-bit probabilities [rows, ldo]
// (middle AttentionBlock, vae.py:239-244).  One CTA per row.
// ---------------------------------------------------------------------------
template <bool kBf16>
__global__ void __launch_bounds__(256)
softmax_rows_kernel(const float* __restrict__ s, long ld, uint16_t* __restrict__ pout, long ldo,
                    int cols) {
  __shared__ float red[8];
  const float* sr = s + static_cast<long>(blockIdx.x) * ld;
  uint16_t* pr = pout + static_cast<long>(blockIdx.x) * ldo;
  float m = -INFINITY;
  for (int c = threadIdx.x; c < cols; c += 256) m = fmaxf(m, sr[c]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  m = red[0];
#pragma unroll
  for (int i = 1; i < 8; ++i) m = fmaxf(m, red[i]);
  __syncthreads();
  float sum = 0.f;
  for (int c = threadIdx.x; c < cols; c += 256) sum += __expf(sr[c] - m);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = sum;
  __syncthreads();
  sum = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) sum += red[i];
  const float inv = 1.0f / sum;
  for (int c = threadIdx.x; c < cols; c += 256) {
    const uint32_t pk = pack16<kBf16>(__expf(sr[c] - m) * inv, 0.f);
    pr[c] = static_cast<uint16_t>(pk & 0xffff);
  }
}

int softmax_rows(int dtype, const float* s, long ld, void* pout, long ldo, int rows, int cols,
                 cudaStream_t stream) {
  if (rows <= 0 || cols <= 0) {
    set_last_error("softmax_rows: empty input");
    return KR_ERR_INVALID_ARG;
  }
  if (dtype == 0)
    softmax_rows_kernel<true><<<rows, 256, 0, stream>>>(s, ld, static_cast<uint16_t*>(pout), ldo, cols);
  else
    softmax_rows_kernel<false><<<rows, 256, 0, stream>>>(s, ld, static_cast<uint16_t*>(pout), ldo, cols);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_last_error("softmax_rows: launch failed: %s", cudaGetErrorString(e));
    return KR_ERR_CUDA;
  }
  return KR_OK;
}


// ---------------------------------------------------------------------------
// frame egress: fp32 pixels [T, 3, H, W] in [-1, 1] -> packed RGB bytes [T, H, W, 3]
//   reference (release_server.py:979-983 + torchvision to_pil_image): on the HOST, after a 57.5 MB fp32
//   device->host copy per 12-frame block,  x.add_(1.0).mul_(0.5).clamp_(0.0, 1.0)  then  .mul(255).byte()
//   (float -> uint8 truncation) and CHW -> HWC.  Here the same fp32 operations run on the device (separate
//   rounded add / mul, no contraction, so every byte is identical) and only 14.4 MB cross PCIe.
// HBM-bound: 12 B read + 3 B written per pixel (71.9 MB per 12-frame 832x480 block).
// ---------------------------------------------------------------------------
__device__ __forceinline__ uint32_t px_to_u8(float x) {
  float v = __fmul_rn(__fadd_rn(x, 1.0f), 0.5f);
  v = fminf(fmaxf(v, 0.0f), 1.0f);
  return __float2uint_rz(__fmul_rn(v, 255.0f));
}

// one thread = 4 consecutive pixels of one row: 3 x float4 in, 12 bytes out
__global__ void __launch_bounds__(256) frames_to_rgb8_vec4(const float* __restrict__ px, uint8_t* __restrict__ out,
                                                           long plane, long quads) {
  const long q = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;   // quad index over T*H*W/4
  if (q >= quads) return;
  const long pix = q * 4;
  const long t = pix / plane, in_plane = pix - t * plane;
  const float* base = px + t * 3 * plane + in_plane;
  const float4 r = __ldg(reinterpret_cast<const float4*>(base));
  const float4 g = __ldg(reinterpret_cast<const float4*>(base + plane));
  const float4 b = __ldg(reinterpret_cast<const float4*>(base + 2 * plane));
  const uint32_t r0 = px_to_u8(r.x), r1 = px_to_u8(r.y), r2 = px_to_u8(r.z), r3 = px_to_u8(r.w);
  const uint32_t g0 = px_to_u8(g.x), g1 = px_to_u8(g.y), g2 = px_to_u8(g.z), g3 = px_to_u8(g.w);
  const uint32_t b0 = px_to_u8(b.x), b1 = px_to_u8(b.y), b2 = px_to_u8(b.z), b3 = px_to_u8(b.w);
  uint3 w;                                                  // bytes r0 g0 b0 r1 | g1 b1 r2 g2 | b2 r3 g3 b3
  w.x = r0 | (g0 << 8) | (b0 << 16) | (r1 << 24);
  w.y = g1 | (b1 << 8) | (r2 << 16) | (g2 << 24);
  w.z = b2 | (r3 << 8) | (g3 << 16) | (b3 << 24);
  uint32_t* o = reinterpret_cast<uint32_t*>(out + pix * 3);   // pix % 4 == 0 -> 12-byte groups, 4-byte aligned
  o[0] = w.x;
  o[1] = w.y;
  o[2] = w.z;
}

__global__ void __launch_bounds__(256) frames_to_rgb8_scalar(const float* __restrict__ px, uint8_t* __restrict__ out,
                                                             long plane, long total) {
  const long pix = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (pix >= total) return;
  const long t = pix / plane, in_plane = pix - t * plane;
  const float* base = px + t * 3 * plane + in_plane;
  out[pix * 3 + 0] = static_cast<uint8_t>(px_to_u8(base[0]));
  out[pix * 3 + 1] = static_cast<uint8_t>(px_to_u8(base[plane]));
  out[pix * 3 + 2] = static_cast<uint8_t>(px_to_u8(base[2 * plane]));
}

int frames_to_rgb8(const float* pixels, uint8_t* rgb, int frames, int height, int width, cudaStream_t stream) {
  if (frames <= 0 || height <= 0 || width <= 0) {
    set_last_error("frames_to_rgb8: non-positive shape T=%d H=%d W=%d", frames, height, width);
    return KR_ERR_INVALID_ARG;
  }
  const long plane = static_cast<long>(height) * width;
  const long total = plane * frames;
  const bool vec = (plane % 4 == 0) && (reinterpret_cast<uintptr_t>(pixels) % 16 == 0) &&
                   (reinterpret_cast<uintptr_t>(rgb) % 4 == 0);
  if (vec) {
    const long quads = total / 4;
    frames_to_rgb8_vec4<<<static_cast<unsigned>((quads + 255) / 256), 256, 0, stream>>>(pixels, rgb, plane, quads);
  } else {
    frames_to_rgb8_scalar<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(pixels, rgb, plane, total);
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_last_error("frames_to_rgb8: launch failed: %s", cudaGetErrorString(e));
    return KR_ERR_CUDA;
  }
  return KR_OK;
}

}  // namespace kr
