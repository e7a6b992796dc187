// kr_vae_halo_kernel.cuh — the body of conv_halo_kernel (kr_vae.cu), included there once per entry-point name
// (KR_CONV_HALO_KERNEL): the decoder and fp16 paths' conv_halo_kernel and the FP8 encoder tier's
// enc_halo_conv_f8n_kernel compile from the same text.  No include guard: it is meant to be included twice.

template <int CIN, int N, bool kBf16, bool kNormF8 = false>
__global__ void __launch_bounds__(kHaloThreads, 1)
KR_CONV_HALO_KERNEL(const __grid_constant__ CUtensorMap tm_in, const __grid_constant__ CUtensorMap tm_w,
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
      conv_epilogue_frag<N, kBf16, kNormF8>(p, acc[mh], t, hh, ww, lane);
    }
  }
}
