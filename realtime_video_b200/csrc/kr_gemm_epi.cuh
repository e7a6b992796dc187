// kr_gemm_epi.cuh — what the data-parallel (kr_gemm.cu), stream-K (kr_gemm_sk.cu) and FP8 (kr_gemm_fp8.cu)
// GEMM kernels share:
//   * gemm_epilogue_row: kW consecutive output columns of ONE output row, fp32 accumulators in registers -> bias ->
//     GELU-tanh / per-frame gate / residual with the reference's 16-bit rounding points (nn.Linear output rounded,
//     then each following elementwise op rounded: causal_model.py:433-435, :466-488) -> 16-bit (or fp32) store,
//     columns >= n_split redirected to the second destination;
//   * gemm_mainloop: the consumer side of the TMA ring, one warpgroup accumulating a 64 x BN slice of a 128-row
//     tile with wgmma (SWIZZLE_128B K-major operands, 128-byte k-blocks);
//   * gemm_frag_epilogue: the wgmma accumulator fragment of one warp (16 rows) -> rows of 16 columns through a
//     small per-warp shared-memory transpose -> gemm_epilogue_row.
#pragma once
#include "kr_common.cuh"
#include "kr_ops.h"

namespace kr {

template <bool kBf16, int kEpi, int kW>
KR_DEVICE void gemm_epilogue_row(float (&v)[kW], const int row, const int col0, const GemmParams& p,
                                 const uint16_t* gate_row) {
    static_assert(kW % 8 == 0, "whole 16-byte groups");
    if (p.bias != nullptr) {
      const uint4* b4 = reinterpret_cast<const uint4*>(
          reinterpret_cast<const uint16_t*>(p.bias) + col0);
#pragma unroll
      for (int q = 0; q < kW / 8; ++q) {
        uint4 bb = __ldg(b4 + q);
        uint32_t w[4] = {bb.x, bb.y, bb.z, bb.w};
#pragma unroll
        for (int h = 0; h < 4; ++h) {
          float2 f = kBf16 ? unpack_bf16x2(w[h]) : unpack_f16x2(w[h]);
          v[q * 8 + h * 2] += f.x;
          v[q * 8 + h * 2 + 1] += f.y;
        }
      }
    }
    if constexpr (kEpi == EPI_F32) {
      float* o = reinterpret_cast<float*>(p.out) + static_cast<size_t>(row) * p.ldc + col0;
#pragma unroll
      for (int q = 0; q < kW / 4; ++q) {
        float4 f4 = make_float4(v[q * 4] * p.alpha, v[q * 4 + 1] * p.alpha,
                                v[q * 4 + 2] * p.alpha, v[q * 4 + 3] * p.alpha);
        reinterpret_cast<float4*>(o)[q] = f4;
      }
    } else {
      auto rnd = [](float x) -> float {
        return kBf16 ? __bfloat162float(__float2bfloat16_rn(x))
                     : __half2float(__float2half_rn(x));
      };
      if constexpr (kEpi == EPI_BIAS_GELU) {
#pragma unroll
        for (int j = 0; j < kW; ++j) v[j] = gelu_tanh(rnd(v[j]));
      }
      if constexpr (kEpi == EPI_BIAS_GATE_RES) {
        const uint4* g4 = reinterpret_cast<const uint4*>(gate_row + col0);
#pragma unroll
        for (int q = 0; q < kW / 8; ++q) {
          uint4 gg = __ldg(g4 + q);
          uint32_t w[4] = {gg.x, gg.y, gg.z, gg.w};
#pragma unroll
          for (int h = 0; h < 4; ++h) {
            float2 f = kBf16 ? unpack_bf16x2(w[h]) : unpack_f16x2(w[h]);
            v[q * 8 + h * 2] = rnd(rnd(v[q * 8 + h * 2]) * f.x);
            v[q * 8 + h * 2 + 1] = rnd(rnd(v[q * 8 + h * 2 + 1]) * f.y);
          }
        }
      }
      if constexpr (kEpi == EPI_BIAS_GATE_RES || kEpi == EPI_BIAS_RES || kEpi == EPI_MUL) {
        const uint4* r4 = reinterpret_cast<const uint4*>(
            reinterpret_cast<const uint16_t*>(p.residual) + static_cast<size_t>(row) * p.ldr +
            col0);
#pragma unroll
        for (int q = 0; q < kW / 8; ++q) {
          uint4 rr = r4[q];
          uint32_t w[4] = {rr.x, rr.y, rr.z, rr.w};
#pragma unroll
          for (int h = 0; h < 4; ++h) {
            float2 f = kBf16 ? unpack_bf16x2(w[h]) : unpack_f16x2(w[h]);
            if constexpr (kEpi == EPI_MUL) {
            v[q * 8 + h * 2] = f.x * rnd(v[q * 8 + h * 2]);
            v[q * 8 + h * 2 + 1] = f.y * rnd(v[q * 8 + h * 2 + 1]);
          } else if constexpr (kEpi == EPI_BIAS_RES) {
              v[q * 8 + h * 2] = f.x + rnd(v[q * 8 + h * 2]);
              v[q * 8 + h * 2 + 1] = f.y + rnd(v[q * 8 + h * 2 + 1]);
            } else {
              v[q * 8 + h * 2] = f.x + v[q * 8 + h * 2];
              v[q * 8 + h * 2 + 1] = f.y + v[q * 8 + h * 2 + 1];
            }
          }
        }
      }
      uint16_t* o = (p.out2 != nullptr && col0 >= p.n_split)
          ? reinterpret_cast<uint16_t*>(p.out2) + static_cast<size_t>(row) * p.ldc2 + (col0 - p.n_split)
          : reinterpret_cast<uint16_t*>(p.out) + static_cast<size_t>(row) * p.ldc + col0;
#pragma unroll
      for (int q = 0; q < kW / 8; ++q) {
        uint4 w;
        if (kBf16) {
          w.x = pack_bf16x2(v[q * 8 + 0], v[q * 8 + 1]);
          w.y = pack_bf16x2(v[q * 8 + 2], v[q * 8 + 3]);
          w.z = pack_bf16x2(v[q * 8 + 4], v[q * 8 + 5]);
          w.w = pack_bf16x2(v[q * 8 + 6], v[q * 8 + 7]);
        } else {
          w.x = pack_f16x2(v[q * 8 + 0], v[q * 8 + 1]);
          w.y = pack_f16x2(v[q * 8 + 2], v[q * 8 + 3]);
          w.z = pack_f16x2(v[q * 8 + 4], v[q * 8 + 5]);
          w.w = pack_f16x2(v[q * 8 + 6], v[q * 8 + 7]);
        }
        reinterpret_cast<uint4*>(o)[q] = w;
      }
    }
}

// 0 = bf16, 1 = fp16, 2 = e4m3, 3 = s8 (K-major operands, 128-byte rows: 64 16-bit or 128 8-bit elements per
// k-block).  s8 accumulates exact s32 sums, held bit for bit in the fp32 accumulator registers until the caller
// converts them.
template <int BN, int kKind>
KR_DEVICE void gemm_k_step(float (&acc)[BN / 2], uint64_t a_desc, uint64_t b_desc, int scale_d) {
  if constexpr (kKind == 3) wgmma_ss_s8<BN>(reinterpret_cast<int32_t*>(acc), a_desc, b_desc, scale_d);
  else if constexpr (kKind == 2) wgmma_ss_e4m3<BN>(acc, a_desc, b_desc, scale_d);
  else wgmma_ss<BN, kKind == 0, 0>(acc, a_desc, b_desc, scale_d);
}

// A consumer warpgroup hands a stage back: one arrive on `empty` of this CTA, or of both CTAs of a 2-CTA cluster
// (the W half that the peer multicast into this CTA is overwritten only when both CTAs are done with the stage).
template <int kCluster>
KR_DEVICE void release_stage(uint64_t* empty) {
  if constexpr (kCluster == 1) {
    mbar_arrive(empty);
  } else {
    mbar_arrive_cluster(empty, 0);
    mbar_arrive_cluster(empty, 1);
  }
}

// Consumer side of the TMA ring for k-blocks [kb0, kb1) of one tile: the warpgroup multiplies its 64-row slice
// (`a_base` already offset to it) of each stage's A tile with the stage's BN-row W tile.  One wgmma group stays in
// flight; a stage is released (one arrive per warpgroup on `empty`) once the group reading it has retired.
// kPromote (e4m3's default) instead retires every k-block into a scratch partial and adds it to `acc` in fp32;
// e4m3 with kPromote = false accumulates in place like the 16-bit kinds (torch._scaled_mm's use_fast_accum).
template <int BN, int kKind, int kCluster = 1, bool kPromote = (kKind == 2)>
KR_DEVICE void gemm_mainloop(float (&acc)[BN / 2], uint32_t a_base, uint32_t b_base, int a_bytes, int b_bytes,
                             int stages, uint64_t* full, uint64_t* empty, int& stage, uint32_t& phase, int kb0,
                             int kb1) {
  const bool leader = (threadIdx.x & 127) == 0;
  if constexpr (kPromote) {
    // e4m3 wgmma accumulates with a reduced-precision adder: each k-block's partial product is added to the fp32
    // accumulator in registers (one wgmma group per k-block, retired before the add)
    float part[BN / 2];
    for (int kb = kb0; kb < kb1; ++kb) {
      mbar_wait(&full[stage], phase);
      const uint32_t a = a_base + stage * a_bytes, b = b_base + stage * b_bytes;
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k)
        gemm_k_step<BN, kKind>(part, make_smem_desc(a + k * 32, 16, 1024), make_smem_desc(b + k * 32, 16, 1024),
                               k != 0 ? 1 : 0);
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence(part);
      if (leader) release_stage<kCluster>(&empty[stage]);
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] = (kb == kb0 ? 0.f : acc[i]) + part[i];
      if (++stage == stages) {
        stage = 0;
        phase ^= 1;
      }
    }
    return;
  }
  int prev = -1;
  for (int kb = kb0; kb < kb1; ++kb) {
    mbar_wait(&full[stage], phase);
    const uint32_t a = a_base + stage * a_bytes, b = b_base + stage * b_bytes;
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k)
      gemm_k_step<BN, kKind>(acc, make_smem_desc(a + k * 32, 16, 1024), make_smem_desc(b + k * 32, 16, 1024),
                             (kb != kb0 || k != 0) ? 1 : 0);
    wgmma_commit();
    wgmma_wait<1>();
    if (prev >= 0 && leader) release_stage<kCluster>(&empty[prev]);
    prev = stage;
    if (++stage == stages) {
      stage = 0;
      phase ^= 1;
    }
  }
  wgmma_wait<0>();
  reg_fence(acc);
  if (prev >= 0 && leader) release_stage<kCluster>(&empty[prev]);
}

// Per-k-block dequantisation scales of the block-scaled FP8 GEMM, as one consumer thread sees them: the activation
// scales of its two accumulator rows (row and row + 8 of its warp's 16) at k-block 0 with k-block pitch `ld` (null
// for a row >= M: it reads no scale), and the tile's weight-block scales, one per k-block.
struct BlockScales {
  const float* __restrict__ sa0;
  const float* __restrict__ sa1;
  long ld;
  const float* __restrict__ sw;
};

// The block-scaled accumulation mode of gemm_mainloop (kBlockScale, promoted e4m3 only): each k-block's partial is
// multiplied by its row's activation scale times the tile's weight scale before the fp32 add
// (acc += part * sa[kb][row] * sw[kb]).  The scales of k-block kb + 1 are loaded while kb's wgmma runs, so the loop
// waits on nothing new.  An overload rather than a branch of the function above: a block-scale argument added to that
// function changed the machine code of the kernels that do not use it.
template <int BN, int kKind, int kCluster, bool kPromote, bool kBlockScale>
KR_DEVICE void gemm_mainloop(float (&acc)[BN / 2], uint32_t a_base, uint32_t b_base, int a_bytes, int b_bytes,
                             int stages, uint64_t* full, uint64_t* empty, int& stage, uint32_t& phase, int kb0,
                             int kb1, const BlockScales& bs) {
  static_assert(kKind == 2 && kPromote && kBlockScale, "block scales are applied at the e4m3 promotion");
  const bool leader = (threadIdx.x & 127) == 0;
  float part[BN / 2];
  float na0 = bs.sa0 != nullptr ? __ldg(bs.sa0 + kb0 * bs.ld) : 0.f;
  float na1 = bs.sa1 != nullptr ? __ldg(bs.sa1 + kb0 * bs.ld) : 0.f;
  float nw = __ldg(bs.sw + kb0);
  for (int kb = kb0; kb < kb1; ++kb) {
    const float s0 = na0 * nw, s1 = na1 * nw;
    if (kb + 1 < kb1) {
      if (bs.sa0 != nullptr) na0 = __ldg(bs.sa0 + (kb + 1) * bs.ld);
      if (bs.sa1 != nullptr) na1 = __ldg(bs.sa1 + (kb + 1) * bs.ld);
      nw = __ldg(bs.sw + kb + 1);
    }
    mbar_wait(&full[stage], phase);
    const uint32_t a = a_base + stage * a_bytes, b = b_base + stage * b_bytes;
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k)
      gemm_k_step<BN, kKind>(part, make_smem_desc(a + k * 32, 16, 1024), make_smem_desc(b + k * 32, 16, 1024),
                             k != 0 ? 1 : 0);
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(part);
    if (leader) release_stage<kCluster>(&empty[stage]);
    // fragment layout of m64nNk32: elements 4j, 4j + 1 belong to the thread's first row, 4j + 2, 4j + 3 to row + 8
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = (kb == kb0 ? 0.f : acc[i]) + part[i] * ((i & 2) ? s1 : s0);
    if (++stage == stages) {
      stage = 0;
      phase ^= 1;
    }
  }
}

constexpr int kEpiScrPitch = 36;                      // floats per scratch row (16-byte aligned, fewer conflicts)
constexpr int kEpiScrFloats = 16 * kEpiScrPitch;       // one warp's 16 x 32 transpose buffer

// The fragment of one warp (rows row0 .. row0+15 of the output, columns col_base + [0, BN)) -> fused epilogue.
// Only the first n_valid columns (a multiple of 32) are stored; every accumulator is multiplied by `scale`, or, with
// kRowScale, by row_scale[row] and then by col_scale[col] (the row-scaled FP8 GEMM; rows >= M read no row scale).
// kS32: the accumulators hold s32 sums bit for bit (the s8 GEMM); each is converted to fp32 (round to nearest) as it
// leaves the transpose, 16 at a time, so no second copy of the fragment is live.
template <int BN, bool kBf16, int kEpi, bool kRowScale = false, bool kS32 = false>
KR_DEVICE void gemm_frag_epilogue(const float (&acc)[BN / 2], float* scr, int row0, int col_base, int n_valid,
                                  float scale, const GemmParams& p, const float* __restrict__ row_scale = nullptr,
                                  const float* __restrict__ col_scale = nullptr) {
  const int lane = threadIdx.x & 31;
  const int row = row0 + (lane >> 1), half = lane & 1;
  const bool row_ok = row < p.M;
  float sa = 0.f;
  if constexpr (kRowScale) {
    if (row_ok) sa = __ldg(row_scale + row);
  }
  const uint16_t* gate_row = nullptr;
  if constexpr (kEpi == EPI_BIAS_GATE_RES) {
    const int g = row_ok ? (row + p.row_offset) / p.rows_per_gate : 0;
    gate_row = reinterpret_cast<const uint16_t*>(p.gate) + static_cast<size_t>(g) * p.gate_stride;
  }
#pragma unroll
  for (int c = 0; c < BN / 32; ++c) {
    if (c * 32 < n_valid) {
      __syncwarp();
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int col = j * 8 + 2 * (lane & 3), r = lane >> 2;
        const float* f = &acc[(4 * c + j) * 4];
        *reinterpret_cast<float2*>(scr + r * kEpiScrPitch + col) = make_float2(f[0], f[1]);
        *reinterpret_cast<float2*>(scr + (r + 8) * kEpiScrPitch + col) = make_float2(f[2], f[3]);
      }
      __syncwarp();
      if (row_ok) {
        float v[16];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          float4 f = *reinterpret_cast<const float4*>(scr + (lane >> 1) * kEpiScrPitch + half * 16 + q * 4);
          if constexpr (kS32)
            f = make_float4(static_cast<float>(__float_as_int(f.x)), static_cast<float>(__float_as_int(f.y)),
                            static_cast<float>(__float_as_int(f.z)), static_cast<float>(__float_as_int(f.w)));
          if constexpr (kRowScale) {
            const float4 sw = __ldg(reinterpret_cast<const float4*>(col_scale + col_base + c * 32 + half * 16) + q);
            v[4 * q] = f.x * sa * sw.x; v[4 * q + 1] = f.y * sa * sw.y;
            v[4 * q + 2] = f.z * sa * sw.z; v[4 * q + 3] = f.w * sa * sw.w;
          } else {
            v[4 * q] = f.x * scale; v[4 * q + 1] = f.y * scale; v[4 * q + 2] = f.z * scale; v[4 * q + 3] = f.w * scale;
          }
        }
        gemm_epilogue_row<kBf16, kEpi, 16>(v, row, col_base + c * 32 + half * 16, p, gate_row);
      }
    }
  }
}

}  // namespace kr
