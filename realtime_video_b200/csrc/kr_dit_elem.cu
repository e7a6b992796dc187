// kr_dit_elem.cu — HBM-bound row kernels of the DiT block (bf16 in / bf16 out, fp32 math).
//
//   ln_modulate       : WanLayerNorm (no affine, eps) then x*(1+scale)+shift per frame
//                       (wan/modules/causal_model.py:466-471, :482-485, :520-522; model.py:88-98)
//   ln_affine         : WanLayerNorm with affine (norm3, causal_model.py:480)
//   qkv_norm_rope     : WanRMSNorm(dim) on q,k (model.py:69-85) + 3-axis RoPE
//                       (causal_model.py:143-171 / model.py:39-66) + KV-cache append
//                       (causal_model.py:310-311, :378-385)
//   rmsnorm_rows      : WanRMSNorm for the cross-attention q / k (model.py:183-190)
//   add_modulation    : e = modulation + e0 (causal_model.py:466, :521)
//   silu / patchify / unpatchify_x0 : small layout kernels around the block stack
//
// Rounding points follow the reference's eager bf16 execution (each torch op rounds its
// result to bf16), so a bf16 reference run and this path agree to ~1 ulp per op.
#include "kr_common.cuh"
#include "kr_ops.h"

#include <cuda_fp8.h>

namespace kr {

static constexpr int kRowThreads = 128;
static constexpr int kMaxVec = 8;   // up to 128*8*8 = 8192 channels

KR_DEVICE float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
// block-wide sum over kRowThreads threads; red must hold 4 floats per call-site slot
KR_DEVICE float block_sum(float v, float* red) {
  v = warp_sum(v);
  const int w = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) red[w] = v;
  __syncthreads();
  float t = red[0] + red[1] + red[2] + red[3];
  __syncthreads();
  return t;
}
// block-wide max over kRowThreads threads (same slot rules as block_sum)
KR_DEVICE float block_max(float v, float* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  const int w = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) red[w] = v;
  __syncthreads();
  float t = fmaxf(fmaxf(red[0], red[1]), fmaxf(red[2], red[3]));
  __syncthreads();
  return t;
}

KR_DEVICE void load8(const uint16_t* p, float (&f)[8]) {
  uint4 u = *reinterpret_cast<const uint4*>(p);
  float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z),
         d = unpack_bf16x2(u.w);
  f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y; f[4] = c.x; f[5] = c.y; f[6] = d.x; f[7] = d.y;
}
KR_DEVICE void store8(uint16_t* p, const float (&f)[8]) {
  uint4 u;
  u.x = pack_bf16x2(f[0], f[1]);
  u.y = pack_bf16x2(f[2], f[3]);
  u.z = pack_bf16x2(f[4], f[5]);
  u.w = pack_bf16x2(f[6], f[7]);
  *reinterpret_cast<uint4*>(p) = u;
}

// ---------------------------------------------------------------------------
// LayerNorm (+ optional affine) (+ optional per-frame modulation)
//   y = bf16(LN(x) [* w + b])                       (torch layer_norm: one rounding)
//   out = bf16(bf16(y * bf16(1 + scale)) + shift)   when mod != nullptr
// mod layout: [frames, mod_rows, D]; scale = row `scale_idx`, shift = row `shift_idx`.
// kFp8: the bf16 output row is also quantised per row to e4m3 (fp8_quantize_row below) for the row-scaled FP8 GEMM;
// the bf16 store happens only when `out` is given.
// ---------------------------------------------------------------------------
// Row data stays PACKED (uint4 = 8 x bf16) in registers and is unpacked per pass: ~3x fewer live
// registers than keeping floats -> more resident CTAs -> more bytes in flight per SM.

// Dynamic per-row e4m3 cast of one row held packed in registers by a kRowThreads CTA (torchao PerRow):
//   amax = max(max|x|, 1e-12), q = sat_e4m3(x * (448 / amax)) (round to nearest even), scale_out = amax / 448.
// `red` holds 4 floats; every thread of the CTA must call it.
template <int kVec>
KR_DEVICE void fp8_quantize_row(const uint4 (&raw)[kVec], int nvec, float* red, uint8_t* __restrict__ qrow,
                                float* __restrict__ scale_out) {
  float m = 0.f;
#pragma unroll
  for (int i = 0; i < kVec; ++i) {
    const int vi = threadIdx.x + i * kRowThreads;
    if (vi < nvec) {
      const uint32_t u[4] = {raw[i].x, raw[i].y, raw[i].z, raw[i].w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = unpack_bf16x2(u[j]);
        m = fmaxf(m, fmaxf(fabsf(f.x), fabsf(f.y)));
      }
    }
  }
  const float amax = fmaxf(block_max(m, red), 1e-12f);
  const float mul = 448.0f / amax;
  if (threadIdx.x == 0) *scale_out = amax / 448.0f;
#pragma unroll
  for (int i = 0; i < kVec; ++i) {
    const int vi = threadIdx.x + i * kRowThreads;
    if (vi < nvec) {
      const uint32_t u[4] = {raw[i].x, raw[i].y, raw[i].z, raw[i].w};
      uint32_t o[2];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = unpack_bf16x2(u[j]);
        const uint32_t h = __nv_cvt_float2_to_fp8x2(make_float2(f.x * mul, f.y * mul), __NV_SATFINITE, __NV_E4M3);
        if (j & 1) o[j >> 1] |= h << 16;
        else o[j >> 1] = h;
      }
      *reinterpret_cast<uint2*>(qrow + vi * 8) = make_uint2(o[0], o[1]);
    }
  }
}

// Dynamic e4m3 cast of one row per 128-channel group (torchao PerBlock [1, 128]), the row held packed in registers by
// a kRowThreads CTA: a group is 16 consecutive 8-channel vectors, i.e. the vectors i of 16 consecutive lanes, so its
// amax is a 16-lane shuffle reduction (no shared memory, no barrier).  Per group g:
//   amax = max(max|x_g|, 1e-12), q_g = sat_e4m3(x_g * (448 / amax)), scale_col[g * ld_s] = amax / 448.
// nvec must be a multiple of 16 (cols % 128 == 0), so a group is either wholly valid or wholly past the row's end.
template <int kVec>
KR_DEVICE void fp8_quantize_row_groups(const uint4 (&raw)[kVec], int nvec, uint8_t* __restrict__ qrow,
                                       float* __restrict__ scale_col, int ld_s) {
#pragma unroll
  for (int i = 0; i < kVec; ++i) {
    const int vi = threadIdx.x + i * kRowThreads;
    const bool valid = vi < nvec;
    const uint32_t u[4] = {raw[i].x, raw[i].y, raw[i].z, raw[i].w};
    float m = 0.f;
    if (valid) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = unpack_bf16x2(u[j]);
        m = fmaxf(m, fmaxf(fabsf(f.x), fabsf(f.y)));
      }
    }
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));   // all lanes take part
    if (valid) {
      const float amax = fmaxf(m, 1e-12f);
      const float mul = 448.0f / amax;
      if ((threadIdx.x & 15) == 0) scale_col[static_cast<size_t>(vi >> 4) * ld_s] = amax / 448.0f;
      uint32_t o[2];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = unpack_bf16x2(u[j]);
        const uint32_t h = __nv_cvt_float2_to_fp8x2(make_float2(f.x * mul, f.y * mul), __NV_SATFINITE, __NV_E4M3);
        if (j & 1) o[j >> 1] |= h << 16;
        else o[j >> 1] = h;
      }
      *reinterpret_cast<uint2*>(qrow + vi * 8) = make_uint2(o[0], o[1]);
    }
  }
}

// Dynamic per-row symmetric s8 cast of one row held packed in registers by a kRowThreads CTA (torchao
// Int8DynamicActivation, per token): amax = max(max|x|, 1e-12), q = clamp(rint(x * (127 / amax)), -127, 127) (round half
// to even), scale_out = amax / 127.  `red` holds 4 floats; every thread of the CTA must call it.
template <int kVec>
KR_DEVICE void i8_quantize_row(const uint4 (&raw)[kVec], int nvec, float* red, int8_t* __restrict__ qrow,
                               float* __restrict__ scale_out) {
  float m = 0.f;
#pragma unroll
  for (int i = 0; i < kVec; ++i) {
    const int vi = threadIdx.x + i * kRowThreads;
    if (vi < nvec) {
      const uint32_t u[4] = {raw[i].x, raw[i].y, raw[i].z, raw[i].w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = unpack_bf16x2(u[j]);
        m = fmaxf(m, fmaxf(fabsf(f.x), fabsf(f.y)));
      }
    }
  }
  const float amax = fmaxf(block_max(m, red), 1e-12f);
  const float mul = 127.0f / amax;
  if (threadIdx.x == 0) *scale_out = amax / 127.0f;
#pragma unroll
  for (int i = 0; i < kVec; ++i) {
    const int vi = threadIdx.x + i * kRowThreads;
    if (vi < nvec) {
      const uint32_t u[4] = {raw[i].x, raw[i].y, raw[i].z, raw[i].w};
      uint32_t o[2] = {0u, 0u};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = unpack_bf16x2(u[j]);
        // the bounds are integers, so clamping before rounding equals clamping after
        const int q0 = __float2int_rn(fminf(fmaxf(f.x * mul, -127.f), 127.f));
        const int q1 = __float2int_rn(fminf(fmaxf(f.y * mul, -127.f), 127.f));
        const uint32_t pair = (static_cast<uint32_t>(q0) & 0xffu) | ((static_cast<uint32_t>(q1) & 0xffu) << 8);
        o[j >> 1] |= pair << (16 * (j & 1));
      }
      *reinterpret_cast<uint2*>(qrow + vi * 8) = make_uint2(o[0], o[1]);
    }
  }
}

// kBlocks (with kFp8): the cast is per 128-channel group (fp8_quantize_row_groups) into q / scale_rows[g * ld_s].
// kI8 (with kFp8, which then names the quantised-output mode): the cast is the per-row s8 one (i8_quantize_row).
template <int kVec, bool kFp8, bool kBlocks = false, bool kI8 = false>
KR_DEVICE void ln_modulate_row(const uint16_t* __restrict__ x, int ldx, uint16_t* __restrict__ out, int ldo,
                               int D, float eps, const uint16_t* __restrict__ w, const uint16_t* __restrict__ b,
                               const uint16_t* __restrict__ mod, int mod_rows, int shift_idx, int scale_idx,
                               int rows_per_frame, int row_offset, uint8_t* __restrict__ q, int ldq,
                               float* __restrict__ scale_rows, int ld_s = 0) {
  __shared__ float red[4];
  const int row = blockIdx.x;
  const uint16_t* xr = x + static_cast<size_t>(row) * ldx;
  const int nvec = D >> 3;
  uint4 raw[kVec];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < kVec; ++i) {
    const int vi = threadIdx.x + i * kRowThreads;
    if (vi < nvec) {
      raw[i] = *reinterpret_cast<const uint4*>(xr + vi * 8);
      const float2 a0 = unpack_bf16x2(raw[i].x), a1 = unpack_bf16x2(raw[i].y),
                   a2 = unpack_bf16x2(raw[i].z), a3 = unpack_bf16x2(raw[i].w);
      s += (a0.x + a0.y) + (a1.x + a1.y) + (a2.x + a2.y) + (a3.x + a3.y);
    }
  }
  const float mean = block_sum(s, red) / D;
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < kVec; ++i) {
    const int vi = threadIdx.x + i * kRowThreads;
    if (vi < nvec) {
      const uint32_t u[4] = {raw[i].x, raw[i].y, raw[i].z, raw[i].w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = unpack_bf16x2(u[j]);
        const float d0 = f.x - mean, d1 = f.y - mean;
        ss += d0 * d0 + d1 * d1;
      }
    }
  }
  const float rstd = rsqrtf(block_sum(ss, red) / D + eps);
  const uint16_t* mrow = nullptr;
  if (mod != nullptr) mrow = mod + static_cast<size_t>((row + row_offset) / rows_per_frame) * mod_rows * D;
  uint16_t* orow = kFp8 && out == nullptr ? nullptr : out + static_cast<size_t>(row) * ldo;
#pragma unroll
  for (int i = 0; i < kVec; ++i) {
    const int vi = threadIdx.x + i * kRowThreads;
    if (vi < nvec) {
      float y[8];
      {
        const float2 a0 = unpack_bf16x2(raw[i].x), a1 = unpack_bf16x2(raw[i].y),
                     a2 = unpack_bf16x2(raw[i].z), a3 = unpack_bf16x2(raw[i].w);
        y[0] = a0.x; y[1] = a0.y; y[2] = a1.x; y[3] = a1.y; y[4] = a2.x; y[5] = a2.y; y[6] = a3.x; y[7] = a3.y;
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) y[j] = (y[j] - mean) * rstd;
      if (w != nullptr) {
        float ww[8], bb[8];
        load8(w + vi * 8, ww);
        load8(b + vi * 8, bb);
#pragma unroll
        for (int j = 0; j < 8; ++j) y[j] = y[j] * ww[j] + bb[j];
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) y[j] = bf16_round(y[j]);
      if (mrow != nullptr) {
        float sc[8], sh[8];
        load8(mrow + static_cast<size_t>(scale_idx) * D + vi * 8, sc);
        load8(mrow + static_cast<size_t>(shift_idx) * D + vi * 8, sh);
#pragma unroll
        for (int j = 0; j < 8; ++j) y[j] = bf16_round(y[j] * bf16_round(1.0f + sc[j])) + sh[j];
      }
      if constexpr (kFp8) {
        // the bf16 output row replaces the input in registers; it is quantised once the whole row is known
        raw[i] = make_uint4(pack_bf16x2(y[0], y[1]), pack_bf16x2(y[2], y[3]), pack_bf16x2(y[4], y[5]),
                            pack_bf16x2(y[6], y[7]));
        if (orow != nullptr) *reinterpret_cast<uint4*>(orow + vi * 8) = raw[i];
      } else {
        store8(orow + vi * 8, y);
      }
    }
  }
  if constexpr (kFp8 && kBlocks)
    fp8_quantize_row_groups<kVec>(raw, nvec, q + static_cast<size_t>(row) * ldq, scale_rows + row, ld_s);
  else if constexpr (kFp8 && kI8)
    i8_quantize_row<kVec>(raw, nvec, red, reinterpret_cast<int8_t*>(q) + static_cast<size_t>(row) * ldq,
                          scale_rows + row);
  else if constexpr (kFp8)
    fp8_quantize_row<kVec>(raw, nvec, red, q + static_cast<size_t>(row) * ldq, scale_rows + row);
}

template <int kVec>
__global__ void __launch_bounds__(kRowThreads, 8)
ln_modulate_kernel(const uint16_t* __restrict__ x, int ldx, uint16_t* __restrict__ out, int ldo,
                   int D, float eps, const uint16_t* __restrict__ w, const uint16_t* __restrict__ b,
                   const uint16_t* __restrict__ mod, int mod_rows, int shift_idx, int scale_idx,
                   int rows_per_frame, int row_offset) {
  ln_modulate_row<kVec, false>(x, ldx, out, ldo, D, eps, w, b, mod, mod_rows, shift_idx, scale_idx, rows_per_frame,
                               row_offset, nullptr, 0, nullptr);
}

template <int kVec>
__global__ void __launch_bounds__(kRowThreads, 8)
ln_modulate_fp8_kernel(const uint16_t* __restrict__ x, int ldx, uint16_t* __restrict__ out, int ldo,
                       int D, float eps, const uint16_t* __restrict__ w, const uint16_t* __restrict__ b,
                       const uint16_t* __restrict__ mod, int mod_rows, int shift_idx, int scale_idx,
                       int rows_per_frame, int row_offset, uint8_t* __restrict__ q, int ldq,
                       float* __restrict__ scale_rows) {
  ln_modulate_row<kVec, true>(x, ldx, out, ldo, D, eps, w, b, mod, mod_rows, shift_idx, scale_idx, rows_per_frame,
                              row_offset, q, ldq, scale_rows);
}

template <int kVec>
__global__ void __launch_bounds__(kRowThreads, 8)
ln_modulate_fp8_blocks_kernel(const uint16_t* __restrict__ x, int ldx, uint16_t* __restrict__ out, int ldo,
                              int D, float eps, const uint16_t* __restrict__ w, const uint16_t* __restrict__ b,
                              const uint16_t* __restrict__ mod, int mod_rows, int shift_idx, int scale_idx,
                              int rows_per_frame, int row_offset, uint8_t* __restrict__ q, int ldq,
                              float* __restrict__ scale, int ld_s) {
  ln_modulate_row<kVec, true, true>(x, ldx, out, ldo, D, eps, w, b, mod, mod_rows, shift_idx, scale_idx,
                                    rows_per_frame, row_offset, q, ldq, scale, ld_s);
}

template <int kVec>
__global__ void __launch_bounds__(kRowThreads, 8)
ln_modulate_i8_kernel(const uint16_t* __restrict__ x, int ldx, uint16_t* __restrict__ out, int ldo,
                      int D, float eps, const uint16_t* __restrict__ w, const uint16_t* __restrict__ b,
                      const uint16_t* __restrict__ mod, int mod_rows, int shift_idx, int scale_idx,
                      int rows_per_frame, int row_offset, uint8_t* __restrict__ q, int ldq,
                      float* __restrict__ scale_rows) {
  ln_modulate_row<kVec, true, false, true>(x, ldx, out, ldo, D, eps, w, b, mod, mod_rows, shift_idx, scale_idx,
                                           rows_per_frame, row_offset, q, ldq, scale_rows);
}

static int ln_check(const char* who, int rows, int D, int ldx, int ldo, const void* w, const void* b, const void* mod,
                    int rows_per_frame) {
  if (D % 8 != 0 || D > kRowThreads * 8 * kMaxVec || rows <= 0 || ldx % 8 != 0 || ldo % 8 != 0) {
    set_last_error("%s: unsupported D=%d rows=%d", who, D, rows);
    return KR_ERR_UNSUPPORTED_SHAPE;
  }
  if ((w == nullptr) != (b == nullptr)) {
    set_last_error("%s: weight and bias must both be given or both be null", who);
    return KR_ERR_INVALID_ARG;
  }
  if (mod != nullptr && rows_per_frame <= 0) {
    set_last_error("%s: rows_per_frame must be positive", who);
    return KR_ERR_INVALID_ARG;
  }
  return KR_OK;
}

static int launch_status(const char* who) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_last_error("%s: launch failed: %s", who, cudaGetErrorString(e));
    return KR_ERR_CUDA;
  }
  return KR_OK;
}

int ln_modulate(const void* x, int ldx, void* out, int ldo, int rows, int D, float eps,
                const void* w, const void* b, const void* mod, int mod_rows, int shift_idx,
                int scale_idx, int rows_per_frame, int row_offset, cudaStream_t stream) {
  const int rc = ln_check("ln_modulate", rows, D, ldx, ldo, w, b, mod, rows_per_frame);
  if (rc != KR_OK) return rc;
  const int nv = (D / 8 + kRowThreads - 1) / kRowThreads;
#define KR_LN_LAUNCH(V)                                                                            \
  ln_modulate_kernel<V><<<rows, kRowThreads, 0, stream>>>(                                         \
      static_cast<const uint16_t*>(x), ldx, static_cast<uint16_t*>(out), ldo, D, eps,              \
      static_cast<const uint16_t*>(w), static_cast<const uint16_t*>(b),                            \
      static_cast<const uint16_t*>(mod), mod_rows, shift_idx, scale_idx, rows_per_frame, row_offset)
  switch (nv) {
    case 1: KR_LN_LAUNCH(1); break;
    case 2: KR_LN_LAUNCH(2); break;
    case 3: KR_LN_LAUNCH(3); break;
    case 4: KR_LN_LAUNCH(4); break;
    case 5: KR_LN_LAUNCH(5); break;
    default: KR_LN_LAUNCH(8); break;
  }
#undef KR_LN_LAUNCH
  return launch_status("ln_modulate");
}

int ln_modulate_fp8(const void* x, int ldx, void* out, int ldo, int rows, int D, float eps,
                    const void* w, const void* b, const void* mod, int mod_rows, int shift_idx,
                    int scale_idx, int rows_per_frame, int row_offset, void* q, int ldq, float* scale_rows,
                    cudaStream_t stream) {
  const int rc = ln_check("ln_modulate_fp8", rows, D, ldx, out != nullptr ? ldo : 8, w, b, mod, rows_per_frame);
  if (rc != KR_OK) return rc;
  if (ldq % 8 != 0 || ldq < D) {
    set_last_error("ln_modulate_fp8: unsupported ldq=%d for D=%d", ldq, D);
    return KR_ERR_UNSUPPORTED_SHAPE;
  }
  const int nv = (D / 8 + kRowThreads - 1) / kRowThreads;
#define KR_LN_LAUNCH(V)                                                                            \
  ln_modulate_fp8_kernel<V><<<rows, kRowThreads, 0, stream>>>(                                     \
      static_cast<const uint16_t*>(x), ldx, static_cast<uint16_t*>(out), ldo, D, eps,              \
      static_cast<const uint16_t*>(w), static_cast<const uint16_t*>(b),                            \
      static_cast<const uint16_t*>(mod), mod_rows, shift_idx, scale_idx, rows_per_frame, row_offset, \
      static_cast<uint8_t*>(q), ldq, scale_rows)
  switch (nv) {
    case 1: KR_LN_LAUNCH(1); break;
    case 2: KR_LN_LAUNCH(2); break;
    case 3: KR_LN_LAUNCH(3); break;
    case 4: KR_LN_LAUNCH(4); break;
    case 5: KR_LN_LAUNCH(5); break;
    default: KR_LN_LAUNCH(8); break;
  }
#undef KR_LN_LAUNCH
  return launch_status("ln_modulate_fp8");
}

int ln_modulate_i8(const void* x, int ldx, void* out, int ldo, int rows, int D, float eps,
                   const void* w, const void* b, const void* mod, int mod_rows, int shift_idx,
                   int scale_idx, int rows_per_frame, int row_offset, void* q, int ldq, float* scale_rows,
                   cudaStream_t stream) {
  const int rc = ln_check("ln_modulate_i8", rows, D, ldx, out != nullptr ? ldo : 8, w, b, mod, rows_per_frame);
  if (rc != KR_OK) return rc;
  if (ldq % 8 != 0 || ldq < D) {
    set_last_error("ln_modulate_i8: unsupported ldq=%d for D=%d", ldq, D);
    return KR_ERR_UNSUPPORTED_SHAPE;
  }
  const int nv = (D / 8 + kRowThreads - 1) / kRowThreads;
#define KR_LN_LAUNCH(V)                                                                            \
  ln_modulate_i8_kernel<V><<<rows, kRowThreads, 0, stream>>>(                                      \
      static_cast<const uint16_t*>(x), ldx, static_cast<uint16_t*>(out), ldo, D, eps,              \
      static_cast<const uint16_t*>(w), static_cast<const uint16_t*>(b),                            \
      static_cast<const uint16_t*>(mod), mod_rows, shift_idx, scale_idx, rows_per_frame, row_offset, \
      static_cast<uint8_t*>(q), ldq, scale_rows)
  switch (nv) {
    case 1: KR_LN_LAUNCH(1); break;
    case 2: KR_LN_LAUNCH(2); break;
    case 3: KR_LN_LAUNCH(3); break;
    case 4: KR_LN_LAUNCH(4); break;
    case 5: KR_LN_LAUNCH(5); break;
    default: KR_LN_LAUNCH(8); break;
  }
#undef KR_LN_LAUNCH
  return launch_status("ln_modulate_i8");
}

int ln_modulate_fp8_blocks(const void* x, int ldx, void* out, int ldo, int rows, int D, float eps,
                           const void* w, const void* b, const void* mod, int mod_rows, int shift_idx,
                           int scale_idx, int rows_per_frame, int row_offset, void* q, int ldq, float* scale,
                           int ld_s, cudaStream_t stream) {
  const int rc = ln_check("ln_modulate_fp8_blocks", rows, D, ldx, out != nullptr ? ldo : 8, w, b, mod,
                          rows_per_frame);
  if (rc != KR_OK) return rc;
  if (D % 128 != 0 || ldq % 16 != 0 || ldq < D || ld_s < rows) {
    set_last_error("ln_modulate_fp8_blocks: unsupported D=%d ldq=%d ld_s=%d rows=%d (need D %% 128 == 0)", D, ldq,
                   ld_s, rows);
    return KR_ERR_UNSUPPORTED_SHAPE;
  }
  const int nv = (D / 8 + kRowThreads - 1) / kRowThreads;
#define KR_LN_LAUNCH(V)                                                                            \
  ln_modulate_fp8_blocks_kernel<V><<<rows, kRowThreads, 0, stream>>>(                              \
      static_cast<const uint16_t*>(x), ldx, static_cast<uint16_t*>(out), ldo, D, eps,              \
      static_cast<const uint16_t*>(w), static_cast<const uint16_t*>(b),                            \
      static_cast<const uint16_t*>(mod), mod_rows, shift_idx, scale_idx, rows_per_frame, row_offset, \
      static_cast<uint8_t*>(q), ldq, scale, ld_s)
  switch (nv) {
    case 1: KR_LN_LAUNCH(1); break;
    case 2: KR_LN_LAUNCH(2); break;
    case 3: KR_LN_LAUNCH(3); break;
    case 4: KR_LN_LAUNCH(4); break;
    case 5: KR_LN_LAUNCH(5); break;
    default: KR_LN_LAUNCH(8); break;
  }
#undef KR_LN_LAUNCH
  return launch_status("ln_modulate_fp8_blocks");
}

// ---------------------------------------------------------------------------
// Dynamic per-row e4m3 activation cast (torchao Float8DynamicActivation, PerRow): one CTA per row, the row in
// registers, one read and one write; scale_rows[r] = amax_r / 448 is the row scale of the row-scaled FP8 GEMM.
// Up to kRowThreads * 8 * kQuantMaxVec = 14336 channels (the FFN width of the 14B model is 13824).
// ---------------------------------------------------------------------------
static constexpr int kQuantMaxVec = 14;

template <int kVec>
__global__ void __launch_bounds__(kRowThreads)
fp8_quantize_rows_kernel(const uint16_t* __restrict__ x, int ldx, int cols, uint8_t* __restrict__ q, int ldq,
                         float* __restrict__ scale_rows) {
  __shared__ float red[4];
  const int row = blockIdx.x;
  const uint16_t* xr = x + static_cast<size_t>(row) * ldx;
  const int nvec = cols >> 3;
  uint4 raw[kVec];
#pragma unroll
  for (int i = 0; i < kVec; ++i) {
    const int vi = threadIdx.x + i * kRowThreads;
    if (vi < nvec) raw[i] = *reinterpret_cast<const uint4*>(xr + vi * 8);
  }
  fp8_quantize_row<kVec>(raw, nvec, red, q + static_cast<size_t>(row) * ldq, scale_rows + row);
}

int fp8_quantize_rows(const void* x, int ldx, int rows, int cols, void* q, int ldq, float* scale_rows,
                      cudaStream_t stream) {
  if (cols <= 0 || cols % 8 != 0 || cols > kRowThreads * 8 * kQuantMaxVec || rows <= 0 || ldx % 8 != 0 ||
      ldq % 8 != 0 || ldx < cols || ldq < cols) {
    set_last_error("fp8_quantize_rows: unsupported rows=%d cols=%d ldx=%d ldq=%d", rows, cols, ldx, ldq);
    return KR_ERR_UNSUPPORTED_SHAPE;
  }
  const int nv = (cols / 8 + kRowThreads - 1) / kRowThreads;
#define KR_Q_LAUNCH(V)                                                                             \
  fp8_quantize_rows_kernel<V><<<rows, kRowThreads, 0, stream>>>(                                   \
      static_cast<const uint16_t*>(x), ldx, cols, static_cast<uint8_t*>(q), ldq, scale_rows)
  switch (nv) {
    case 1: KR_Q_LAUNCH(1); break;
    case 2: KR_Q_LAUNCH(2); break;
    case 3: KR_Q_LAUNCH(3); break;
    case 4: KR_Q_LAUNCH(4); break;
    case 5: KR_Q_LAUNCH(5); break;
    case 6: KR_Q_LAUNCH(6); break;
    case 7: case 8: KR_Q_LAUNCH(8); break;
    case 9: case 10: KR_Q_LAUNCH(10); break;
    default: KR_Q_LAUNCH(14); break;
  }
#undef KR_Q_LAUNCH
  return launch_status("fp8_quantize_rows");
}

// Dynamic per-row symmetric s8 activation cast (torchao Int8DynamicActivation, per token): the e4m3 row quantiser's
// layout, i8_quantize_row's numerics; scale_rows[r] = amax_r / 127 is the row scale of the s8 GEMM.
template <int kVec>
__global__ void __launch_bounds__(kRowThreads)
i8_quantize_rows_kernel(const uint16_t* __restrict__ x, int ldx, int cols, int8_t* __restrict__ q, int ldq,
                        float* __restrict__ scale_rows) {
  __shared__ float red[4];
  const int row = blockIdx.x;
  const uint16_t* xr = x + static_cast<size_t>(row) * ldx;
  const int nvec = cols >> 3;
  uint4 raw[kVec];
#pragma unroll
  for (int i = 0; i < kVec; ++i) {
    const int vi = threadIdx.x + i * kRowThreads;
    if (vi < nvec) raw[i] = *reinterpret_cast<const uint4*>(xr + vi * 8);
  }
  i8_quantize_row<kVec>(raw, nvec, red, q + static_cast<size_t>(row) * ldq, scale_rows + row);
}

int i8_quantize_rows(const void* x, int ldx, int rows, int cols, void* q, int ldq, float* scale_rows,
                     cudaStream_t stream) {
  if (cols <= 0 || cols % 8 != 0 || cols > kRowThreads * 8 * kQuantMaxVec || rows <= 0 || ldx % 8 != 0 ||
      ldq % 8 != 0 || ldx < cols || ldq < cols) {
    set_last_error("i8_quantize_rows: unsupported rows=%d cols=%d ldx=%d ldq=%d", rows, cols, ldx, ldq);
    return KR_ERR_UNSUPPORTED_SHAPE;
  }
  const int nv = (cols / 8 + kRowThreads - 1) / kRowThreads;
#define KR_Q_LAUNCH(V)                                                                             \
  i8_quantize_rows_kernel<V><<<rows, kRowThreads, 0, stream>>>(                                    \
      static_cast<const uint16_t*>(x), ldx, cols, static_cast<int8_t*>(q), ldq, scale_rows)
  switch (nv) {
    case 1: KR_Q_LAUNCH(1); break;
    case 2: KR_Q_LAUNCH(2); break;
    case 3: KR_Q_LAUNCH(3); break;
    case 4: KR_Q_LAUNCH(4); break;
    case 5: KR_Q_LAUNCH(5); break;
    case 6: KR_Q_LAUNCH(6); break;
    case 7: case 8: KR_Q_LAUNCH(8); break;
    case 9: case 10: KR_Q_LAUNCH(10); break;
    default: KR_Q_LAUNCH(14); break;
  }
#undef KR_Q_LAUNCH
  return launch_status("i8_quantize_rows");
}

// Dynamic per-group e4m3 activation cast (torchao PerBlock [1, 128]): the row quantiser's CTA-per-row layout, one
// scale per 128-channel group stored k-block-major (scale[g * ld_s + r]: one k-block's row scales are contiguous for
// the block-scaled GEMM).  One read, one write, no atomics, no memset.
template <int kVec>
__global__ void __launch_bounds__(kRowThreads)
fp8_quantize_blocks_kernel(const uint16_t* __restrict__ x, int ldx, int cols, uint8_t* __restrict__ q, int ldq,
                           float* __restrict__ scale, int ld_s) {
  const int row = blockIdx.x;
  const uint16_t* xr = x + static_cast<size_t>(row) * ldx;
  const int nvec = cols >> 3;
  uint4 raw[kVec];
#pragma unroll
  for (int i = 0; i < kVec; ++i) {
    const int vi = threadIdx.x + i * kRowThreads;
    if (vi < nvec) raw[i] = *reinterpret_cast<const uint4*>(xr + vi * 8);
  }
  fp8_quantize_row_groups<kVec>(raw, nvec, q + static_cast<size_t>(row) * ldq, scale + row, ld_s);
}

int fp8_quantize_blocks(const void* x, int ldx, int rows, int cols, void* q, int ldq, float* scale, int ld_s,
                        cudaStream_t stream) {
  if (cols <= 0 || cols % 128 != 0 || cols > kRowThreads * 8 * kQuantMaxVec || rows <= 0 || ldx % 8 != 0 ||
      ldq % 16 != 0 || ldx < cols || ldq < cols || ld_s < rows) {
    set_last_error("fp8_quantize_blocks: unsupported rows=%d cols=%d ldx=%d ldq=%d ld_s=%d", rows, cols, ldx, ldq,
                   ld_s);
    return KR_ERR_UNSUPPORTED_SHAPE;
  }
  const int nv = (cols / 8 + kRowThreads - 1) / kRowThreads;
#define KR_Q_LAUNCH(V)                                                                             \
  fp8_quantize_blocks_kernel<V><<<rows, kRowThreads, 0, stream>>>(                                 \
      static_cast<const uint16_t*>(x), ldx, cols, static_cast<uint8_t*>(q), ldq, scale, ld_s)
  switch (nv) {
    case 1: KR_Q_LAUNCH(1); break;
    case 2: KR_Q_LAUNCH(2); break;
    case 3: KR_Q_LAUNCH(3); break;
    case 4: KR_Q_LAUNCH(4); break;
    case 5: KR_Q_LAUNCH(5); break;
    case 6: KR_Q_LAUNCH(6); break;
    case 7: case 8: KR_Q_LAUNCH(8); break;
    case 9: case 10: KR_Q_LAUNCH(10); break;
    default: KR_Q_LAUNCH(14); break;
  }
#undef KR_Q_LAUNCH
  return launch_status("fp8_quantize_blocks");
}

// ---------------------------------------------------------------------------
// q/k RMSNorm + RoPE + KV append.  One CTA per token row.
//   qkv row layout: q = qkv + row*ldqkv, k = q + D, v = q + 2D (fused to_qkv output), or three
//   separate pointers with their own leading dimensions.
//   rope table: float2 (cos, sin) [max_pos, head_dim/2]; per pair index i inside a head the
//   position used is  f (i < c_t) | h (i < c_t + c_h) | w  with c_t = c - 2*(c/3), c_h = c/3.
// ---------------------------------------------------------------------------

template <int kVec>
__global__ void __launch_bounds__(kRowThreads, 6) qkv_post_kernel(const QkvPostParams p) {
  __shared__ float red[4];
  const int row = blockIdx.x;
  const int nvec = p.D >> 3;
  const uint16_t* qr = p.q + static_cast<size_t>(row) * p.ldq;
  const uint16_t* kr_ = p.k + static_cast<size_t>(row) * p.ldk;
  uint4 qraw[kVec], kraw[kVec];          // packed bf16, unpacked per pass (see ln_modulate_kernel)
  float sq = 0.f, sk = 0.f;
#pragma unroll
  for (int i = 0; i < kVec; ++i) {
    const int vi = threadIdx.x + i * kRowThreads;
    if (vi < nvec) {
      qraw[i] = *reinterpret_cast<const uint4*>(qr + vi * 8);
      kraw[i] = *reinterpret_cast<const uint4*>(kr_ + vi * 8);
      const uint32_t uq[4] = {qraw[i].x, qraw[i].y, qraw[i].z, qraw[i].w};
      const uint32_t uk[4] = {kraw[i].x, kraw[i].y, kraw[i].z, kraw[i].w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 a = unpack_bf16x2(uq[j]), b = unpack_bf16x2(uk[j]);
        sq += a.x * a.x + a.y * a.y;
        sk += b.x * b.x + b.y * b.y;
      }
    }
  }
  const float rq = rsqrtf(block_sum(sq, red) / p.D + p.eps);
  const float rk = rsqrtf(block_sum(sk, red) / p.D + p.eps);

  const int hw = p.grid_h * p.grid_w;
  const int grow = row + p.row_offset;
  const int pf = grow / hw + p.start_frame;
  const int ph = (grow % hw) / p.grid_w;
  const int pw = grow % p.grid_w;
  const int c = p.head_dim >> 1;
  const int c_h = c / 3, c_t = c - 2 * c_h;

  const bool peers = p.peer_cols > 0;
  uint16_t* qo = peers ? nullptr : p.q_out + static_cast<size_t>(row) * p.ldqo;
  uint16_t* ko = peers ? nullptr : p.k_out + static_cast<size_t>(row) * p.ldko;
#pragma unroll
  for (int i = 0; i < kVec; ++i) {
    const int vi = threadIdx.x + i * kRowThreads;
    if (vi < nvec) {
      float wq[8], wk[8], a[8], b[8];
      load8(p.wq + vi * 8, wq);
      load8(p.wk + vi * 8, wk);
      {
        const uint32_t uq[4] = {qraw[i].x, qraw[i].y, qraw[i].z, qraw[i].w};
        const uint32_t uk[4] = {kraw[i].x, kraw[i].y, kraw[i].z, kraw[i].w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 fa = unpack_bf16x2(uq[j]), fb = unpack_bf16x2(uk[j]);
          a[2 * j] = fa.x; a[2 * j + 1] = fa.y;
          b[2 * j] = fb.x; b[2 * j + 1] = fb.y;
        }
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        a[j] = bf16_round(bf16_round(a[j] * rq) * wq[j]);
        b[j] = bf16_round(bf16_round(b[j] * rk) * wk[j]);
      }
      if (p.rope != nullptr) {
        const int pair0 = ((vi * 8) % p.head_dim) >> 1;   // first of 4 complex pairs
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int pi = pair0 + j;
          const int pos = pi < c_t ? pf : (pi < c_t + c_h ? ph : pw);
          const float2 cs = __ldg(p.rope + static_cast<size_t>(pos) * c + pi);
          const float a0 = a[2 * j], a1 = a[2 * j + 1];
          a[2 * j] = a0 * cs.x - a1 * cs.y;
          a[2 * j + 1] = a0 * cs.y + a1 * cs.x;
          const float b0 = b[2 * j], b1 = b[2 * j + 1];
          b[2 * j] = b0 * cs.x - b1 * cs.y;
          b[2 * j + 1] = b0 * cs.y + b1 * cs.x;
        }
      }
      if (peers) {
        // heads [d*peer_cols/head_dim, ...) belong to rank d: remote 16-byte stores over NVLink
        const int d = (vi * 8) / p.peer_cols, col = (vi * 8) - d * p.peer_cols;
        store8(p.q_peer[d] + static_cast<size_t>(row) * p.ldqo + col, a);
        store8(p.k_peer[d] + static_cast<size_t>(row) * p.ldko + col, b);
      } else {
        store8(qo + vi * 8, a);
        store8(ko + vi * 8, b);
      }
    }
  }
  if (p.v != nullptr) {
    const uint16_t* vr = p.v + static_cast<size_t>(row) * p.ldv;
    if (peers) {
      for (int vi = threadIdx.x; vi < nvec; vi += kRowThreads) {
        const int d = (vi * 8) / p.peer_cols, col = (vi * 8) - d * p.peer_cols;
        *reinterpret_cast<uint4*>(p.v_peer[d] + static_cast<size_t>(row) * p.ldvo + col) =
            *reinterpret_cast<const uint4*>(vr + vi * 8);
      }
    } else {
      uint16_t* vo = p.v_out + static_cast<size_t>(row) * p.ldvo;
      for (int vi = threadIdx.x; vi < nvec; vi += kRowThreads)
        *reinterpret_cast<uint4*>(vo + vi * 8) = *reinterpret_cast<const uint4*>(vr + vi * 8);
    }
  }
}

// ---------------------------------------------------------------------------
// KV-cache roll (rolling-window eviction, causal_model.py:363-373): rows [src_row, src_row + rows) move down to
// [dst_row, dst_row + rows), dst_row < src_row, ranges may overlap.  The reference does it with a `.clone()` of
// the whole window per tensor; here every thread owns ONE 16-byte column of the row and walks the rows in
// ascending order (reads of a batch of rows precede the writes of that batch), so an overlapping shift needs no
// temporary and no ordering between threads: a column is only ever touched by its own thread.
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
kv_roll_kernel(uint4* __restrict__ base, long pitch_vec, int vecs_per_row, int dst_row, int src_row, int rows) {
  const int col = blockIdx.x * blockDim.x + threadIdx.x;
  if (col >= vecs_per_row) return;
  constexpr int U = 8;
  uint4* d = base + static_cast<size_t>(dst_row) * pitch_vec + col;
  const uint4* s = base + static_cast<size_t>(src_row) * pitch_vec + col;
  int r = 0;
  for (; r + U <= rows; r += U) {
    uint4 t[U];
#pragma unroll
    for (int j = 0; j < U; ++j) t[j] = s[static_cast<size_t>(r + j) * pitch_vec];
#pragma unroll
    for (int j = 0; j < U; ++j) d[static_cast<size_t>(r + j) * pitch_vec] = t[j];
  }
  for (; r < rows; ++r) d[static_cast<size_t>(r) * pitch_vec] = s[static_cast<size_t>(r) * pitch_vec];
}

int kv_roll(void* cache, int ld, int width, int dst_row, int src_row, int rows, cudaStream_t stream) {
  if (ld % 8 != 0 || width % 8 != 0 || width > ld || rows < 0 || dst_row < 0 || src_row < dst_row) {
    set_last_error("kv_roll: unsupported ld=%d width=%d dst=%d src=%d rows=%d", ld, width, dst_row, src_row, rows);
    return KR_ERR_INVALID_ARG;
  }
  if (rows == 0 || src_row == dst_row) return KR_OK;
  const int vecs = width / 8;
  kv_roll_kernel<<<(vecs + 255) / 256, 256, 0, stream>>>(static_cast<uint4*>(cache), ld / 8, vecs, dst_row, src_row,
                                                         rows);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_last_error("kv_roll: launch failed: %s", cudaGetErrorString(e));
    return KR_ERR_CUDA;
  }
  return KR_OK;
}

// ---------------------------------------------------------------------------
// rows of src -> the peer that owns them (attention output back from head-sharded to row-sharded)
// ---------------------------------------------------------------------------
struct ScatterPeers { uint16_t* dst[8]; };
__global__ void __launch_bounds__(128)
p2p_scatter_rows_kernel(const uint16_t* __restrict__ src, int ld_src, const ScatterPeers peers, int ld_dst,
                        int cols, int rows_per_peer) {
  const int row = blockIdx.x;
  const int d = row / rows_per_peer, r = row - d * rows_per_peer;
  const uint4* s = reinterpret_cast<const uint4*>(src + static_cast<size_t>(row) * ld_src);
  uint4* o = reinterpret_cast<uint4*>(peers.dst[d] + static_cast<size_t>(r) * ld_dst);
  for (int vi = threadIdx.x; vi < (cols >> 3); vi += blockDim.x) o[vi] = s[vi];
}

int p2p_scatter_rows(const void* src, int ld_src, void* const* dst_peer, int ld_dst, int rows, int cols,
                     int rows_per_peer, int world, cudaStream_t stream) {
  if (world < 1 || world > 8 || cols % 8 != 0 || ld_src % 8 != 0 || ld_dst % 8 != 0 || rows <= 0 ||
      rows_per_peer <= 0 || rows > rows_per_peer * world) {
    set_last_error("p2p_scatter_rows: unsupported rows=%d cols=%d rows_per_peer=%d world=%d", rows, cols,
                   rows_per_peer, world);
    return KR_ERR_INVALID_ARG;
  }
  ScatterPeers sp;
  for (int i = 0; i < 8; ++i) sp.dst[i] = i < world ? static_cast<uint16_t*>(dst_peer[i]) : nullptr;
  p2p_scatter_rows_kernel<<<rows, 128, 0, stream>>>(static_cast<const uint16_t*>(src), ld_src, sp, ld_dst, cols,
                                                    rows_per_peer);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_last_error("p2p_scatter_rows: launch failed: %s", cudaGetErrorString(e));
    return KR_ERR_CUDA;
  }
  return KR_OK;
}

int qkv_post(const QkvPostParams& p, int rows, cudaStream_t stream) {
  if (p.D % 8 != 0 || p.D > kRowThreads * 8 * kMaxVec || p.head_dim % 8 != 0 || rows <= 0 ||
      p.D % p.head_dim != 0) {
    set_last_error("qkv_post: unsupported D=%d head_dim=%d rows=%d", p.D, p.head_dim, rows);
    return KR_ERR_UNSUPPORTED_SHAPE;
  }
  if (p.rope != nullptr && (p.grid_h <= 0 || p.grid_w <= 0)) {
    set_last_error("qkv_post: rope needs grid_h/grid_w");
    return KR_ERR_INVALID_ARG;
  }
  const int nv = (p.D / 8 + kRowThreads - 1) / kRowThreads;
  switch (nv) {
    case 1: qkv_post_kernel<1><<<rows, kRowThreads, 0, stream>>>(p); break;
    case 2: qkv_post_kernel<2><<<rows, kRowThreads, 0, stream>>>(p); break;
    case 3: qkv_post_kernel<3><<<rows, kRowThreads, 0, stream>>>(p); break;
    case 4: qkv_post_kernel<4><<<rows, kRowThreads, 0, stream>>>(p); break;
    case 5: qkv_post_kernel<5><<<rows, kRowThreads, 0, stream>>>(p); break;
    default: qkv_post_kernel<8><<<rows, kRowThreads, 0, stream>>>(p); break;
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_last_error("qkv_post: launch failed: %s", cudaGetErrorString(e));
    return KR_ERR_CUDA;
  }
  return KR_OK;
}

// ---------------------------------------------------------------------------
// RMSNorm rows: out = bf16(bf16(x * rsqrt(mean(x^2)+eps)) * w)
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(kRowThreads)
rmsnorm_rows_kernel(const uint16_t* __restrict__ x, int ldx, uint16_t* __restrict__ out, int ldo,
                    const uint16_t* __restrict__ w, int D, float eps) {
  __shared__ float red[4];
  const int row = blockIdx.x;
  const int nvec = D >> 3;
  const uint16_t* xr = x + static_cast<size_t>(row) * ldx;
  float v[kMaxVec][8];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < kMaxVec; ++i) {
    const int vi = threadIdx.x + i * kRowThreads;
    if (vi < nvec) {
      load8(xr + vi * 8, v[i]);
#pragma unroll
      for (int j = 0; j < 8; ++j) s += v[i][j] * v[i][j];
    }
  }
  const float r = rsqrtf(block_sum(s, red) / D + eps);
  uint16_t* orow = out + static_cast<size_t>(row) * ldo;
#pragma unroll
  for (int i = 0; i < kMaxVec; ++i) {
    const int vi = threadIdx.x + i * kRowThreads;
    if (vi < nvec) {
      float ww[8], y[8];
      load8(w + vi * 8, ww);
#pragma unroll
      for (int j = 0; j < 8; ++j) y[j] = bf16_round(v[i][j] * r) * ww[j];
      store8(orow + vi * 8, y);
    }
  }
}

int rmsnorm_rows(const void* x, int ldx, void* out, int ldo, const void* w, int rows, int D,
                 float eps, cudaStream_t stream) {
  if (D % 8 != 0 || D > kRowThreads * 8 * kMaxVec || rows <= 0) {
    set_last_error("rmsnorm_rows: unsupported D=%d rows=%d", D, rows);
    return KR_ERR_UNSUPPORTED_SHAPE;
  }
  rmsnorm_rows_kernel<<<rows, kRowThreads, 0, stream>>>(
      static_cast<const uint16_t*>(x), ldx, static_cast<uint16_t*>(out), ldo,
      static_cast<const uint16_t*>(w), D, eps);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_last_error("rmsnorm_rows: launch failed: %s", cudaGetErrorString(e));
    return KR_ERR_CUDA;
  }
  return KR_OK;
}

// ---------------------------------------------------------------------------
// e[f, r, :] = bf16(modulation[r, :] + e0[f, r, :])   (r < mod_rows)
// ---------------------------------------------------------------------------
__global__ void add_modulation_kernel(const uint16_t* __restrict__ modulation,
                                      const uint16_t* __restrict__ e0, int lde0_frame,
                                      uint16_t* __restrict__ out, int frames, int mod_rows, int D) {
  const int per_frame = mod_rows * D;
  const int idx = (blockIdx.x * blockDim.x + threadIdx.x) * 8;
  if (idx >= frames * per_frame) return;
  const int f = idx / per_frame, r = idx % per_frame;
  float a[8], b[8];
  load8(modulation + r, a);
  load8(e0 + static_cast<size_t>(f) * lde0_frame + r, b);
#pragma unroll
  for (int j = 0; j < 8; ++j) a[j] += b[j];
  store8(out + idx, a);
}

int add_modulation(const void* modulation, const void* e0, int lde0_frame, void* out, int frames,
                   int mod_rows, int D, cudaStream_t stream) {
  if (D % 8 != 0 || frames <= 0 || mod_rows <= 0) {
    set_last_error("add_modulation: unsupported D=%d", D);
    return KR_ERR_UNSUPPORTED_SHAPE;
  }
  const int n = frames * mod_rows * D / 8;
  add_modulation_kernel<<<(n + 255) / 256, 256, 0, stream>>>(
      static_cast<const uint16_t*>(modulation), static_cast<const uint16_t*>(e0), lde0_frame,
      static_cast<uint16_t*>(out), frames, mod_rows, D);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_last_error("add_modulation: launch failed: %s", cudaGetErrorString(e));
    return KR_ERR_CUDA;
  }
  return KR_OK;
}

// ---------------------------------------------------------------------------
// elementwise activations on bf16: 0 = SiLU, 1 = GELU(tanh)
// ---------------------------------------------------------------------------
__global__ void act_kernel(const uint16_t* __restrict__ x, uint16_t* __restrict__ y, size_t n8,
                           int kind) {
  const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n8) return;
  float v[8];
  load8(x + i * 8, v);
#pragma unroll
  for (int j = 0; j < 8; ++j)
    v[j] = kind == 0 ? v[j] / (1.0f + __expf(-v[j])) : gelu_tanh(v[j]);
  store8(y + i * 8, v);
}

int activation(const void* x, void* y, size_t n, int kind, cudaStream_t stream) {
  if (n % 8 != 0) {
    set_last_error("activation: n=%zu not a multiple of 8", n);
    return KR_ERR_UNSUPPORTED_SHAPE;
  }
  const size_t n8 = n / 8;
  act_kernel<<<static_cast<unsigned>((n8 + 255) / 256), 256, 0, stream>>>(
      static_cast<const uint16_t*>(x), static_cast<uint16_t*>(y), n8, kind);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_last_error("activation: launch failed: %s", cudaGetErrorString(e));
    return KR_ERR_CUDA;
  }
  return KR_OK;
}

// ---------------------------------------------------------------------------
// patchify: x [C, F, H, W] (strided) -> tokens [F*(H/2)*(W/2), C*4] with column order
// (c, ph, pw) = the flattened Conv3d(k=s=(1,2,2)) weight order (causal_model.py:614-615, :874-877)
// ---------------------------------------------------------------------------
__global__ void patchify_kernel(const uint16_t* __restrict__ x, long sc, long sf, long sh, long sw,
                                uint16_t* __restrict__ out, int C, int F, int H, int W) {
  const int h2 = H / 2, w2 = W / 2;
  const int K = C * 4;
  const long total = static_cast<long>(F) * h2 * w2 * K;
  const long idx = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int col = idx % K;
  const long tok = idx / K;
  const int c = col >> 2, ph = (col >> 1) & 1, pw = col & 1;
  const int ww = tok % w2, hh = (tok / w2) % h2, f = tok / (static_cast<long>(w2) * h2);
  out[idx] = x[c * sc + f * sf + (2 * hh + ph) * sh + (2 * ww + pw) * sw];
}

int patchify(const void* x, long sc, long sf, long sh, long sw, void* out, int C, int F, int H,
             int W, cudaStream_t stream) {
  if (H % 2 != 0 || W % 2 != 0) {
    set_last_error("patchify: odd H/W");
    return KR_ERR_UNSUPPORTED_SHAPE;
  }
  const long total = static_cast<long>(F) * (H / 2) * (W / 2) * C * 4;
  patchify_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(
      static_cast<const uint16_t*>(x), sc, sf, sh, sw, static_cast<uint16_t*>(out), C, F, H, W);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_last_error("patchify: launch failed: %s", cudaGetErrorString(e));
    return KR_ERR_CUDA;
  }
  return KR_OK;
}

// ---------------------------------------------------------------------------
// unpatchify + flow->x0:
//   head_out [F*h2*w2, 4*C] with column order (ph, pw, c) (causal_model.py:1145-1147)
//   flow[f, c, 2hh+ph, 2ww+pw] = head_out[...]
//   x0 = bf16( double(xt) - sigma[f] * double(flow) )   (utils/wan_wrapper.py:181-205)
// flow / x0 / xt are [F, C, H, W] contiguous.
// ---------------------------------------------------------------------------
__global__ void unpatchify_x0_kernel(const uint16_t* __restrict__ head_out, int ldh,
                                     const uint16_t* __restrict__ xt, const double* __restrict__ sigma,
                                     uint16_t* __restrict__ flow, uint16_t* __restrict__ x0, int C,
                                     int F, int H, int W) {
  const long total = static_cast<long>(F) * C * H * W;
  const long idx = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int w = idx % W, h = (idx / W) % H;
  const int c = (idx / (static_cast<long>(W) * H)) % C;
  const int f = idx / (static_cast<long>(W) * H * C);
  const int h2 = H / 2, w2 = W / 2;
  const long tok = (static_cast<long>(f) * h2 + h / 2) * w2 + w / 2;
  const int col = ((h & 1) * 2 + (w & 1)) * C + c;
  const uint16_t fv = head_out[tok * ldh + col];
  flow[idx] = fv;
  if (x0 != nullptr) {
    const double fl = static_cast<double>(__bfloat162float(*reinterpret_cast<const __nv_bfloat16*>(&fv)));
    const double xv = static_cast<double>(
        __bfloat162float(*reinterpret_cast<const __nv_bfloat16*>(&xt[idx])));
    const float r = static_cast<float>(xv - sigma[f] * fl);
    // double -> bf16: round-to-nearest-even from the double value (via float is exact enough:
    // the difference of two bf16-scale numbers fits float's 24-bit mantissa except in rare
    // double-rounding ties, which torch's double->bf16 cast also resolves through float)
    __nv_bfloat16 o = __float2bfloat16_rn(r);
    x0[idx] = *reinterpret_cast<uint16_t*>(&o);
  }
}

int unpatchify_x0(const void* head_out, int ldh, const void* xt, const double* sigma, void* flow,
                  void* x0, int C, int F, int H, int W, cudaStream_t stream) {
  if (H % 2 != 0 || W % 2 != 0) {
    set_last_error("unpatchify_x0: odd H/W");
    return KR_ERR_UNSUPPORTED_SHAPE;
  }
  const long total = static_cast<long>(F) * C * H * W;
  unpatchify_x0_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(
      static_cast<const uint16_t*>(head_out), ldh, static_cast<const uint16_t*>(xt), sigma,
      static_cast<uint16_t*>(flow), static_cast<uint16_t*>(x0), C, F, H, W);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_last_error("unpatchify_x0: launch failed: %s", cudaGetErrorString(e));
    return KR_ERR_CUDA;
  }
  return KR_OK;
}

}  // namespace kr
