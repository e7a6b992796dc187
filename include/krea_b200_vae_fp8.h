/* krea_b200_vae_fp8.h — C ABI of the FP8 (e4m3) tier of the VAE decoder's and encoder's convolutions (included by krea_b200.h;
 * the conventions of krea_b200.h apply: device pointers, caller-owned memory, 0 or a negative KR_ERR_* code). */
#ifndef KREA_B200_VAE_FP8_H_
#define KREA_B200_VAE_FP8_H_

#ifdef __cplusplus
extern "C" {
#endif

/* The convs whose input is a normalised tensor (residual.2 / residual.6 of every ResidualBlock, head.2) read e4m3 bytes
 * e4m3(v * s) of the fp16 value v = SiLU(RMS_norm(x) * sqrt(C) * gamma), with the static per-conv scale
 * s = 448 / (sqrt(C) * max|gamma|) (no amax pass: |v| <= sqrt(C) max|gamma|, nothing saturates), and per-output-channel
 * e4m3 weights w_q [w_rows, taps*cin] with fp32 dequantisation scales w_scale [n] (w ~ w_q * w_scale[row]).
 *
 * kr_vae_conv_fp8: kr_vae_conv3d's contract (same geometry, strides and epilogues; fp16 only, no sub2) with
 *   in_fp8 = 1: in / weight are e4m3, acc = sum(in_q * w_q) in fp32 (promoted every <= 128 k), then
 *               out = acc * (1 / in_scale) * w_scale[c] + bias, and the fp16 epilogue as kr_vae_conv3d.
 *               (cin, n) in (192,192) (96,96) (96,192) [3x3 spatial taps], (384,384) (192,384) (96,16) (384,32).
 *   in_fp8 = 0: in / weight are fp16 (kr_vae_conv3d) and out_norm is required.
 *               (cin, n) in (64,384) (64,96) (192,192) (384,384), and (384,192) (192,96) (96,96) with 3x3 spatial
 *               taps.
 *   out_norm, when given, holds e4m3 bytes e4m3_satfinite(fp16(SiLU(...)) * norm_q_scale) (element strides = bytes).
 * kr_vae_conv_fp8_sub2: kr_vae_conv_fp8 with kr_vae_conv3d's sub2 = 1 epilogue (the encoder's stride-2 conv behind
 *   ZeroPad2d((0,1,0,1)): H x W input, H/2 x W/2 outputs); in_fp8 = 0, 3x3 spatial taps, kt = 1, no out_pix.
 * kr_vae_rmsnorm_silu_fp8: kr_vae_rmsnorm_silu (fp16, SiLU on) with y as e4m3 bytes e4m3_satfinite(fp16(y) * q_scale).
 * Bad arguments return KR_ERR_INVALID_ARG before any CUDA call. */
int kr_vae_conv_fp8(int in_fp8, int cin, int n, const void* in, int t_in, const void* weight, const float* w_scale,
                    float in_scale, int w_rows, const void* bias, int cout, int T, int H, int W, int tile_w,
                    int tile_h, int kt, int kh, int kw, void* out_raw, long raw_pix, long raw_frame, void* out_norm,
                    long norm_pix, long norm_frame, float norm_q_scale, const void* gamma, const void* residual,
                    long res_pix, long res_frame, float* out_pix, void* stream);
int kr_vae_conv_fp8_sub2(int in_fp8, int cin, int n, const void* in, int t_in, const void* weight,
                         const float* w_scale, float in_scale, int w_rows, const void* bias, int cout, int T, int H,
                         int W, int tile_w, int tile_h, int kt, int kh, int kw, void* out_raw, long raw_pix,
                         long raw_frame, void* out_norm, long norm_pix, long norm_frame, float norm_q_scale,
                         const void* gamma, const void* residual, long res_pix, long res_frame, float* out_pix,
                         void* stream);
int kr_vae_rmsnorm_silu_fp8(const void* x, void* y, const void* gamma, long pixels, int C, float q_scale,
                            void* stream);

#ifdef __cplusplus
}
#endif
#endif /* KREA_B200_VAE_FP8_H_ */
