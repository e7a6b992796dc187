/* krea_b200_fp8_blocks.h — C ABI of the block-scaled FP8 linears of libkrea_b200.so (included by krea_b200.h; the
 * conventions of krea_b200.h apply: device pointers, caller-owned memory, 0 or a negative KR_ERR_* code). */
#ifndef KREA_B200_FP8_BLOCKS_H_
#define KREA_B200_FP8_BLOCKS_H_

#ifdef __cplusplus
extern "C" {
#endif

/* Block-scaled FP8 = torchao Float8DynamicActivationFloat8WeightConfig(granularity=[PerBlock([1, 128]),
 * PerBlock([128, 128])]), the DeepSeek-V3 recipe: one scale per 1 x 128 group of an activation row and one per
 * 128 x 128 block of the weight, so an outlier channel sets the scale of its own 128-channel group only.
 * Activation scales are stored k-block-major, fp32 [cols / 128, ld_s] with ld_s >= rows: scale[g * ld_s + r] is the
 * scale of channels [128 g, 128 g + 128) of row r (one k-block's row scales are contiguous).
 *   kr_fp8_quantize_blocks    : x [rows, cols] bf16 -> q e4m3 bytes [rows, ldq], q[r, g] = sat(x[r, g] * 448 / amax)
 *                               with amax = max(max|x[r, g]|, 1e-12) (a true fp32 division, round to nearest even),
 *                               scale[g * ld_s + r] = amax / 448.  One read, one write; cols % 128 == 0,
 *                               cols <= 14336, ldq % 16 == 0.
 *   kr_ln_modulate_fp8_blocks : kr_ln_modulate whose bf16 output row is cast like kr_fp8_quantize_blocks into q /
 *                               scale (bit-identical to quantising kr_ln_modulate's output); out may be NULL, then only
 *                               the e4m3 bytes and scales are written.  D % 128 == 0.
 *   kr_gemm_fp8_blockwise     : out = epilogue(sum_kb (a_q[:, kb] @ w_q[:, kb]^T) * scale_a[kb][m] * scale_w[n/128][kb]
 *                               + bias), scale_w fp32 [N / 128, K / 128]; every 128-wide k-block's partial is scaled
 *                               and added in fp32 (promoted accumulation only).  The epilogues of kr_gemm_fp8 plus
 *                               KR_EPI_F32 (alpha 1); N % 128 == 0, K % 128 == 0, lda / ldw % 16 == 0, ldc % 8 == 0,
 *                               ld_sa >= M, else KR_ERR_INVALID_ARG before any CUDA call. */
int kr_fp8_quantize_blocks(const void* x, int ldx, int rows, int cols, void* q, int ldq, float* scale, int ld_s,
                           void* stream);
int kr_ln_modulate_fp8_blocks(const void* x, int ldx, void* out, int ldo, int rows, int D, float eps,
                              const void* w, const void* b, const void* mod, int mod_rows, int shift_idx,
                              int scale_idx, int rows_per_frame, int row_offset, void* q, int ldq, float* scale,
                              int ld_s, void* stream);
int kr_gemm_fp8_blockwise(int epilogue, const void* a, int lda, const void* w, int ldw, const float* scale_a,
                          int ld_sa, const float* scale_w, const void* bias, void* out, int ldc, int M, int N, int K,
                          const void* residual, int ldr, const void* gate, int gate_stride, int rows_per_gate,
                          void* out2, int ldc2, int n_split, int row_offset, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* KREA_B200_FP8_BLOCKS_H_ */
