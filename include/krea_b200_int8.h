/* krea_b200_int8.h — C ABI of the INT8 linears of libkrea_b200.so (included by krea_b200.h; the conventions of
 * krea_b200.h apply: device pointers, caller-owned memory, 0 or a negative KR_ERR_* code). */
#ifndef KREA_B200_INT8_H_
#define KREA_B200_INT8_H_

#ifdef __cplusplus
extern "C" {
#endif

/* INT8 = torchao Int8DynamicActivationInt8WeightConfig: symmetric per-token s8 activations, symmetric per-channel s8
 * weights, an s8 tensor-core GEMM whose s32 sums are exact.
 *   kr_i8_quantize_rows : x [rows, cols] bf16 -> q s8 [rows, ldq], q[r] = clamp(rint(x[r] * (127 / amax_r)), -127, 127)
 *                         with amax_r = max(max|x[r]|, 1e-12) (a true fp32 division, round half to even);
 *                         scale_rows [rows] fp32 receives amax_r / 127.  One read, one write; cols % 8 == 0,
 *                         cols <= 14336.
 *   kr_ln_modulate_i8   : kr_ln_modulate whose bf16 output row is also cast like kr_i8_quantize_rows into q /
 *                         scale_rows (bit-identical to quantising kr_ln_modulate's output); out may be NULL, then only
 *                         the s8 bytes and scales are written.
 *   kr_gemm_i8_rowwise  : out = epilogue((float(a_q @ w_q^T) * scale_a[m]) * scale_w[n] + bias), the product summed
 *                         exactly in s32; scale_w [N] fp32 is 16-byte aligned.  The epilogues of kr_gemm_fp8 plus
 *                         KR_EPI_F32 (the scaled sums as fp32, no rounding to bf16).  A 128 x 256 tile: N % 256 == 0,
 *                         K % 16 == 0, K <= 132104 (so |sum| <= 127 * 128 * K < 2^31), lda / ldw % 16 == 0,
 *                         ldc % 8 == 0, else KR_ERR_INVALID_ARG before any CUDA call. */
int kr_i8_quantize_rows(const void* x, int ldx, int rows, int cols, void* q, int ldq, float* scale_rows,
                        void* stream);
int kr_ln_modulate_i8(const void* x, int ldx, void* out, int ldo, int rows, int D, float eps,
                      const void* w, const void* b, const void* mod, int mod_rows, int shift_idx,
                      int scale_idx, int rows_per_frame, int row_offset, void* q, int ldq, float* scale_rows,
                      void* stream);
int kr_gemm_i8_rowwise(int epilogue, const void* a, int lda, const void* w, int ldw, const float* scale_a,
                       const float* scale_w, const void* bias, void* out, int ldc, int M, int N, int K,
                       const void* residual, int ldr, const void* gate, int gate_stride, int rows_per_gate,
                       void* out2, int ldc2, int n_split, int row_offset, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* KREA_B200_INT8_H_ */
