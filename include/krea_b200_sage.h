/* krea_b200_sage.h — C ABI of the quantised attention tier of libkrea_b200.so (included by krea_b200.h; the
 * conventions of krea_b200.h apply: device pointers, caller-owned memory, 0 or a negative KR_ERR_* code). */
#ifndef KREA_B200_SAGE_H_
#define KREA_B200_SAGE_H_

#ifdef __cplusplus
extern "C" {
#endif

/* Quantised attention tier = what the reference runs on an H100 with the sageattention wheel installed
 * (wan/modules/attention.py:166-180, model.py:201-213: sageattn -> sageattn_qk_int8_pv_fp8_cuda_sm90 with per-thread
 * INT8 Q/K, smoothed K and e4m3 P.V with fp32 accumulation) for the cached self-attention and the cross-attention.
 * No mask; head_dim 128; q/k/v bf16 [L, heads*128] with free row pitches (K/V read in place from cache views).
 * Buffers (device memory, caller-owned; nqb = ceil(Lq/16), nkb = ceil(Lkv/128), W = heads*128):
 *   q_i8    int8  [Lq, W]         trunc(q/s + 0.5 sign(q)), s = q_scale of the row's group
 *   q_scale fp32  [heads, nqb, 8]  group (h, b, t) = rows 16b+t and 16b+8+t: amax/127 + 1e-7
 *   k_mean  bf16  [W]              bf16(mean of k over the Lkv rows), summed in a fixed order
 *   k_i8    int8  [Lkv, W]         the same rule on bf16(k - k_mean)
 *   k_scale fp32  [heads, nkb, 4]  group (h, c, t) = keys 128c + 8i + 2t + {0,1}, i < 16
 *   v_t8    e4m3  [W, nkb*128]     e4m3_satfinite(v / v_scale), transposed (keys contiguous); within every 16 keys
 *                                  stored position p holds key {0,1,8,9,2,3,10,11,4,5,12,13,6,7,14,15}[p]; keys >= Lkv 0
 *   v_scale fp32  [W]              max(amax_rows |v|, 1e-12) / 448
 * kr_sage_quantize: three launches, no host sync.  kr_sage_attn: out bf16 [Lq, ldo] = softmax(scale q k^T) v with
 * S = s32(q_i8 k_i8^T) * q_scale * k_scale, P~ = e4m3(448 P), O = sum over 128-key tiles of P~ v_t8 in fp32,
 * out = O * v_scale / (448 l).  Bad arguments return KR_ERR_INVALID_ARG before any CUDA call. */
int kr_sage_quantize(const void* q, int ldq, const void* k, int ldk, const void* v, int ldv, int Lq, int Lkv, int heads,
                     void* q_i8, float* q_scale, void* k_mean, void* k_i8, float* k_scale, void* v_t8, float* v_scale,
                     void* stream);
int kr_sage_attn(const void* q_i8, const float* q_scale, const void* k_i8, const float* k_scale, const void* v_t8,
                 const float* v_scale, void* out, int ldo, int Lq, int Lkv, int heads, float softmax_scale, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* KREA_B200_SAGE_H_ */
