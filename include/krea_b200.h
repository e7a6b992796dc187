/* krea_b200.h — C ABI of libkrea_b200.so (H100 / sm_90a kernels for the Self-Forcing
 * causal-inference hot path of krea-ai/realtime-video).
 *
 * The reference has no FFI of its own (it is pure Python over torch; SURVEY.md §8b), so this
 * ABI is the boundary a maintainer binds with ctypes (INTEGRATION.md shows the stub).  Each
 * entry point names the reference code it replaces (paths relative to the reference repo).
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless stated; the caller (PyTorch) owns all memory,
 *     kernels never allocate; `stream` is a cudaStream_t passed as void*.
 *   - 16-bit tensors: dtype 0 = bfloat16, 1 = float16.  "ld*" = leading dimension in elements.
 *   - return 0 on success, negative KR_ERR_* otherwise; kr_last_error() gives the message of
 *     the calling thread's last failure.  Nothing throws across the ABI.
 *   - calls are asynchronous on `stream`; re-entrant, but two calls must not touch the same
 *     KV cache concurrently (the reference is single-threaded on GPU work,
 *     release_server.py:918).
 */
#ifndef KREA_B200_H_
#define KREA_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define KR_OK 0
#define KR_ERR_INVALID_ARG (-1)
#define KR_ERR_UNSUPPORTED_SHAPE (-2)
#define KR_ERR_CUDA (-3)
#define KR_ERR_NO_DEVICE (-4)
#define KR_ERR_TENSORMAP (-5)

/* library version (major*10000 + minor*100 + patch) and last error string */
int kr_version(void);
const char* kr_last_error(void);

/* GEMM epilogues of kr_gemm */
#define KR_EPI_BIAS 0          /* out = cast(acc + bias)                                         */
#define KR_EPI_BIAS_GELU 1     /* out = cast(gelu_tanh(cast(acc + bias)))                        */
#define KR_EPI_BIAS_GATE_RES 2 /* out = cast(res + cast(cast(acc+bias) * gate[row/rows_per_gate])) */
#define KR_EPI_BIAS_RES 3      /* out = cast(res + cast(acc + bias))                             */
#define KR_EPI_F32 4           /* out(fp32) = (acc + bias) * alpha                               */
#define KR_EPI_MUL 5           /* out = cast(cast(acc + bias) * res)  (UMT5 gated FFN, t5.py:138-140) */

/* out[M,N] = epilogue(a[M,K] @ w[N,K]^T + bias[N]); wgmma tensor-core GEMM.
 * Replaces nn.Linear (cuBLASLt) + the elementwise ops that follow it:
 *   to_qkv / q / k / v / o      wan/modules/causal_model.py:246-253, :396
 *   gate + residual             wan/modules/causal_model.py:476, :487-488
 *   ffn.0 + GELU(tanh), ffn.2   wan/modules/causal_model.py:433-435
 *   cross-attn q/k/v/o          wan/modules/model.py:183-190, :226-227
 *   patch/text/time embeddings, time_projection, head   causal_model.py:874-902, :507-522
 * Needs K % 8 == 0, N % 32 == 0, ld* % 8 == 0.  bias/residual/gate may be NULL when unused.
 * out2 (optional): output columns >= n_split (a multiple of 256) are written to out2 instead,
 * starting at its column 0 with leading dimension ldc2 — the V third of to_qkv goes straight
 * into the KV-cache slot (causal_model.py:385).  row_offset: global index of local row 0 when the
 * token rows are sharded across GPUs (gate row = (row + row_offset) / rows_per_gate). */
int kr_gemm(int dtype, int epilogue, const void* a, int lda, const void* w, int ldw,
            const void* bias, void* out, int ldc, int M, int N, int K, const void* residual,
            int ldr, const void* gate, int gate_stride, int rows_per_gate, float alpha,
            void* out2, int ldc2, int n_split, int row_offset, void* stream);

/* kr_gemm with a caller-owned workspace: kr_gemm_workspace_bytes() bytes of device memory, zero-filled ONCE by the
 * caller and then private to the stream the calls are issued on.  With it, shapes whose output-tile count does not
 * fill the SMs (e.g. the M = 4680/N-row shards of the multi-GPU mode) run on the stream-K kernel: equal shares of
 * (tile, k-block) MMA iterations per SM, fp32 partial tiles exchanged through the workspace, the last contributor
 * of a tile sums them in CTA order and runs the fused epilogue.  workspace == NULL behaves exactly like kr_gemm. */
int kr_gemm_ws(int dtype, int epilogue, const void* a, int lda, const void* w, int ldw,
               const void* bias, void* out, int ldc, int M, int N, int K, const void* residual,
               int ldr, const void* gate, int gate_stride, int rows_per_gate, float alpha,
               void* out2, int ldc2, int n_split, int row_offset, void* workspace, size_t workspace_bytes,
               void* stream);
size_t kr_gemm_workspace_bytes(void);

/* FP8 path = what `enable_fp8: true` does to the reference's transformer (release_server.py:179-182: torchao
 * quantize_(..., Float8DynamicActivationFloat8WeightConfig(granularity=PerTensor()))): every nn.Linear becomes
 * a dynamic per-tensor e4m3 cast of its input followed by an FP8 matmul with fp32 accumulation and bf16 output.
 *   kr_fp8_quantize : x [rows, cols] bf16 -> q e4m3 bytes [rows, ldq] = sat(x * 448 / amax(|x|)); state (2 floats of
 *                     device memory) receives [amax, amax / 448]; &state[1] is the scale_a of the following GEMM.
 *   kr_gemm_fp8     : out = epilogue((a_q @ w_q^T) * (*scale_a) * scale_w + bias), e4m3 wgmma, bf16
 *                     output, the epilogues of kr_gemm except KR_EPI_F32 / KR_EPI_MUL; N % 256 == 0, K % 16 == 0.
 * Weights are quantised once by the caller (w_q = sat(w * 448 / amax(|w|)), scale_w = amax / 448). */
int kr_fp8_quantize(const void* x, int ldx, int rows, int cols, void* q, int ldq, float* state, void* stream);
int kr_gemm_fp8(int epilogue, const void* a, int lda, const void* w, int ldw, const float* scale_a, float scale_w,
                const void* bias, void* out, int ldc, int M, int N, int K, const void* residual, int ldr,
                const void* gate, int gate_stride, int rows_per_gate, void* out2, int ldc2, int n_split, int row_offset,
                void* stream);

/* Which kernel kr_gemm launches for this epilogue and shape: 1 = the single-CTA kernel, 2 = the 2-CTA
 * cluster kernel (128x256 tile per CTA, W multicast to both), 3 = the stream-K kernel (only with a workspace), 4 = the
 * single-CTA kernel with a runtime tile width fitted to whole waves of SMs (small-M shards).  Host-only
 * queries (no launch), used by bench.py to attribute launch time per kernel. */
int kr_gemm_kernel_id(int epilogue, int M, int N, int K);
int kr_gemm_kernel_id_ws(int epilogue, int M, int N, int K, int have_workspace);

/* softmax(scale * q k^T) v, head_dim 128, [L, heads, 128] layout, bf16/fp16, fp32 softmax.
 * mask_mode 0: none (cached self-attention causal_model.py:386-390, cross-attention
 * model.py:214-215); mask_mode 1: block-causal rule of get_block_mask (causal_model.py:109-141)
 * with block_len = frame_seqlen*num_frame_per_block tokens and window = local_attn_size *
 * frame_seqlen tokens (0 = global); pad_keys = zero-padded key rows (ceil(L/128)*128 - L) that
 * queries of an incomplete last block also attend on the reference's FlexAttention path
 * (causal_model.py:316-348).  Replaces flash_attn_func / flex_attention. */
int kr_attn_fwd(int dtype, const void* q, int ldq, const void* k, int ldk, const void* v, int ldv,
                void* out, int ldo, int Lq, int Lkv, int heads, float softmax_scale, int mask_mode,
                int block_len, int window, int pad_keys, void* stream);

/* UMT5 encoder self-attention, one launch per layer: head_dim 64, bf16, L <= 1024, no 1/sqrt(d) scaling;
 *   out[q,h,:] = softmax_k( bf16(bf16(q.k) + bias_delta[h, k - q + L-1]) ) v[k,h,:],  masked keys (key_mask[k] == 0)
 * get finfo(bf16).min like the reference.  bias_delta [heads, 2L-1] bf16 = the layer's relative-position embedding
 * gathered by offset (T5RelativeEmbedding, wan/modules/t5.py:221-264); key_mask [L] uint8 or NULL.
 * Replaces T5Attention.forward's einsum / bias / fp32 softmax / einsum (wan/modules/t5.py:86-120). */
int kr_t5_attn(const void* q, int ldq, const void* k, int ldk, const void* v, int ldv, void* out, int ldo, int L,
               int heads, const void* bias_delta, const void* key_mask, void* stream);

/* WanLayerNorm (+affine) (+per-frame modulation x*(1+scale)+shift).
 * mod: [frames, mod_rows, D] 16-bit or NULL; w,b: [D] or NULL.
 * Replaces wan/modules/model.py:88-98 + causal_model.py:466-471, :482-485, :520-522 (bf16). */
int kr_ln_modulate(const void* x, int ldx, void* out, int ldo, int rows, int D, float eps,
                   const void* w, const void* b, const void* mod, int mod_rows, int shift_idx,
                   int scale_idx, int rows_per_frame, int row_offset, void* stream);

/* q,k: WanRMSNorm over D (model.py:69-85) then 3-axis RoPE (causal_model.py:143-171) written to
 * q_out and to the K cache slot; v copied to the V cache slot (causal_model.py:378-385, :310-311).
 * rope: float2 (cos,sin) [max_pos, head_dim/2] or NULL (no rotation, v may be NULL too). */
int kr_qkv_norm_rope(const void* q, int ldq, const void* k, int ldk, const void* v, int ldv,
                     const void* wq, const void* wk, void* q_out, int ldqo, void* k_out, int ldko,
                     void* v_out, int ldvo, const void* rope, int rows, int D, int head_dim,
                     int grid_h, int grid_w, int start_frame, int row_offset, float eps, void* stream);

/* Multi-GPU single-stream mode (SURVEY.md 8e option 3: token rows sharded, heads sharded for self-attention).
 * kr_qkv_norm_rope_p2p = kr_qkv_norm_rope whose stores ARE the rows->heads exchange: the columns of rank d's heads
 * ([d*peer_cols, (d+1)*peer_cols)) of every local row are written straight into rank d's q buffer / K-cache slot /
 * V-cache slot over NVLink peer memory (16-byte remote stores); *_peer[d] addresses this rank's first row inside
 * rank d's buffer (caller-owned symmetric allocations whose peer addresses the caller exchanged, e.g. through
 * torch.distributed._symmetric_memory); world <= 8.  kr_comm_scatter_rows is the way back: rows
 * [r*rows_per_peer, (r+1)*rows_per_peer) of the attention output of MY heads go to rank r's row-sharded buffer at
 * MY column block.  Both replace an NCCL all_to_all + pack/unpack copies; ordering across ranks is the caller's
 * (a barrier between the exchange and its consumer).  The reference is single-GPU (release_server.py:111-119 only
 * replicates models); these entry points have no reference counterpart. */
int kr_qkv_norm_rope_p2p(const void* q, int ldq, const void* k, int ldk, const void* v, int ldv,
                         const void* wq, const void* wk, void* const* q_peer, int ldqo, void* const* k_peer,
                         int ldko, void* const* v_peer, int ldvo, int world, int peer_cols, const void* rope,
                         int rows, int D, int head_dim, int grid_h, int grid_w, int start_frame, int row_offset,
                         float eps, void* stream);
int kr_comm_scatter_rows(const void* src, int ld_src, void* const* dst_peer, int ld_dst, int rows, int cols,
                         int rows_per_peer, int world, void* stream);

/* Rolling-window eviction of the self-attention KV cache (causal_model.py:363-373: `cache[sink : sink+rolled] =
 * cache[sink+evicted : sink+evicted+rolled].clone()`): rows [src_row, src_row+rows) of a 16-bit [*, ld] cache move
 * down to [dst_row, ...) in place (ranges may overlap, dst_row <= src_row), only the first `width` columns. */
int kr_kv_roll(void* cache, int ld, int width, int dst_row, int src_row, int rows, void* stream);

/* WanRMSNorm rows (cross-attention q / k): model.py:69-85, :183-190 */
int kr_rmsnorm(const void* x, int ldx, void* out, int ldo, const void* w, int rows, int D,
               float eps, void* stream);

/* e = modulation[mod_rows, D] + e0[frames, mod_rows, D]  (causal_model.py:466, :521) */
int kr_add_modulation(const void* modulation, const void* e0, int lde0_frame, void* out,
                      int frames, int mod_rows, int D, void* stream);

/* elementwise activation on bf16: kind 0 = SiLU, 1 = GELU(tanh)  (causal_model.py:617-623) */
int kr_activation(const void* x, void* y, size_t n, int kind, void* stream);

/* Conv3d(k=s=(1,2,2)) patch embedding as im2col: x[C,F,H,W] (element strides sc,sf,sh,sw) ->
 * tokens [F*(H/2)*(W/2), 4C]  (causal_model.py:614-615, :874-877) */
int kr_patchify(const void* x, long sc, long sf, long sh, long sw, void* out, int C, int F, int H,
                int W, void* stream);

/* unpatchify (causal_model.py:1126-1149) fused with flow->x0 in fp64
 * (utils/wan_wrapper.py:181-205): flow,x0,xt are [F,C,H,W]; sigma: double[F]; x0 may be NULL */
int kr_unpatchify_x0(const void* head_out, int ldh, const void* xt, const double* sigma,
                     void* flow, void* x0, int C, int F, int H, int W, void* stream);

/* ---- causal 3D VAE decoder (channels-last activations [frames, H, W, C], fp16 or bf16) ---- */

/* CausalConv3d / Conv2d / 1x1x1 conv as a wgmma implicit GEMM (wan/modules/vae.py:17-36,
 * :175-209; demo_utils/vae_block3.py:46-91, :386-443).  `in` holds t_in >= T + kt - 1 frames:
 * the (kt-1) cached frames in front of the T new ones (read in place, no cat/pad); spatial zero
 * padding is the TMA out-of-bounds fill.  weight: [w_rows, kt*kh*kw*cin] (tap-major, cin
 * contiguous).  (cin, n) must be one of the decoder's channel pairs: (64,384) (384,384)
 * (192,384) (384,192) (192,192) (192,96) (96,96) (96,16); n is the padded Cout, cout the real
 * one.  tile_w*tile_h == 128.  Outputs (any subset), element strides per pixel / per frame:
 *   out_raw  = cast(acc + bias [+ residual])
 *   out_norm = SiLU(RMS_norm_C(out_raw) * sqrt(cout) * gamma)     (vae.py:39-54, :184-186)
 *   out_pix  = clamp(out_raw, -1, 1) as fp32 [T, cout, H, W]       (vae_block3.py:226)
 * sub2 = 1: the encoder's stride-2 Conv2d behind ZeroPad2d((0,1,0,1)) (vae.py:84-92): only the odd
 * (h, w) positions of the stride-1 result are kept, compacted to an H/2 x W/2 output.
 * Extra (cin, n) pairs for the encoder: (64,96) (96,192) (384,32). */
int kr_vae_conv3d(int dtype, int cin, int n, const void* in, int t_in, const void* weight,
                  int w_rows, const void* bias, int cout, int T, int H, int W, int tile_w, int tile_h,
                  int kt, int kh, int kw, void* out_raw, long raw_pix, long raw_frame, void* out_norm,
                  long norm_pix, long norm_frame, const void* gamma, const void* residual,
                  long res_pix, long res_frame, float* out_pix, int sub2, void* stream);

/* y = RMS_norm_C(x) * sqrt(C) * gamma [-> SiLU], x,y [pixels, C]  (vae.py:39-54) */
int kr_vae_rmsnorm_silu(int dtype, const void* x, void* y, const void* gamma, long pixels, int C,
                        int do_silu, void* stream);

/* nearest-neighbour 2x spatial upsample [T,H,W,C] -> [T,2H,2W,C]  (vae.py:57-63) */
int kr_vae_upsample2x(const void* in, void* out, int T, int H, int W, int C, void* stream);

/* z [T,16,H,W] (element strides zt,zc,zh,zw): x = z/inv_std + mean, y = conv2_1x1x1(x), written
 * channels-last and zero-padded to 64 channels  (demo_utils/vae_block3.py:205-214) */
int kr_vae_scale_input(int dtype, const void* z, long zt, long zc, long zh, long zw,
                       const void* mean, const void* inv_std, const void* w2, const void* b2,
                       void* out, int T, int H, int W, void* stream);

/* p[r, :cols] = softmax(s[r, :cols]) ; fp32 in, 16-bit out  (vae.py:239-244 attention block) */
int kr_softmax_rows(int dtype, const float* s, long ld, void* p, long ldo, int rows, int cols,
                    void* stream);

/* One whole CausalWanAttentionBlock forward (causal_model.py:440-492: AdaLN-modulated self-attention with KV-cache
 * append (:218-397), T5 cross-attention (model.py:171-228), GELU FFN) as ONE call: the same 14 launches, with the same
 * arguments, as the per-op schedule above (kr_add_modulation, kr_ln_modulate, kr_gemm split into the V-cache slot,
 * kr_qkv_norm_rope into the K-cache slot, kr_attn_fwd, kr_gemm gate+residual, kr_ln_modulate affine, kr_gemm,
 * kr_rmsnorm, kr_attn_fwd over the prompt K/V, kr_gemm residual, kr_ln_modulate, kr_gemm GELU, kr_gemm gate+residual).
 * bf16, fused to_qkv ([3D, D], causal_model.py:204-216), one GPU, prompt K/V already projected (crossattn_cache
 * is_init); all weights [out, in] contiguous.  The cache index algebra of causal_model.py:349-392 stays with the
 * caller, which passes the resolved slot: rows [local_start, local_end) of the K / V cache receive this call's keys /
 * values; the queries attend rows [attn_lo, local_end) (cache branch, mask_mode 0) or rows [0, L) under the
 * block-causal rule (recompute branch, mask_mode 1: block_len / window / pad_keys as in kr_attn_fwd).
 * x [L, D] is updated in place.  workspace: kr_dit_block_workspace_bytes(L, D, ffn, frames) bytes, 256-byte aligned,
 * private to the stream; gemm_workspace: optional stream-K workspace exactly as in kr_gemm_ws (may be NULL). */
typedef struct KrDitBlockParams {
  int L, D, ffn, heads, head_dim;          /* tokens of this call, model width, FFN width, heads, 128 */
  int frames, rows_per_frame;              /* L == frames * rows_per_frame (modulation / gate rows change per frame) */
  int grid_h, grid_w, start_frame;         /* RoPE positions: token grid and the absolute index of the first frame */
  int cross_attn_norm;                     /* 1: norm3 is an affine LayerNorm, 0: identity */
  float eps_block, eps_qk, eps_norm3, eps_cross;
  void* x; int ldx;                        /* residual stream, in place */
  const void* e0; int lde0_frame;          /* time projection [frames, 6, D]; elements between frames */
  const void* modulation;                  /* blocks.N.modulation [6, D] */
  const void* rope;                        /* float2 (cos, sin) [1024, 64] */
  const void* w_qkv; const void* b_qkv;    /* self_attn.to_qkv */
  const void* norm_q; const void* norm_k;  /* self_attn.norm_q / norm_k weights [D] */
  const void* w_o; const void* b_o;        /* self_attn.o */
  void* k_cache; void* v_cache; int ld_cache;   /* row 0 of this layer's caches viewed as [rows, D] */
  int local_start, local_end, attn_lo;
  int mask_mode, block_len, window, pad_keys;
  const void* norm3_w; const void* norm3_b;
  const void* w_cq; const void* b_cq; const void* norm_cq;      /* cross_attn.q, cross_attn.norm_q */
  const void* ck; const void* cv; int ld_ck, ld_cv, text_len;   /* projected + normalised prompt K, V [text_len, D] */
  const void* w_co; const void* b_co;      /* cross_attn.o */
  const void* w_ffn0; const void* b_ffn0; const void* w_ffn2; const void* b_ffn2;
  void* workspace; size_t workspace_bytes;
  void* gemm_workspace; size_t gemm_workspace_bytes;
} KrDitBlockParams;
size_t kr_dit_block_workspace_bytes(int L, int D, int ffn, int frames);
int kr_dit_block_fwd(const KrDitBlockParams* params, void* stream);

/* Frame egress (SURVEY.md 8f.2): decoder pixels fp32 [frames, 3, H, W] in [-1, 1] -> packed RGB bytes
 * [frames, H, W, 3], byte = trunc(clamp((x + 1) * 0.5, 0, 1) * 255) in fp32 — the arithmetic the reference
 * runs on the host after the device->host copy (release_server.py:979-983 `add_(1.0).mul_(0.5).clamp_(0,1)`,
 * then torchvision `to_pil_image`: `.mul(255).byte()`), so 14.4 MB instead of 57.5 MB leave the device per
 * 12-frame 832x480 block.  `pixels` must be contiguous. */
int kr_frames_to_rgb8(const float* pixels, unsigned char* rgb, int frames, int height, int width, void* stream);

/* Frame egress, second half (SURVEY.md 8f.2): the JPEG files the reference produces on the host for every frame,
 * `TF.to_pil_image(frames[0, idx], "RGB").save(io, format='JPEG', quality=90)` (release_server.py:973; Pillow ->
 * libjpeg-turbo in a 24-thread pool), encoded on the device and BYTE-IDENTICAL to Pillow's output: integer
 * RGB->YCbCr, 4:2:0 box downsampling, "islow" DCT, round-half-away quantisation with the Annex K tables scaled by
 * `quality`, baseline Huffman coding, 0xFF stuffing, libjpeg's marker layout.  Per 12-frame 832x480 block ~1-3 MB
 * leave the device instead of 57.5 MB (fp32) or 14.4 MB (RGB8).
 *   kr_frames_to_jpeg : pixels fp32 [frames, 3, H, W] in [-1, 1], contiguous, 16-byte aligned (the decoder's
 *                       output; normalised exactly like kr_frames_to_rgb8)
 *   kr_rgb8_to_jpeg   : rgb bytes [frames, H, W, 3], contiguous, 8-byte aligned
 * H and W must be multiples of 16 (true for every resolution of the path: pixels = 8 x latent, latent dims even).
 * out: [frames, cap] bytes (cap % 4 == 0, out 4-byte aligned); file f starts at out + f * cap and has sizes[f]
 * bytes; sizes[f] < 0 means the file needs -sizes[f] bytes and did not fit (nothing is written past cap).
 * workspace: kr_jpeg_workspace_bytes(frames, H, W) bytes of device memory, 256-byte aligned, private to the stream
 * for the duration of the call (coefficients, bit offsets, the unstuffed bit stream).  Four launches, no host sync. */
size_t kr_jpeg_workspace_bytes(int frames, int height, int width);
int kr_frames_to_jpeg(const float* pixels, int frames, int height, int width, int quality, unsigned char* out,
                      long cap, int* sizes, void* workspace, size_t workspace_bytes, void* stream);
int kr_rgb8_to_jpeg(const unsigned char* rgb, int frames, int height, int width, int quality, unsigned char* out,
                    long cap, int* sizes, void* workspace, size_t workspace_bytes, void* stream);

#ifdef __cplusplus
}
#endif

/* The quantised attention tier (kr_sage_quantize / kr_sage_attn) is declared in its own header: its entry points and
 * kernels are one translation unit, kr_sage.cu, outside the API layer above. */
#include "krea_b200_sage.h"

#endif /* KREA_B200_H_ */
