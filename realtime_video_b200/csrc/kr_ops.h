// kr_ops.h — internal C++ interface between the kernels' host launchers and kr_api.cu.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stddef.h>

namespace kr {
const char* last_error();

enum GemmEpilogue : int {
  EPI_BIAS = 0,           // out = cast(acc + bias)
  EPI_BIAS_GELU = 1,      // out = cast(gelu_tanh(cast(acc + bias)))
  EPI_BIAS_GATE_RES = 2,  // out = cast(res + cast(cast(acc + bias) * gate[row / rows_per_gate]))
  EPI_BIAS_RES = 3,       // out = cast(res + cast(acc + bias))
  EPI_F32 = 4,            // out(fp32) = (acc + bias) * alpha
  EPI_MUL = 5,            // out = cast(cast(acc + bias) * res)   (gated FFN: fc1(x) * gelu(gate(x)), t5.py:138-140)
};

struct GemmParams {
  void* out;
  const void* bias;      // [N] 16-bit or nullptr
  const void* residual;  // [M, ldr] 16-bit (EPI_*_RES)
  const void* gate;      // [G, gate_stride] 16-bit (EPI_BIAS_GATE_RES)
  int M, N, K;
  int ldc;               // elements
  int ldr;               // elements
  int gate_stride;       // elements between consecutive gate rows
  int rows_per_gate;     // consecutive output rows sharing one gate row
  int row_offset;        // global index of local row 0 (sequence-parallel shards): gate row = (row + row_offset) / rows_per_gate
  float alpha;
  // optional second destination: output columns >= n_split go to out2 (column 0 = n_split),
  // e.g. the V third of the fused QKV projection straight into the KV-cache slot
  void* out2;
  int ldc2;
  int n_split;
};
// workspace (optional): gemm_sk_workspace_bytes() bytes, zero-filled once, private to the stream -> enables the
// stream-K kernel for shapes whose tile count leaves SMs idle (kr_gemm_sk.cu)
int gemm_tn(int dtype, int epi, const void* a, int lda, const void* w, int ldw, const GemmParams& p,
            cudaStream_t stream, void* workspace = nullptr, size_t workspace_bytes = 0);
int gemm_sk_tn(int dtype, int epi, const void* a, int lda, const void* w, int ldw, const GemmParams& p,
               void* workspace, size_t workspace_bytes, cudaStream_t stream);
size_t gemm_sk_workspace_bytes();
bool gemm_sk_preferred(int epi, int M, int N, int K);
// FP8 (e4m3) path, kr_gemm_fp8.cu: dynamic per-tensor activation quantisation + e4m3 wgmma GEMM.
// state: 2 floats of device memory [amax, dequant scale = amax / 448]; the GEMM reads state[1] as scale_a.
int fp8_quantize(const void* x, long ld, int rows, int cols, void* q, long ldq, float* state, cudaStream_t stream);
int gemm_fp8_tn(int epi, const void* a, int lda, const void* w, int ldw, const GemmParams& p, const float* scale_a,
                float scale_w, cudaStream_t stream);
// 2-CTA cluster variant (W multicast to both CTAs, 128x256 tile per CTA), kr_gemm2.cu; N % 256 == 0
int gemm2_tn(int dtype, int epi, const void* a, int lda, const void* w, int ldw, const GemmParams& p,
             cudaStream_t stream);
int gemm_plan(int epi, int M, int N, int K, bool have_workspace = false);   // 0 fixed-width kernel, 1 2-CTA cluster kernel, 2 stream-K, 3 runtime-width kernel
int gemm_flex_bn(int epi, int M, int N, int K);

struct AttnParams {
  void* out;           // [Lq, heads*128] 16-bit
  int ldo;             // elements
  int Lq, Lkv, heads;
  float scale_log2;    // softmax_scale * log2(e)
  // mask: 0 none; 1 block-causal: key k visible to query q iff lo(q) <= k < hi(q),
  //   hi(q) = min(Lkv, (q / block_len + 1) * block_len), lo(q) = window>0 ? max(0, hi'(q)-window) : 0
  int mask_mode;
  int block_len;       // tokens per causal block (frame_len * frames_per_block)
  int window;          // tokens (local_attn_size * frame_len) or 0
  // FlexAttention-path quirk (causal_model.py:316-348): q/k/v are zero-padded to a multiple of
  // 128 rows and queries of an incomplete last block also see those padded keys (score 0,
  // value 0).  pad_keys = number of such phantom keys after Lkv (0 = off).
  int pad_keys;
};
int attn_fwd(int dtype, const void* q, int ldq, const void* k, int ldk, const void* v, int ldv,
             const AttnParams& p, cudaStream_t stream);

// UMT5 self-attention (kr_t5attn.cu): head_dim 64, bf16, bias by (head, k - q), key mask, no scaling
struct T5AttnParams {
  void* out; int ldo;            // [L, heads*64] bf16
  int L, heads;
  const void* bias_delta;        // [heads, 2L-1] bf16: entry d = position bias of relative offset k - q = d - (L-1)
  const void* key_mask;          // [L] uint8 (1 = token, 0 = padding) or null
};
int t5_attn(const void* q, int ldq, const void* k, int ldk, const void* v, int ldv, const T5AttnParams& p,
            cudaStream_t stream);

int ln_modulate(const void* x, int ldx, void* out, int ldo, int rows, int D, float eps,
                const void* w, const void* b, const void* mod, int mod_rows, int shift_idx,
                int scale_idx, int rows_per_frame, int row_offset, cudaStream_t stream);

struct QkvPostParams {
  const uint16_t* q; const uint16_t* k; const uint16_t* v;
  int ldq, ldk, ldv;
  const uint16_t* wq; const uint16_t* wk;   // RMSNorm weights [D]
  uint16_t* q_out; int ldqo;                // [rows, D]
  uint16_t* k_out; int ldko;                // cache slot base (already offset to first row)
  uint16_t* v_out; int ldvo;
  const float2* rope;                       // may be null -> no rotation
  int D, head_dim;
  int grid_h, grid_w, start_frame;
  int row_offset;                           // global token index of local row 0
  float eps;
  // sequence-parallel exchange fused into the store (kr_comm, SURVEY.md 8e option 3): peer_cols > 0 sends the
  // columns [d*peer_cols, (d+1)*peer_cols) (= the heads owned by rank d) of every row to rank d's buffers over
  // NVLink peer memory instead of the local q_out / k_out / v_out.  The *_peer pointers address THIS rank's first
  // row inside each destination buffer (row pitch ldqo / ldko / ldvo).
  int peer_cols;
  uint16_t* q_peer[8]; uint16_t* k_peer[8]; uint16_t* v_peer[8];
};
int qkv_post(const QkvPostParams& p, int rows, cudaStream_t stream);
// rows [r*rows_per_peer, (r+1)*rows_per_peer) of src [rows, cols] -> peer r's buffer dst_peer[r] (pitch ld_dst):
// the attention output of MY heads scattered back to the ranks that own the token rows
int p2p_scatter_rows(const void* src, int ld_src, void* const* dst_peer, int ld_dst, int rows, int cols,
                     int rows_per_peer, int world, cudaStream_t stream);
// in-place downward shift of cache rows (16-bit elements): [src_row, src_row+rows) -> [dst_row, ...), dst_row <= src_row
int kv_roll(void* cache, int ld, int width, int dst_row, int src_row, int rows, cudaStream_t stream);
int rmsnorm_rows(const void* x, int ldx, void* out, int ldo, const void* w, int rows, int D,
                 float eps, cudaStream_t stream);
int add_modulation(const void* modulation, const void* e0, int lde0_frame, void* out, int frames,
                   int mod_rows, int D, cudaStream_t stream);
int activation(const void* x, void* y, size_t n, int kind, cudaStream_t stream);
int patchify(const void* x, long sc, long sf, long sh, long sw, void* out, int C, int F, int H,
             int W, cudaStream_t stream);
int unpatchify_x0(const void* head_out, int ldh, const void* xt, const double* sigma, void* flow,
                  void* x0, int C, int F, int H, int W, cudaStream_t stream);
struct ConvParams {
  int T, H, W;          // output frames / height / width
  int TW, TH;           // spatial tile, TW * TH == 128
  int KT, KH, KW;       // taps
  int cout;             // real output channels (<= N)
  void* out_raw; long raw_pix, raw_frame;       // 16-bit; element strides per pixel / frame
  void* out_norm; long norm_pix, norm_frame;    // 16-bit, RMS_norm*gamma -> SiLU
  float* out_pix;                               // fp32 [T, cout, H, W], clamp(-1, 1)
  const void* bias;                             // [cout] 16-bit or null
  const void* residual; long res_pix, res_frame;
  const void* gamma;                            // [cout] for out_norm
  float norm_scale;                             // sqrt(C)
  int sub2;                                     // 1: keep only odd (h, w) outputs, compacted to H/2 x W/2
};
int vae_conv(int dtype, int cin, int n, const void* in, int t_in, const void* wgt, int w_rows,
             const ConvParams& p, cudaStream_t stream);
int vae_rmsnorm_silu(int dtype, const void* x, void* y, const void* gamma, long pixels, int C,
                     int do_silu, cudaStream_t stream);
int vae_upsample2x(const void* in, void* out, int T, int H, int W, int C, cudaStream_t stream);
int vae_scale_input(int dtype, const void* z, long zt, long zc, long zh, long zw, const void* mean,
                    const void* inv_std, const void* w2, const void* b2, void* out, int T, int H,
                    int W, cudaStream_t stream);
int softmax_rows(int dtype, const float* s, long ld, void* pout, long ldo, int rows, int cols,
                 cudaStream_t stream);
int frames_to_rgb8(const float* pixels, uint8_t* rgb, int frames, int height, int width, cudaStream_t stream);
// device-side baseline JPEG (kr_jpeg.cu): byte-identical to Pillow's save(format='JPEG', quality=q) of each frame.
// src_kind 0: fp32 planar [frames, 3, H, W] in [-1, 1] (normalised like frames_to_rgb8); 1: RGB bytes [frames, H, W, 3].
// out [frames, cap] bytes, sizes[frames] = bytes of each file (negative: -(bytes needed), the file did not fit in cap).
size_t jpeg_workspace_bytes(int frames, int height, int width);
int frames_to_jpeg(const void* src, int src_kind, int frames, int height, int width, int quality, uint8_t* out,
                   long cap, int* sizes, void* workspace, size_t workspace_bytes, cudaStream_t stream);
}  // namespace kr
