// Launch wrappers shared by engine.cu and the kernel-level C-ABI entry points.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>

namespace stk {

// Epilogue description common to the fp32-FFMA and the tensor-core GEMMs:  y = act(A W^T + bias)
//   mode EPI_STORE : out[orow, n] = y (+ addtab[(m % add_period) * add_ld + n])
//   mode EPI_RESID : out[orow, n] = resid[orow, n] + gate[(m % gate_period) * gate_ld + n] * y   (gate NULL -> 1)
//   mode EPI_SPLIT : out_hi/out_lo[orow, n] = bf16 split of y            (tensor-core A-operand planes)
// Row remap (joint attention buffer):  orow = (m / rpb_in) * rpb_out + row_off + m % rpb_in   (rpb_in == 0: orow = m)
// Token-range plan (plan != NULL, QKV epilogues only): per image b an (a_b, c_b) pair -- its live context rows are stream rows
// [a_b, a_b + c_b).  The image's slot of rpb_out rows then holds its live context rows, its image rows, and last its other
// context rows (computed, never visible): plan_ctx = 1 (context stream, rpb_in = Kc): row r -> r - a_b when live, else the tail;
// plan_ctx = 0 (image stream, rpb_in = N): row r -> c_b + r.
// Per-row indices (packed step calls, NULL otherwise): tab_rows[m] replaces m % period as the gate / addtab row, and row_map[m]
// replaces the remap above as the output row.
// e4m3 operands (NSPLIT_E4M3): A and W hold e4m3 codes with one fp32 scale per row (per GEMM row of A, per output channel of W),
// and y = act(fma(acc, s_a[m] * s_w[n], bias)) -- the product s_a[m] * s_w[n] rounded to fp32 first, then one fma -- before the
// mode above.  m is the GEMM row before any remap (plan, row_map, rpb_in), so the scale travels with the A row it belongs to.
//
// Quantization contract (per row x of K fp32 values; launch_quant_e4m3_rows, the e4m3 mode of launch_ln_mod_pair):
//   amax   = max |x_i|, NaN when the row holds a NaN (a NaN-propagating max, never fmaxf)
//   inv    = __fdiv_rn(448, amax), scale = __fdiv_rn(amax, 448); amax == 0: inv = 0, scale = 0 (all codes 0)
//   code_i = cvt.rn.satfinite.e4m3(__fmul_rn(x_i, inv))
// A non-finite amax is not sanitised: the row comes out non-finite downstream.
enum EpiMode { EPI_STORE = 0, EPI_RESID = 1, EPI_SPLIT = 2 };
constexpr int NSPLIT_E4M3 = 4;           // launch_gemm_tc* nsplit value of the e4m3 single-pass mode
struct Epilogue {
  int mode = EPI_STORE;
  int act = 0;
  const float* bias = nullptr;
  float* out = nullptr;
  int64_t ldo = 0;
  const float* resid = nullptr;          // EPI_RESID (may alias out)
  const float* gate = nullptr;
  int64_t gate_ld = 0;
  int gate_period = 1;
  const float* addtab = nullptr;         // EPI_STORE
  int64_t add_ld = 0;
  int add_period = 1;
  __nv_bfloat16* out_hi = nullptr;       // EPI_SPLIT
  __nv_bfloat16* out_lo = nullptr;       // may be NULL (single-pass bf16); must be NULL with fp16
  int rpb_in = 0, rpb_out = 0, row_off = 0;
  int fp16 = 0;                          // EPI_SPLIT: planes hold IEEE half (single-pass fp16 mode) instead of bf16
  const int* plan = nullptr;             // token-range plan of this step, [B][2] int32 (a, c); NULL: plain remap
  int plan_ctx = 0;
  const int* tab_rows = nullptr;         // [M] gate (EPI_RESID) / addtab (EPI_STORE) row of GEMM row m
  const int* row_map = nullptr;          // [M] output row of GEMM row m
  const float* s_a = nullptr;            // e4m3 only: [M] row scales of A
  const float* s_w = nullptr;            // e4m3 only: [N] row scales of W (per output channel)
};
// slot row of stream row r of an image with plan pair (a, c); n_img = image rows per slot
__host__ __device__ __forceinline__ int plan_slot_row(int r, int a, int c, int n_img, bool ctx) {
  if (!ctx) return c + r;
  return r < a ? c + n_img + r : (r < a + c ? r - a : n_img + r);
}
// Host-side checks of an epilogue that both GEMM launchers make before any launch (SELFTOK_ERR_BAD_ARG on failure): the
// pointers its mode needs are set, periods are >= 1, the fp32 bases (bias, out, resid, gate, addtab) are 8-byte aligned and
// the 16-bit plane bases 4-byte aligned (the wgmma epilogue moves column pairs), and the fp16 split mode has no out_lo plane.
int check_epilogue(const Epilogue& ep, const char* who);

// ---- fp32 FFMA kernels (kernels_simt.cu) ---------------------------------------------------------------------
int launch_linear_f32(const float* A, int64_t lda, const float* W, int64_t ldw, int64_t M, int N, int K,
                      const Epilogue& ep, cudaStream_t s);
// LN (no affine, eps) + modulate; writes fp32 and/or bf16 planes.  shift/scale NULL -> plain LN.  rows != NULL: row m uses
// table row rows[m] instead of m % period.
int launch_ln_mod(const float* x, int64_t ldx, const float* shift, const float* scale, int64_t ld_mod, int period,
                  float* out_f32, __nv_bfloat16* out_hi, __nv_bfloat16* out_lo, int64_t ldo, int64_t M, int D,
                  float eps, cudaStream_t s, int fp16 = 0, const int* rows = nullptr);
// Two LN + modulate problems (the context- and the image-row pass of one MMDiT layer stage) in ONE launch, 16-bit plane
// output (IEEE half when fp16, else bf16 hi [+ lo]).  period > 1: rows are [image][position] with a per-position table row
// (M must be a multiple of period); period <= 1: one table row for all rows.
struct LnProblem {
  const float* x = nullptr;          // [M, D] fp32, contiguous rows
  const float* shift = nullptr;
  const float* scale = nullptr;
  int64_t ld_mod = 0;
  int period = 1;
  __nv_bfloat16* out_hi = nullptr;
  __nv_bfloat16* out_lo = nullptr;
  int64_t M = 0;
  const int* rows = nullptr;         // [M] table row of every row (packed step calls; then for every problem of the launch)
  float* out_scale = nullptr;        // e4m3 output: out_hi holds [M, D] e4m3 codes (D bytes per row) and this [M] fp32 row
                                     // scales (quantization contract above); then for every problem of the launch
  int imgs = 0;                      // filled by the launcher
};
int launch_ln_mod_pair(const LnProblem* probs, int n, int D, float eps, cudaStream_t s, int fp16);
// Attention output routing: query rows [0,split) of every image go to the compact buffer A ([B*split, ld]),
// rows [split,Sq) to buffer B ([B*(Sq-split), ld]).  split == Sq -> everything in A.  Each buffer is fp32 and/or
// bf16 hi(/lo) planes (NULL pointers are skipped).
struct AttnOut {
  float* f32_a = nullptr; __nv_bfloat16* hi_a = nullptr; __nv_bfloat16* lo_a = nullptr;
  float* f32_b = nullptr; __nv_bfloat16* hi_b = nullptr; __nv_bfloat16* lo_b = nullptr;
  int split = 0;
  int64_t ld = 0;
  int fp16 = 0;                          // planes hold IEEE half instead of bf16
};
// Token-range plan of the joint attention (plan != NULL): image b's slot of S rows holds c_b live context rows, n_img image rows,
// then its S - c_b - n_img other context rows (see Epilogue).  Image rows see keys [0, c_b + n_img); context rows the same, or
// [0, c_b) with ctx_self; a row with no visible key writes 0.  route != 0: output rows go back to the streams (inverse of the
// QKV remap; AttnOut.split = Kc = S - n_img), else AttnOut's own routing applies.
// packed: the plan pairs are (off_b, c_b) of a packed context stream (selftok_decode_step): slot row r < c_b goes to context row
// off_b + r, image rows to b * n_img + r - c_b; rows >= c_b + n_img hold nothing and are not written.
struct AttnPlan {
  const int* plan = nullptr;             // [B][2] int32 (a, c) of this step
  int n_img = 0;
  int ctx_self = 0;
  int route = 1;
  int packed = 0;
};
// stream row of slot row `row` of an image with plan pair (a, c); ctx = whether it is a context row
__host__ __device__ __forceinline__ int plan_stream_row(int row, int a, int c, int n_img, bool& ctx) {
  if (row < c) { ctx = true; return a + row; }
  if (row < c + n_img) { ctx = false; return row - c; }
  ctx = true;
  const int t = row - c - n_img;
  return t < a ? t : t + c;
}
// softmax(q k^T / sqrt(hd)) v in fp32.  q rows: q + b*q_bs + s*q_ld + h*hd; keys = segment 1 (S1 rows) followed by
// segment 2 (S2 rows).  Rows < ctx_rows only see keys < ctx_keys (renderer rule); ctx_rows = 0 -> dense.
int launch_attention_f32(const float* q, int64_t q_ld, int64_t q_bs, const float* k1, const float* v1, int64_t kv1_ld,
                         int64_t kv1_bs, int S1, const float* k2, const float* v2, int64_t kv2_ld, int64_t kv2_bs,
                         int S2, const AttnOut& out, int B, int Sq, int H, int hd, int ctx_rows, int ctx_keys,
                         cudaStream_t s, const AttnPlan& plan = AttnPlan());
// Fused VQ: project_in + l2norm + argmax over the codebook + gather + final_layer_norm3.
int launch_vq(const float* z, int64_t R, int Q, const float* w_in, const float* b_in, const float* codebook,
              const float* codebook_t, int n_codes, int code_dim, const float* ln_w, const float* ln_b,
              int64_t* ids, float* outs_q, cudaStream_t s);
// ids outside [0, n_codes): row poisoned with NaN and counted in *bad_ids (may be NULL).  range != NULL: [R / K][2] int32 (lo, hi)
// token windows; positions outside an image's window are not read and write a zero row.  gather != NULL: output row m reads
// ids[gather[m]] (packed context stream).
int launch_lookup_ln3(const int64_t* ids, int64_t R, const float* codebook, int n_codes, int code_dim,
                      const float* ln_w, const float* ln_b, float* outs_q, int* bad_ids, cudaStream_t s,
                      const int* range = nullptr, int K = 0, const int* gather = nullptr);
// [B,C,Hh,Ww] latents -> [B*(Hh/p)*(Ww/p), C*p*p] patch rows ((c,ph,pw) fastest-last, Conv2d weight order)
int launch_patchify(const float* x, float* out, int B, int C, int Hh, int Ww, int p, cudaStream_t s);
// x_lat[b,c,h*p+ph,w*p+pw] = x_in[...] - dt * o[b, h*gw+w, (ph*p+pw)*C + c]   (unpatchify of a gh x gw patch grid + Euler; dt = -1
// & x_in NULL: plain unpatchify).  o_u != NULL (guided sampler): v = o_u + cfg_scale * (o - o_u) first.  dt_img / scale_img != NULL:
// device [B] per-image dt and cfg_scale instead of the scalars
int launch_unpatchify_axpy(const float* o, const float* x_in, float* x_out, float dt, int B, int C, int gh, int gw, int p,
                           cudaStream_t s, const float* o_u = nullptr, float cfg_scale = 1.f, const float* dt_img = nullptr,
                           const float* scale_img = nullptr);
// Per-row maps of a packed step call from its per-image block blk = [B][2] (off_b, c_b) | [B] lo_b | [B] step_b: context row
// m = off_b + r (r < c_b) gets ctx_tok = b K + lo_b + r, ctx_pos = lo_b + r, ctx_step = step_b, ctx_dst = b S + r; image row
// b N + r gets x_step = step_b.
int launch_expand_packed(const int* blk, int B, int K, int N, int S, int* ctx_tok, int* ctx_pos, int* ctx_step, int* ctx_dst,
                         int* x_step, cudaStream_t s);
// zero the rows [c_b + n_img, S) of slot b up to its next 64-row boundary (pair = [B][2] (off_b, c_b)) in a [B*S] x row_bytes buffer
int launch_zero_slot_tails(const int* pair, int B, int S, int n_img, void* buf, int64_t row_bytes, cudaStream_t s);
// e4m3 codes [M, K] (K bytes per row) + fp32 scales [M] of fp32 rows x [M, K] under the quantization contract above
int launch_quant_e4m3_rows(const float* x, int64_t M, int K, uint8_t* codes, float* scales, cudaStream_t s);
int launch_transpose(const float* in, float* out, int rows, int cols, cudaStream_t s);
int launch_split_bf16(const float* in, __nv_bfloat16* hi, __nv_bfloat16* lo, int64_t n, cudaStream_t s, int fp16 = 0);
// out[b, r, :] = src[r, :] for b in 0..B-1 (broadcast rows), optionally + add[r,:]
int launch_bcast_rows(const float* src, const float* add, float* out, int B, int64_t rows, int64_t cols, cudaStream_t s);
// window [top, top + gh) x [left, left + gw) of a [max,max,D] positional grid -> [gh,gw,D]
int launch_crop_pos(const float* pos, float* out, int max_size, int gh, int gw, int top, int left, int D, cudaStream_t s);
int launch_copy_rows(const float* src, int64_t src_bs, float* dst, int64_t dst_bs, int B, int64_t n_per_batch, cudaStream_t s);

// ---- wgmma GEMM (gemm_tc.cu) ----------------------------------------------------------------------------------
// A planes [M,K] bf16 row-major (lo NULL iff nsplit == 1), W planes [N,K] bf16 row-major.
// fp16 != 0: operands are IEEE half planes (nsplit must be 1).
// nsplit == NSPLIT_E4M3: A_hi / W_hi hold e4m3 codes (K bytes per row, K % 16 == 0), lo planes unused, and every problem's
// epilogue carries both row-scale arrays s_a / s_w (no other mode may carry them, so one launch never mixes operand types).
// No convolution in this mode.
int launch_gemm_tc(const __nv_bfloat16* A_hi, const __nv_bfloat16* A_lo, const __nv_bfloat16* W_hi,
                   const __nv_bfloat16* W_lo, int64_t M, int N, int K, int nsplit, const Epilogue& ep,
                   cudaStream_t s, int fp16 = 0);
struct TcProblem {
  const __nv_bfloat16* A_hi; const __nv_bfloat16* A_lo; const __nv_bfloat16* W_hi; const __nv_bfloat16* W_lo;
  int64_t M; int N; int K;
  Epilogue ep;
  // conv_C > 0: implicit-GEMM 3x3 convolution (stride 1, pad 1): A planes are NHWC activations [M / (H W), H, W, C], W planes
  // [N, 9 C] with K index = (ky * 3 + kx) * C + c, M = output pixels, K = 9 C.  conv_stride == 2: A planes are the four
  // polyphase components of the input [images * 4, H_out, W_out, C] (pad right / bottom), conv_H / conv_W = output dims.
  // conv_edge == 0: the 128-pixel A tiles must tile each image exactly (part of a row, whole rows, or whole images; stride 2: not
  // whole images); != 0: any H, W -- tiles then overhang the right / bottom edge and their outside rows are dropped.
  int conv_C = 0, conv_H = 0, conv_W = 0, conv_stride = 1, conv_edge = 0;
};
// one launch for one or two independent problems of the same operand type
int launch_gemm_tc_grouped(const TcProblem* probs, int n, int nsplit, cudaStream_t s, int fp16 = 0);
// the host-side checks launch_gemm_tc_grouped makes of each problem (no CUDA call)
int check_gemm_tc_problem(const TcProblem& q, int nsplit, int fp16);
int gemm_tc_init();   // resolves cuTensorMapEncodeTiled, sets smem attributes; idempotent
void gemm_tc_set_ctas(int n);   // 2 (default): two-CTA clusters sharing the W tile by TMA multicast; 1: one CTA per tile

// ---- tensor-core attention -----------------------------------------------------------------------------------
// qkv planes: packed 16-bit [B,S,3,H,64] (hi, and lo for the split mode), written by the QKV GEMM epilogue
// wgmma attention (attn_tc5.cu): single-pass 16-bit operands (fp16 != 0: IEEE half, else bf16), or -- with the lo
// planes given -- the fp32-faithful split-bf16 mode (three MMAs per product, P split in registers)
int launch_attention_tc5(const __nv_bfloat16* qkv16, int B, int S, int H, int ctx_rows, int ctx_keys, const AttnOut& out,
                         cudaStream_t s, int fp16, const __nv_bfloat16* qkv_lo = nullptr, const AttnPlan& plan = AttnPlan());

}  // namespace stk
