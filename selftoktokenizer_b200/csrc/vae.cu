// SD3 16-channel VAE on the device (SURVEY 8f rank 1): the steps either side of the token path in SelftokPipeline --
// `self.vae.encode(images)[0].mode()` before the encoder (SelftokPipeline.py:215) and `self.vae.decode(pred_x0_out)` after the
// sampler / renderer (:288,316).  Architecture as vendored in the reference tree (mimogpt/models/selftok/sd3/sd3_impls.py):
//   VAEDecoder (:388-444)  conv_in -> mid (ResnetBlock, AttnBlock, ResnetBlock) -> 4 levels of 3 ResnetBlocks (+ nearest-2x
//                          Upsample + conv) -> GroupNorm -> SiLU -> conv_out
//   VAEEncoder (:314-385)  conv_in -> 4 levels of 2 ResnetBlocks (+ Downsample: zero pad right / bottom, 3x3 stride-2 conv) -> mid
//                          -> GroupNorm -> SiLU -> conv_out (mean | logvar)
//
//   layout        NHWC.  The residual stream is fp32 [B, H, W, C]; every convolution / 1x1 projection reads its input as
//                 16-bit operand planes (bf16 hi + lo: the fp32-faithful split mode, three MMAs per product) written by the
//                 kernel that produces it (GroupNorm+SiLU, nearest upsample, softmax, GEMM epilogues).
//   3x3 convs     implicit GEMM on the wgmma kernel of gemm_tc.cu: A tile = 4-D TMA box of the NHWC planes shifted by
//                 the tap offset (the TMA unit's out-of-bounds zero fill IS the padding), K = 9 C, weights repacked to
//                 [Cout, (ky, kx), Cin]; bias and the residual add (x + h, ResnetBlock.forward :256) in the GEMM epilogue.
//                 Any image size: where no 128-pixel box tiles the image exactly, the boxes overhang its right / bottom edge.
//   stride-2 conv the input is written as its four polyphase planes (space_to_depth_planes_kernel); every tap is then a
//                 unit-stride box of one phase plane, and the zero fill past the last row / column is the one-sided padding.
//   GroupNorm     32 groups, eps 1e-6, affine; two deterministic passes (per-chunk partial sums in a fixed order, then
//                 normalise + SiLU + plane output) -- no atomics.
//   attention     the single-head 512-channel block of the middle (AttnBlock.forward :276-287): per image S = Q K^T and
//                 O = P V on the same wgmma GEMM (V^T comes straight out of its projection GEMM with the operands swapped; its
//                 bias is added after P V, rows of P sum to one), row softmax in fp32.
//
// Weights under the reference's own SDVAE key names ("decoder.up.3.block.0.conv1.weight", ...).
#include "../../include/selftok_b200.h"
#include "common.cuh"
#include "kernels.h"

#include <math.h>
#include <string>
#include <unordered_map>
#include <vector>

using namespace stk;
typedef __nv_bfloat16 bf16;

namespace {

// ------------------------------------------------------------------------------------------------ kernels
// z [B, Cz, h, w] fp32 NCHW -> bf16 hi / lo planes [B, h, w, 64] NHWC (channels >= Cz are zero: the 16-channel conv_in runs
// through the same 64-channel-chunk implicit GEMM, its weights are zero-padded to match)
__global__ void latent_to_planes_kernel(const float* __restrict__ z, bf16* __restrict__ hi, bf16* __restrict__ lo, int B, int Cz, int h, int w) {
  const int64_t total = (int64_t)B * h * w * 64;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % 64);
    const int64_t pix = i / 64;
    const int x = (int)(pix % w), y = (int)((pix / w) % h), b = (int)(pix / ((int64_t)w * h));
    const float v = c < Cz ? z[(((int64_t)b * Cz + c) * h + y) * w + x] : 0.f;
    uint16_t a, r;
    split16(v, false, a, r);
    reinterpret_cast<uint16_t*>(hi)[i] = a;
    reinterpret_cast<uint16_t*>(lo)[i] = r;
  }
}

// GroupNorm statistics, pass 1: per (image, pixel chunk) partial (sum, sum of squares) of every group.  A float4 of channels
// never straddles two groups (channels per group is a multiple of 4 for C in {128, 256, 512}).
constexpr int GN_GROUPS = 32;
__global__ void __launch_bounds__(256) gn_partial_kernel(const float* __restrict__ x, float* __restrict__ part, int HW, int C, int chunk_pix) {
  __shared__ float red_s[256], red_q[256];
  const int b = blockIdx.y, chunk = blockIdx.x, nchunk = gridDim.x;
  const int c4n = C >> 2, cpg = C / GN_GROUPS;
  const int p0 = chunk * chunk_pix, p1 = min(HW, p0 + chunk_pix);
  const float4* xb = reinterpret_cast<const float4*>(x + (int64_t)b * HW * C);
  const int lane_c4 = threadIdx.x % c4n, pstep = blockDim.x / c4n;              // blockDim.x is a multiple of c4n (32 / 64 / 128)
  float s = 0.f, q = 0.f;
  for (int p = p0 + threadIdx.x / c4n; p < p1; p += pstep) {
    const float4 v = xb[(int64_t)p * c4n + lane_c4];
    s += (v.x + v.y) + (v.z + v.w);
    q += (v.x * v.x + v.y * v.y) + (v.z * v.z + v.w * v.w);
  }
  red_s[threadIdx.x] = s;
  red_q[threadIdx.x] = q;
  __syncthreads();
  if (threadIdx.x < GN_GROUPS) {                  // fixed-order combine of the block's 256 partials: bit-reproducible, no atomics
    const int g = threadIdx.x;
    float ts = 0.f, tq = 0.f;
    for (int t = 0; t < 256; ++t)
      if (((t % c4n) * 4) / cpg == g) { ts += red_s[t]; tq += red_q[t]; }
    part[(((int64_t)b * nchunk + chunk) * 2 + 0) * GN_GROUPS + g] = ts;
    part[(((int64_t)b * nchunk + chunk) * 2 + 1) * GN_GROUPS + g] = tq;
  }
}
// pass 2: (mean, rstd) per (image, group) in double over the chunk partials, fixed order
__global__ void gn_finalize_kernel(const float* __restrict__ part, float* __restrict__ stats, int nchunk, int64_t n_per_group, float eps) {
  const int b = blockIdx.x, g = threadIdx.x;
  if (g >= GN_GROUPS) return;
  double s = 0.0, q = 0.0;
  for (int c = 0; c < nchunk; ++c) {
    s += (double)part[(((int64_t)b * nchunk + c) * 2 + 0) * GN_GROUPS + g];
    q += (double)part[(((int64_t)b * nchunk + c) * 2 + 1) * GN_GROUPS + g];
  }
  const double mean = s / (double)n_per_group;
  const double var = fmax(q / (double)n_per_group - mean * mean, 0.0);
  stats[((int64_t)b * GN_GROUPS + g) * 2 + 0] = (float)mean;
  stats[((int64_t)b * GN_GROUPS + g) * 2 + 1] = (float)(1.0 / sqrt(var + (double)eps));
}
// pass 3: y = (x - mean) * rstd * gamma + beta, optional SiLU, -> bf16 hi / lo planes (same NHWC shape)
template <bool SILU>
__global__ void __launch_bounds__(256) gn_apply_kernel(const float* __restrict__ x, const float* __restrict__ stats, const float* __restrict__ gamma,
                                                       const float* __restrict__ beta, bf16* __restrict__ hi, bf16* __restrict__ lo,
                                                       int64_t HW, int C, int64_t total4) {
  const int c4n = C >> 2, cpg = C / GN_GROUPS;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total4; i += (int64_t)gridDim.x * blockDim.x) {
    const int c4 = (int)(i % c4n);
    const int64_t b = i / ((int64_t)c4n * HW);
    const int g = (c4 * 4) / cpg;
    const float mean = stats[(b * GN_GROUPS + g) * 2], rstd = stats[(b * GN_GROUPS + g) * 2 + 1];
    const float4 v = reinterpret_cast<const float4*>(x)[i];
    const float4 ga = reinterpret_cast<const float4*>(gamma)[c4], be = reinterpret_cast<const float4*>(beta)[c4];
    float y[4] = {(v.x - mean) * rstd * ga.x + be.x, (v.y - mean) * rstd * ga.y + be.y, (v.z - mean) * rstd * ga.z + be.z,
                  (v.w - mean) * rstd * ga.w + be.w};
    if (SILU) {
#pragma unroll
      for (int k = 0; k < 4; ++k) y[k] = silu(y[k]);
    }
    const uint32_t p0 = pack2_sat16(y[0], y[1], false), p1 = pack2_sat16(y[2], y[3], false);
    reinterpret_cast<uint2*>(hi)[i] = make_uint2(p0, p1);
    reinterpret_cast<uint2*>(lo)[i] = make_uint2(pack2_resid_bf16(y[0], y[1], p0), pack2_resid_bf16(y[2], y[3], p1));
  }
}
// nearest-neighbour 2x upsample (F.interpolate(scale_factor=2, mode="nearest"), sd3_impls.py:311) of the fp32 NHWC stream into
// the operand planes of the convolution that follows it
__global__ void __launch_bounds__(256) upsample2x_planes_kernel(const float* __restrict__ x, bf16* __restrict__ hi, bf16* __restrict__ lo, int B, int H, int W,
                                                                int C) {
  const int c4n = C >> 2, H2 = 2 * H, W2 = 2 * W;
  const int64_t total4 = (int64_t)B * H2 * W2 * c4n;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total4; i += (int64_t)gridDim.x * blockDim.x) {
    const int c4 = (int)(i % c4n);
    const int64_t pix = i / c4n;
    const int x2 = (int)(pix % W2), y2 = (int)((pix / W2) % H2);
    const int64_t b = pix / ((int64_t)W2 * H2);
    const float4 v = reinterpret_cast<const float4*>(x)[((b * H + (y2 >> 1)) * W + (x2 >> 1)) * c4n + c4];
    const uint32_t p0 = pack2_sat16(v.x, v.y, false), p1 = pack2_sat16(v.z, v.w, false);
    reinterpret_cast<uint2*>(hi)[i] = make_uint2(p0, p1);
    reinterpret_cast<uint2*>(lo)[i] = make_uint2(pack2_resid_bf16(v.x, v.y, p0), pack2_resid_bf16(v.z, v.w, p1));
  }
}
// Downsample input: fp32 NHWC [B, H, W, C] -> polyphase operand planes [B * 4 + (py * 2 + px)][H / 2][W / 2][C] with
// phase(py, px)[y][x] = in[2y + py][2x + px] (the A operand layout of the stride-2 implicit GEMM, gemm_tc.cu)
__global__ void __launch_bounds__(256) space_to_depth_planes_kernel(const float* __restrict__ x, bf16* __restrict__ hi, bf16* __restrict__ lo, int B, int H,
                                                                    int W, int C) {
  const int c4n = C >> 2, Ho = H >> 1, Wo = W >> 1;
  const int64_t total4 = (int64_t)B * H * W * c4n;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total4; i += (int64_t)gridDim.x * blockDim.x) {
    const int c4 = (int)(i % c4n);
    const int64_t pix = i / c4n;                                   // output order: (b, phase, yo, xo)
    const int xo = (int)(pix % Wo), yo = (int)((pix / Wo) % Ho);
    const int ph = (int)((pix / ((int64_t)Wo * Ho)) & 3);
    const int64_t b = pix / ((int64_t)Wo * Ho * 4);
    const float4 v = reinterpret_cast<const float4*>(x)[((b * H + (2 * yo + (ph >> 1))) * W + (2 * xo + (ph & 1))) * c4n + c4];
    const uint32_t p0 = pack2_sat16(v.x, v.y, false), p1 = pack2_sat16(v.z, v.w, false);
    reinterpret_cast<uint2*>(hi)[i] = make_uint2(p0, p1);
    reinterpret_cast<uint2*>(lo)[i] = make_uint2(pack2_resid_bf16(v.x, v.y, p0), pack2_resid_bf16(v.z, v.w, p1));
  }
}
// row softmax of the attention scores: P = softmax(S * scale) over the n real columns of S [rows, ld] fp32 -> bf16 hi / lo
// planes [rows, ld] whose columns [n, ld) (the pad to a 16-byte row pitch) are zero; one warp per row
__global__ void __launch_bounds__(256) softmax_rows_kernel(const float* __restrict__ s, bf16* __restrict__ hi, bf16* __restrict__ lo, int64_t rows, int n,
                                                           int ld, float scale) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const float* sr = s + row * ld;
  float mx = -INFINITY;
  for (int i = lane; i < n; i += 32) mx = fmaxf(mx, sr[i]);
  mx = warp_max(mx) * scale;
  float sum = 0.f;
  for (int i = lane; i < n; i += 32) sum += expf(sr[i] * scale - mx);
  const float inv = 1.0f / warp_sum(sum);
  for (int i = lane; i < n; i += 32) {
    const float p = expf(sr[i] * scale - mx) * inv;
    uint16_t a, r;
    split16(p, false, a, r);
    reinterpret_cast<uint16_t*>(hi)[row * ld + i] = a;
    reinterpret_cast<uint16_t*>(lo)[row * ld + i] = r;
  }
  for (int i = n + lane; i < ld; i += 32) {
    reinterpret_cast<uint16_t*>(hi)[row * ld + i] = 0;
    reinterpret_cast<uint16_t*>(lo)[row * ld + i] = 0;
  }
}
// conv_out result [B, H, W, 4] fp32 NHWC (3 real channels) -> [B, 3, H, W] NCHW, optionally norm_ip(., -1, 1) (clamp to [-1, 1],
// rescale to [0, 1]; SelftokPipeline.py:135-137,293)
__global__ void nhwc4_to_nchw3_kernel(const float* __restrict__ x, float* __restrict__ out, int B, int HW, int norm) {
  const int64_t total = (int64_t)B * 3 * HW;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t p = i % HW;
    const int c = (int)((i / HW) % 3);
    const int64_t b = i / ((int64_t)3 * HW);
    float v = x[(b * HW + p) * 4 + c];
    if (norm) v = (fminf(fmaxf(v, -1.f), 1.f) + 1.f) * 0.5f;
    out[i] = v;
  }
}
// channels [c0, c0 + Cn) of an fp32 NHWC tensor [B, HW, Cs] -> NCHW [B, Cn, HW] (the mean / logvar halves of the encoder's conv_out)
__global__ void nhwc_to_nchw_kernel(const float* __restrict__ x, float* __restrict__ out, int B, int HW, int Cs, int c0, int Cn) {
  const int64_t total = (int64_t)B * Cn * HW;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t p = i % HW;
    const int c = (int)((i / HW) % Cn);
    const int64_t b = i / ((int64_t)Cn * HW);
    out[i] = x[(b * HW + p) * Cs + c0 + c];
  }
}
// conv weight [Cout, Cin, kh, kw] fp32 -> GEMM operand [Npad, kh*kw*Cpad] fp32 with K index (ky*kw + kx) * Cpad + c (zero padding)
__global__ void repack_conv_kernel(const float* __restrict__ w, float* __restrict__ out, int Cout, int Cin, int taps, int Npad, int Cpad) {
  const int64_t total = (int64_t)Npad * taps * Cpad;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % Cpad), t = (int)((i / Cpad) % taps), n = (int)(i / ((int64_t)Cpad * taps));
    out[i] = (n < Cout && c < Cin) ? w[((int64_t)n * Cin + c) * taps + t] : 0.f;
  }
}

inline unsigned blocks_for(int64_t n, int per = 256, int64_t cap = 132 * 32) { return (unsigned)std::max<int64_t>(1, std::min<int64_t>((n + per - 1) / per, cap)); }

}  // namespace

// ------------------------------------------------------------------------------------------------ handle
struct VaeW {            // one convolution / projection: packed planes + fp32 bias
  bf16 *hi = nullptr, *lo = nullptr;
  float* bias = nullptr;
  int N = 0, Npad = 0, K = 0, Cpad = 0, taps = 1;
};
struct selftok_vae {
  int device = 0, ch = 128;
  int mult[4] = {1, 2, 4, 4};
  bool finalized = false, has_dec = false, has_enc = false;
  std::unordered_map<std::string, std::pair<float*, std::vector<int64_t>>> raw;      // loaded fp32 tensors (freed at finalize unless norm / bias)
  std::unordered_map<std::string, VaeW> conv;
  std::vector<void*> allocs;
  // workspace (sized for the last batch / latent size that did not fit the one before)
  int wsB = 0, wsh = 0, wsw = 0;
  std::vector<void*> ws_allocs;
  float *xa = nullptr, *xb = nullptr, *sc = nullptr, *part = nullptr, *stats = nullptr, *s_attn = nullptr, *out4 = nullptr;
  bf16 *p_hi = nullptr, *p_lo = nullptr, *q_hi = nullptr, *q_lo = nullptr, *k_hi = nullptr, *k_lo = nullptr, *vt_hi = nullptr, *vt_lo = nullptr,
       *pr_hi = nullptr, *pr_lo = nullptr, *o_hi = nullptr, *o_lo = nullptr;
  int64_t bytes = 0;
};

#define VAE_CUDA(expr) STK_CUDA(expr)

static int v_alloc(selftok_vae* v, std::vector<void*>& pool, void** p, size_t bytes) {
  VAE_CUDA(cudaMalloc(p, bytes ? bytes : 16));
  pool.push_back(*p);
  v->bytes += (int64_t)bytes;
  return 0;
}
template <typename T> static int v_alloc_t(selftok_vae* v, std::vector<void*>& pool, T** p, int64_t n) {
  return v_alloc(v, pool, reinterpret_cast<void**>(p), sizeof(T) * (size_t)n);
}

extern "C" __attribute__((visibility("default"))) int selftok_vae_create(int ch, int device, selftok_vae_t* out) {
  STK_CHECK(out && ch == 128, SELFTOK_ERR_UNSUPPORTED, "selftok_vae_create: ch must be 128 (the SD3 VAE; GroupNorm groups of >= 4 channels)");
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) {
    set_error("no CUDA device visible: selftok_b200 has no CPU fallback");
    return SELFTOK_ERR_NO_DEVICE;
  }
  STK_CHECK(device >= 0 && device < ndev, SELFTOK_ERR_BAD_ARG, "bad device ordinal");
  cudaDeviceProp prop;
  STK_CUDA(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0) {
    set_error("device is not sm_90 (Hopper H100): kernels are built for sm_90a only");
    return SELFTOK_ERR_NO_DEVICE;
  }
  STK_CUDA(cudaSetDevice(device));
  STK_TRY(gemm_tc_init());
  selftok_vae* v = new selftok_vae();
  v->device = device;
  v->ch = ch;
  *out = v;
  return SELFTOK_OK;
}

extern "C" __attribute__((visibility("default"))) int selftok_vae_destroy(selftok_vae_t v) {
  if (!v) return SELFTOK_OK;
  cudaSetDevice(v->device);
  cudaDeviceSynchronize();
  for (auto& kv : v->raw) cudaFree(kv.second.first);
  for (void* p : v->allocs) cudaFree(p);
  for (void* p : v->ws_allocs) cudaFree(p);
  delete v;
  return SELFTOK_OK;
}

extern "C" __attribute__((visibility("default"))) int selftok_vae_load_tensor(selftok_vae_t v, const char* name, const void* data, int ndim, const int64_t* shape,
                                       int is_device) {
  STK_CHECK(v && name && data && shape && ndim >= 1 && ndim <= 4, SELFTOK_ERR_BAD_ARG, "selftok_vae_load_tensor: bad argument");
  STK_CHECK(!v->finalized, SELFTOK_ERR_STATE, "load_tensor after finalize");
  STK_CUDA(cudaSetDevice(v->device));
  int64_t n = 1;
  std::vector<int64_t> sh(shape, shape + ndim);
  for (int64_t d : sh) n *= d;
  STK_CHECK(n > 0, SELFTOK_ERR_BAD_ARG, "empty tensor");
  auto it = v->raw.find(name);
  if (it != v->raw.end()) { cudaFree(it->second.first); v->raw.erase(it); }
  float* d;
  STK_CUDA(cudaMalloc(&d, sizeof(float) * (size_t)n));
  STK_CUDA(cudaMemcpy(d, data, sizeof(float) * (size_t)n, is_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice));
  v->raw[name] = {d, sh};
  return SELFTOK_OK;
}

// pack one conv ("<name>.weight" [Cout, Cin, k, k] + "<name>.bias"): GEMM operand planes [Npad, taps * Cpad], K-major
static int pack_conv(selftok_vae* v, const std::string& name, cudaStream_t s) {
  auto wi = v->raw.find(name + ".weight"), bi = v->raw.find(name + ".bias");
  if (wi == v->raw.end() || bi == v->raw.end()) {
    set_error("VAE checkpoint key not loaded: " + name + ".weight / .bias");
    return SELFTOK_ERR_MISSING_TENSOR;
  }
  const std::vector<int64_t>& sh = wi->second.second;
  STK_CHECK(sh.size() == 4 && sh[2] == sh[3] && (sh[2] == 1 || sh[2] == 3), SELFTOK_ERR_UNSUPPORTED, "VAE conv weights must be [Cout, Cin, 1|3, 1|3]");
  VaeW w;
  w.N = (int)sh[0];
  w.taps = (int)(sh[2] * sh[3]);
  const int Cin = (int)sh[1];
  w.Cpad = (Cin + 63) / 64 * 64;
  w.Npad = (w.N + 3) / 4 * 4;
  w.K = w.taps * w.Cpad;
  float* tmp;
  STK_CUDA(cudaMalloc(&tmp, sizeof(float) * (size_t)w.Npad * w.K));
  repack_conv_kernel<<<blocks_for((int64_t)w.Npad * w.K), 256, 0, s>>>(wi->second.first, tmp, w.N, Cin, w.taps, w.Npad, w.Cpad);
  count_launch();
  STK_TRY(v_alloc_t(v, v->allocs, &w.hi, (int64_t)w.Npad * w.K));
  STK_TRY(v_alloc_t(v, v->allocs, &w.lo, (int64_t)w.Npad * w.K));
  STK_TRY(launch_split_bf16(tmp, w.hi, w.lo, (int64_t)w.Npad * w.K, s, 0));
  STK_TRY(v_alloc_t(v, v->allocs, &w.bias, w.Npad));
  STK_CUDA(cudaMemsetAsync(w.bias, 0, sizeof(float) * w.Npad, s));
  STK_CUDA(cudaMemcpyAsync(w.bias, bi->second.first, sizeof(float) * w.N, cudaMemcpyDeviceToDevice, s));
  STK_CUDA(cudaStreamSynchronize(s));
  cudaFree(tmp);
  cudaFree(wi->second.first);
  v->raw.erase(wi);
  v->conv[name] = w;
  return 0;
}

static std::vector<std::string> resnet_names(const std::string& p, bool shortcut) {
  std::vector<std::string> n = {p + ".conv1", p + ".conv2"};
  if (shortcut) n.push_back(p + ".nin_shortcut");
  return n;
}

extern "C" __attribute__((visibility("default"))) int selftok_vae_finalize(selftok_vae_t v, void* stream) {
  STK_CHECK(v && !v->finalized, SELFTOK_ERR_STATE, "selftok_vae_finalize: bad state");
  STK_CUDA(cudaSetDevice(v->device));
  cudaStream_t s = (cudaStream_t)stream;
  const int ch = v->ch;
  v->has_dec = v->raw.count("decoder.conv_in.weight") > 0;
  v->has_enc = v->raw.count("encoder.conv_in.weight") > 0;
  STK_CHECK(v->has_dec || v->has_enc, SELFTOK_ERR_MISSING_TENSOR, "selftok_vae_finalize: neither decoder.* nor encoder.* tensors were loaded");
  std::vector<std::string> convs;
  auto add_mid = [&](const std::string& p) {
    for (const char* n : {".conv_in", ".conv_out", ".mid.attn_1.q", ".mid.attn_1.k", ".mid.attn_1.v", ".mid.attn_1.proj_out"}) convs.push_back(p + n);
    for (const char* b : {".mid.block_1", ".mid.block_2"})
      for (auto& n : resnet_names(p + b, false)) convs.push_back(n);
  };
  if (v->has_dec) {
    add_mid("decoder");
    int cin = ch * v->mult[3];
    for (int lvl = 3; lvl >= 0; --lvl) {
      const int cout = ch * v->mult[lvl];
      for (int b = 0; b < 3; ++b) {
        for (auto& n : resnet_names("decoder.up." + std::to_string(lvl) + ".block." + std::to_string(b), cin != cout)) convs.push_back(n);
        cin = cout;
      }
      if (lvl != 0) convs.push_back("decoder.up." + std::to_string(lvl) + ".upsample.conv");
    }
  }
  if (v->has_enc) {
    add_mid("encoder");
    int cin = ch;
    for (int lvl = 0; lvl < 4; ++lvl) {
      const int cout = ch * v->mult[lvl];
      for (int b = 0; b < 2; ++b) {
        for (auto& n : resnet_names("encoder.down." + std::to_string(lvl) + ".block." + std::to_string(b), cin != cout)) convs.push_back(n);
        cin = cout;
      }
      if (lvl != 3) convs.push_back("encoder.down." + std::to_string(lvl) + ".downsample.conv");
    }
  }
  for (auto& n : convs) STK_TRY(pack_conv(v, n, s));
  v->finalized = true;
  return SELFTOK_OK;
}

// ------------------------------------------------------------------------------------------------ forward
struct VaeCtx {
  selftok_vae* v;
  cudaStream_t s;
  int B;
};
static const float* vget(selftok_vae* v, const std::string& name) {
  auto it = v->raw.find(name);
  return it == v->raw.end() ? nullptr : it->second.first;
}
// y = conv(planes) (+ resid) -> out (fp32 NHWC [M, N]); taps == 9: implicit GEMM over [B, H, W, Cpad] planes, at any H, W (its
// 128-pixel tiles may overhang the image edge; their outside rows are neither stored nor loaded, so the fp32 stream only ever
// holds the H W real pixels of each image)
static int vconv(VaeCtx& c, const std::string& name, const bf16* a_hi, const bf16* a_lo, int H, int W, float* out, const float* resid, int stride = 1) {
  auto it = c.v->conv.find(name);
  STK_CHECK(it != c.v->conv.end(), SELFTOK_ERR_STATE, "VAE conv not packed");
  const VaeW& w = it->second;
  Epilogue ep;
  ep.bias = w.bias; ep.out = out; ep.ldo = w.Npad;
  if (resid) { ep.mode = EPI_RESID; ep.resid = resid; }
  TcProblem q{a_hi, a_lo, w.hi, w.lo, (int64_t)c.B * H * W, w.Npad, w.K, ep};
  if (w.taps == 9) { q.conv_C = w.Cpad; q.conv_H = H; q.conv_W = W; q.conv_stride = stride; q.conv_edge = 1; }   // stride 2: H, W = output dims
  return launch_gemm_tc_grouped(&q, 1, 3, c.s, 0);
}
// GroupNorm (+ SiLU) of the fp32 NHWC stream x [B, HW, C] into the operand planes.  The statistics cover exactly the H W real
// pixels of each image: the stream is dense [B, H, W, C], and the rows of a convolution tile that overhang the image edge
// never reach it (vconv).
static int vnorm(VaeCtx& c, const std::string& name, const float* x, int64_t HW, int C, bool silu_act) {
  selftok_vae* v = c.v;
  const float *g = vget(v, name + ".weight"), *b = vget(v, name + ".bias");
  STK_CHECK(g && b, SELFTOK_ERR_MISSING_TENSOR, "VAE GroupNorm parameters missing");
  STK_CHECK(C % 128 == 0 && 256 % (C / 4) == 0, SELFTOK_ERR_UNSUPPORTED, "VAE GroupNorm: channels must be 128, 256 or 512");
  const int chunk_pix = 1024;
  const int nchunk = (int)((HW + chunk_pix - 1) / chunk_pix);
  gn_partial_kernel<<<dim3(nchunk, c.B), 256, 0, c.s>>>(x, v->part, (int)HW, C, chunk_pix);
  count_launch();
  gn_finalize_kernel<<<c.B, 32, 0, c.s>>>(v->part, v->stats, nchunk, HW * (C / GN_GROUPS), 1e-6f);
  count_launch();
  const int64_t total4 = (int64_t)c.B * HW * (C / 4);
  if (silu_act) gn_apply_kernel<true><<<blocks_for(total4, 256, 132 * 16), 256, 0, c.s>>>(x, v->stats, g, b, v->p_hi, v->p_lo, HW, C, total4);
  else gn_apply_kernel<false><<<blocks_for(total4, 256, 132 * 16), 256, 0, c.s>>>(x, v->stats, g, b, v->p_hi, v->p_lo, HW, C, total4);
  count_launch();
  STK_CUDA(cudaGetLastError());
  return 0;
}
// ResnetBlock.forward (sd3_impls.py:245-256): x (fp32, C_in) -> y (fp32, C_out) = shortcut(x) + conv2(silu(norm2(conv1(silu(norm1(x))))))
static int vresnet(VaeCtx& c, const std::string& p, float*& x, float*& y, int H, int W, int Cin, int Cout) {
  selftok_vae* v = c.v;
  const int64_t HW = (int64_t)H * W;
  STK_TRY(vnorm(c, p + ".norm1", x, HW, Cin, true));
  STK_TRY(vconv(c, p + ".conv1", v->p_hi, v->p_lo, H, W, y, nullptr));                 // y = conv1(.)          [C_out]
  STK_TRY(vnorm(c, p + ".norm2", y, HW, Cout, true));
  if (Cin != Cout) {
    // 1x1 shortcut of the raw x: needs x as planes -- upsample kernel with factor 1 is not available, so use the split kernel
    STK_TRY(launch_split_bf16(x, v->q_hi, v->q_lo, (int64_t)c.B * HW * Cin, c.s, 0));
    STK_TRY(vconv(c, p + ".nin_shortcut", v->q_hi, v->q_lo, H, W, v->sc, nullptr));
    STK_TRY(vconv(c, p + ".conv2", v->p_hi, v->p_lo, H, W, y, v->sc));                 // y = sc + conv2(.)
  } else {
    STK_TRY(vconv(c, p + ".conv2", v->p_hi, v->p_lo, H, W, y, x));                     // y = x + conv2(.)   (y != x: conv1 output consumed)
  }
  std::swap(x, y);
  return 0;
}

// the middle of both networks: ResnetBlock, AttnBlock, ResnetBlock at Cm channels on the [B, H, W] grid
static int vmid(VaeCtx& c, const std::string& pre, float*& x, float*& y, int H, int W, int Cm) {
  selftok_vae* v = c.v;
  cudaStream_t s = c.s;
  const int B = c.B;
  STK_TRY(vresnet(c, pre + ".mid.block_1", x, y, H, W, Cm, Cm));
  {
    // AttnBlock (sd3_impls.py:276-287): h = norm(x); q, k, v = 1x1 convs; softmax(q k^T / sqrt(C)) v; x + proj_out(.)
    // The key axis of S, P and V^T is padded to Tp, a multiple of 8 (16-byte rows for TMA and the GEMM pitch checks).  S's pad
    // columns are products with the rows after image b's keys (the next image's, or the workspace's slack rows) and are never
    // read; P's pad columns are written as zero by the softmax and V^T's are cleared, so that they add exactly 0 to P V (0 x NaN
    // would be NaN).
    const int64_t T = (int64_t)H * W, Tp = (T + 7) / 8 * 8;
    STK_TRY(vnorm(c, pre + ".mid.attn_1.norm", x, T, Cm, false));
    auto lin_planes = [&](const std::string& name, bf16* oh, bf16* ol) -> int {       // [B T, C] planes -> [B T, C] planes (+ bias)
      const VaeW& wq = v->conv[name];
      Epilogue ep;
      ep.mode = EPI_SPLIT; ep.bias = wq.bias; ep.out_hi = oh; ep.out_lo = ol; ep.ldo = Cm;
      TcProblem q{v->p_hi, v->p_lo, wq.hi, wq.lo, (int64_t)B * T, Cm, Cm, ep};
      return launch_gemm_tc_grouped(&q, 1, 3, s, 0);
    };
    STK_TRY(lin_planes(pre + ".mid.attn_1.q", v->q_hi, v->q_lo));
    STK_TRY(lin_planes(pre + ".mid.attn_1.k", v->k_hi, v->k_lo));
    const VaeW& wv = v->conv[pre + ".mid.attn_1.v"];
    for (int b = 0; b < B; ++b) {
      const int64_t off = (int64_t)b * T * Cm, off_vt = (int64_t)b * Cm * Tp;
      // V^T [C, Tp] = W_v [C, C] . h_b^T  (operands swapped; the bias is added after P V: the rows of P sum to one)
      Epilogue ev;
      ev.mode = EPI_SPLIT; ev.out_hi = v->vt_hi + off_vt; ev.out_lo = v->vt_lo + off_vt; ev.ldo = Tp;
      TcProblem qv{wv.hi, wv.lo, v->p_hi + off, v->p_lo + off, Cm, (int)Tp, Cm, ev};
      STK_TRY(launch_gemm_tc_grouped(&qv, 1, 3, s, 0));
      if (Tp > T) {
        STK_CUDA(cudaMemset2DAsync(v->vt_hi + off_vt + T, Tp * sizeof(bf16), 0, (Tp - T) * sizeof(bf16), Cm, s));
        STK_CUDA(cudaMemset2DAsync(v->vt_lo + off_vt + T, Tp * sizeof(bf16), 0, (Tp - T) * sizeof(bf16), Cm, s));
      }
      // S = Q_b K_b^T  [T, Tp] fp32
      Epilogue es;
      es.out = v->s_attn; es.ldo = Tp;
      TcProblem qs{v->q_hi + off, v->q_lo + off, v->k_hi + off, v->k_lo + off, T, (int)Tp, Cm, es};
      STK_TRY(launch_gemm_tc_grouped(&qs, 1, 3, s, 0));
      softmax_rows_kernel<<<(unsigned)((T + 7) / 8), 256, 0, s>>>(v->s_attn, v->pr_hi, v->pr_lo, T, (int)T, (int)Tp, 1.0f / sqrtf((float)Cm));
      count_launch();
      // O_b = P V + b_v  [T, C] -> planes (A operand of proj_out)
      Epilogue eo;
      eo.mode = EPI_SPLIT; eo.bias = wv.bias; eo.out_hi = v->o_hi + off; eo.out_lo = v->o_lo + off; eo.ldo = Cm;
      TcProblem qo{v->pr_hi, v->pr_lo, v->vt_hi + off_vt, v->vt_lo + off_vt, T, Cm, (int)Tp, eo};
      STK_TRY(launch_gemm_tc_grouped(&qo, 1, 3, s, 0));
    }
    STK_TRY(vconv(c, pre + ".mid.attn_1.proj_out", v->o_hi, v->o_lo, H, W, y, x));     // y = x + proj_out(o)
    std::swap(x, y);
  }
  STK_TRY(vresnet(c, pre + ".mid.block_2", x, y, H, W, Cm, Cm));
  return 0;
}

// workspace for B images of latent size h x w (a decode of [B, 16, h, w], or an encode of [B, 3, 8h, 8w]); kept while a call fits
static int vae_ensure_ws(selftok_vae* v, int B, int h, int w) {
  if (v->wsB >= B && v->wsh >= h && v->wsw >= w) return 0;
  for (void* p : v->ws_allocs) cudaFree(p);
  v->ws_allocs.clear();
  auto& P = v->ws_allocs;
  const int ch = v->ch;
  // the largest fp32 tensor: max over levels of H W C (level l: h * 2^(3-l) x w * 2^(3-l), channels ch * mult[l]); and the
  // padded conv_in input
  int64_t big = (int64_t)h * w * 64;
  for (int l = 0; l < 4; ++l) {
    const int64_t hs = (int64_t)h << (3 - l), ws = (int64_t)w << (3 - l);
    big = std::max(big, hs * ws * ch * v->mult[l]);
    if (l > 0) big = std::max(big, (hs * 2) * (ws * 2) * ch * v->mult[l]);           // upsampled planes keep the level's channels
  }
  big *= B;
  // attention (vmid): key axis padded to Tp; the S and V^T GEMMs read Tp rows of image b's keys / normalised input, so the last
  // image reads up to 7 rows past B T: k gets 8 slack rows, and the p planes (big >= B 8h 8w 128 = 16 B T Cm) have them already
  const int64_t T = (int64_t)h * w, Tp = (T + 7) / 8 * 8, Cm = (int64_t)ch * v->mult[3];
  STK_TRY(v_alloc_t(v, P, &v->xa, big));
  STK_TRY(v_alloc_t(v, P, &v->xb, big));
  STK_TRY(v_alloc_t(v, P, &v->sc, big));
  STK_TRY(v_alloc_t(v, P, &v->p_hi, big));
  STK_TRY(v_alloc_t(v, P, &v->p_lo, big));
  STK_TRY(v_alloc_t(v, P, &v->q_hi, big));
  STK_TRY(v_alloc_t(v, P, &v->q_lo, big));
  STK_TRY(v_alloc_t(v, P, &v->k_hi, ((int64_t)B * T + 8) * Cm));
  STK_TRY(v_alloc_t(v, P, &v->k_lo, ((int64_t)B * T + 8) * Cm));
  STK_TRY(v_alloc_t(v, P, &v->vt_hi, (int64_t)B * Cm * Tp));
  STK_TRY(v_alloc_t(v, P, &v->vt_lo, (int64_t)B * Cm * Tp));
  STK_TRY(v_alloc_t(v, P, &v->pr_hi, T * Tp));
  STK_TRY(v_alloc_t(v, P, &v->pr_lo, T * Tp));
  STK_TRY(v_alloc_t(v, P, &v->o_hi, (int64_t)B * T * Cm));
  STK_TRY(v_alloc_t(v, P, &v->o_lo, (int64_t)B * T * Cm));
  STK_TRY(v_alloc_t(v, P, &v->s_attn, T * Tp));
  const int64_t HWmax = ((int64_t)h * 8) * ((int64_t)w * 8);
  STK_TRY(v_alloc_t(v, P, &v->part, (int64_t)B * ((HWmax + 1023) / 1024) * 2 * GN_GROUPS));
  STK_TRY(v_alloc_t(v, P, &v->stats, (int64_t)B * GN_GROUPS * 2));
  STK_TRY(v_alloc_t(v, P, &v->out4, (int64_t)B * HWmax * 4));
  v->wsB = B; v->wsh = h; v->wsw = w;
  return 0;
}

// z_dev [B, 16, h, w] fp32 (VAE latent space, i.e. AFTER SD3LatentFormat.process_out), 1 <= h, w <= 128 -> out_dev [B, 3, 8h, 8w]
// fp32; norm_ip != 0: clamp to [-1, 1] and rescale to [0, 1] (SelftokPipeline.py:293).  Each image's result does not depend on
// the batch: every kernel works per pixel or per image, and the convolution tiles are chosen from (h, w) alone.
extern "C" __attribute__((visibility("default"))) int selftok_vae_decode(selftok_vae_t v, const float* z_dev, int B, int h, int w, float* out_dev, int norm_ip,
                                  void* stream) {
  STK_CHECK(v && z_dev && out_dev && B > 0, SELFTOK_ERR_BAD_ARG, "selftok_vae_decode: bad argument");
  STK_CHECK(v->finalized, SELFTOK_ERR_STATE, "selftok_vae_finalize has not been called");
  STK_CHECK(v->has_dec, SELFTOK_ERR_MISSING_TENSOR, "selftok_vae_decode: no decoder.* tensors were loaded");
  STK_CHECK(h >= 1 && h <= 128 && w >= 1 && w <= 128, SELFTOK_ERR_UNSUPPORTED, "VAE decode: latent sides must be in [1, 128]");
  STK_CUDA(cudaSetDevice(v->device));
  cudaStream_t s = (cudaStream_t)stream;
  STK_TRY(vae_ensure_ws(v, B, h, w));
  VaeCtx c{v, s, B};
  const int ch = v->ch, Cm = ch * v->mult[3];
  int H = h, W = w;
  // conv_in: 16 latent channels zero-padded to one 64-channel chunk
  latent_to_planes_kernel<<<blocks_for((int64_t)B * H * W * 64), 256, 0, s>>>(z_dev, v->p_hi, v->p_lo, B, 16, H, W);
  count_launch();
  float *x = v->xa, *y = v->xb;
  STK_TRY(vconv(c, "decoder.conv_in", v->p_hi, v->p_lo, H, W, x, nullptr));
  STK_TRY(vmid(c, "decoder", x, y, H, W, Cm));
  // upsampling
  int cin = Cm;
  for (int lvl = 3; lvl >= 0; --lvl) {
    const int cout = ch * v->mult[lvl];
    for (int b = 0; b < 3; ++b) {
      STK_TRY(vresnet(c, "decoder.up." + std::to_string(lvl) + ".block." + std::to_string(b), x, y, H, W, cin, cout));
      cin = cout;
    }
    if (lvl != 0) {
      upsample2x_planes_kernel<<<blocks_for((int64_t)B * 4 * H * W * (cin / 4), 256, 132 * 16), 256, 0, s>>>(x, v->p_hi, v->p_lo, B, H, W, cin);
      count_launch();
      H *= 2; W *= 2;
      STK_TRY(vconv(c, "decoder.up." + std::to_string(lvl) + ".upsample.conv", v->p_hi, v->p_lo, H, W, y, nullptr));
      std::swap(x, y);
    }
  }
  STK_TRY(vnorm(c, "decoder.norm_out", x, (int64_t)H * W, cin, true));
  STK_TRY(vconv(c, "decoder.conv_out", v->p_hi, v->p_lo, H, W, v->out4, nullptr));
  nhwc4_to_nchw3_kernel<<<blocks_for((int64_t)B * 3 * H * W), 256, 0, s>>>(v->out4, out_dev, B, H * W, norm_ip);
  count_launch();
  STK_CUDA(cudaGetLastError());
  return SELFTOK_OK;
}

// images_dev [B, 3, H, W] fp32 in [-1, 1], H and W multiples of 8 in [8, 1024] -> the latent distribution's parameters
// [B, 16, H/8, W/8] fp32 NCHW each (VAE latent space, i.e. BEFORE SD3LatentFormat.process_in): mean_out_dev = `.mode()`
// (SelftokPipeline.py:215), logvar_out_dev optional.  Every downsampled level has even sides (H / 8 may be odd), so the stride-2
// convolutions keep the polyphase layout.  Batch-invariant as selftok_vae_decode.
extern "C" __attribute__((visibility("default"))) int selftok_vae_encode(selftok_vae_t v, const float* images_dev, int B, int H, int W, float* mean_out_dev,
                                  float* logvar_out_dev, void* stream) {
  STK_CHECK(v && images_dev && mean_out_dev && B > 0, SELFTOK_ERR_BAD_ARG, "selftok_vae_encode: bad argument");
  STK_CHECK(v->finalized, SELFTOK_ERR_STATE, "selftok_vae_finalize has not been called");
  STK_CHECK(v->has_enc, SELFTOK_ERR_MISSING_TENSOR, "selftok_vae_encode: no encoder.* tensors were loaded");
  STK_CHECK(H % 8 == 0 && W % 8 == 0 && H >= 8 && H <= 1024 && W >= 8 && W <= 1024, SELFTOK_ERR_UNSUPPORTED,
            "VAE encode: image sides must be multiples of 8 in [8, 1024]");
  STK_CUDA(cudaSetDevice(v->device));
  cudaStream_t s = (cudaStream_t)stream;
  STK_TRY(vae_ensure_ws(v, B, H / 8, W / 8));
  VaeCtx c{v, s, B};
  const int ch = v->ch, Cm = ch * v->mult[3];
  // conv_in: 3 image channels zero-padded to one 64-channel chunk
  latent_to_planes_kernel<<<blocks_for((int64_t)B * H * W * 64), 256, 0, s>>>(images_dev, v->p_hi, v->p_lo, B, 3, H, W);
  count_launch();
  float *x = v->xa, *y = v->xb;
  STK_TRY(vconv(c, "encoder.conv_in", v->p_hi, v->p_lo, H, W, x, nullptr));
  int cin = ch;
  for (int lvl = 0; lvl < 4; ++lvl) {
    const int cout = ch * v->mult[lvl];
    for (int b = 0; b < 2; ++b) {
      STK_TRY(vresnet(c, "encoder.down." + std::to_string(lvl) + ".block." + std::to_string(b), x, y, H, W, cin, cout));
      cin = cout;
    }
    if (lvl != 3) {
      space_to_depth_planes_kernel<<<blocks_for((int64_t)B * H * W * (cin / 4), 256, 132 * 16), 256, 0, s>>>(x, v->p_hi, v->p_lo, B, H, W, cin);
      count_launch();
      H /= 2; W /= 2;
      STK_TRY(vconv(c, "encoder.down." + std::to_string(lvl) + ".downsample.conv", v->p_hi, v->p_lo, H, W, y, nullptr, 2));
      std::swap(x, y);
    }
  }
  STK_TRY(vmid(c, "encoder", x, y, H, W, Cm));
  STK_TRY(vnorm(c, "encoder.norm_out", x, (int64_t)H * W, Cm, true));
  STK_TRY(vconv(c, "encoder.conv_out", v->p_hi, v->p_lo, H, W, v->out4, nullptr));       // [B, h, w, 32] = (mean | logvar)
  nhwc_to_nchw_kernel<<<blocks_for((int64_t)B * 16 * H * W), 256, 0, s>>>(v->out4, mean_out_dev, B, H * W, 32, 0, 16);
  count_launch();
  if (logvar_out_dev) {
    nhwc_to_nchw_kernel<<<blocks_for((int64_t)B * 16 * H * W), 256, 0, s>>>(v->out4, logvar_out_dev, B, H * W, 32, 16, 16);
    count_launch();
  }
  STK_CUDA(cudaGetLastError());
  return SELFTOK_OK;
}

extern "C" __attribute__((visibility("default"))) int64_t selftok_vae_device_bytes(selftok_vae_t v) { return v ? v->bytes : -1; }
