// selftok_b200 engine: the C ABI of include/selftok_b200.h.
//
// Host-side orchestration of the encode / decode hot path of mimogpt/infer/SelftokPipeline.py — weights under the
// reference's checkpoint key names, every input-independent table built once at finalize, one workspace per batch
// size, and the 50-step sampler captured in one CUDA graph.  All arithmetic is in the kernels of kernels_simt.cu
// (fp32 FFMA: encoder, VQ, tables), gemm_tc.cu (wgmma GEMMs of the MMDiT) and attn_tc5.cu (wgmma joint attention).
#include "../../include/selftok_b200.h"
#include "common.cuh"
#include "kernels.h"

#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <map>
#include <string>
#include <tuple>
#include <unordered_map>
#include <vector>

namespace stk {
static thread_local std::string g_error;
thread_local int64_t g_launch_count = 0;
void set_error(const std::string& msg) { g_error = msg; }
}  // namespace stk

using namespace stk;
typedef __nv_bfloat16 bf16;

struct Tensor {
  float* d = nullptr;
  std::vector<int64_t> shape;
  int64_t numel = 0;
};
struct WPack {
  bf16* hi = nullptr;                   // fp8 mode, qkv / fc1: e4m3 codes [N, K] (one byte each)
  bf16* lo = nullptr;
  float* scale = nullptr;               // fp8 mode, qkv / fc1: [N] per-output-channel scales of the codes
};

// Bump allocator over ONE block of device memory: the activation workspaces are carved from it.  The block is either the
// caller's (selftok_set_workspace: PyTorch keeps ownership, nothing is allocated behind its caching allocator) or one
// cudaMalloc of exactly selftok_workspace_bytes.  dry = sizing pass only.
struct Arena {
  char* base = nullptr;
  size_t cap = 0, off = 0;
  bool dry = false;
  template <typename T> int take(T** p, int64_t n) {
    const size_t bytes = (sizeof(T) * (size_t)(n > 0 ? n : 1) + 255) & ~(size_t)255;
    if (!dry) {
      if (off + bytes > cap) { set_error("workspace too small"); return SELFTOK_ERR_BAD_ARG; }
      *p = reinterpret_cast<T*>(base + off);
    }
    off += bytes;
    return 0;
  }
};

struct DecodeWs {       // activation workspace of the MMDiT, carved for one batch size and latent geometry
  int B = 0, lh = 0, lw = 0;
  char* base = nullptr;                          // the block it is carved from (the caller's or `own`) and its size
  size_t cap = 0;
  int64_t* tokens = nullptr;
  float *outs_q = nullptr, *x_lat = nullptr, *patch = nullptr, *ctx0 = nullptr, *ctx = nullptr, *x = nullptr;
  float *qkv = nullptr, *o_final = nullptr;      // qkv: fp32 joint buffer (fp32 mode only)
  float* o_final_u = nullptr;                    // final-layer output of the unconditional branch (guided sampler)
  // split-bf16 operand planes of the two skinny fp32-faithful GEMMs of every evaluation (patch embedding K = 64, final layer N = 64)
  bf16 *patch_hi = nullptr, *patch_lo = nullptr, *fin_hi = nullptr, *fin_lo = nullptr;
  bf16 *qkv_hi = nullptr, *qkv_lo = nullptr;     // joint q/k/v as 16-bit planes [B,S,3,H,64] (tensor-core modes)
  // fp32 mode activations
  float *a_c = nullptr, *a_x = nullptr, *attn_c = nullptr, *attn_x = nullptr, *h_c = nullptr, *h_x = nullptr;
  // tensor-core mode activations (bf16 planes)
  bf16 *a_c_hi = nullptr, *a_c_lo = nullptr, *a_x_hi = nullptr, *a_x_lo = nullptr;
  bf16 *attn_c_hi = nullptr, *attn_c_lo = nullptr, *attn_x_hi = nullptr, *attn_x_lo = nullptr;
  bf16 *h_c_hi = nullptr, *h_c_lo = nullptr, *h_x_hi = nullptr, *h_x_lo = nullptr;
  float *sa_c = nullptr, *sa_x = nullptr;        // fp8 mode: row scales of the e4m3 codes in a_c_hi / a_x_hi
  int* plan = nullptr;                           // token-range calls: [B][2] windows (lo, hi), then the plan [steps][B][2] (a, c)
  int* pk = nullptr;                             // step calls: the per-image block (see Packed), then the per-row maps
  void* own = nullptr;                           // the library's own block (NULL when the caller's workspace is in use)
  size_t own_bytes = 0;
};
struct EncodeWs {
  int B = 0, lh = 0, lw = 0;
  char* base = nullptr;
  size_t cap = 0;
  float *x0 = nullptr, *patch = nullptr, *x = nullptr, *q = nullptr, *xn = nullptr, *qn = nullptr, *xqkv = nullptr,
        *xkv = nullptr, *qqkv = nullptr, *xattn = nullptr, *qattn = nullptr, *xh = nullptr, *qh = nullptr, *outs_q = nullptr;
  int64_t* tokens = nullptr;
  void* own = nullptr;
  size_t own_bytes = 0;
};

struct selftok_engine {
  selftok_config_t cfg;
  int D = 0, H = 0;
  // latent geometry of the hot-path calls (selftok_set_latent_size; default cfg.latent x cfg.latent) and its patch counts
  int lat_h = 0, lat_w = 0, Nimg = 0, Nenc = 0;
  bool finalized = false;
  bool use_graph = true;
  std::unordered_map<std::string, Tensor> w;
  std::unordered_map<std::string, WPack> wp;
  std::vector<void*> allocs;            // tables + packed weights
  int64_t bytes = 0;
  // schedule
  int steps = 0;
  std::vector<float> t, dt;
  std::vector<int> k;
  float *t_freq = nullptr, *pos_freq = nullptr;
  float* t_freq_u = nullptr;            // classifier-free guidance: features of floor(1000 t).clamp(0, 999) (MMDiT.cfg_inference)
  // tables
  float *enc_mod = nullptr, *enc_pos = nullptr, *cbt = nullptr;
  float *ctx_mod = nullptr, *x_mod = nullptr, *ctx_last_mod = nullptr, *final_mod = nullptr, *dit_pos = nullptr;
  float *x_mod_u = nullptr, *final_mod_u = nullptr;     // unconditional branch of the guided sampler (optional)
  float* rend_x0 = nullptr;
  // centre crops of encoder.pos_embed [0] / model.pos_embed [1] for the geometries other than the default one, keyed by the
  // patch grid (gh, gw); the default crops are enc_pos / dit_pos.  pos_cur: the tables of the current geometry (pos_table)
  std::map<std::pair<int, int>, float*> pos_crops[2];
  const float* pos_cur[2] = {nullptr, nullptr};
  bool has_cfg = false;                 // unconditional-branch tables built (selftok_set_cfg_schedule before finalize)
  int* bad_ids = nullptr;               // device counter of out-of-range token ids seen by the lookup kernel
  DecodeWs dws;
  EncodeWs ews;
  void* user_ws[2] = {nullptr, nullptr};          // caller-provided workspaces (selftok_set_workspace): [0] encode, [1] decode / render
  size_t user_ws_bytes[2] = {0, 0};
  std::map<std::tuple<int, int, int, int>, std::pair<cudaGraphExec_t, int64_t>> graphs;   // (B, steps, lat_h, lat_w) -> (exec, launches)
  // token ranges: (B, steps, Lo, Hi, lat_h, lat_w)
  std::map<std::tuple<int, int, int, int, int, int>, std::pair<cudaGraphExec_t, int64_t>> range_graphs;
  std::vector<int> plan_host;           // token-range plan of the current call, built on the host
  int* plan_pinned = nullptr;           // pinned staging copy of it (an H2D copy from pageable memory would block the host)
  size_t plan_pinned_n = 0;
  cudaEvent_t plan_copied = nullptr;    // recorded after each upload: the staging buffer is reused only once it has completed
  std::map<std::tuple<int, int, int>, std::pair<cudaGraphExec_t, int64_t>> enc_graphs;   // encode, (B, lat_h, lat_w) -> (exec, launches)
  int64_t last_launches = 0;
  // optional per-kernel-class timing (CUDA events around every launch; only meaningful with graphs disabled)
  bool prof_on = false;
  std::vector<cudaEvent_t> prof_ev;     // pairs (start, stop)
  std::vector<int> prof_cat;
};

enum ProfCat { PC_GEMM_TC = 0, PC_ATTN = 1, PC_LN = 2, PC_LINEAR_F32 = 3, PC_VQ = 4, PC_OTHER = 5, PC_COUNT = 8 };
struct ProfScope {
  selftok_engine* e; cudaStream_t s; bool on;
  ProfScope(selftok_engine* e_, int cat, cudaStream_t s_) : e(e_), s(s_), on(e_->prof_on) {
    if (!on) return;
    cudaEvent_t a, b;
    cudaEventCreate(&a); cudaEventCreate(&b);
    e->prof_ev.push_back(a); e->prof_ev.push_back(b); e->prof_cat.push_back(cat);
    cudaEventRecord(a, s);
  }
  void end() { if (on) cudaEventRecord(e->prof_ev.back(), s); }
};
#define PROF(cat, expr)                         \
  do {                                          \
    ProfScope _ps(e, (cat), s);                 \
    int _st = (expr);                           \
    _ps.end();                                  \
    if (_st != 0) return _st;                   \
  } while (0)

static int dmalloc(selftok_engine* e, std::vector<void*>& pool, void** p, size_t bytes) {
  STK_CUDA(cudaMalloc(p, bytes ? bytes : 16));
  pool.push_back(*p);
  e->bytes += (int64_t)bytes;
  return 0;
}
template <typename T>
static int dalloc(selftok_engine* e, std::vector<void*>& pool, T** p, int64_t n) {
  return dmalloc(e, pool, reinterpret_cast<void**>(p), sizeof(T) * (size_t)n);
}
static void free_pool(selftok_engine* e, std::vector<void*>& pool) {
  for (void* p : pool) cudaFree(p);
  pool.clear();
}

static const Tensor* find(selftok_engine* e, const std::string& name) {
  auto it = e->w.find(name);
  return it == e->w.end() ? nullptr : &it->second;
}
#define GETW(var, name)                                                             \
  const Tensor* var = find(e, (name));                                              \
  if (!var) {                                                                       \
    set_error(std::string("checkpoint key not loaded: ") + (name));                 \
    return SELFTOK_ERR_MISSING_TENSOR;                                              \
  }

static bool tc_mode(const selftok_engine* e) { return e->cfg.precision != SELFTOK_PREC_FP32_SIMT; }
static int nsplit(const selftok_engine* e) { return e->cfg.precision == SELFTOK_PREC_BF16X3 ? 3 : 1; }
// the fp8 mode is the fp16 mode with e4m3 QKV and fc1 GEMMs: every 16-bit plane of it holds IEEE half
static int is_fp16(const selftok_engine* e) { return e->cfg.precision == SELFTOK_PREC_FP16 || e->cfg.precision == SELFTOK_PREC_FP8 ? 1 : 0; }
static bool is_fp8(const selftok_engine* e) { return e->cfg.precision == SELFTOK_PREC_FP8; }
// the linears that run on e4m3 operands in the fp8 mode: the two whose A operand comes from LayerNorm + modulate
static bool e4m3_linear(const std::string& name) {
  return name.find(".attn.qkv.") != std::string::npos || name.find(".mlp.fc1.") != std::string::npos;
}

// y = act(A W^T + b) with weights looked up by checkpoint prefix (fp32 FFMA path)
static int lin32(selftok_engine* e, const std::string& prefix, const float* A, int64_t lda, int64_t M, Epilogue ep,
                 cudaStream_t s) {
  GETW(W, prefix + ".weight");
  GETW(Bv, prefix + ".bias");
  int N = (int)W->shape[0];
  int K = (int)(W->numel / W->shape[0]);
  ep.bias = Bv->d;
  if (ep.ldo == 0) ep.ldo = N;
  PROF(PC_LINEAR_F32, launch_linear_f32(A, lda, W->d, K, M, N, K, ep, s));
  return 0;
}
// tensor-core path: A given as bf16 planes
static int lintc(selftok_engine* e, const std::string& prefix, const bf16* A_hi, const bf16* A_lo, int64_t M,
                 Epilogue ep, cudaStream_t s) {
  GETW(W, prefix + ".weight");
  GETW(Bv, prefix + ".bias");
  auto it = e->wp.find(prefix + ".weight");
  STK_CHECK(it != e->wp.end(), SELFTOK_ERR_STATE, "packed weight missing");
  int N = (int)W->shape[0];
  int K = (int)(W->numel / W->shape[0]);
  ep.bias = Bv->d;
  if (ep.ldo == 0) ep.ldo = N;
  ep.fp16 = is_fp16(e);
  PROF(PC_GEMM_TC, launch_gemm_tc(A_hi, A_lo, it->second.hi, it->second.lo, M, N, K, nsplit(e), ep, s, is_fp16(e)));
  return 0;
}

// tensor-core problem descriptor for a checkpoint linear (weights already packed at finalize).  e4m3-packed weights (fp8 mode):
// A_hi holds e4m3 codes and s_a their row scales.
static int tc_problem(selftok_engine* e, const std::string& prefix, const bf16* A_hi, const bf16* A_lo, int64_t M, Epilogue ep,
                      TcProblem* out, const float* s_a = nullptr) {
  GETW(W, prefix + ".weight");
  GETW(Bv, prefix + ".bias");
  auto it = e->wp.find(prefix + ".weight");
  STK_CHECK(it != e->wp.end(), SELFTOK_ERR_STATE, "packed weight missing");
  const int N = (int)W->shape[0];
  const int K = (int)(W->numel / W->shape[0]);
  ep.bias = Bv->d;
  if (ep.ldo == 0) ep.ldo = N;
  ep.fp16 = is_fp16(e);
  if (it->second.scale) {
    STK_CHECK(s_a, SELFTOK_ERR_STATE, "e4m3 weights need the row scales of A");
    ep.s_a = s_a; ep.s_w = it->second.scale;
  }
  *out = TcProblem{A_hi, A_lo, it->second.hi, it->second.lo, M, N, K, ep};
  return 0;
}
// the context- and image-stream GEMM of a layer in ONE launch (n == 1: image stream only); e4m3: the fp8 mode's QKV / fc1
static int lintc2(selftok_engine* e, const TcProblem* probs, int n, cudaStream_t s, bool e4m3 = false) {
  if (e4m3) PROF(PC_GEMM_TC, launch_gemm_tc_grouped(probs, n, NSPLIT_E4M3, s, 0));
  else PROF(PC_GEMM_TC, launch_gemm_tc_grouped(probs, n, nsplit(e), s, is_fp16(e)));
  return 0;
}

// ------------------------------------------------------------------------------------------------ C ABI: lifetime
extern "C" __attribute__((visibility("default"))) const char* selftok_last_error(void) { return g_error.c_str(); }
extern "C" __attribute__((visibility("default"))) const char* selftok_version(void) { return "selftok_b200 abi1 sm_90a (fp32-ffma + wgmma)"; }

extern "C" __attribute__((visibility("default"))) int selftok_create(const selftok_config_t* cfg, selftok_handle_t* out) {
  STK_CHECK(cfg && out, SELFTOK_ERR_BAD_ARG, "selftok_create: null argument");
  int ndev = 0;
  cudaError_t ce = cudaGetDeviceCount(&ndev);
  if (ce != cudaSuccess || ndev <= 0) {
    set_error("no CUDA device visible: selftok_b200 has no CPU fallback");
    return SELFTOK_ERR_NO_DEVICE;
  }
  STK_CHECK(cfg->device >= 0 && cfg->device < ndev, SELFTOK_ERR_BAD_ARG, "bad device ordinal");
  cudaDeviceProp prop;
  STK_CUDA(cudaGetDeviceProperties(&prop, cfg->device));
  if (prop.major != 9 || prop.minor != 0) {
    set_error("device is not sm_90 (Hopper H100): kernels are built for sm_90a only");
    return SELFTOK_ERR_NO_DEVICE;
  }
  STK_CHECK(cfg->K > 0 && cfg->latent > 0 && cfg->dit_depth > 0 && cfg->enc_depth > 0, SELFTOK_ERR_BAD_ARG, "bad dims");
  STK_CHECK(cfg->code_dim == 16, SELFTOK_ERR_UNSUPPORTED, "code_dim must be 16");
  STK_CHECK(cfg->enc_hidden % cfg->enc_heads == 0 && cfg->enc_qdim % cfg->enc_qheads == 0, SELFTOK_ERR_BAD_ARG, "bad heads");
  int hd1 = cfg->enc_hidden / cfg->enc_heads, hd2 = cfg->enc_qdim / cfg->enc_qheads;
  STK_CHECK((hd1 == 16 || hd1 == 32 || hd1 == 64) && (hd2 == 16 || hd2 == 32 || hd2 == 64), SELFTOK_ERR_UNSUPPORTED,
            "encoder head_dim must be 16/32/64");
  STK_CHECK(cfg->precision >= 0 && cfg->precision <= SELFTOK_PREC_FP8, SELFTOK_ERR_BAD_ARG, "bad precision");
  STK_CUDA(cudaSetDevice(cfg->device));
  selftok_engine* e = new selftok_engine();
  e->cfg = *cfg;
  e->D = 64 * cfg->dit_depth;
  e->H = cfg->dit_depth;
  e->lat_h = e->lat_w = cfg->latent;
  e->Nimg = (cfg->latent / cfg->dit_patch) * (cfg->latent / cfg->dit_patch);
  e->Nenc = (cfg->latent / cfg->enc_patch) * (cfg->latent / cfg->enc_patch);
  if (tc_mode(e)) {
    int st = gemm_tc_init();
    if (st != 0) { delete e; return st; }
  }
  if (cudaMalloc(&e->bad_ids, sizeof(int)) != cudaSuccess || cudaMemset(e->bad_ids, 0, sizeof(int)) != cudaSuccess) {
    set_error("cudaMalloc failed in selftok_create");
    delete e;
    return SELFTOK_ERR_CUDA;
  }
  *out = e;
  return SELFTOK_OK;
}

static void free_dws(selftok_engine* e) {
  if (e->dws.own) { cudaFree(e->dws.own); e->bytes -= (int64_t)e->dws.own_bytes; }
  e->dws = DecodeWs();
}
static void drop_encode_graphs(selftok_engine* e) {
  for (auto& g : e->enc_graphs) cudaGraphExecDestroy(g.second.first);
  e->enc_graphs.clear();
}
static void free_ews(selftok_engine* e) {
  drop_encode_graphs(e);                                                      // graphs hold pointers into the workspace
  if (e->ews.own) { cudaFree(e->ews.own); e->bytes -= (int64_t)e->ews.own_bytes; }
  e->ews = EncodeWs();
}

extern "C" __attribute__((visibility("default"))) int selftok_destroy(selftok_handle_t e) {
  if (!e) return SELFTOK_OK;
  cudaSetDevice(e->cfg.device);
  cudaDeviceSynchronize();
  for (auto& g : e->graphs) cudaGraphExecDestroy(g.second.first);
  for (auto& g : e->range_graphs) cudaGraphExecDestroy(g.second.first);
  if (e->plan_pinned) cudaFreeHost(e->plan_pinned);
  if (e->plan_copied) cudaEventDestroy(e->plan_copied);
  for (auto& kv : e->w) cudaFree(kv.second.d);
  free_pool(e, e->allocs);
  if (e->bad_ids) cudaFree(e->bad_ids);
  free_dws(e);
  free_ews(e);
  delete e;
  return SELFTOK_OK;
}

extern "C" __attribute__((visibility("default"))) int selftok_load_tensor(selftok_handle_t e, const char* name, const void* data, int dtype, int ndim,
                                   const int64_t* shape, int is_device) {
  STK_CHECK(e && name && data && shape && ndim >= 0 && ndim <= 8, SELFTOK_ERR_BAD_ARG, "selftok_load_tensor: bad argument");
  STK_CHECK(dtype == SELFTOK_F32, SELFTOK_ERR_UNSUPPORTED, "only fp32 checkpoint tensors are supported");
  STK_CHECK(!e->finalized, SELFTOK_ERR_STATE, "load_tensor after finalize");
  STK_CUDA(cudaSetDevice(e->cfg.device));
  Tensor t;
  t.numel = 1;
  for (int i = 0; i < ndim; ++i) { t.shape.push_back(shape[i]); t.numel *= shape[i]; }
  STK_CHECK(t.numel > 0, SELFTOK_ERR_BAD_ARG, "empty tensor");
  auto it = e->w.find(name);
  if (it != e->w.end()) { cudaFree(it->second.d); e->bytes -= it->second.numel * 4; e->w.erase(it); }
  STK_CUDA(cudaMalloc(&t.d, sizeof(float) * (size_t)t.numel));
  e->bytes += t.numel * 4;
  STK_CUDA(cudaMemcpy(t.d, data, sizeof(float) * (size_t)t.numel, is_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice));
  e->w[name] = t;
  return SELFTOK_OK;
}

extern "C" __attribute__((visibility("default"))) int selftok_set_schedule(selftok_handle_t e, int steps, const float* t_host, const float* dt_host,
                                    const int32_t* k_host, const float* t_freq_host, const float* pos_freq_host) {
  STK_CHECK(e && steps > 0 && t_host && dt_host && k_host && t_freq_host && pos_freq_host, SELFTOK_ERR_BAD_ARG,
            "selftok_set_schedule: bad argument");
  STK_CHECK(!e->finalized, SELFTOK_ERR_STATE, "set_schedule after finalize");
  STK_CUDA(cudaSetDevice(e->cfg.device));
  e->steps = steps;
  e->t.assign(t_host, t_host + steps);
  e->dt.assign(dt_host, dt_host + steps);
  e->k.assign(k_host, k_host + steps);
  for (int i = 0; i < steps; ++i)
    STK_CHECK(e->k[i] >= 0 && e->k[i] < e->cfg.K, SELFTOK_ERR_BAD_ARG, "schedule k out of range");
  STK_TRY(dalloc(e, e->allocs, &e->t_freq, (int64_t)steps * 256));
  STK_TRY(dalloc(e, e->allocs, &e->pos_freq, (int64_t)e->cfg.K * 256));
  STK_CUDA(cudaMemcpy(e->t_freq, t_freq_host, sizeof(float) * steps * 256, cudaMemcpyHostToDevice));
  STK_CUDA(cudaMemcpy(e->pos_freq, pos_freq_host, sizeof(float) * e->cfg.K * 256, cudaMemcpyHostToDevice));
  return SELFTOK_OK;
}

// Optional, before finalize: sinusoidal features [steps,256] of floor(1000 t_i).clamp(0, 999), the timestep the unconditional
// branch of the guided sampler is embedded with (MMDiT.cfg_inference, sd3/mmdit.py:1127).  Enables selftok_decode_cfg.
extern "C" __attribute__((visibility("default"))) int selftok_set_cfg_schedule(selftok_handle_t e, const float* t_freq_uncond_host) {
  STK_CHECK(e && t_freq_uncond_host, SELFTOK_ERR_BAD_ARG, "selftok_set_cfg_schedule: bad argument");
  STK_CHECK(!e->finalized && e->steps > 0, SELFTOK_ERR_STATE, "selftok_set_cfg_schedule: after selftok_set_schedule, before selftok_finalize");
  STK_CHECK(!e->cfg.renderer, SELFTOK_ERR_STATE, "the renderer has no guided path");
  STK_CUDA(cudaSetDevice(e->cfg.device));
  if (!e->t_freq_u) STK_TRY(dalloc(e, e->allocs, &e->t_freq_u, (int64_t)e->steps * 256));
  STK_CUDA(cudaMemcpy(e->t_freq_u, t_freq_uncond_host, sizeof(float) * e->steps * 256, cudaMemcpyHostToDevice));
  return SELFTOK_OK;
}

// ------------------------------------------------------------------------------------------------ finalize
// adaLN table of a position-indexed block:  Linear(SiLU(t_embedder(pos_freq)))  (modules.py:311-318; mmdit.py:446-458)
static int build_pos_table(selftok_engine* e, const std::string& blk, const float* freq, int rows, float* tmp1, float* tmp2,
                           float* out, cudaStream_t s) {
  Epilogue ep;
  ep.act = ACT_SILU; ep.out = tmp1;
  STK_TRY(lin32(e, blk + "t_embedder.mlp.0", freq, 256, rows, ep, s));
  GETW(W2, blk + "t_embedder.mlp.2.weight");
  int dim = (int)W2->shape[0];
  ep.out = tmp2;                                            // SiLU applied here: t_emb is only consumed through SiLU
  STK_TRY(lin32(e, blk + "t_embedder.mlp.2", tmp1, dim, rows, ep, s));
  Epilogue ep2;
  ep2.out = out;
  STK_TRY(lin32(e, blk + "adaLN_modulation.1", tmp2, dim, rows, ep2, s));
  return 0;
}

extern "C" __attribute__((visibility("default"))) int selftok_finalize(selftok_handle_t e, void* stream) {
  STK_CHECK(e, SELFTOK_ERR_BAD_ARG, "null handle");
  STK_CHECK(!e->finalized, SELFTOK_ERR_STATE, "already finalized");
  STK_CHECK(e->steps > 0, SELFTOK_ERR_STATE, "selftok_set_schedule must precede finalize");
  STK_CUDA(cudaSetDevice(e->cfg.device));
  cudaStream_t s = (cudaStream_t)stream;
  const selftok_config_t& c = e->cfg;
  const int K = c.K, Q = c.enc_qdim, D = e->D, L = c.dit_depth, T = e->steps;
  // scratch for the table MLPs
  float *tmp1, *tmp2;
  int64_t rows_max = K > T ? K : T, dim_max = D > Q ? D : Q;
  std::vector<void*> scratch;
  STK_TRY(dalloc(e, scratch, &tmp1, rows_max * dim_max));
  STK_TRY(dalloc(e, scratch, &tmp2, rows_max * dim_max));
  // ---- encoder: adaLN tables [depth][K][6Q], cropped positional grid, transposed codebook
  STK_TRY(dalloc(e, e->allocs, &e->enc_mod, (int64_t)c.enc_depth * K * 6 * Q));
  for (int i = 0; i < c.enc_depth; ++i)
    STK_TRY(build_pos_table(e, "encoder.blocks." + std::to_string(i) + ".", e->pos_freq, K, tmp1, tmp2,
                            e->enc_mod + (int64_t)i * K * 6 * Q, s));
  {
    GETW(pe, "encoder.pos_embed");
    STK_CHECK(pe->numel == (int64_t)c.enc_pos_max * c.enc_pos_max * c.enc_hidden, SELFTOK_ERR_BAD_ARG, "encoder.pos_embed shape");
    int g = c.latent / c.enc_patch;
    STK_TRY(dalloc(e, e->allocs, &e->enc_pos, (int64_t)g * g * c.enc_hidden));
    PROF(PC_OTHER, launch_crop_pos(pe->d, e->enc_pos, c.enc_pos_max, g, g, (c.enc_pos_max - g) / 2, (c.enc_pos_max - g) / 2, c.enc_hidden, s));
    GETW(cb, "encoder.quantizer._codebook.embed");
    STK_CHECK(cb->numel == (int64_t)c.codebook_size * c.code_dim, SELFTOK_ERR_BAD_ARG, "codebook shape");
    STK_TRY(dalloc(e, e->allocs, &e->cbt, cb->numel));
    PROF(PC_OTHER, launch_transpose(cb->d, e->cbt, c.codebook_size, c.code_dim, s));
  }
  // ---- decoder tables
  STK_TRY(dalloc(e, e->allocs, &e->ctx_mod, (int64_t)(L - 1 > 0 ? L - 1 : 1) * K * 6 * D));
  for (int j = 0; j < L - 1; ++j)
    STK_TRY(build_pos_table(e, "model.joint_blocks." + std::to_string(j) + ".context_block.", e->pos_freq, K, tmp1, tmp2,
                            e->ctx_mod + (int64_t)j * K * 6 * D, s));
  {
    // csil = SiLU(t_embedder(t_freq)) [T, D]  (mmdit.py:1022; every consumer is Sequential(SiLU, Linear))
    float* csil;
    STK_TRY(dalloc(e, scratch, &csil, (int64_t)T * D));
    Epilogue ep;
    ep.act = ACT_SILU; ep.out = tmp1;
    STK_TRY(lin32(e, "model.t_embedder.mlp.0", e->t_freq, 256, T, ep, s));
    ep.out = csil;
    STK_TRY(lin32(e, "model.t_embedder.mlp.2", tmp1, D, T, ep, s));
    STK_TRY(dalloc(e, e->allocs, &e->x_mod, (int64_t)L * T * 6 * D));
    for (int j = 0; j < L; ++j) {
      Epilogue e2;
      e2.out = e->x_mod + (int64_t)j * T * 6 * D;
      STK_TRY(lin32(e, "model.joint_blocks." + std::to_string(j) + ".x_block.adaLN_modulation.1", csil, D, T, e2, s));
    }
    STK_TRY(dalloc(e, e->allocs, &e->ctx_last_mod, (int64_t)T * 2 * D));
    Epilogue e3;
    e3.out = e->ctx_last_mod;
    STK_TRY(lin32(e, "model.joint_blocks." + std::to_string(L - 1) + ".context_block.adaLN_modulation.1", csil, D, T, e3, s));
    STK_TRY(dalloc(e, e->allocs, &e->final_mod, (int64_t)T * 2 * D));
    Epilogue e4;
    e4.out = e->final_mod;
    STK_TRY(lin32(e, "model.final_layer.adaLN_modulation.1", csil, D, T, e4, s));
    if (e->t_freq_u) {
      // unconditional branch of the guided sampler: same MLPs on the integer-floored timestep (mmdit.py:1127-1130), image
      // stream only (every row of that pass is blind to the context keys, so the context stream never reaches the output)
      ep.act = ACT_SILU; ep.out = tmp1;
      STK_TRY(lin32(e, "model.t_embedder.mlp.0", e->t_freq_u, 256, T, ep, s));
      ep.out = csil;
      STK_TRY(lin32(e, "model.t_embedder.mlp.2", tmp1, D, T, ep, s));
      STK_TRY(dalloc(e, e->allocs, &e->x_mod_u, (int64_t)L * T * 6 * D));
      for (int j = 0; j < L; ++j) {
        Epilogue e2;
        e2.out = e->x_mod_u + (int64_t)j * T * 6 * D;
        STK_TRY(lin32(e, "model.joint_blocks." + std::to_string(j) + ".x_block.adaLN_modulation.1", csil, D, T, e2, s));
      }
      STK_TRY(dalloc(e, e->allocs, &e->final_mod_u, (int64_t)T * 2 * D));
      Epilogue e5;
      e5.out = e->final_mod_u;
      STK_TRY(lin32(e, "model.final_layer.adaLN_modulation.1", csil, D, T, e5, s));
    }
  }
  if (c.renderer) {
    GETW(pe, "model.positional_embedding");
    GETW(mt, "model.mask_token");
    STK_CHECK(pe->numel == (int64_t)e->Nimg * D && mt->numel == D, SELFTOK_ERR_UNSUPPORTED,
              "renderer expects positional_embedding [N,D] and mask_token [1,1,D] (repeat=True)");
    float* tmp;
    STK_TRY(dalloc(e, scratch, &tmp, (int64_t)e->Nimg * D));
    STK_TRY(dalloc(e, e->allocs, &e->rend_x0, (int64_t)e->Nimg * D));
    PROF(PC_OTHER, launch_bcast_rows(mt->d, nullptr, tmp, e->Nimg, 1, D, s));
    PROF(PC_OTHER, launch_bcast_rows(tmp, pe->d, e->rend_x0, 1, e->Nimg, D, s));
  } else {
    GETW(pe, "model.pos_embed");
    STK_CHECK(pe->numel == (int64_t)c.dit_pos_max * c.dit_pos_max * D, SELFTOK_ERR_BAD_ARG, "model.pos_embed shape");
    int g = c.latent / c.dit_patch;
    STK_TRY(dalloc(e, e->allocs, &e->dit_pos, (int64_t)g * g * D));
    PROF(PC_OTHER, launch_crop_pos(pe->d, e->dit_pos, c.dit_pos_max, g, g, (c.dit_pos_max - g) / 2, (c.dit_pos_max - g) / 2, D, s));
  }
  // ---- tensor-core operand planes of the MMDiT linears
  std::vector<std::string> packed_names;
  if (tc_mode(e)) {
    const char* blocks[2] = {"context_block", "x_block"};
    const char* lins[4] = {"attn.qkv", "attn.proj", "mlp.fc1", "mlp.fc2"};
    for (int j = 0; j < L; ++j)
      for (int b = 0; b < 2; ++b)
        for (int l = 0; l < 4; ++l) {
          if (j == L - 1 && b == 0 && l > 0) continue;          // pre_only context block: qkv only
          std::string name = "model.joint_blocks." + std::to_string(j) + "." + blocks[b] + "." + lins[l] + ".weight";
          GETW(W, name);
          WPack p;
          if (is_fp8(e) && e4m3_linear(name)) {                 // e4m3 codes + one scale per output channel
            const int64_t N = W->shape[0];
            uint8_t* codes;
            STK_TRY(dalloc(e, e->allocs, &codes, W->numel));
            STK_TRY(dalloc(e, e->allocs, &p.scale, N));
            PROF(PC_OTHER, launch_quant_e4m3_rows(W->d, N, (int)(W->numel / N), codes, p.scale, s));
            p.hi = reinterpret_cast<bf16*>(codes);
            e->wp[name] = p;
            packed_names.push_back(name);
            continue;
          }
          STK_TRY(dalloc(e, e->allocs, &p.hi, W->numel));
          if (nsplit(e) == 3) STK_TRY(dalloc(e, e->allocs, &p.lo, W->numel));
          PROF(PC_OTHER, launch_split_bf16(W->d, p.hi, p.lo, W->numel, s, is_fp16(e)));
          e->wp[name] = p;
          packed_names.push_back(name);
        }
  }
  if (tc_mode(e)) {
    // the patch embedding (K = 64) and the final layer (N = 64) stay fp32-faithful in every tensor-core mode: split-bf16 planes
    // (hi + lo, three MMAs per product); their fp32 copies are kept (the fp32 FFMA mode and the table MLPs read them)
    for (const char* nm : {"model.x_embedder.proj.weight", "model.final_layer.linear.weight"}) {
      if (c.renderer && std::string(nm) == "model.x_embedder.proj.weight") continue;      // the renderer has no x_embedder
      GETW(W, nm);
      WPack p;
      STK_TRY(dalloc(e, e->allocs, &p.hi, W->numel));
      STK_TRY(dalloc(e, e->allocs, &p.lo, W->numel));
      PROF(PC_OTHER, launch_split_bf16(W->d, p.hi, p.lo, W->numel, s, 0));
      e->wp[nm] = p;
    }
  }
  STK_CUDA(cudaStreamSynchronize(s));
  for (void* p : scratch) cudaFree(p);
  // the fp32 staging copies of the packed MMDiT weights are not read again (their shapes are): release 8.3 GB
  for (const std::string& name : packed_names) {
    Tensor& t = e->w[name];
    cudaFree(t.d);
    t.d = nullptr;
    e->bytes -= t.numel * 4;
  }
  e->has_cfg = e->x_mod_u != nullptr;
  e->finalized = true;
  return SELFTOK_OK;
}

// ------------------------------------------------------------------------------------------------ prepack cache
// The finalized device state (fp32 tensors that stay fp32, 16-bit operand planes, every static table, the schedule) as ONE
// file, so that a later process skips torch.load of the fp32 checkpoint, the per-tensor uploads, the table MLPs and the
// packing (SURVEY 8f rank 2: checkpoint loader + prepack cache; SelftokPipeline.py:188-199 reloads 8.3 GB of fp32 per process).
struct TableRef { const char* tag; float** ptr; int64_t numel; };
static std::vector<TableRef> table_refs(selftok_engine* e) {
  const selftok_config_t& c = e->cfg;
  const int64_t K = c.K, Q = c.enc_qdim, D = e->D, L = c.dit_depth, T = e->steps;
  const int64_t ge = c.latent / c.enc_patch, gd = c.latent / c.dit_patch;
  std::vector<TableRef> t = {
      {"t_freq", &e->t_freq, T * 256}, {"pos_freq", &e->pos_freq, K * 256},
      {"enc_mod", &e->enc_mod, (int64_t)c.enc_depth * K * 6 * Q}, {"enc_pos", &e->enc_pos, ge * ge * c.enc_hidden},
      {"cbt", &e->cbt, (int64_t)c.codebook_size * c.code_dim},
      {"ctx_mod", &e->ctx_mod, (L - 1 > 0 ? L - 1 : 1) * K * 6 * D}, {"x_mod", &e->x_mod, L * T * 6 * D},
      {"ctx_last_mod", &e->ctx_last_mod, T * 2 * D}, {"final_mod", &e->final_mod, T * 2 * D}};
  if (c.renderer) t.push_back({"rend_x0", &e->rend_x0, (int64_t)e->Nimg * D});
  else t.push_back({"dit_pos", &e->dit_pos, gd * gd * D});
  if (e->has_cfg) {
    t.push_back({"x_mod_u", &e->x_mod_u, L * T * 6 * D});
    t.push_back({"final_mod_u", &e->final_mod_u, T * 2 * D});
  }
  return t;
}
static const char kPackMagic[8] = {'S', 'T', 'K', 'P', 'A', 'C', 'K', '3'};
static bool same_model(const selftok_config_t& a, const selftok_config_t& b) {
  selftok_config_t x = a, y = b;
  x.device = y.device = 0;
  return memcmp(&x, &y, sizeof(x)) == 0;
}
namespace {
struct PackIO {
  FILE* f = nullptr;
  void* bounce = nullptr;                                     // pinned staging buffer
  static constexpr size_t CH = 64u << 20;
  ~PackIO() { if (f) fclose(f); if (bounce) cudaFreeHost(bounce); }
  bool w(const void* p, size_t n) { return fwrite(p, 1, n, f) == n; }
  bool r(void* p, size_t n) { return fread(p, 1, n, f) == n; }
  bool wdev(const void* d, size_t n) {
    for (size_t o = 0; o < n; o += CH) {
      const size_t m = n - o < CH ? n - o : CH;
      if (cudaMemcpy(bounce, (const char*)d + o, m, cudaMemcpyDeviceToHost) != cudaSuccess || !w(bounce, m)) return false;
    }
    return true;
  }
  bool rdev(void* d, size_t n) {
    for (size_t o = 0; o < n; o += CH) {
      const size_t m = n - o < CH ? n - o : CH;
      if (!r(bounce, m) || cudaMemcpy((char*)d + o, bounce, m, cudaMemcpyHostToDevice) != cudaSuccess) return false;
    }
    return true;
  }
  bool wstr(const std::string& s) { uint32_t n = (uint32_t)s.size(); return w(&n, 4) && w(s.data(), n); }
  bool rstr(std::string& s) { uint32_t n = 0; if (!r(&n, 4) || n > 4096) return false; s.resize(n); return r(&s[0], n); }
};
}  // namespace

extern "C" __attribute__((visibility("default"))) int selftok_export_packed(selftok_handle_t e, const char* path) {
  STK_CHECK(e && path, SELFTOK_ERR_BAD_ARG, "selftok_export_packed: bad argument");
  STK_CHECK(e->finalized, SELFTOK_ERR_STATE, "selftok_export_packed: finalize first");
  STK_CUDA(cudaSetDevice(e->cfg.device));
  STK_CUDA(cudaDeviceSynchronize());
  PackIO io;
  const std::string tmp = std::string(path) + ".tmp";
  io.f = fopen(tmp.c_str(), "wb");
  STK_CHECK(io.f, SELFTOK_ERR_BAD_ARG, "selftok_export_packed: cannot open the file for writing");
  STK_CUDA(cudaMallocHost(&io.bounce, PackIO::CH));
  bool ok = io.w(kPackMagic, 8);
  const uint32_t cfg_bytes = sizeof(selftok_config_t), steps = (uint32_t)e->steps, has_cfg = e->has_cfg ? 1u : 0u;
  ok = ok && io.w(&cfg_bytes, 4) && io.w(&e->cfg, cfg_bytes) && io.w(&has_cfg, 4) && io.w(&steps, 4) && io.w(e->t.data(), 4 * steps) &&
       io.w(e->dt.data(), 4 * steps) && io.w(e->k.data(), 4 * steps);
  const uint32_t n_w = (uint32_t)e->w.size(), n_p = (uint32_t)e->wp.size();
  ok = ok && io.w(&n_w, 4);
  for (auto& kv : e->w) {
    if (!ok) break;
    const Tensor& t = kv.second;
    const uint32_t nd = (uint32_t)t.shape.size(), has = t.d != nullptr;
    ok = io.wstr(kv.first) && io.w(&nd, 4) && io.w(t.shape.data(), 8 * nd) && io.w(&has, 4);
    if (ok && has) ok = io.wdev(t.d, sizeof(float) * (size_t)t.numel);
  }
  ok = ok && io.w(&n_p, 4);
  for (auto& kv : e->wp) {
    if (!ok) break;
    const int64_t numel = e->w[kv.first].numel;
    // kind 0: one 16-bit plane, 1: hi + lo planes, 2: e4m3 codes (1 byte each) + [N] fp32 scales
    const uint32_t kind = kv.second.scale ? 2u : kv.second.lo != nullptr ? 1u : 0u;
    ok = io.wstr(kv.first) && io.w(&numel, 8) && io.w(&kind, 4) && io.wdev(kv.second.hi, (kind == 2 ? 1 : 2) * (size_t)numel);
    if (ok && kind == 1) ok = io.wdev(kv.second.lo, 2 * (size_t)numel);
    if (ok && kind == 2) {
      const int64_t n = e->w[kv.first].shape[0];
      ok = io.w(&n, 8) && io.wdev(kv.second.scale, sizeof(float) * (size_t)n);
    }
  }
  for (const TableRef& t : table_refs(e)) {
    if (!ok) break;
    ok = io.wstr(t.tag) && io.w(&t.numel, 8) && io.wdev(*t.ptr, sizeof(float) * (size_t)t.numel);
  }
  fclose(io.f);
  io.f = nullptr;
  if (!ok) { remove(tmp.c_str()); set_error("selftok_export_packed: write failed"); return SELFTOK_ERR_CUDA; }
  STK_CHECK(rename(tmp.c_str(), path) == 0, SELFTOK_ERR_BAD_ARG, "selftok_export_packed: rename failed");
  return SELFTOK_OK;
}

// Fresh handle (selftok_create only) -> the finalized state of the file.  The file must have been exported for the same
// model configuration, precision and schedule length; anything else is SELFTOK_ERR_BAD_ARG and the handle stays fresh.
extern "C" __attribute__((visibility("default"))) int selftok_import_packed(selftok_handle_t e, const char* path) {
  STK_CHECK(e && path, SELFTOK_ERR_BAD_ARG, "selftok_import_packed: bad argument");
  STK_CHECK(!e->finalized && e->w.empty() && e->steps == 0, SELFTOK_ERR_STATE, "selftok_import_packed: the handle is not fresh");
  STK_CUDA(cudaSetDevice(e->cfg.device));
  PackIO io;
  io.f = fopen(path, "rb");
  STK_CHECK(io.f, SELFTOK_ERR_BAD_ARG, "selftok_import_packed: cannot open the file");
  char magic[8];
  uint32_t cfg_bytes = 0, steps = 0;
  selftok_config_t fc;
  STK_CHECK(io.r(magic, 8) && memcmp(magic, kPackMagic, 8) == 0 && io.r(&cfg_bytes, 4) && cfg_bytes == sizeof(fc) && io.r(&fc, cfg_bytes),
            SELFTOK_ERR_BAD_ARG, "selftok_import_packed: not a selftok_b200 pack file of this ABI");
  STK_CHECK(same_model(fc, e->cfg), SELFTOK_ERR_BAD_ARG, "selftok_import_packed: the file was exported for another configuration / precision");
  uint32_t has_cfg = 0;
  STK_CHECK(io.r(&has_cfg, 4) && io.r(&steps, 4) && steps > 0 && steps < 100000, SELFTOK_ERR_BAD_ARG, "selftok_import_packed: bad header");
  e->has_cfg = has_cfg != 0;
  STK_CUDA(cudaMallocHost(&io.bounce, PackIO::CH));
  e->steps = (int)steps;
  e->t.resize(steps); e->dt.resize(steps); e->k.resize(steps);
  bool ok = io.r(e->t.data(), 4 * steps) && io.r(e->dt.data(), 4 * steps) && io.r(e->k.data(), 4 * steps);
  uint32_t n_w = 0, n_p = 0;
  ok = ok && io.r(&n_w, 4) && n_w < 100000;
  for (uint32_t i = 0; ok && i < n_w; ++i) {
    std::string name;
    uint32_t nd = 0, has = 0;
    Tensor t;
    ok = io.rstr(name) && io.r(&nd, 4) && nd <= 8;
    if (!ok) break;
    t.shape.resize(nd);
    ok = io.r(t.shape.data(), 8 * nd) && io.r(&has, 4);
    t.numel = 1;
    for (int64_t d : t.shape) t.numel *= d;
    if (ok && has) {
      ok = cudaMalloc(&t.d, sizeof(float) * (size_t)t.numel) == cudaSuccess && io.rdev(t.d, sizeof(float) * (size_t)t.numel);
      e->bytes += t.numel * 4;
    }
    e->w[name] = t;
  }
  ok = ok && io.r(&n_p, 4) && n_p < 100000;
  for (uint32_t i = 0; ok && i < n_p; ++i) {
    std::string name;
    int64_t numel = 0;
    uint32_t kind = 0;
    WPack pk;
    ok = io.rstr(name) && io.r(&numel, 8) && io.r(&kind, 4) && numel > 0 && kind <= 2;
    if (!ok) break;
    if (kind == 2) {                                          // e4m3 codes + per-channel scales
      uint8_t* codes = nullptr;
      int64_t n = 0;
      ok = dalloc(e, e->allocs, &codes, numel) == 0 && io.rdev(codes, (size_t)numel) && io.r(&n, 8) && n > 0 && numel % n == 0 &&
           dalloc(e, e->allocs, &pk.scale, n) == 0 && io.rdev(pk.scale, sizeof(float) * (size_t)n);
      pk.hi = reinterpret_cast<bf16*>(codes);
    } else {
      ok = dalloc(e, e->allocs, &pk.hi, numel) == 0 && io.rdev(pk.hi, 2 * (size_t)numel);
      if (ok && kind == 1) ok = dalloc(e, e->allocs, &pk.lo, numel) == 0 && io.rdev(pk.lo, 2 * (size_t)numel);
    }
    e->wp[name] = pk;
  }
  for (const TableRef& t : table_refs(e)) {
    if (!ok) break;
    std::string tag;
    int64_t numel = 0;
    ok = io.rstr(tag) && tag == t.tag && io.r(&numel, 8) && numel == t.numel && dalloc(e, e->allocs, t.ptr, numel) == 0 &&
         io.rdev(*t.ptr, sizeof(float) * (size_t)numel);
  }
  if (!ok) {
    set_error("selftok_import_packed: truncated or mismatching pack file (destroy the handle)");
    return SELFTOK_ERR_BAD_ARG;
  }
  e->finalized = true;
  return SELFTOK_OK;
}

// ------------------------------------------------------------------------------------------------ encode
static int64_t lat_elems(const selftok_engine* e) { return (int64_t)e->cfg.in_channels * e->lat_h * e->lat_w; }   // per image

static int layout_ews(selftok_engine* e, EncodeWs& w, int64_t B, Arena& A) {
  const selftok_config_t& c = e->cfg;
  const int64_t Ni = e->Nenc, K = c.K, Hh = c.enc_hidden, Q = c.enc_qdim;
  STK_TRY(A.take(&w.x0, B * lat_elems(e)));
  STK_TRY(A.take(&w.patch, B * Ni * c.in_channels * c.enc_patch * c.enc_patch));
  STK_TRY(A.take(&w.x, B * Ni * Hh));
  STK_TRY(A.take(&w.q, B * K * Q));
  STK_TRY(A.take(&w.xn, B * Ni * Hh));
  STK_TRY(A.take(&w.qn, B * K * Q));
  STK_TRY(A.take(&w.xqkv, B * Ni * 3 * Hh));
  STK_TRY(A.take(&w.xkv, B * Ni * 2 * Q));
  STK_TRY(A.take(&w.qqkv, B * K * 3 * Q));
  STK_TRY(A.take(&w.xattn, B * Ni * Hh));
  STK_TRY(A.take(&w.qattn, B * K * Q));
  STK_TRY(A.take(&w.xh, B * Ni * 4 * Hh));
  STK_TRY(A.take(&w.qh, B * K * 4 * Q));
  STK_TRY(A.take(&w.outs_q, B * K * c.code_dim));
  STK_TRY(A.take(&w.tokens, B * K));
  return 0;
}
// Carve the workspace of `op` (0 encode, 1 decode / render) for batch B at the current geometry.  The carve is a function of
// (block, B, geometry) alone, so a graph captured for a (B, geometry) finds its buffers where it left them as long as the block
// stays.  The block stays while the layout fits in it; otherwise every graph pointing into it is dropped and the layout moves to
// the caller's block if that is large enough, else to one cudaMalloc of exactly the needed size.
template <typename WS, typename LAYOUT, typename DROP>
static int place_ws(selftok_engine* e, int op, WS& w, int B, LAYOUT layout, DROP drop_graphs) {
  if (w.base && w.B == B && w.lh == e->lat_h && w.lw == e->lat_w) return 0;
  Arena dry;
  dry.dry = true;
  WS scratch;
  STK_TRY(layout(scratch, (int64_t)B, dry));
  if (!w.base || w.cap < dry.off) {
    drop_graphs();
    if (w.own) { cudaFree(w.own); e->bytes -= (int64_t)w.own_bytes; }
    w.own = nullptr; w.own_bytes = 0; w.base = nullptr; w.cap = 0; w.B = 0;
    if (e->user_ws[op] && e->user_ws_bytes[op] >= dry.off) {
      w.base = reinterpret_cast<char*>(e->user_ws[op]);
      w.cap = e->user_ws_bytes[op];
    } else {
      STK_CUDA(cudaMalloc(&w.own, dry.off));
      w.own_bytes = dry.off;
      e->bytes += (int64_t)dry.off;
      w.base = reinterpret_cast<char*>(w.own);
      w.cap = dry.off;
    }
  }
  Arena A;
  A.base = w.base;
  A.cap = w.cap;
  STK_TRY(layout(w, (int64_t)B, A));
  w.B = B; w.lh = e->lat_h; w.lw = e->lat_w;
  return 0;
}
static int ensure_ews(selftok_engine* e, int B) {
  return place_ws(e, 0, e->ews, B, [&](EncodeWs& w, int64_t b, Arena& A) { return layout_ews(e, w, b, A); },
                  [&] { drop_encode_graphs(e); });
}

// The patch grid of the current geometry must fit the positional grid of the encoder (enc = true) or the MMDiT.
static int check_grid(selftok_engine* e, bool enc, const char* who) {
  const selftok_config_t& c = e->cfg;
  const int p = enc ? c.enc_patch : c.dit_patch, mx = enc ? c.enc_pos_max : c.dit_pos_max;
  if (e->lat_h / p > mx || e->lat_w / p > mx) {
    set_error(std::string(who) + ": latent " + std::to_string(e->lat_h) + " x " + std::to_string(e->lat_w) + " is a " +
              std::to_string(e->lat_h / p) + " x " + std::to_string(e->lat_w / p) + " patch grid, beyond the " +
              (enc ? "encoder" : "MMDiT") + " positional grid of " + std::to_string(mx) + " x " + std::to_string(mx) +
              " (latent sides up to " + std::to_string(mx * p) + ")");
    return SELFTOK_ERR_UNSUPPORTED;
  }
  return 0;
}

// Points e->pos_cur[enc ? 0 : 1] at the centre crop of the encoder's / MMDiT's positional grid for the current geometry
// (top = (max - gh) / 2, left = (max - gw) / 2: cropped_pos_embed, models_ours.py:183-202, sd3/mmdit.py:877-896).  The default
// geometry uses the table built at finalize; any other one is cropped from the full grid once, on the calling stream (so never
// inside a capture: call this before one), and kept until selftok_destroy.
static int pos_table(selftok_engine* e, bool enc, cudaStream_t s) {
  const selftok_config_t& c = e->cfg;
  const int i = enc ? 0 : 1;
  if (e->lat_h == c.latent && e->lat_w == c.latent) {
    e->pos_cur[i] = enc ? e->enc_pos : e->dit_pos;
    return 0;
  }
  STK_TRY(check_grid(e, enc, "positional table"));
  const int p = enc ? c.enc_patch : c.dit_patch, mx = enc ? c.enc_pos_max : c.dit_pos_max, dim = enc ? c.enc_hidden : e->D;
  const int gh = e->lat_h / p, gw = e->lat_w / p;
  auto it = e->pos_crops[i].find(std::make_pair(gh, gw));
  if (it == e->pos_crops[i].end()) {
    GETW(pe, enc ? "encoder.pos_embed" : "model.pos_embed");
    float* t;
    STK_TRY(dalloc(e, e->allocs, &t, (int64_t)gh * gw * dim));
    const int64_t l0 = g_launch_count;                      // a one-time table build, not a launch of the call
    STK_TRY(launch_crop_pos(pe->d, t, mx, gh, gw, (mx - gh) / 2, (mx - gw) / 2, dim, s));
    g_launch_count = l0;
    it = e->pos_crops[i].emplace(std::make_pair(gh, gw), t).first;
  }
  e->pos_cur[i] = it->second;
  return 0;
}

extern "C" __attribute__((visibility("default"))) int selftok_set_latent_size(selftok_handle_t e, int lat_h, int lat_w) {
  STK_CHECK(e, SELFTOK_ERR_BAD_ARG, "null handle");
  const selftok_config_t& c = e->cfg;
  const std::string hw = std::to_string(lat_h) + " x " + std::to_string(lat_w);
  if (lat_h <= 0 || lat_w <= 0 || lat_h % c.dit_patch || lat_w % c.dit_patch || lat_h % c.enc_patch || lat_w % c.enc_patch) {
    set_error("selftok_set_latent_size: latent " + hw + ": both sides must be positive multiples of dit_patch (" +
              std::to_string(c.dit_patch) + ") and enc_patch (" + std::to_string(c.enc_patch) + ")");
    return SELFTOK_ERR_BAD_ARG;
  }
  const bool dit_ok = lat_h / c.dit_patch <= c.dit_pos_max && lat_w / c.dit_patch <= c.dit_pos_max;
  const bool enc_ok = lat_h / c.enc_patch <= c.enc_pos_max && lat_w / c.enc_patch <= c.enc_pos_max;
  if (!dit_ok && !enc_ok) {
    set_error("selftok_set_latent_size: latent " + hw + " is beyond both positional grids (latent sides up to " +
              std::to_string(c.dit_pos_max * c.dit_patch) + " for decode, " + std::to_string(c.enc_pos_max * c.enc_patch) +
              " for encode)");
    return SELFTOK_ERR_UNSUPPORTED;
  }
  if (c.renderer && (lat_h != c.latent || lat_w != c.latent)) {
    set_error("selftok_set_latent_size: a renderer handle serves " + std::to_string(c.latent) + " x " + std::to_string(c.latent) +
              " latents only (model.positional_embedding has a fixed number of rows), got " + hw);
    return SELFTOK_ERR_UNSUPPORTED;
  }
  e->lat_h = lat_h;
  e->lat_w = lat_w;
  e->Nimg = (lat_h / c.dit_patch) * (lat_w / c.dit_patch);
  e->Nenc = (lat_h / c.enc_patch) * (lat_w / c.enc_patch);
  return SELFTOK_OK;
}

// Encoder.forward up to the quantizer input (models_ours.py:204-219,315-343; modules.py:310-327)
static int encoder_features(selftok_engine* e, const float* x0, int B, cudaStream_t s) {
  EncodeWs& w = e->ews;
  const selftok_config_t& c = e->cfg;
  const int Ni = e->Nenc, K = c.K, Hh = c.enc_hidden, Q = c.enc_qdim;
  const int64_t Mx = (int64_t)B * Ni, Mq = (int64_t)B * K;
  const float eps = 1e-6f;
  PROF(PC_OTHER, launch_patchify(x0, w.patch, B, c.in_channels, e->lat_h, e->lat_w, c.enc_patch, s));
  {
    Epilogue ep;
    ep.out = w.x; ep.addtab = e->pos_cur[0]; ep.add_ld = Hh; ep.add_period = Ni;
    STK_TRY(lin32(e, "encoder.x_embedder.proj", w.patch, c.in_channels * c.enc_patch * c.enc_patch, Mx, ep, s));
    GETW(qt, "encoder.query_tokens");
    STK_CHECK(qt->numel == (int64_t)K * Q, SELFTOK_ERR_BAD_ARG, "query_tokens shape");
    PROF(PC_OTHER, launch_bcast_rows(qt->d, nullptr, w.q, B, K, Q, s));
  }
  for (int i = 0; i < c.enc_depth; ++i) {
    const std::string p = "encoder.blocks." + std::to_string(i) + ".";
    const float* mod = e->enc_mod + (int64_t)i * K * 6 * Q;     // [K][shift_msa|scale_msa|gate_msa|shift_mlp|scale_mlp|gate_mlp]
    PROF(PC_LN, launch_ln_mod(w.x, Hh, nullptr, nullptr, 0, 1, w.xn, nullptr, nullptr, Hh, Mx, Hh, eps, s));
    PROF(PC_LN, launch_ln_mod(w.q, Q, mod, mod + Q, 6 * Q, K, w.qn, nullptr, nullptr, Q, Mq, Q, eps, s));
    Epilogue ep;
    ep.out = w.xqkv; STK_TRY(lin32(e, p + "attn.qkv", w.xn, Hh, Mx, ep, s));
    ep.out = w.xkv; STK_TRY(lin32(e, p + "attn.to_query_kv", w.xn, Hh, Mx, ep, s));
    ep.out = w.qqkv; STK_TRY(lin32(e, p + "attn.query_linear", w.qn, Q, Mq, ep, s));
    AttnOut ox;
    ox.f32_a = w.xattn; ox.split = Ni; ox.ld = Hh;
    PROF(PC_ATTN, launch_attention_f32(w.xqkv, 3 * Hh, (int64_t)Ni * 3 * Hh, w.xqkv + Hh, w.xqkv + 2 * Hh, 3 * Hh, (int64_t)Ni * 3 * Hh, Ni,
                                 nullptr, nullptr, 0, 0, 0, ox, B, Ni, c.enc_heads, Hh / c.enc_heads, 0, 0, s));
    AttnOut oq;
    oq.f32_a = w.qattn; oq.split = K; oq.ld = Q;
    PROF(PC_ATTN, launch_attention_f32(w.qqkv, 3 * Q, (int64_t)K * 3 * Q, w.xkv, w.xkv + Q, 2 * Q, (int64_t)Ni * 2 * Q, Ni,
                                 w.qqkv + Q, w.qqkv + 2 * Q, 3 * Q, (int64_t)K * 3 * Q, K, oq, B, K, c.enc_qheads,
                                 Q / c.enc_qheads, 0, 0, s));
    // image stream: x += proj(x_attn); x += mlp(norm2(x))
    Epilogue er;
    er.mode = EPI_RESID; er.out = w.x; er.resid = w.x; er.ldo = Hh;
    STK_TRY(lin32(e, p + "attn.proj", w.xattn, Hh, Mx, er, s));
    PROF(PC_LN, launch_ln_mod(w.x, Hh, nullptr, nullptr, 0, 1, w.xn, nullptr, nullptr, Hh, Mx, Hh, eps, s));
    Epilogue eg;
    eg.act = ACT_GELU; eg.out = w.xh;
    STK_TRY(lin32(e, p + "mlp.fc1", w.xn, Hh, Mx, eg, s));
    STK_TRY(lin32(e, p + "mlp.fc2", w.xh, 4 * Hh, Mx, er, s));
    // query stream: q += gate_msa * query_proj(q_attn); q += gate_mlp * q_mlp(modulate(norm2(q)))
    Epilogue eq;
    eq.mode = EPI_RESID; eq.out = w.q; eq.resid = w.q; eq.ldo = Q; eq.gate = mod + 2 * Q; eq.gate_ld = 6 * Q; eq.gate_period = K;
    STK_TRY(lin32(e, p + "attn.query_proj", w.qattn, Q, Mq, eq, s));
    PROF(PC_LN, launch_ln_mod(w.q, Q, mod + 3 * Q, mod + 4 * Q, 6 * Q, K, w.qn, nullptr, nullptr, Q, Mq, Q, eps, s));
    eg.out = w.qh;
    STK_TRY(lin32(e, p + "q_mlp.fc1", w.qn, Q, Mq, eg, s));
    eq.gate = mod + 5 * Q;
    STK_TRY(lin32(e, p + "q_mlp.fc2", w.qh, 4 * Q, Mq, eq, s));
  }
  return 0;
}

static int run_vq(selftok_engine* e, const float* z, int64_t R, int64_t* ids, float* outs_q, cudaStream_t s) {
  const selftok_config_t& c = e->cfg;
  GETW(wi, "encoder.quantizer.project_in.weight");
  GETW(bi, "encoder.quantizer.project_in.bias");
  GETW(cb, "encoder.quantizer._codebook.embed");
  GETW(lw, "encoder.final_layer_norm3.weight");
  GETW(lb, "encoder.final_layer_norm3.bias");
  PROF(PC_VQ, launch_vq(z, R, c.enc_qdim, wi->d, bi->d, cb->d, e->cbt, c.codebook_size, c.code_dim, lw->d, lb->d, ids, outs_q, s));
  return 0;
}

#define HOT_PROLOGUE(e)                                                                  \
  STK_CHECK(e, SELFTOK_ERR_BAD_ARG, "null handle");                                      \
  STK_CHECK(e->finalized, SELFTOK_ERR_STATE, "selftok_finalize has not been called");    \
  STK_CUDA(cudaSetDevice(e->cfg.device));                                                \
  cudaStream_t s = (cudaStream_t)stream;                                                 \
  const int64_t launches0 = g_launch_count;

extern "C" __attribute__((visibility("default"))) int selftok_encode(selftok_handle_t e, const float* x0_dev, int B, int64_t* tokens_dev, float* outs_q_dev,
                              float* feats_dev, void* stream) {
  HOT_PROLOGUE(e);
  STK_CHECK(x0_dev && tokens_dev && B > 0, SELFTOK_ERR_BAD_ARG, "selftok_encode: bad argument");
  STK_TRY(check_grid(e, true, "selftok_encode"));
  STK_TRY(ensure_ews(e, B));
  STK_TRY(pos_table(e, true, s));
  const int64_t R = (int64_t)B * e->cfg.K;
  EncodeWs& w = e->ews;
  if (!e->use_graph || e->prof_on) {                       // eager (per-launch profiling needs real launches)
    STK_TRY(encoder_features(e, x0_dev, B, s));
    STK_TRY(run_vq(e, w.q, R, tokens_dev, outs_q_dev ? outs_q_dev : w.outs_q, s));
    e->last_launches = g_launch_count - launches0;
  } else {
    // one CUDA graph per batch size over the workspace's own input / output buffers (the ~250 launches of the 16 dual blocks
    // dominate a small-batch encode when issued one by one); the caller's buffers are copied in and out around the replay
    const int64_t nlat = (int64_t)B * lat_elems(e);
    if (x0_dev != w.x0) STK_CUDA(cudaMemcpyAsync(w.x0, x0_dev, sizeof(float) * nlat, cudaMemcpyDeviceToDevice, s));
    const auto key = std::make_tuple(B, e->lat_h, e->lat_w);
    auto it = e->enc_graphs.find(key);
    if (it == e->enc_graphs.end()) {
      cudaStream_t cs;
      STK_CUDA(cudaStreamCreateWithFlags(&cs, cudaStreamNonBlocking));
      {
        const cudaError_t be = cudaStreamBeginCapture(cs, cudaStreamCaptureModeThreadLocal);
        if (be != cudaSuccess) {
          cudaStreamDestroy(cs);
          STK_CUDA(be);
        }
      }
      const int64_t l0 = g_launch_count;
      int st = encoder_features(e, w.x0, B, cs);
      if (!st) st = run_vq(e, w.q, R, w.tokens, w.outs_q, cs);
      cudaGraph_t graph = nullptr;
      cudaError_t ce = cudaStreamEndCapture(cs, &graph);
      cudaStreamDestroy(cs);
      if (st != 0) { if (graph) cudaGraphDestroy(graph); return st; }
      STK_CUDA(ce);
      cudaGraphExec_t exec;
      STK_CUDA(cudaGraphInstantiate(&exec, graph, 0));
      cudaGraphDestroy(graph);
      it = e->enc_graphs.emplace(key, std::make_pair(exec, g_launch_count - l0)).first;
    }
    STK_CUDA(cudaGraphLaunch(it->second.first, s));
    e->last_launches = it->second.second;
    if (tokens_dev != w.tokens) STK_CUDA(cudaMemcpyAsync(tokens_dev, w.tokens, sizeof(int64_t) * R, cudaMemcpyDeviceToDevice, s));
    if (outs_q_dev && outs_q_dev != w.outs_q)
      STK_CUDA(cudaMemcpyAsync(outs_q_dev, w.outs_q, sizeof(float) * R * e->cfg.code_dim, cudaMemcpyDeviceToDevice, s));
  }
  if (feats_dev) STK_CUDA(cudaMemcpyAsync(feats_dev, w.q, sizeof(float) * R * e->cfg.enc_qdim, cudaMemcpyDeviceToDevice, s));
  return SELFTOK_OK;
}

extern "C" __attribute__((visibility("default"))) int selftok_vq_argmax(selftok_handle_t e, const float* z_dev, int64_t R, int64_t* ids_dev, float* outs_q_dev,
                                 void* stream) {
  HOT_PROLOGUE(e);
  STK_CHECK(z_dev && ids_dev && R > 0, SELFTOK_ERR_BAD_ARG, "selftok_vq_argmax: bad argument");
  STK_TRY(run_vq(e, z_dev, R, ids_dev, outs_q_dev, s));
  e->last_launches = g_launch_count - launches0;
  return SELFTOK_OK;
}

// range != NULL: device [B][2] token windows; ids outside an image's window are not read (zero rows)
// gather != NULL: R rows of a packed context stream, row m from tokens[gather[m]]
static int run_lookup(selftok_engine* e, const int64_t* tokens, int B, float* outs_q, cudaStream_t s, const int* range = nullptr,
                      const int* gather = nullptr, int64_t R = 0) {
  GETW(cb, "encoder.quantizer._codebook.embed");
  GETW(lw, "encoder.final_layer_norm3.weight");
  GETW(lb, "encoder.final_layer_norm3.bias");
  PROF(PC_OTHER, launch_lookup_ln3(tokens, gather ? R : (int64_t)B * e->cfg.K, cb->d, e->cfg.codebook_size, e->cfg.code_dim, lw->d, lb->d,
                                   outs_q, e->bad_ids, s, range, e->cfg.K, gather));
  return 0;
}

// Synchronises `stream`, returns how many token ids outside [0, codebook_size) the lookups on this handle have seen since
// the last call (their rows were poisoned with NaN) and resets the counter; < 0 on a CUDA error.
extern "C" __attribute__((visibility("default"))) int64_t selftok_id_errors(selftok_handle_t e, void* stream) {
  if (!e || !e->bad_ids) return -1;
  int n = 0;
  if (cudaSetDevice(e->cfg.device) != cudaSuccess) return -1;
  cudaStream_t s = (cudaStream_t)stream;
  if (cudaMemcpyAsync(&n, e->bad_ids, sizeof(int), cudaMemcpyDeviceToHost, s) != cudaSuccess) return -1;
  if (cudaMemsetAsync(e->bad_ids, 0, sizeof(int), s) != cudaSuccess) return -1;
  if (cudaStreamSynchronize(s) != cudaSuccess) return -1;
  return n;
}
static int check_ids_after_sync(selftok_engine* e, void* stream, const char* who) {
  const int64_t n = selftok_id_errors(e, stream);
  STK_CHECK(n >= 0, SELFTOK_ERR_CUDA, "selftok_id_errors failed");
  if (n > 0) {
    set_error(std::string(who) + ": " + std::to_string(n) + " token id(s) outside [0, codebook_size)");
    return SELFTOK_ERR_BAD_ARG;
  }
  return 0;
}

extern "C" __attribute__((visibility("default"))) int selftok_lookup(selftok_handle_t e, const int64_t* tokens_dev, int B, float* outs_q_dev, void* stream) {
  HOT_PROLOGUE(e);
  STK_CHECK(tokens_dev && outs_q_dev && B > 0, SELFTOK_ERR_BAD_ARG, "selftok_lookup: bad argument");
  STK_TRY(run_lookup(e, tokens_dev, B, outs_q_dev, s));
  e->last_launches = g_launch_count - launches0;
  return SELFTOK_OK;
}

// ------------------------------------------------------------------------------------------------ decode
// A step call (selftok_decode_step) runs one Euler step for images at their own schedule rows over a PACKED context stream: image
// b contributes exactly its c_b visible rows, at stream rows [off_b, off_b + c_b).  Its joint-attention slot of S = max c + N rows
// holds those c_b rows, then its N image rows.  Per-image block uploaded once per call (ws.pk, int32):
//   [B][2] (off_b, c_b) | [B] lo_b | [B] step_b | [B] dt of step_b (float) | [B] cfg scale (float)
// followed by the per-row maps launch_expand_packed derives from it on the device.
constexpr int PK_IMG_INTS = 6;
struct Packed {
  int Mc = 0, S = 0;                                   // context stream rows (sum of c_b), joint slot rows
  const int* pair = nullptr;                           // [B][2] (off_b, c_b)
  const float *dt = nullptr, *scale = nullptr;         // [B]
  const int *ctx_tok = nullptr, *ctx_pos = nullptr, *ctx_step = nullptr, *ctx_dst = nullptr;   // [Mc]
  const int* x_step = nullptr;                         // [B N]
};
static int layout_dws(selftok_engine* e, DecodeWs& w, int64_t B, Arena& A) {
  const selftok_config_t& c = e->cfg;
  const int64_t K = c.K, N = e->Nimg, D = e->D, S = K + N;
  STK_TRY(A.take(&w.tokens, B * K));
  STK_TRY(A.take(&w.outs_q, B * K * c.code_dim));
  STK_TRY(A.take(&w.x_lat, B * lat_elems(e)));
  STK_TRY(A.take(&w.patch, B * N * c.in_channels * c.dit_patch * c.dit_patch));
  STK_TRY(A.take(&w.ctx0, B * K * D));
  STK_TRY(A.take(&w.ctx, B * K * D));
  STK_TRY(A.take(&w.x, B * N * D));
  STK_TRY(A.take(&w.o_final, B * N * c.dit_patch * c.dit_patch * c.in_channels));
  STK_TRY(A.take(&w.o_final_u, B * N * c.dit_patch * c.dit_patch * c.in_channels));
  STK_TRY(A.take(&w.a_x, B * N * D));                       // fp32 LN output of the final layer (both modes)
  STK_TRY(A.take(&w.plan, B * 2 * (1 + (int64_t)e->steps)));
  STK_TRY(A.take(&w.pk, B * (PK_IMG_INTS + 4 * K + N)));
  if (!tc_mode(e)) {
    STK_TRY(A.take(&w.qkv, B * S * 3 * D));
    STK_TRY(A.take(&w.a_c, B * K * D));
    STK_TRY(A.take(&w.attn_c, B * K * D));
    STK_TRY(A.take(&w.attn_x, B * N * D));
    STK_TRY(A.take(&w.h_c, B * K * 4 * D));
    STK_TRY(A.take(&w.h_x, B * N * 4 * D));
  } else {
    const bool lo = nsplit(e) == 3;
    STK_TRY(A.take(&w.patch_hi, B * N * c.in_channels * c.dit_patch * c.dit_patch));
    STK_TRY(A.take(&w.patch_lo, B * N * c.in_channels * c.dit_patch * c.dit_patch));
    STK_TRY(A.take(&w.fin_hi, B * N * D));
    STK_TRY(A.take(&w.fin_lo, B * N * D));
    STK_TRY(A.take(&w.qkv_hi, B * S * 3 * D));
    if (lo) STK_TRY(A.take(&w.qkv_lo, B * S * 3 * D));
    STK_TRY(A.take(&w.a_c_hi, B * K * D));
    STK_TRY(A.take(&w.a_x_hi, B * N * D));
    STK_TRY(A.take(&w.attn_c_hi, B * K * D));
    STK_TRY(A.take(&w.attn_x_hi, B * N * D));
    STK_TRY(A.take(&w.h_c_hi, B * K * 4 * D));
    STK_TRY(A.take(&w.h_x_hi, B * N * 4 * D));
    if (is_fp8(e)) {                                          // row scales of the e4m3 LN outputs (QKV / fc1 A operands)
      STK_TRY(A.take(&w.sa_c, B * K));
      STK_TRY(A.take(&w.sa_x, B * N));
    }
    if (lo) {
      STK_TRY(A.take(&w.a_c_lo, B * K * D));
      STK_TRY(A.take(&w.a_x_lo, B * N * D));
      STK_TRY(A.take(&w.attn_c_lo, B * K * D));
      STK_TRY(A.take(&w.attn_x_lo, B * N * D));
      STK_TRY(A.take(&w.h_c_lo, B * K * 4 * D));
      STK_TRY(A.take(&w.h_x_lo, B * N * 4 * D));
    }
  }
  return 0;
}
static void drop_decode_graphs(selftok_engine* e) {
  for (auto& g : e->graphs) cudaGraphExecDestroy(g.second.first);
  e->graphs.clear();
  for (auto& g : e->range_graphs) cudaGraphExecDestroy(g.second.first);
  e->range_graphs.clear();
}
static int ensure_dws(selftok_engine* e, int B) {
  return place_ws(e, 1, e->dws, B, [&](DecodeWs& w, int64_t b, Arena& A) { return layout_dws(e, w, b, A); },
                  [&] { drop_decode_graphs(e); });
}

// One stream of one JointBlock: LN+modulate -> qkv GEMM into the joint buffer   (mmdit.py:441-483, 521-529)
static int pre_attention(selftok_engine* e, const std::string& blk, const float* resid, int64_t M, const float* shift,
                         const float* scale, int64_t ld_mod, int period, float* a32, bf16* a_hi, bf16* a_lo, int rpb_in,
                         int S, int row_off, cudaStream_t s, const int* plan = nullptr, int plan_ctx = 0, const int* rows = nullptr,
                         const int* row_map = nullptr) {
  const int D = e->D;
  DecodeWs& w = e->dws;
  Epilogue ep;
  ep.out = w.qkv; ep.ldo = 3 * D; ep.rpb_in = rpb_in; ep.rpb_out = S; ep.row_off = row_off;
  ep.plan = plan; ep.plan_ctx = plan_ctx; ep.row_map = row_map;
  if (!tc_mode(e)) {
    PROF(PC_LN, launch_ln_mod(resid, D, shift, scale, ld_mod, period, a32, nullptr, nullptr, D, M, D, 1e-6f, s, 0, rows));
    return lin32(e, blk + "attn.qkv", a32, D, M, ep, s);
  }
  PROF(PC_LN, launch_ln_mod(resid, D, shift, scale, ld_mod, period, nullptr, a_hi, a_lo, D, M, D, 1e-6f, s, is_fp16(e), rows));
  ep.mode = EPI_SPLIT; ep.out = nullptr; ep.out_hi = w.qkv_hi; ep.out_lo = w.qkv_lo;      // q/k/v leave the GEMM as 16-bit planes
  return lintc(e, blk + "attn.qkv", a_hi, a_lo, M, ep, s);
}

// post_attention (mmdit.py:485-496): x += gate_msa*proj(attn); x += gate_mlp*mlp(modulate(norm2(x)))
static int post_attention(selftok_engine* e, const std::string& blk, float* resid, int64_t M, const float* mod, int64_t ld_mod,
                          int period, const float* attn32, const bf16* attn_hi, const bf16* attn_lo, float* a32, bf16* a_hi,
                          bf16* a_lo, float* h32, bf16* h_hi, bf16* h_lo, cudaStream_t s, const int* rows = nullptr) {
  const int D = e->D;
  Epilogue er;
  er.mode = EPI_RESID; er.out = resid; er.resid = resid; er.ldo = D;
  er.gate = mod + 2 * D; er.gate_ld = ld_mod; er.gate_period = period; er.tab_rows = rows;
  Epilogue eh;
  eh.act = ACT_GELU;
  if (!tc_mode(e)) {
    STK_TRY(lin32(e, blk + "attn.proj", attn32, D, M, er, s));
    PROF(PC_LN, launch_ln_mod(resid, D, mod + 3 * D, mod + 4 * D, ld_mod, period, a32, nullptr, nullptr, D, M, D, 1e-6f, s, 0, rows));
    eh.out = h32; eh.ldo = 4 * D;
    STK_TRY(lin32(e, blk + "mlp.fc1", a32, D, M, eh, s));
    er.gate = mod + 5 * D;
    return lin32(e, blk + "mlp.fc2", h32, 4 * D, M, er, s);
  }
  STK_TRY(lintc(e, blk + "attn.proj", attn_hi, attn_lo, M, er, s));
  PROF(PC_LN, launch_ln_mod(resid, D, mod + 3 * D, mod + 4 * D, ld_mod, period, nullptr, a_hi, a_lo, D, M, D, 1e-6f, s, is_fp16(e), rows));
  eh.mode = EPI_SPLIT; eh.out_hi = h_hi; eh.out_lo = h_lo; eh.ldo = 4 * D;
  STK_TRY(lintc(e, blk + "mlp.fc1", a_hi, a_lo, M, eh, s));
  er.gate = mod + 5 * D;
  return lintc(e, blk + "mlp.fc2", h_hi, h_lo, M, er, s);
}

// x = x_embedder(patches) + cropped pos_embed (mmdit.py:1000-1001) from ws.patch into ws.x.  Tensor-core modes: the K = 64 GEMM on
// the tensor-core kernel with split-bf16 operands (fp32-faithful) instead of the fp32 FFMA kernel (0.3 ms -> ~20 us per evaluation).
static int x_embed(selftok_engine* e, int B, cudaStream_t s) {
  const selftok_config_t& c = e->cfg;
  DecodeWs& w = e->dws;
  const int D = e->D, N = e->Nimg, Kp = c.in_channels * c.dit_patch * c.dit_patch;
  Epilogue ep;
  ep.out = w.x; ep.addtab = e->pos_cur[1]; ep.add_ld = D; ep.add_period = N;
  if (!tc_mode(e) || Kp % 8 != 0) return lin32(e, "model.x_embedder.proj", w.patch, Kp, (int64_t)B * N, ep, s);
  PROF(PC_OTHER, launch_split_bf16(w.patch, w.patch_hi, w.patch_lo, (int64_t)B * N * Kp, s, 0));
  GETW(Bv, "model.x_embedder.proj.bias");
  auto it = e->wp.find("model.x_embedder.proj.weight");
  STK_CHECK(it != e->wp.end(), SELFTOK_ERR_STATE, "packed x_embedder missing");
  ep.bias = Bv->d; ep.ldo = D;
  PROF(PC_GEMM_TC, launch_gemm_tc(w.patch_hi, w.patch_lo, it->second.hi, it->second.lo, (int64_t)B * N, D, Kp, 3, ep, s, 0));
  return 0;
}
// FinalLayer (mmdit.py:641-645): LN + modulate, then the N = p*p*C = 64 column linear -> o_out [B*N, 64] fp32
// rows != NULL: per-row rows of the fm table (packed step calls), else its single row
static int final_layer(selftok_engine* e, int B, const float* fm, float* o_out, cudaStream_t s, const int* rows = nullptr) {
  DecodeWs& w = e->dws;
  const int D = e->D;
  const int64_t Mx = (int64_t)B * e->Nimg;
  if (!tc_mode(e)) {
    PROF(PC_LN, launch_ln_mod(w.x, D, fm, fm + D, 2 * D, 1, w.a_x, nullptr, nullptr, D, Mx, D, 1e-6f, s, 0, rows));
    Epilogue ep;
    ep.out = o_out;
    return lin32(e, "model.final_layer.linear", w.a_x, D, Mx, ep, s);
  }
  LnProblem lp;
  lp.x = w.x; lp.shift = fm; lp.scale = fm + D; lp.ld_mod = 2 * D; lp.period = 1; lp.out_hi = w.fin_hi; lp.out_lo = w.fin_lo; lp.M = Mx;
  lp.rows = rows;
  PROF(PC_LN, launch_ln_mod_pair(&lp, 1, D, 1e-6f, s, 0));
  GETW(W, "model.final_layer.linear.weight");
  GETW(Bv, "model.final_layer.linear.bias");
  auto it = e->wp.find("model.final_layer.linear.weight");
  STK_CHECK(it != e->wp.end(), SELFTOK_ERR_STATE, "packed final layer missing");
  Epilogue ep;
  ep.out = o_out; ep.bias = Bv->d; ep.ldo = (int)W->shape[0];
  PROF(PC_GEMM_TC, launch_gemm_tc(w.fin_hi, w.fin_lo, it->second.hi, it->second.lo, Mx, (int)W->shape[0], D, 3, ep, s, 0));
  return 0;
}

// forward_core_with_concat (mmdit.py:918-933) on the residual streams already initialised in ws.ctx / ws.x.
//   Kc         visible context rows (prefix; rows >= Kc are dropped — exact, SURVEY 8a note)
//   step       row of the per-step tables (x adaLN, final adaLN, last-layer context adaLN)
//   ctx_self   context rows attend to context keys only (renderer; mmdit.py:1581)
//   uncond     unconditional branch of the guided sampler (MMDiT.cfg_inference, mmdit.py:1117-1163): Kc must be 0 (no row of
//              that pass sees a context key, so the context stream is dropped -- exact), x-stream adaLN from the integer timestep
//   o_out      final-layer output [B*N, p*p*C]
//   plan, Lo   token-range call: the context stream holds positions [Lo, Lo + Kc), and `plan` ([B][2] (a, c) of this step, device)
//              tells where each image's live rows are (Epilogue / AttnPlan); NULL: the prefix [0, Kc) of every image is live
//   pk         step call (Kc, step, plan and Lo unused): packed context stream of pk->Mc rows (Mc = 0: none), every table row
//              taken from the per-row maps
static int joint_blocks(selftok_engine* e, int B, int Kc, int step, bool ctx_self, cudaStream_t s, bool uncond = false,
                        float* o_out = nullptr, const int* plan = nullptr, int Lo = 0, const Packed* pk = nullptr) {
  const selftok_config_t& c = e->cfg;
  DecodeWs& w = e->dws;
  if (pk) { step = 0; Lo = 0; plan = pk->pair; Kc = pk->S - e->Nimg; }
  const int D = e->D, N = e->Nimg, L = c.dit_depth, T = e->steps, S = Kc + N;
  const int64_t Mc = pk ? pk->Mc : (int64_t)B * Kc, Mx = (int64_t)B * N;
  const bool ctx = Mc > 0;                                                      // is there a context stream in this pass at all
  STK_CHECK(!uncond || (!ctx && e->x_mod_u), SELFTOK_ERR_STATE, "unconditional pass needs the guided-sampler tables and no context");
  if (!ctx) plan = nullptr;
  AttnPlan ap;
  ap.plan = plan; ap.n_img = N; ap.ctx_self = ctx_self; ap.packed = pk && ctx;
  const float* x_mod_base = uncond ? e->x_mod_u : e->x_mod;
  // per-row table rows of a step call: context rows by position (last layer: by step), image rows by step
  const int* rows_c = pk ? pk->ctx_pos : nullptr;
  const int* rows_cl = pk ? pk->ctx_step : nullptr;
  const int* rows_x = pk ? pk->x_step : nullptr;
  const int* map_c = pk ? pk->ctx_dst : nullptr;
  for (int j = 0; j < L; ++j) {
    const bool last = j == L - 1;
    const bool ctx_post = ctx && !last;                                         // the last context block is pre_only
    const std::string pc = "model.joint_blocks." + std::to_string(j) + ".context_block.";
    const std::string px = "model.joint_blocks." + std::to_string(j) + ".x_block.";
    const float* cmod = e->ctx_mod + ((int64_t)j * c.K + Lo) * 6 * D;           // [K][6D], from position Lo
    const float* xmod = x_mod_base + ((int64_t)j * T + step) * 6 * D;           // [6D]
    if (tc_mode(e)) {
      // ---- tensor-core path: the two streams' GEMMs of every stage share one launch (lintc2)
      const int fp16 = is_fp16(e);
      // fp8 mode: the LN launches write e4m3 codes + row scales into a_*_hi, and the QKV / fc1 GEMMs run on e4m3
      const bool fp8 = is_fp8(e);
      const int ln16 = fp8 ? 0 : fp16;
      const float* lm = e->ctx_last_mod + (int64_t)step * 2 * D;                // last layer: pre_only (shift, scale) from c
      // LN + modulate of both streams in one launch (context rows: per-position adaLN table; image rows: the step's row)
      LnProblem lp[2];
      lp[0].x = w.ctx; lp[0].out_hi = w.a_c_hi; lp[0].out_lo = w.a_c_lo; lp[0].M = Mc;
      if (!last) { lp[0].shift = cmod; lp[0].scale = cmod + D; lp[0].ld_mod = 6 * D; lp[0].period = Kc; lp[0].rows = rows_c; }
      else { lp[0].shift = lm; lp[0].scale = lm + D; lp[0].ld_mod = 2 * D; lp[0].period = 1; lp[0].rows = rows_cl; }
      lp[1].x = w.x; lp[1].out_hi = w.a_x_hi; lp[1].out_lo = w.a_x_lo; lp[1].M = Mx;
      lp[1].shift = xmod; lp[1].scale = xmod + D; lp[1].ld_mod = 6 * D; lp[1].period = 1; lp[1].rows = rows_x;
      if (fp8) { lp[0].out_scale = w.sa_c; lp[1].out_scale = w.sa_x; }
      if (ctx) PROF(PC_LN, launch_ln_mod_pair(lp, 2, D, 1e-6f, s, ln16));
      else PROF(PC_LN, launch_ln_mod_pair(lp + 1, 1, D, 1e-6f, s, ln16));
      TcProblem pr[2];
      Epilogue eq;                                                              // q/k/v leave the GEMM as 16-bit planes in the joint buffer
      eq.mode = EPI_SPLIT; eq.out_hi = w.qkv_hi; eq.out_lo = w.qkv_lo; eq.ldo = 3 * D; eq.rpb_out = S; eq.plan = plan;
      int np = 0;
      eq.rpb_in = Kc; eq.row_off = 0; eq.plan_ctx = 1; eq.row_map = map_c;
      if (ctx) STK_TRY(tc_problem(e, pc + "attn.qkv", w.a_c_hi, w.a_c_lo, Mc, eq, &pr[np++], w.sa_c));
      eq.rpb_in = N; eq.row_off = Kc; eq.plan_ctx = 0; eq.row_map = nullptr;
      STK_TRY(tc_problem(e, px + "attn.qkv", w.a_x_hi, w.a_x_lo, Mx, eq, &pr[np++], w.sa_x));
      STK_TRY(lintc2(e, pr, np, s, fp8));
      AttnOut ao;
      ao.split = Kc; ao.ld = D;
      ao.hi_a = w.attn_c_hi; ao.lo_a = w.attn_c_lo; ao.hi_b = w.attn_x_hi; ao.lo_b = w.attn_x_lo;
      ao.fp16 = fp16;
      const int ctx_rows = ctx_self ? Kc : 0, ctx_keys = ctx_self ? Kc : 0;
      PROF(PC_ATTN, launch_attention_tc5(w.qkv_hi, B, S, e->H, ctx_rows, ctx_keys, ao, s, fp16, nsplit(e) == 3 ? w.qkv_lo : nullptr, ap));
      // post_attention (mmdit.py:485-496); the pre_only context block of the last layer stops here
      Epilogue erx, erc;
      erx.mode = EPI_RESID; erx.out = w.x; erx.resid = w.x; erx.ldo = D; erx.gate = xmod + 2 * D; erx.gate_ld = 6 * D; erx.gate_period = 1;
      erc.mode = EPI_RESID; erc.out = w.ctx; erc.resid = w.ctx; erc.ldo = D; erc.gate = cmod + 2 * D; erc.gate_ld = 6 * D; erc.gate_period = Kc;
      erx.tab_rows = rows_x; erc.tab_rows = rows_c;
      np = 0;
      if (ctx_post) STK_TRY(tc_problem(e, pc + "attn.proj", w.attn_c_hi, w.attn_c_lo, Mc, erc, &pr[np++]));
      STK_TRY(tc_problem(e, px + "attn.proj", w.attn_x_hi, w.attn_x_lo, Mx, erx, &pr[np++]));
      STK_TRY(lintc2(e, pr, np, s));
      lp[0].shift = cmod + 3 * D; lp[0].scale = cmod + 4 * D; lp[0].ld_mod = 6 * D; lp[0].period = Kc; lp[0].rows = rows_c;
      lp[1].shift = xmod + 3 * D; lp[1].scale = xmod + 4 * D;
      if (ctx_post) PROF(PC_LN, launch_ln_mod_pair(lp, 2, D, 1e-6f, s, ln16));
      else PROF(PC_LN, launch_ln_mod_pair(lp + 1, 1, D, 1e-6f, s, ln16));
      Epilogue ehc, ehx;
      ehc.mode = EPI_SPLIT; ehc.act = ACT_GELU; ehc.out_hi = w.h_c_hi; ehc.out_lo = w.h_c_lo; ehc.ldo = 4 * D;
      ehx = ehc; ehx.out_hi = w.h_x_hi; ehx.out_lo = w.h_x_lo;
      np = 0;
      if (ctx_post) STK_TRY(tc_problem(e, pc + "mlp.fc1", w.a_c_hi, w.a_c_lo, Mc, ehc, &pr[np++], w.sa_c));
      STK_TRY(tc_problem(e, px + "mlp.fc1", w.a_x_hi, w.a_x_lo, Mx, ehx, &pr[np++], w.sa_x));
      STK_TRY(lintc2(e, pr, np, s, fp8));
      erc.gate = cmod + 5 * D; erx.gate = xmod + 5 * D;
      np = 0;
      if (ctx_post) STK_TRY(tc_problem(e, pc + "mlp.fc2", w.h_c_hi, w.h_c_lo, Mc, erc, &pr[np++]));
      STK_TRY(tc_problem(e, px + "mlp.fc2", w.h_x_hi, w.h_x_lo, Mx, erx, &pr[np++]));
      STK_TRY(lintc2(e, pr, np, s));
      continue;
    }
    if (ctx && !last) {
      STK_TRY(pre_attention(e, pc, w.ctx, Mc, cmod, cmod + D, 6 * D, Kc, w.a_c, w.a_c_hi, w.a_c_lo, Kc, S, 0, s, plan, 1, rows_c, map_c));
    } else if (ctx) {
      const float* lm = e->ctx_last_mod + (int64_t)step * 2 * D;                // pre_only: (shift, scale) from c
      STK_TRY(pre_attention(e, pc, w.ctx, Mc, lm, lm + D, 2 * D, 1, w.a_c, w.a_c_hi, w.a_c_lo, Kc, S, 0, s, plan, 1, rows_cl, map_c));
    }
    STK_TRY(pre_attention(e, px, w.x, Mx, xmod, xmod + D, 6 * D, 1, w.a_x, w.a_x_hi, w.a_x_lo, N, S, Kc, s, plan, 0, rows_x));
    AttnOut ao;
    ao.split = Kc; ao.ld = D;
    const int ctx_rows = ctx_self ? Kc : 0, ctx_keys = ctx_self ? Kc : 0;
    if (!tc_mode(e)) {
      ao.f32_a = w.attn_c; ao.f32_b = w.attn_x;
      PROF(PC_ATTN, launch_attention_f32(w.qkv, 3 * D, (int64_t)S * 3 * D, w.qkv + D, w.qkv + 2 * D, 3 * D, (int64_t)S * 3 * D, S,
                                   nullptr, nullptr, 0, 0, 0, ao, B, S, e->H, 64, ctx_rows, ctx_keys, s, ap));
    } else {
      ao.hi_a = w.attn_c_hi; ao.lo_a = w.attn_c_lo; ao.hi_b = w.attn_x_hi; ao.lo_b = w.attn_x_lo;
      ao.fp16 = is_fp16(e);
      PROF(PC_ATTN, launch_attention_tc5(w.qkv_hi, B, S, e->H, ctx_rows, ctx_keys, ao, s, is_fp16(e), nsplit(e) == 3 ? w.qkv_lo : nullptr, ap));
    }
    if (ctx_post)
      STK_TRY(post_attention(e, pc, w.ctx, Mc, cmod, 6 * D, Kc, w.attn_c, w.attn_c_hi, w.attn_c_lo, w.a_c, w.a_c_hi, w.a_c_lo,
                             w.h_c, w.h_c_hi, w.h_c_lo, s, rows_c));
    STK_TRY(post_attention(e, px, w.x, Mx, xmod, 6 * D, 1, w.attn_x, w.attn_x_hi, w.attn_x_lo, w.a_x, w.a_x_hi, w.a_x_lo,
                           w.h_x, w.h_x_hi, w.h_x_lo, s, rows_x));
  }
  const float* fm = (uncond ? e->final_mod_u : e->final_mod) + (int64_t)step * 2 * D;
  return final_layer(e, B, fm, o_out ? o_out : w.o_final, s, rows_x);
}

// context_embedder(outs_q) + context_pos_embed (mmdit.py:1026) — step invariant, computed once per call
static int context_embed(selftok_engine* e, int B, cudaStream_t s) {
  DecodeWs& w = e->dws;
  GETW(cp, "model.context_pos_embed");
  STK_CHECK(cp->numel == (int64_t)e->cfg.K * e->D, SELFTOK_ERR_BAD_ARG, "context_pos_embed shape");
  Epilogue ep;
  ep.out = w.ctx0; ep.addtab = cp->d; ep.add_ld = e->D; ep.add_period = e->cfg.K;
  return lin32(e, "model.context_embedder", w.outs_q, e->cfg.code_dim, (int64_t)B * e->cfg.K, ep, s);
}

// Token-range call (selftok_*_range): per-image windows [lo_b, hi_b), rounded outward to 64 tokens for the whole batch so that one
// captured graph serves many range sets.  Step i's context stream holds positions [Lo, Lo + Kc[i]); the per-image plan says where
// each image's visible rows [lo_b, min(hi_b, k_i + 1)) lie in it.  Both arrays live in ws.plan (one upload per call).
struct Window {
  int Lo = 0, Hi = 0;
  std::vector<int> Kc;                   // context rows per step
  const int* range = nullptr;            // device [B][2] (lo, hi)
  const int* plan = nullptr;             // device [steps][B][2] (a, c)
};
static void window_step(const Window* win, int B, int step, int k_default, int* Kc, const int** plan, int* Lo) {
  if (!win) { *Kc = k_default; *plan = nullptr; *Lo = 0; return; }
  *Kc = win->Kc[step];
  *plan = *Kc > 0 ? win->plan + (int64_t)step * B * 2 : nullptr;
  *Lo = win->Lo;
}

// One MMDiT.forward (mmdit.py:992-1101) at schedule row `step` on ws.x_lat; leaves the patch outputs in ws.o_final.
static int dit_forward(selftok_engine* e, int B, int step, cudaStream_t s, const Window* win = nullptr) {
  const selftok_config_t& c = e->cfg;
  DecodeWs& w = e->dws;
  const int D = e->D;
  int Kc, Lo;
  const int* plan;
  window_step(win, B, step, e->k[step] + 1, &Kc, &plan, &Lo);
  PROF(PC_OTHER, launch_patchify(w.x_lat, w.patch, B, c.in_channels, e->lat_h, e->lat_w, c.dit_patch, s));
  STK_TRY(x_embed(e, B, s));
  if (Kc > 0) PROF(PC_OTHER, launch_copy_rows(w.ctx0 + (int64_t)Lo * D, (int64_t)c.K * D, w.ctx, (int64_t)Kc * D, B, (int64_t)Kc * D, s));
  // context rows see the image keys unless the handle was created with context_see_xt = 0 (sd3/mmdit.py:1012,1060; the
  // reference pipeline's sampler passes context_see_xt=True, SelftokPipeline.py:259)
  return joint_blocks(e, B, Kc, step, /*ctx_self=*/e->cfg.context_see_xt == 0, s, false, nullptr, plan, Lo);
}

// The two evaluations of one guided step (sample_one_step with cfg_scale != 1, rectified_flow.py:280-289): the conditional
// one -- called there WITHOUT context_see_xt, i.e. context rows only see the visible context keys -- into ws.o_final, and
// MMDiT.cfg_inference (context = zeros, every context key masked for every row: the image stream alone, integer timestep)
// into ws.o_final_u.
static int dit_forward_cfg(selftok_engine* e, int B, int step, cudaStream_t s, const Window* win = nullptr) {
  const selftok_config_t& c = e->cfg;
  DecodeWs& w = e->dws;
  const int D = e->D;
  int Kc, Lo;
  const int* plan;
  window_step(win, B, step, e->k[step] + 1, &Kc, &plan, &Lo);
  STK_CHECK(e->has_cfg, SELFTOK_ERR_STATE, "guided sampling needs selftok_set_cfg_schedule before selftok_finalize");
  STK_CHECK(Kc > 0, SELFTOK_ERR_BAD_ARG, "guided sampling needs a visible context token at every step");
  PROF(PC_OTHER, launch_patchify(w.x_lat, w.patch, B, c.in_channels, e->lat_h, e->lat_w, c.dit_patch, s));
  STK_TRY(x_embed(e, B, s));
  PROF(PC_OTHER, launch_copy_rows(w.ctx0 + (int64_t)Lo * D, (int64_t)c.K * D, w.ctx, (int64_t)Kc * D, B, (int64_t)Kc * D, s));
  STK_TRY(joint_blocks(e, B, Kc, step, /*ctx_self=*/true, s, /*uncond=*/false, w.o_final, plan, Lo));
  STK_TRY(x_embed(e, B, s));
  return joint_blocks(e, B, 0, step, /*ctx_self=*/false, s, /*uncond=*/true, w.o_final_u);
}

static int decode_body(selftok_engine* e, int B, int steps, cudaStream_t s, bool guided = false, float cfg_scale = 1.f,
                       const Window* win = nullptr) {
  const selftok_config_t& c = e->cfg;
  DecodeWs& w = e->dws;
  STK_TRY(run_lookup(e, w.tokens, B, w.outs_q, s, win ? win->range : nullptr));
  STK_TRY(context_embed(e, B, s));
  for (int i = 0; i < steps; ++i) {
    // euler_step (rectified_flow.py:301-303): x <- x - (t_i - t_{i+1}) * v, fused with unpatchify
    if (!guided) {
      STK_TRY(dit_forward(e, B, i, s, win));
      PROF(PC_OTHER, launch_unpatchify_axpy(w.o_final, w.x_lat, w.x_lat, e->dt[i], B, c.in_channels, e->lat_h / c.dit_patch,
                                            e->lat_w / c.dit_patch, c.dit_patch, s));
    } else {
      STK_TRY(dit_forward_cfg(e, B, i, s, win));
      PROF(PC_OTHER, launch_unpatchify_axpy(w.o_final, w.x_lat, w.x_lat, e->dt[i], B, c.in_channels, e->lat_h / c.dit_patch,
                                            e->lat_w / c.dit_patch, c.dit_patch, s, w.o_final_u, cfg_scale));
    }
  }
  return 0;
}

// Bytes of activation workspace op (0: selftok_encode*, 1: selftok_decode* / selftok_render* / selftok_dit_velocity) needs for batch B.
extern "C" __attribute__((visibility("default"))) int64_t selftok_workspace_bytes(selftok_handle_t e, int B, int op) {
  if (!e || B <= 0 || (op != 0 && op != 1)) return -1;
  Arena dry;
  dry.dry = true;
  if (op == 0) { EncodeWs w; if (layout_ews(e, w, B, dry) != 0) return -1; }
  else { DecodeWs w; if (layout_dws(e, w, B, dry) != 0) return -1; }
  return (int64_t)dry.off;
}
// Hand the library a caller-owned device block for workspace `op` (NULL / 0 returns to library-owned memory).  While it is at
// least selftok_workspace_bytes(h, B, op) large, calls with batch <= B allocate nothing; the block must stay alive and must not
// be used by anything else while a call on this handle is in flight.  Captured CUDA graphs of the decode loop are dropped.
extern "C" __attribute__((visibility("default"))) int selftok_set_workspace(selftok_handle_t e, int op, void* ws_dev, size_t bytes) {
  STK_CHECK(e && (op == 0 || op == 1), SELFTOK_ERR_BAD_ARG, "selftok_set_workspace: bad argument");
  STK_CHECK((reinterpret_cast<uintptr_t>(ws_dev) & 255) == 0, SELFTOK_ERR_BAD_ARG, "selftok_set_workspace: the block must be 256-byte aligned");
  STK_CUDA(cudaSetDevice(e->cfg.device));
  STK_CUDA(cudaDeviceSynchronize());
  e->user_ws[op] = bytes ? ws_dev : nullptr;
  e->user_ws_bytes[op] = ws_dev ? bytes : 0;
  if (op == 0) free_ews(e);
  else {
    drop_decode_graphs(e);
    free_dws(e);
  }
  return SELFTOK_OK;
}

extern "C" __attribute__((visibility("default"))) int selftok_set_use_graph(selftok_handle_t e, int enable) {
  STK_CHECK(e, SELFTOK_ERR_BAD_ARG, "null handle");
  e->use_graph = enable != 0;
  return SELFTOK_OK;
}

static int decode_impl(selftok_handle_t e, const int64_t* tokens_dev, const float* noise_dev, int B, int steps, float* x0_out_dev,
                       void* stream, bool guided, float cfg_scale, const int32_t* range_host = nullptr);

// Validates the host windows of a token-range call (before any launch) and builds its plan on the host: e->plan_host = [B][2]
// windows then [steps][B][2] (a, c).  render: one pass, the window is not clipped by the schedule.  guided: every window must keep
// a visible token at every executed step (the reference's conditional branch is NaN on an empty one).
static int plan_window(selftok_engine* e, const int32_t* range_host, int B, int steps, bool render, bool guided, Window* win) {
  STK_CHECK(range_host, SELFTOK_ERR_BAD_ARG, "token range: null range array");
  const int K = e->cfg.K;
  int min_k = K;
  for (int i = 0; i < steps && !render; ++i) min_k = e->k[i] < min_k ? e->k[i] : min_k;
  int lo_min = K, hi_max = 0;
  for (int b = 0; b < B; ++b) {
    const int lo = range_host[2 * b], hi = range_host[2 * b + 1];
    if (!(0 <= lo && lo < hi && hi <= K)) {
      set_error("token range of image " + std::to_string(b) + ": [" + std::to_string(lo) + ", " + std::to_string(hi) +
                ") is not a window 0 <= lo < hi <= K = " + std::to_string(K));
      return SELFTOK_ERR_BAD_ARG;
    }
    if (guided && lo > min_k) {
      set_error("token range of image " + std::to_string(b) + ": the guided sampler needs lo <= k of the last step (" +
                std::to_string(min_k) + "), got lo = " + std::to_string(lo));
      return SELFTOK_ERR_BAD_ARG;
    }
    lo_min = lo < lo_min ? lo : lo_min;
    hi_max = hi > hi_max ? hi : hi_max;
  }
  win->Lo = lo_min / 64 * 64;
  win->Hi = (hi_max + 63) / 64 * 64 < K ? (hi_max + 63) / 64 * 64 : K;
  std::vector<int>& h = e->plan_host;
  h.assign((size_t)B * 2 * (1 + steps), 0);
  std::copy(range_host, range_host + 2 * B, h.begin());
  win->Kc.assign(steps, 0);
  for (int i = 0; i < steps; ++i) {
    const int vis_end = render ? K : e->k[i] + 1;                 // visible positions [lo_b, min(hi_b, vis_end))
    const int end = vis_end < win->Hi ? vis_end : win->Hi;
    win->Kc[i] = end > win->Lo ? end - win->Lo : 0;
    for (int b = 0; b < B; ++b) {
      const int lo = range_host[2 * b], hi = range_host[2 * b + 1];
      const int c = (hi < vis_end ? hi : vis_end) - lo;
      int* pr = &h[(size_t)2 * B * (1 + i) + 2 * b];
      pr[0] = lo - win->Lo;
      pr[1] = c > 0 ? c : 0;
    }
  }
  return 0;
}
// uploads e->plan_host to dst on the call's stream (kernels, and graphs, read it from that fixed address) through a pinned staging
// buffer, so that the call stays asynchronous; the buffer is rewritten only after the previous upload has completed
static int upload_plan(selftok_engine* e, int* dst, cudaStream_t s) {
  const size_t n = e->plan_host.size();
  if (!e->plan_copied) STK_CUDA(cudaEventCreateWithFlags(&e->plan_copied, cudaEventDisableTiming));
  else STK_CUDA(cudaEventSynchronize(e->plan_copied));
  if (e->plan_pinned_n < n) {
    if (e->plan_pinned) STK_CUDA(cudaFreeHost(e->plan_pinned));
    e->plan_pinned = nullptr;
    e->plan_pinned_n = 0;
    STK_CUDA(cudaMallocHost(&e->plan_pinned, sizeof(int) * n));
    e->plan_pinned_n = n;
  }
  memcpy(e->plan_pinned, e->plan_host.data(), sizeof(int) * n);
  STK_CUDA(cudaMemcpyAsync(dst, e->plan_pinned, sizeof(int) * n, cudaMemcpyHostToDevice, s));
  STK_CUDA(cudaEventRecord(e->plan_copied, s));
  return 0;
}
static int upload_window(selftok_engine* e, Window* win, int B, cudaStream_t s) {
  DecodeWs& w = e->dws;
  STK_TRY(upload_plan(e, w.plan, s));
  win->range = w.plan;
  win->plan = w.plan + 2 * B;
  return 0;
}

extern "C" __attribute__((visibility("default"))) int selftok_decode(selftok_handle_t e, const int64_t* tokens_dev, const float* noise_dev, int B, int steps,
                              float* x0_out_dev, void* stream) {
  return decode_impl(e, tokens_dev, noise_dev, B, steps, x0_out_dev, stream, false, 1.f);
}

// Guided sampler: p_sample_loop(..., uncond_scale = cfg_scale) of the reference (rectified_flow.py:165-294): two MMDiT
// evaluations per step, v = v_u + cfg_scale (v_c - v_u).  Needs selftok_set_cfg_schedule before finalize.
extern "C" __attribute__((visibility("default"))) int selftok_decode_cfg(selftok_handle_t e, const int64_t* tokens_dev, const float* noise_dev, int B, int steps,
                                  float cfg_scale, float* x0_out_dev, void* stream) {
  return decode_impl(e, tokens_dev, noise_dev, B, steps, x0_out_dev, stream, true, cfg_scale);
}

// Token-range entries: image b decodes from its ids [lo_b, hi_b) only (range_host: host int32 [B][2]); ids outside the window are
// not read.  At step i the visible tokens are [lo_b, min(hi_b, k_i + 1)), the reference's `mask & super_mask`.
extern "C" __attribute__((visibility("default"))) int selftok_decode_range(selftok_handle_t e, const int64_t* tokens_dev, const int32_t* range_host,
                                    const float* noise_dev, int B, int steps, float* x0_out_dev, void* stream) {
  STK_CHECK(range_host, SELFTOK_ERR_BAD_ARG, "selftok_decode_range: null range array");
  return decode_impl(e, tokens_dev, noise_dev, B, steps, x0_out_dev, stream, false, 1.f, range_host);
}
extern "C" __attribute__((visibility("default"))) int selftok_decode_cfg_range(selftok_handle_t e, const int64_t* tokens_dev, const int32_t* range_host,
                                        const float* noise_dev, int B, int steps, float cfg_scale, float* x0_out_dev,
                                        void* stream) {
  STK_CHECK(range_host, SELFTOK_ERR_BAD_ARG, "selftok_decode_cfg_range: null range array");
  return decode_impl(e, tokens_dev, noise_dev, B, steps, x0_out_dev, stream, true, cfg_scale, range_host);
}

static int decode_impl(selftok_handle_t e, const int64_t* tokens_dev, const float* noise_dev, int B, int steps, float* x0_out_dev,
                       void* stream, bool guided, float cfg_scale, const int32_t* range_host) {
  HOT_PROLOGUE(e);
  STK_CHECK(!guided || e->has_cfg, SELFTOK_ERR_STATE, "selftok_decode_cfg: selftok_set_cfg_schedule was not called before finalize");
  STK_CHECK(tokens_dev && noise_dev && x0_out_dev && B > 0, SELFTOK_ERR_BAD_ARG, "selftok_decode: bad argument");
  STK_CHECK(!e->cfg.renderer, SELFTOK_ERR_STATE, "handle was created for the renderer; use selftok_render");
  STK_CHECK(steps > 0 && steps <= e->steps, SELFTOK_ERR_BAD_ARG, "steps exceeds the schedule");
  STK_TRY(check_grid(e, false, guided ? "selftok_decode_cfg" : "selftok_decode"));
  Window win;
  if (range_host) STK_TRY(plan_window(e, range_host, B, steps, false, guided, &win));
  STK_TRY(ensure_dws(e, B));
  STK_TRY(pos_table(e, false, s));
  DecodeWs& w = e->dws;
  if (range_host) STK_TRY(upload_window(e, &win, B, s));
  const Window* wp = range_host ? &win : nullptr;
  const int64_t nlat = (int64_t)B * lat_elems(e);
  if (tokens_dev != w.tokens) STK_CUDA(cudaMemcpyAsync(w.tokens, tokens_dev, sizeof(int64_t) * B * e->cfg.K, cudaMemcpyDeviceToDevice, s));
  if (noise_dev != w.x_lat) STK_CUDA(cudaMemcpyAsync(w.x_lat, noise_dev, sizeof(float) * nlat, cudaMemcpyDeviceToDevice, s));
  // eager when asked to, for the guided loop (cfg_scale is a kernel argument) and whenever per-launch profiling is on (events
  // recorded inside a capture never execute on a real stream: their elapsed times would be garbage)
  if (!e->use_graph || guided || e->prof_on) {
    STK_TRY(decode_body(e, B, steps, s, guided, cfg_scale, wp));
    e->last_launches = g_launch_count - launches0;
  } else {
    // token-range calls have their own graphs, keyed by the rounded window bounds: the plan itself is read at run time, so one
    // graph serves every range set with the same (Lo, Hi)
    const auto rkey = std::make_tuple(B, steps, win.Lo, win.Hi, e->lat_h, e->lat_w);
    const auto dkey = std::make_tuple(B, steps, e->lat_h, e->lat_w);
    std::pair<cudaGraphExec_t, int64_t>* g = nullptr;
    if (wp) {
      auto f = e->range_graphs.find(rkey);
      if (f != e->range_graphs.end()) g = &f->second;
    } else {
      auto f = e->graphs.find(dkey);
      if (f != e->graphs.end()) g = &f->second;
    }
    if (!g) {
      cudaStream_t cs;
      STK_CUDA(cudaStreamCreateWithFlags(&cs, cudaStreamNonBlocking));
      {
        const cudaError_t be = cudaStreamBeginCapture(cs, cudaStreamCaptureModeThreadLocal);
        if (be != cudaSuccess) {
          cudaStreamDestroy(cs);                                       // no leak on the error path
          STK_CUDA(be);
        }
      }
      const int64_t l0 = g_launch_count;
      int st = decode_body(e, B, steps, cs, false, 1.f, wp);
      cudaGraph_t graph = nullptr;
      cudaError_t ce = cudaStreamEndCapture(cs, &graph);
      cudaStreamDestroy(cs);
      if (st != 0) { if (graph) cudaGraphDestroy(graph); return st; }
      STK_CUDA(ce);
      cudaGraphExec_t exec;
      STK_CUDA(cudaGraphInstantiate(&exec, graph, 0));
      cudaGraphDestroy(graph);
      const auto val = std::make_pair(exec, g_launch_count - l0);
      g = wp ? &e->range_graphs.emplace(rkey, val).first->second : &e->graphs.emplace(dkey, val).first->second;
    }
    STK_CUDA(cudaGraphLaunch(g->first, s));
    e->last_launches = g->second;
  }
  if (x0_out_dev != w.x_lat) STK_CUDA(cudaMemcpyAsync(x0_out_dev, w.x_lat, sizeof(float) * nlat, cudaMemcpyDeviceToDevice, s));
  return SELFTOK_OK;
}

// One Euler step per image at its own schedule row (continuous batching): x_out[b] = x[b] - dt[s_b] v_b, eager, over a packed
// context stream (see Packed).  Bitwise what selftok_decode(_cfg)(_range) computes for that image at step s_b.
extern "C" __attribute__((visibility("default"))) int selftok_decode_step(selftok_handle_t e, const int64_t* tokens_dev, const int32_t* range_host,
                                   const int32_t* step_host, const float* cfg_scale_host, const float* x_dev, int B,
                                   float* x_out_dev, void* stream) {
  HOT_PROLOGUE(e);
  STK_CHECK(tokens_dev && step_host && x_dev && x_out_dev && B > 0, SELFTOK_ERR_BAD_ARG, "selftok_decode_step: bad argument");
  STK_CHECK(!e->cfg.renderer, SELFTOK_ERR_STATE, "selftok_decode_step: handle was created for the renderer");
  const bool guided = cfg_scale_host != nullptr;
  STK_CHECK(!guided || e->has_cfg, SELFTOK_ERR_STATE, "selftok_decode_step: guided steps need selftok_set_cfg_schedule before finalize");
  STK_TRY(check_grid(e, false, "selftok_decode_step"));
  const selftok_config_t& c = e->cfg;
  const int K = c.K, N = e->Nimg;
  // the per-image block, validated before anything is launched
  std::vector<int>& h = e->plan_host;
  h.assign((size_t)B * PK_IMG_INTS, 0);
  int Mc = 0, cmax = 0;
  for (int b = 0; b < B; ++b) {
    const int st = step_host[b];
    if (st < 0 || st >= e->steps) {
      set_error("selftok_decode_step: step of image " + std::to_string(b) + " is " + std::to_string(st) + ", not in [0, " +
                std::to_string(e->steps) + ")");
      return SELFTOK_ERR_BAD_ARG;
    }
    const int lo = range_host ? range_host[2 * b] : 0, hi = range_host ? range_host[2 * b + 1] : K;
    if (!(0 <= lo && lo < hi && hi <= K)) {
      set_error("selftok_decode_step: token range of image " + std::to_string(b) + ": [" + std::to_string(lo) + ", " +
                std::to_string(hi) + ") is not a window 0 <= lo < hi <= K = " + std::to_string(K));
      return SELFTOK_ERR_BAD_ARG;
    }
    const int end = hi < e->k[st] + 1 ? hi : e->k[st] + 1;
    const int cb = end > lo ? end - lo : 0;
    if (guided && cb == 0) {
      set_error("selftok_decode_step: image " + std::to_string(b) + " has no visible token at step " + std::to_string(st) +
                " (the guided sampler needs lo <= k = " + std::to_string(e->k[st]) + ", got lo = " + std::to_string(lo) + ")");
      return SELFTOK_ERR_BAD_ARG;
    }
    h[2 * b] = Mc; h[2 * b + 1] = cb; h[2 * B + b] = lo; h[3 * B + b] = st;
    memcpy(&h[4 * B + b], &e->dt[st], sizeof(float));
    if (guided) memcpy(&h[5 * B + b], &cfg_scale_host[b], sizeof(float));
    Mc += cb;
    cmax = cb > cmax ? cb : cmax;
  }
  STK_TRY(ensure_dws(e, B));
  STK_TRY(pos_table(e, false, s));
  DecodeWs& w = e->dws;
  STK_TRY(upload_plan(e, w.pk, s));
  int* rows = w.pk + (int64_t)PK_IMG_INTS * B;
  const int64_t BK = (int64_t)B * K;
  Packed pk;
  pk.Mc = Mc; pk.S = cmax + N; pk.pair = w.pk;
  pk.dt = reinterpret_cast<const float*>(w.pk + 4 * B); pk.scale = reinterpret_cast<const float*>(w.pk + 5 * B);
  pk.ctx_tok = rows; pk.ctx_pos = rows + BK; pk.ctx_step = rows + 2 * BK; pk.ctx_dst = rows + 3 * BK; pk.x_step = rows + 4 * BK;
  PROF(PC_OTHER, launch_expand_packed(w.pk, B, K, N, pk.S, rows, rows + BK, rows + 2 * BK, rows + 3 * BK, rows + 4 * BK, s));
  const int64_t row_bytes = (int64_t)3 * e->D * (tc_mode(e) ? 2 : 4);
  if (!tc_mode(e)) PROF(PC_OTHER, launch_zero_slot_tails(pk.pair, B, pk.S, N, w.qkv, row_bytes, s));
  if (w.qkv_hi) PROF(PC_OTHER, launch_zero_slot_tails(pk.pair, B, pk.S, N, w.qkv_hi, row_bytes, s));
  if (w.qkv_lo) PROF(PC_OTHER, launch_zero_slot_tails(pk.pair, B, pk.S, N, w.qkv_lo, row_bytes, s));
  if (Mc > 0) {
    // context_embedder(outs_q) + context_pos_embed of the visible rows only, straight into the context stream
    STK_TRY(run_lookup(e, tokens_dev, B, w.outs_q, s, nullptr, pk.ctx_tok, Mc));
    GETW(cp, "model.context_pos_embed");
    STK_CHECK(cp->numel == (int64_t)K * e->D, SELFTOK_ERR_BAD_ARG, "context_pos_embed shape");
    Epilogue ep;
    ep.out = w.ctx; ep.addtab = cp->d; ep.add_ld = e->D; ep.tab_rows = pk.ctx_pos;
    STK_TRY(lin32(e, "model.context_embedder", w.outs_q, c.code_dim, Mc, ep, s));
  }
  PROF(PC_OTHER, launch_patchify(x_dev, w.patch, B, c.in_channels, e->lat_h, e->lat_w, c.dit_patch, s));
  STK_TRY(x_embed(e, B, s));
  if (!guided) {
    STK_TRY(joint_blocks(e, B, 0, 0, /*ctx_self=*/c.context_see_xt == 0, s, false, w.o_final, nullptr, 0, &pk));
  } else {
    // as dit_forward_cfg: the conditional pass with context rows blind to image keys, then the image stream alone
    STK_TRY(joint_blocks(e, B, 0, 0, /*ctx_self=*/true, s, false, w.o_final, nullptr, 0, &pk));
    STK_TRY(x_embed(e, B, s));
    Packed pu = pk;
    pu.Mc = 0; pu.S = N;
    STK_TRY(joint_blocks(e, B, 0, 0, /*ctx_self=*/false, s, /*uncond=*/true, w.o_final_u, nullptr, 0, &pu));
  }
  PROF(PC_OTHER, launch_unpatchify_axpy(w.o_final, x_dev, x_out_dev, 0.f, B, c.in_channels, e->lat_h / c.dit_patch, e->lat_w / c.dit_patch,
                                        c.dit_patch, s, guided ? w.o_final_u : nullptr, 1.f, pk.dt, guided ? pk.scale : nullptr));
  e->last_launches = g_launch_count - launches0;
  return SELFTOK_OK;
}

extern "C" __attribute__((visibility("default"))) int selftok_dit_velocity(selftok_handle_t e, const int64_t* tokens_dev, const float* x_dev, int B, int step,
                                    float* v_out_dev, void* stream) {
  HOT_PROLOGUE(e);
  STK_CHECK(tokens_dev && x_dev && v_out_dev && B > 0, SELFTOK_ERR_BAD_ARG, "selftok_dit_velocity: bad argument");
  STK_CHECK(!e->cfg.renderer, SELFTOK_ERR_STATE, "renderer handle");
  STK_CHECK(step >= 0 && step < e->steps, SELFTOK_ERR_BAD_ARG, "step out of range");
  STK_TRY(check_grid(e, false, "selftok_dit_velocity"));
  STK_TRY(ensure_dws(e, B));
  STK_TRY(pos_table(e, false, s));
  DecodeWs& w = e->dws;
  const selftok_config_t& c = e->cfg;
  const int64_t nlat = (int64_t)B * lat_elems(e);
  STK_CUDA(cudaMemcpyAsync(w.tokens, tokens_dev, sizeof(int64_t) * B * c.K, cudaMemcpyDeviceToDevice, s));
  STK_CUDA(cudaMemcpyAsync(w.x_lat, x_dev, sizeof(float) * nlat, cudaMemcpyDeviceToDevice, s));
  STK_TRY(run_lookup(e, w.tokens, B, w.outs_q, s));
  STK_TRY(context_embed(e, B, s));
  STK_TRY(dit_forward(e, B, step, s));
  PROF(PC_OTHER, launch_unpatchify_axpy(w.o_final, nullptr, v_out_dev, -1.f, B, c.in_channels, e->lat_h / c.dit_patch,
                                        e->lat_w / c.dit_patch, c.dit_patch, s));
  e->last_launches = g_launch_count - launches0;
  return SELFTOK_OK;
}

static int render_impl(selftok_handle_t e, const int64_t* tokens_dev, int B, float* x0_out_dev, void* stream, const int32_t* range_host) {
  HOT_PROLOGUE(e);
  STK_CHECK(tokens_dev && x0_out_dev && B > 0, SELFTOK_ERR_BAD_ARG, "selftok_render: bad argument");
  STK_CHECK(e->cfg.renderer, SELFTOK_ERR_STATE, "handle was not created for the renderer");
  Window win;
  if (range_host) STK_TRY(plan_window(e, range_host, B, 1, true, false, &win));
  STK_TRY(ensure_dws(e, B));
  DecodeWs& w = e->dws;
  const selftok_config_t& c = e->cfg;
  if (range_host) STK_TRY(upload_window(e, &win, B, s));
  // the renderer's context: all K rows, or the rounded window [Lo, Hi) of a token-range call (no schedule clipping)
  const int Lo = range_host ? win.Lo : 0, Kc = range_host ? win.Kc[0] : c.K;
  if (tokens_dev != w.tokens) STK_CUDA(cudaMemcpyAsync(w.tokens, tokens_dev, sizeof(int64_t) * B * c.K, cudaMemcpyDeviceToDevice, s));
  STK_TRY(run_lookup(e, w.tokens, B, w.outs_q, s, range_host ? win.range : nullptr));
  STK_TRY(context_embed(e, B, s));
  // x = mask_token + positional_embedding (mmdit.py:1518-1522); context rows see context only
  PROF(PC_OTHER, launch_bcast_rows(e->rend_x0, nullptr, w.x, B, e->Nimg, e->D, s));
  PROF(PC_OTHER, launch_copy_rows(w.ctx0 + (int64_t)Lo * e->D, (int64_t)c.K * e->D, w.ctx, (int64_t)Kc * e->D, B, (int64_t)Kc * e->D, s));
  STK_TRY(joint_blocks(e, B, Kc, 0, /*ctx_self=*/true, s, false, nullptr, range_host ? win.plan : nullptr, Lo));
  PROF(PC_OTHER, launch_unpatchify_axpy(w.o_final, nullptr, x0_out_dev, -1.f, B, c.in_channels, e->lat_h / c.dit_patch,
                                        e->lat_w / c.dit_patch, c.dit_patch, s));
  e->last_launches = g_launch_count - launches0;
  return SELFTOK_OK;
}
extern "C" __attribute__((visibility("default"))) int selftok_render(selftok_handle_t e, const int64_t* tokens_dev, int B, float* x0_out_dev, void* stream) {
  return render_impl(e, tokens_dev, B, x0_out_dev, stream, nullptr);
}
// Renderer over per-image token windows (range_host: host int32 [B][2]): MMDiT_Renderer.forward(..., mask = the window).
extern "C" __attribute__((visibility("default"))) int selftok_render_range(selftok_handle_t e, const int64_t* tokens_dev, const int32_t* range_host, int B,
                                    float* x0_out_dev, void* stream) {
  STK_CHECK(range_host, SELFTOK_ERR_BAD_ARG, "selftok_render_range: null range array");
  return render_impl(e, tokens_dev, B, x0_out_dev, stream, range_host);
}

// ------------------------------------------------------------------------------------------------ host-buffer variants
extern "C" __attribute__((visibility("default"))) int selftok_encode_host(selftok_handle_t e, const float* x0_host, int B, int64_t* tokens_host, void* stream) {
  STK_CHECK(e && x0_host && tokens_host && B > 0, SELFTOK_ERR_BAD_ARG, "selftok_encode_host: bad argument");
  STK_CHECK(e->finalized, SELFTOK_ERR_STATE, "selftok_finalize has not been called");
  STK_CUDA(cudaSetDevice(e->cfg.device));
  cudaStream_t s = (cudaStream_t)stream;
  STK_TRY(check_grid(e, true, "selftok_encode_host"));
  STK_TRY(ensure_ews(e, B));
  const int64_t nlat = (int64_t)B * lat_elems(e);
  STK_CUDA(cudaMemcpyAsync(e->ews.x0, x0_host, sizeof(float) * nlat, cudaMemcpyHostToDevice, s));
  STK_TRY(selftok_encode(e, e->ews.x0, B, e->ews.tokens, nullptr, nullptr, stream));
  STK_CUDA(cudaMemcpyAsync(tokens_host, e->ews.tokens, sizeof(int64_t) * B * e->cfg.K, cudaMemcpyDeviceToHost, s));
  STK_CUDA(cudaStreamSynchronize(s));
  return SELFTOK_OK;
}

extern "C" __attribute__((visibility("default"))) int selftok_decode_host(selftok_handle_t e, const int64_t* tokens_host, const float* noise_host, int B, int steps,
                                   float* x0_out_host, void* stream) {
  STK_CHECK(e && tokens_host && noise_host && x0_out_host && B > 0, SELFTOK_ERR_BAD_ARG, "selftok_decode_host: bad argument");
  STK_CHECK(e->finalized, SELFTOK_ERR_STATE, "selftok_finalize has not been called");
  STK_CUDA(cudaSetDevice(e->cfg.device));
  cudaStream_t s = (cudaStream_t)stream;
  STK_TRY(check_grid(e, false, "selftok_decode_host"));
  STK_TRY(ensure_dws(e, B));
  DecodeWs& w = e->dws;
  const int64_t nlat = (int64_t)B * lat_elems(e);
  STK_CUDA(cudaMemcpyAsync(w.tokens, tokens_host, sizeof(int64_t) * B * e->cfg.K, cudaMemcpyHostToDevice, s));
  STK_CUDA(cudaMemcpyAsync(w.x_lat, noise_host, sizeof(float) * nlat, cudaMemcpyHostToDevice, s));
  STK_TRY(selftok_decode(e, w.tokens, w.x_lat, B, steps, w.x_lat, stream));
  STK_CUDA(cudaMemcpyAsync(x0_out_host, w.x_lat, sizeof(float) * nlat, cudaMemcpyDeviceToHost, s));
  STK_CUDA(cudaStreamSynchronize(s));
  return check_ids_after_sync(e, stream, "selftok_decode_host");
}

extern "C" __attribute__((visibility("default"))) int selftok_render_host(selftok_handle_t e, const int64_t* tokens_host, int B, float* x0_out_host, void* stream) {
  STK_CHECK(e && tokens_host && x0_out_host && B > 0, SELFTOK_ERR_BAD_ARG, "selftok_render_host: bad argument");
  STK_CHECK(e->finalized, SELFTOK_ERR_STATE, "selftok_finalize has not been called");
  STK_CUDA(cudaSetDevice(e->cfg.device));
  cudaStream_t s = (cudaStream_t)stream;
  STK_TRY(ensure_dws(e, B));
  DecodeWs& w = e->dws;
  const int64_t nlat = (int64_t)B * lat_elems(e);
  STK_CUDA(cudaMemcpyAsync(w.tokens, tokens_host, sizeof(int64_t) * B * e->cfg.K, cudaMemcpyHostToDevice, s));
  STK_TRY(selftok_render(e, w.tokens, B, w.x_lat, stream));
  STK_CUDA(cudaMemcpyAsync(x0_out_host, w.x_lat, sizeof(float) * nlat, cudaMemcpyDeviceToHost, s));
  STK_CUDA(cudaStreamSynchronize(s));
  return check_ids_after_sync(e, stream, "selftok_render_host");
}

extern "C" __attribute__((visibility("default"))) int selftok_set_profile(selftok_handle_t e, int enable) {
  STK_CHECK(e, SELFTOK_ERR_BAD_ARG, "null handle");
  e->prof_on = enable != 0;
  return SELFTOK_OK;
}

// Synchronises the device, sums the recorded event pairs per kernel class and clears them.
extern "C" __attribute__((visibility("default"))) int selftok_get_profile(selftok_handle_t e, double* ms_out, int64_t* count_out) {
  STK_CHECK(e && ms_out && count_out, SELFTOK_ERR_BAD_ARG, "selftok_get_profile: bad argument");
  STK_CUDA(cudaSetDevice(e->cfg.device));
  STK_CUDA(cudaDeviceSynchronize());
  for (int i = 0; i < PC_COUNT; ++i) { ms_out[i] = 0.0; count_out[i] = 0; }
  for (size_t i = 0; i < e->prof_cat.size(); ++i) {
    float ms = 0.f;
    cudaEventElapsedTime(&ms, e->prof_ev[2 * i], e->prof_ev[2 * i + 1]);
    ms_out[e->prof_cat[i]] += ms;
    count_out[e->prof_cat[i]] += 1;
    cudaEventDestroy(e->prof_ev[2 * i]);
    cudaEventDestroy(e->prof_ev[2 * i + 1]);
  }
  e->prof_ev.clear();
  e->prof_cat.clear();
  return SELFTOK_OK;
}

extern "C" __attribute__((visibility("default"))) int64_t selftok_last_launch_count(selftok_handle_t e) { return e ? e->last_launches : -1; }
extern "C" __attribute__((visibility("default"))) int64_t selftok_device_bytes(selftok_handle_t e) { return e ? e->bytes : -1; }

// ------------------------------------------------------------------------------------------------ kernel-level ABI
static Epilogue k_epilogue(const selftok_k_epilogue_t& d) {
  Epilogue ep;
  ep.mode = d.mode; ep.act = d.act; ep.bias = d.bias; ep.out = d.out; ep.ldo = d.ldo;
  ep.resid = d.resid; ep.gate = d.gate; ep.gate_ld = d.gate_ld; ep.gate_period = d.gate_period;
  ep.addtab = d.addtab; ep.add_ld = d.add_ld; ep.add_period = d.add_period;
  ep.out_hi = (bf16*)d.out_hi; ep.out_lo = (bf16*)d.out_lo;
  ep.rpb_in = d.rpb_in; ep.rpb_out = d.rpb_out; ep.row_off = d.row_off; ep.fp16 = d.fp16;
  ep.plan = d.plan; ep.plan_ctx = d.plan_ctx; ep.tab_rows = d.tab_rows; ep.row_map = d.row_map;
  return ep;
}

// fp32 elements of a problem's A operand in the layout the kernel reads (stride-2 convolutions: four polyphase planes per image)
static int64_t k_gemm_a_elems(const selftok_k_gemm_problem_t& q) {
  if (q.conv_C <= 0) return q.M * q.K;
  return q.M * q.conv_C * (q.conv_stride == 2 ? 4 : 1);
}

extern "C" __attribute__((visibility("default"))) int selftok_k_gemm(int path, int ns, const selftok_k_gemm_problem_t* probs, int n, void* stream) {
  STK_CHECK(probs && (path == 0 || path == 1) && n >= 1 && n <= (path == 0 ? 1 : 2), SELFTOK_ERR_BAD_ARG,
            "selftok_k_gemm: path 0 takes one problem, path 1 one or two");
  STK_CHECK(path == 0 || ns == 0 || ns == 1 || ns == 3 || ns == NSPLIT_E4M3, SELFTOK_ERR_BAD_ARG, "selftok_k_gemm: nsplit must be 4, 3, 1 or 0");
  const bool e4m3 = path == 1 && ns == NSPLIT_E4M3;
  Epilogue eps[2];
  for (int i = 0; i < n; ++i) {
    const selftok_k_gemm_problem_t& q = probs[i];
    STK_CHECK(q.A && q.W && q.M > 0 && q.N > 0 && q.K > 0, SELFTOK_ERR_BAD_ARG, "selftok_k_gemm: bad operands or shape");
    STK_CHECK(path == 1 || q.conv_C == 0, SELFTOK_ERR_BAD_ARG, "selftok_k_gemm: the fp32 FFMA path has no convolution mode");
    STK_CHECK(!e4m3 || q.conv_C == 0, SELFTOK_ERR_BAD_ARG, "selftok_k_gemm: the e4m3 mode has no convolution");
    eps[i] = k_epilogue(q.ep);
    STK_TRY(check_epilogue(eps[i], "selftok_k_gemm"));   // before any CUDA call
  }
  cudaStream_t s = (cudaStream_t)stream;
  if (path == 0) {
    const selftok_k_gemm_problem_t& q = probs[0];
    STK_TRY(launch_linear_f32(q.A, q.K, q.W, q.K, q.M, q.N, q.K, eps[0], s));
    STK_CUDA(cudaStreamSynchronize(s));
    return SELFTOK_OK;
  }
  const int fp16 = ns == 0;
  const int nsplit = e4m3 ? NSPLIT_E4M3 : ns == 3 ? 3 : 1;
  STK_TRY(gemm_tc_init());
  bf16* planes[2][4] = {};                                // per problem: A hi, A lo, W hi, W lo (e4m3: A codes, A scales, W codes, W scales)
  TcProblem tp[2];
  int st = 0;
  for (int i = 0; i < n && !st; ++i) {
    const selftok_k_gemm_problem_t& q = probs[i];
    const int64_t na = k_gemm_a_elems(q), nw = (int64_t)q.N * q.K;
    for (int p = 0; p < 4 && !st; ++p) {
      if ((p & 1) && nsplit != 3 && !e4m3) continue;
      // e4m3: one byte per code, one fp32 scale per row
      const size_t bytes = e4m3 ? ((p & 1) ? sizeof(float) * (size_t)(p < 2 ? q.M : q.N) : (size_t)(p < 2 ? na : nw))
                                : sizeof(bf16) * (size_t)(p < 2 ? na : nw);
      if (cudaMalloc(&planes[i][p], bytes) != cudaSuccess) {
        set_error("selftok_k_gemm: cudaMalloc of the operand planes failed");
        st = SELFTOK_ERR_CUDA;
      }
    }
    if (st) break;
    if (e4m3) {
      eps[i].s_a = reinterpret_cast<const float*>(planes[i][1]);
      eps[i].s_w = reinterpret_cast<const float*>(planes[i][3]);
      tp[i] = TcProblem{planes[i][0], nullptr, planes[i][2], nullptr, q.M, q.N, q.K, eps[i]};
    } else {
      tp[i] = TcProblem{planes[i][0], planes[i][1], planes[i][2], planes[i][3], q.M, q.N, q.K, eps[i]};
    }
    tp[i].conv_C = q.conv_C; tp[i].conv_H = q.conv_H; tp[i].conv_W = q.conv_W; tp[i].conv_stride = q.conv_stride;
    tp[i].conv_edge = q.conv_edge;
    st = check_gemm_tc_problem(tp[i], nsplit, fp16);      // shape / geometry errors before any launch
  }
  for (int i = 0; i < n && !st; ++i) {
    if (e4m3) {                                           // A per GEMM row, W per output channel (kernels.h contract)
      st = launch_quant_e4m3_rows(probs[i].A, probs[i].M, probs[i].K, reinterpret_cast<uint8_t*>(planes[i][0]),
                                  reinterpret_cast<float*>(planes[i][1]), s);
      if (!st) st = launch_quant_e4m3_rows(probs[i].W, probs[i].N, probs[i].K, reinterpret_cast<uint8_t*>(planes[i][2]),
                                           reinterpret_cast<float*>(planes[i][3]), s);
      continue;
    }
    st = launch_split_bf16(probs[i].A, planes[i][0], planes[i][1], k_gemm_a_elems(probs[i]), s, fp16);
    if (!st) st = launch_split_bf16(probs[i].W, planes[i][2], planes[i][3], (int64_t)probs[i].N * probs[i].K, s, fp16);
  }
  if (!st) st = launch_gemm_tc_grouped(tp, n, nsplit, s, fp16);
  if (cudaStreamSynchronize(s) != cudaSuccess && !st) {
    set_error("selftok_k_gemm: the stream failed");
    st = SELFTOK_ERR_CUDA;
  }
  for (auto& pl : planes)
    for (bf16* p : pl)
      if (p) cudaFree(p);
  return st;
}

extern "C" __attribute__((visibility("default"))) int selftok_k_set_gemm_ctas(int n) {
  STK_CHECK(n == 1 || n == 2, SELFTOK_ERR_BAD_ARG, "selftok_k_set_gemm_ctas: n must be 1 or 2");
  gemm_tc_set_ctas(n);
  return SELFTOK_OK;
}

extern "C" __attribute__((visibility("default"))) int selftok_k_ln_mod_f32(const float* x, const float* shift, const float* scale, int64_t ld_mod, int period,
                                    float* out, int64_t M, int D, void* stream) {
  return launch_ln_mod(x, D, shift, scale, ld_mod, period, out, nullptr, nullptr, D, M, D, 1e-6f, (cudaStream_t)stream);
}

extern "C" __attribute__((visibility("default"))) int selftok_k_quant_e4m3(const float* x, int64_t M, int K, void* codes_out,
                                                                          float* scales_out, void* stream) {
  return launch_quant_e4m3_rows(x, M, K, static_cast<uint8_t*>(codes_out), scales_out, (cudaStream_t)stream);
}

// the fp8 decoder's LN + modulate -> e4m3 launch (launch_ln_mod_pair, one problem)
extern "C" __attribute__((visibility("default"))) int selftok_k_ln_mod_e4m3(const float* x, const float* shift, const float* scale, int64_t ld_mod,
                                                                           int period, void* codes_out, float* scales_out, int64_t M, int D,
                                                                           void* stream) {
  LnProblem lp;
  lp.x = x; lp.shift = shift; lp.scale = scale; lp.ld_mod = ld_mod; lp.period = period;
  lp.out_hi = static_cast<bf16*>(codes_out); lp.out_scale = scales_out; lp.M = M;
  return launch_ln_mod_pair(&lp, 1, D, 1e-6f, (cudaStream_t)stream, 0);
}

extern "C" __attribute__((visibility("default"))) int selftok_k_attention_f32(const float* q, int64_t q_ld, const float* k1, const float* v1, int64_t kv1_ld, int S1,
                                       const float* k2, const float* v2, int64_t kv2_ld, int S2, float* out, int64_t out_ld,
                                       int B, int Sq, int H, int hd, void* stream) {
  AttnOut ao;
  ao.f32_a = out; ao.split = Sq; ao.ld = out_ld;
  return launch_attention_f32(q, q_ld, (int64_t)Sq * q_ld, k1, v1, kv1_ld, (int64_t)S1 * kv1_ld, S1, k2, v2, kv2_ld,
                              (int64_t)S2 * kv2_ld, S2, ao, B, Sq, H, hd, 0, 0, (cudaStream_t)stream);
}

extern "C" __attribute__((visibility("default"))) int selftok_k_attention_tc(const float* qkv, float* out, int B, int S, int H, int ns, int ctx_rows, int ctx_keys,
                                      void* stream) {
  STK_CHECK(qkv && out && (ns == 0 || ns == 1 || ns == 3), SELFTOK_ERR_BAD_ARG, "selftok_k_attention_tc: bad argument");
  const int fp16 = ns == 0;                     // 0: IEEE half, 1: bf16, 3: split bf16 (hi + lo planes, three MMAs per product)
  cudaStream_t s = (cudaStream_t)stream;
  const int64_t n = (int64_t)B * S * 3 * H * 64;
  bf16 *qh, *ql = nullptr;
  STK_CUDA(cudaMalloc(&qh, sizeof(bf16) * n));
  if (ns == 3) STK_CUDA(cudaMalloc(&ql, sizeof(bf16) * n));
  int st = launch_split_bf16(qkv, qh, ql, n, s, fp16);
  AttnOut ao;
  ao.f32_a = out; ao.split = S; ao.ld = (int64_t)H * 64;
  if (!st) st = launch_attention_tc5(qh, B, S, H, ctx_rows, ctx_keys, ao, s, fp16, ql);
  cudaStreamSynchronize(s);
  cudaFree(qh);
  if (ql) cudaFree(ql);
  return st;
}

// Joint attention with per-image live context counts (the token-range plan with a = 0), output in slot order [B,S,H*64].
// live_host: host int32 [1 + B] = {Kc, c_0, ..., c_{B-1}}: every slot has Kc context rows and S - Kc image rows.
extern "C" __attribute__((visibility("default"))) int selftok_k_attention_tc_range(const float* qkv, float* out, int B, int S, int H, int ns, int ctx_self,
                                            const int32_t* live_host, void* stream) {
  STK_CHECK(qkv && out && live_host && B > 0 && (ns == 0 || ns == 1 || ns == 3), SELFTOK_ERR_BAD_ARG,
            "selftok_k_attention_tc_range: bad argument");
  const int Kc = live_host[0];
  STK_CHECK(Kc >= 0 && Kc < S, SELFTOK_ERR_BAD_ARG, "selftok_k_attention_tc_range: need 0 <= Kc < S");
  std::vector<int> plan((size_t)2 * B);
  for (int b = 0; b < B; ++b) {
    STK_CHECK(live_host[1 + b] >= 0 && live_host[1 + b] <= Kc, SELFTOK_ERR_BAD_ARG, "selftok_k_attention_tc_range: need 0 <= c_b <= Kc");
    plan[2 * b + 1] = live_host[1 + b];
  }
  const int fp16 = ns == 0;
  cudaStream_t s = (cudaStream_t)stream;
  const int64_t n = (int64_t)B * S * 3 * H * 64;
  bf16 *qh, *ql = nullptr;
  int* plan_dev;
  STK_CUDA(cudaMalloc(&plan_dev, sizeof(int) * plan.size()));
  STK_CUDA(cudaMemcpy(plan_dev, plan.data(), sizeof(int) * plan.size(), cudaMemcpyHostToDevice));
  STK_CUDA(cudaMalloc(&qh, sizeof(bf16) * n));
  if (ns == 3) STK_CUDA(cudaMalloc(&ql, sizeof(bf16) * n));
  int st = launch_split_bf16(qkv, qh, ql, n, s, fp16);
  AttnOut ao;
  ao.f32_a = out; ao.split = S; ao.ld = (int64_t)H * 64;
  AttnPlan ap;
  ap.plan = plan_dev; ap.n_img = S - Kc; ap.ctx_self = ctx_self != 0; ap.route = 0;
  if (!st) st = launch_attention_tc5(qh, B, S, H, 0, 0, ao, s, fp16, ql, ap);
  cudaStreamSynchronize(s);
  cudaFree(qh);
  if (ql) cudaFree(ql);
  cudaFree(plan_dev);
  return st;
}
