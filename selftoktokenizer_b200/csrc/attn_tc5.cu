// Joint attention of the MMDiT on Hopper tensor cores (sm_90a, wgmma), head_dim 64, fp32 softmax in registers.
// Operands: single-pass 16-bit (IEEE half or bf16), or split bf16 ("bf16x3": hi*hi + hi*lo + lo*hi into the same fp32
// accumulators for both products, fp32-faithful).
//
//   grid           one CTA per work item (image, head, 128-query tile), query tile fastest so that the CTAs running side by
//                  side share one (image, head)'s K / V in L2; two CTAs per SM
//   warp 8         TMA producer: the Q tile once, then K and V tiles (64 keys x 64 dims) through a ring of KV_STAGES stages
//   warpgroups 0-1 64 query rows each: S = Q K^T (wgmma m64n64k16, both operands from shared memory) into registers; online
//                  softmax on the accumulator fragment (a row lives in a quad of lanes: max / sum exchanged with two
//                  shuffles); P rounded to 16 bits in registers is the A operand of O += P V (wgmma m64n64k16, A from
//                  registers, V MN-major straight from the TMA tile) -- no shared-memory round trip for P
//   epilogue       O / l -> fp32 and / or the 16-bit A-operand planes of the proj GEMM
//
// Contract (sd3/mmdit.py:521-531, sd3/other_impls.py:37-45): dense non-causal attention over the joint
// [context prefix ; image] sequence; rows < ctx_rows only see keys < ctx_keys (renderer rule, mmdit.py:1581).  With a
// token-range plan (AttnPlan) every image has its own number of live context rows and keys; the key loop of the producer and of
// the consumers stops at the image's last visible key.
#include "common.cuh"
#include "hopper.cuh"
#include "kernels.h"

#include <algorithm>

namespace stk {

// provided by gemm_tc.cu
int make_tensor_map_2d(CUtensorMap* map, const void* ptr, uint64_t rows, uint64_t cols, uint32_t box_rows, uint32_t box_cols,
                       int fp16);

namespace {

using namespace hop;

constexpr int HD = 64, BQ = 128, BKV = 64;
constexpr int Q_BYTES = BQ * HD * 2, KV_TILE_BYTES = BKV * HD * 2;
constexpr int NUM_THREADS = 2 * 128 + 32;       // two consumer warpgroups, one producer warp
// NSPLIT == 1: single-pass 16-bit operands.  NSPLIT == 3 ("bf16x3", fp32-faithful): Q, K, V arrive as hi and lo planes
// (twice the shared memory per stage), P is split in registers.  Both keep two CTAs per SM.
template <int NSPLIT> struct A5 {
  static constexpr int PL = NSPLIT == 3 ? 2 : 1;                        // operand planes
  static constexpr int KV_STAGES = NSPLIT == 3 ? 2 : 4;
  static constexpr int Q_STAGE = PL * Q_BYTES;                          // [hi | lo]
  static constexpr int KV_STAGE = PL * 2 * KV_TILE_BYTES;               // [K hi | V hi | K lo | V lo]
  static constexpr int SMEM_BYTES = Q_STAGE + KV_STAGES * KV_STAGE + 1024 + 256;   // tiles + alignment slack + barriers
};

// V tile descriptor (MN-major, 64 head dims = one 128 B swizzle row per key): the K direction steps over 8-key atoms.  LBO and
// SBO both carry the 1024 B atom stride -- with a single 64-element atom across N only that stride is ever applied.
__device__ __forceinline__ uint64_t make_v_desc(uint32_t smem_addr) { return make_smem_desc(smem_addr) | ((uint64_t)(1024 >> 4) << 16); }

__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// two fp32 -> packed 16-bit pair (IEEE half or bf16), one cvt instruction
__device__ __forceinline__ uint32_t pack2_16(float lo, float hi, bool fp16) {
  uint32_t r;
  if (fp16) asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  else asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}

template <bool FP16>
__device__ __forceinline__ void mma_qk(float (&d)[32], uint64_t da, uint64_t db, uint32_t acc) {
  if (FP16) wgmma_m64n64k16_ss_f16(d, da, db, acc);
  else wgmma_m64n64k16_ss_bf16(d, da, db, acc);
}
template <bool FP16>
__device__ __forceinline__ void mma_pv(float (&d)[32], const uint32_t (&a)[4], uint64_t db) {
  if (FP16) wgmma_m64n64k16_rs_f16(d, a, db, 1u);
  else wgmma_m64n64k16_rs_bf16(d, a, db, 1u);
}

struct Attn5Params {
  AttnOut out;
  int B, S, H, ctx_rows, ctx_keys, fp16;
  float scale_log2e;
  AttnPlan pl;
};

template <bool FP16, int NSPLIT>
__global__ void __launch_bounds__(NUM_THREADS, 2)
attention_tc5_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_kv,
                     const __grid_constant__ CUtensorMap map_q_lo, const __grid_constant__ CUtensorMap map_kv_lo, const Attn5Params p) {
  static_assert(NSPLIT == 1 || (NSPLIT == 3 && !FP16), "split mode uses bf16 planes");
  using C = A5<NSPLIT>;
  constexpr int KV_STAGES = C::KV_STAGES;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t q_s = base;                                  // Q hi (, Q lo)
  const uint32_t kv_s = base + C::Q_STAGE;                    // stage st at kv_s + st * KV_STAGE: K hi, V hi (, K lo, V lo)
  const uint32_t bars = kv_s + KV_STAGES * C::KV_STAGE;
  const uint32_t q_full = bars;
  auto kv_full = [&](int st) { return bars + 8 + 8u * st; };
  auto kv_empty = [&](int st) { return bars + 8 + 8u * KV_STAGES + 8u * st; };

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int S = p.S;
  const int nq = (S + BQ - 1) / BQ;
  const int item = blockIdx.x;
  const int qt = item % nq, h = (item / nq) % p.H, b = item / (nq * p.H);
  // token-range plan: this image's live context rows pc and live keys [0, live); a tile of context rows only stops at pc
  const int pc = p.pl.plan ? p.pl.plan[2 * b + 1] : 0, live = p.pl.plan ? pc + p.pl.n_img : S;
  const int kmax_cta = !p.pl.plan ? (((qt + 1) * BQ <= p.ctx_rows) ? p.ctx_keys : S)   // every row of the tile is a context row
                                  : ((p.pl.ctx_self && ((qt + 1) * BQ <= pc || qt * BQ >= live)) ? pc : live);
  const int n_tiles = (kmax_cta + BKV - 1) / BKV;
  const int row0 = b * S;                                     // first row of this image in the [B*S, 3*H*64] matrix
  if (p.pl.packed && qt * BQ >= live) return;                 // packed slot: no row of this tile holds anything

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&map_q);
    tma_prefetch_desc(&map_kv);
    mbar_init(q_full, 1);
    for (int st = 0; st < KV_STAGES; ++st) { mbar_init(kv_full(st), 1); mbar_init(kv_empty(st), 2); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == 8) {
    // =========================================================== TMA producer
    if (lane == 0) {
      mbar_expect_tx(q_full, C::Q_STAGE);
      tma_load_2d(q_s, &map_q, q_full, h * HD, row0 + qt * BQ);
      if (NSPLIT == 3) tma_load_2d(q_s + Q_BYTES, &map_q_lo, q_full, h * HD, row0 + qt * BQ);
      for (int j = 0; j < n_tiles; ++j) {
        const int st = j % KV_STAGES;
        mbar_wait(kv_empty(st), ((j / KV_STAGES) & 1) ^ 1);
        const uint32_t ks = kv_s + st * C::KV_STAGE;
        mbar_expect_tx(kv_full(st), C::KV_STAGE);
        tma_load_2d(ks, &map_kv, kv_full(st), (p.H + h) * HD, row0 + j * BKV);
        tma_load_2d(ks + KV_TILE_BYTES, &map_kv, kv_full(st), (2 * p.H + h) * HD, row0 + j * BKV);
        if (NSPLIT == 3) {
          tma_load_2d(ks + 2 * KV_TILE_BYTES, &map_kv_lo, kv_full(st), (p.H + h) * HD, row0 + j * BKV);
          tma_load_2d(ks + 3 * KV_TILE_BYTES, &map_kv_lo, kv_full(st), (2 * p.H + h) * HD, row0 + j * BKV);
        }
      }
    }
    return;
  }
  // =========================================================== consumer warpgroups
  const int wg = warp >> 2, wl = threadIdx.x & 127;
  const int quad = lane & 3;
  // this thread's two rows of the tile (accumulator fragment rows r and r + 8) and its key / dim columns 8 i + 2 quad + {0, 1}
  const int rt = wg * 64 + (wl >> 5) * 16 + (lane >> 2);
  int kmax[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int row = qt * BQ + rt + 8 * r;
    kmax[r] = !p.pl.plan ? ((row < p.ctx_rows) ? p.ctx_keys : S) : ((p.pl.ctx_self && (row < pc || row >= live)) ? pc : live);
  }
  float m_run[2] = {-INFINITY, -INFINITY}, l_part[2] = {0.f, 0.f};
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  const uint32_t qs = q_s + wg * (64 * 128);                  // this warpgroup's 64 Q rows (8 swizzle atoms)
  mbar_wait(q_full, 0);
  for (int j = 0; j < n_tiles; ++j) {
    const int st = j % KV_STAGES;
    mbar_wait(kv_full(st), (j / KV_STAGES) & 1);
    const uint32_t ks = kv_s + st * C::KV_STAGE, vs = ks + KV_TILE_BYTES;
    float s[32];
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < HD / 16; ++k) {                       // K dimension = head dim: 32 B per k-step inside the row
      mma_qk<FP16>(s, make_smem_desc(qs + k * 32), make_smem_desc(ks + k * 32), k > 0 ? 1u : 0u);
      if (NSPLIT == 3) {                                      // + Q_hi K_lo^T + Q_lo K_hi^T
        mma_qk<FP16>(s, make_smem_desc(qs + k * 32), make_smem_desc(ks + 2 * KV_TILE_BYTES + k * 32), 1u);
        mma_qk<FP16>(s, make_smem_desc(qs + Q_BYTES + k * 32), make_smem_desc(ks + k * 32), 1u);
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(s);
    // ---- online softmax (log2 domain); a row's 64 keys are spread over the 4 lanes of a quad
    uint32_t ph[16], pl[16];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      float mx = -INFINITY;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          const int key = j * BKV + 8 * i + 2 * quad + c;
          float& v = s[4 * i + 2 * r + c];
          if (key >= kmax[r]) v = -INFINITY;
          mx = fmaxf(mx, v);
        }
      }
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m_run[r], mx * p.scale_log2e);
      const float sub = (m_new == -INFINITY) ? 0.f : m_new;
      const float corr = (m_new == m_run[r] || m_new == -INFINITY) ? 1.f : ex2_approx(m_run[r] - m_new);
      float rs = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float e0 = ex2_approx(fmaf(s[4 * i + 2 * r], p.scale_log2e, -sub));
        const float e1 = ex2_approx(fmaf(s[4 * i + 2 * r + 1], p.scale_log2e, -sub));
        rs += e0 + e1;
        // A fragment of k-step i / 2: registers {row r, keys 2 quad..} then {row r, keys 8 + 2 quad..}
        const int ai = 4 * (i >> 1) + 2 * (i & 1) + r;
        ph[ai] = pack2_16(e0, e1, FP16);
        if (NSPLIT == 3) pl[ai] = pack2_resid_bf16(e0, e1, ph[ai]);   // lo plane: rn(p - rn_bf16(p))
      }
      l_part[r] = l_part[r] * corr + rs;
      m_run[r] = m_new;
#pragma unroll
      for (int i = 0; i < 8; ++i) { o[4 * i + 2 * r] *= corr; o[4 * i + 2 * r + 1] *= corr; }
    }
    // ---- O += P V
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < BKV / 16; ++k) {                      // 16 keys = 2 atoms of 8 key rows of the V tile
      const uint32_t a_hi[4] = {ph[4 * k], ph[4 * k + 1], ph[4 * k + 2], ph[4 * k + 3]};
      mma_pv<FP16>(o, a_hi, make_v_desc(vs + k * 2048));
      if (NSPLIT == 3) {                                      // + P_hi V_lo + P_lo V_hi
        const uint32_t a_lo[4] = {pl[4 * k], pl[4 * k + 1], pl[4 * k + 2], pl[4 * k + 3]};
        mma_pv<FP16>(o, a_hi, make_v_desc(vs + 2 * KV_TILE_BYTES + k * 2048));
        mma_pv<FP16>(o, a_lo, make_v_desc(vs + k * 2048));
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(o);
    if (wl == 0) mbar_arrive(kv_empty(st));                   // this warpgroup's reads of the stage have completed
  }
  // ---- epilogue: O / l -> fp32 and / or 16-bit planes
  const AttnOut& t = p.out;
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    float l = l_part[r];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const int row = qt * BQ + rt + 8 * r;
    if (row >= S) continue;
    const float inv = l > 0.f ? 1.0f / l : 0.f;                // a row with no visible key (token-range plan) writes 0
    bool inA = row < t.split;
    int64_t orow = inA ? ((int64_t)b * t.split + row) : ((int64_t)b * (S - t.split) + (row - t.split));
    if (p.pl.packed) {
      if (row >= live) continue;
      inA = row < pc;
      orow = inA ? (int64_t)p.pl.plan[2 * b] + row : (int64_t)b * p.pl.n_img + row - pc;
    } else if (p.pl.plan && p.pl.route) {
      const int sr = plan_stream_row(row, p.pl.plan[2 * b], pc, p.pl.n_img, inA);
      orow = inA ? (int64_t)b * t.split + sr : (int64_t)b * p.pl.n_img + sr;
    }
    float* of = inA ? t.f32_a : t.f32_b;
    __nv_bfloat16* oh = inA ? t.hi_a : t.hi_b;
    __nv_bfloat16* ol = inA ? t.lo_a : t.lo_b;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int64_t off = orow * t.ld + (int64_t)h * HD + 8 * i + 2 * quad;
      const float y0 = o[4 * i + 2 * r] * inv, y1 = o[4 * i + 2 * r + 1] * inv;
      if (of) *reinterpret_cast<float2*>(of + off) = make_float2(y0, y1);
      if (oh) {
        const uint32_t hp = pack2_sat16(y0, y1, FP16);
        *reinterpret_cast<uint32_t*>(oh + off) = hp;
        if (!FP16 && ol) *reinterpret_cast<uint32_t*>(ol + off) = pack2_resid_bf16(y0, y1, hp);   // bf16 residual planes
      }
    }
  }
}

bool g_attr_dev[64];       // cudaFuncSetAttribute is per device: one handle per GPU may live in the same process

}  // namespace

int launch_attention_tc5(const __nv_bfloat16* qkv16, int B, int S, int H, int ctx_rows, int ctx_keys, const AttnOut& out,
                         cudaStream_t s, int fp16, const __nv_bfloat16* qkv_lo, const AttnPlan& plan) {
  STK_CHECK(qkv16 && B > 0 && S > 0 && H > 0, -1, "attention_tc5: bad arguments");
  STK_CHECK(out.ld % 8 == 0, -1, "attention_tc5: output pitch must be a multiple of 8");
  STK_CHECK(ctx_keys <= S && ctx_rows <= S && ctx_keys >= 0 && ctx_rows >= 0, -1, "attention_tc5: context limits exceed the sequence");
  STK_CHECK(!(fp16 && qkv_lo), -1, "attention_tc5: the split mode uses bf16 planes");
  STK_CHECK(!plan.plan || (plan.n_img > 0 && plan.n_img <= S && (!plan.route || out.split == S - plan.n_img)), -1,
            "attention_tc5: inconsistent token-range plan");
  STK_TRY(gemm_tc_init());
  int dev = 0;
  STK_CUDA(cudaGetDevice(&dev));
  STK_CHECK(dev >= 0 && dev < 64, -1, "attention_tc5: device ordinal out of range");
  if (!g_attr_dev[dev]) {
    STK_CUDA(cudaFuncSetAttribute(attention_tc5_kernel<true, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, A5<1>::SMEM_BYTES));
    STK_CUDA(cudaFuncSetAttribute(attention_tc5_kernel<false, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, A5<1>::SMEM_BYTES));
    STK_CUDA(cudaFuncSetAttribute(attention_tc5_kernel<false, 3>, cudaFuncAttributeMaxDynamicSharedMemorySize, A5<3>::SMEM_BYTES));
    g_attr_dev[dev] = true;
  }
  CUtensorMap mq, mkv, mql, mkvl;
  const uint64_t rows = (uint64_t)B * S, cols = (uint64_t)3 * H * HD;
  STK_TRY(make_tensor_map_2d(&mq, qkv16, rows, cols, BQ, HD, fp16));
  STK_TRY(make_tensor_map_2d(&mkv, qkv16, rows, cols, BKV, HD, fp16));
  mql = mq; mkvl = mkv;
  if (qkv_lo) {
    STK_TRY(make_tensor_map_2d(&mql, qkv_lo, rows, cols, BQ, HD, 0));
    STK_TRY(make_tensor_map_2d(&mkvl, qkv_lo, rows, cols, BKV, HD, 0));
  }
  Attn5Params p{out, B, S, H, ctx_rows, ctx_keys, fp16, 0.125f * 1.4426950408889634f, plan};
  const int n_items = ((S + BQ - 1) / BQ) * H * B;
  if (qkv_lo) attention_tc5_kernel<false, 3><<<n_items, NUM_THREADS, A5<3>::SMEM_BYTES, s>>>(mq, mkv, mql, mkvl, p);
  else if (fp16) attention_tc5_kernel<true, 1><<<n_items, NUM_THREADS, A5<1>::SMEM_BYTES, s>>>(mq, mkv, mql, mkvl, p);
  else attention_tc5_kernel<false, 1><<<n_items, NUM_THREADS, A5<1>::SMEM_BYTES, s>>>(mq, mkv, mql, mkvl, p);
  count_launch();
  STK_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace stk
