// Tensor-core GEMM of the MMDiT linears (sm_90a):  y = A W^T (+bias, fused epilogue), fp32 accumulation in registers.
//
//   operands   bf16 planes, K-major.  NSPLIT == 1: y = A_hi W_hi^T.  NSPLIT == 3 ("bf16x3", fp32-faithful to ~2^-17):
//              y = A_hi W_hi^T + A_hi W_lo^T + A_lo W_hi^T, all three products accumulated into the same registers.
//              E4M3: e4m3 codes with per-row scales (kernels.h), wgmma m64n256k32; a k-block is 128 elements, so the tiles, TMA
//              boxes and descriptors (128 B per K row) are byte for byte those of the 16-bit modes.
//   tile       128 x 256 x 64 per pipeline stage per CTA; two consumer warpgroups, each wgmma m64n256k16 on its 64 rows
//   staging    TMA (cp.async.bulk.tensor, SWIZZLE_128B) -> shared memory ring, mbarrier full/empty pairs
//   roles      warpgroups 0-1: wgmma + epilogue (registers -> HBM) | warpgroup 2: TMA producer (1 thread)
//   cluster    CL == 2: two CTAs (rows 256 apart in M) share the W tile: each loads half of it and multicasts it to both,
//              halving the L2 -> SM traffic of the weights; CL == 1: one CTA loads the whole tile
//   schedule   persistent CTAs (grid = #SMs), tiles rasterised in groups of M-blocks for L2 reuse of W
//
// Replaces the cuBLAS SGEMMs behind nn.Linear in DismantledBlock (sd3/mmdit.py:266,269,293,301; other_impls.py:82-84)
// together with the elementwise kernels around them (bias, GELU-tanh, gate*y + residual; mmdit.py:485-496).
#include "common.cuh"
#include "hopper.cuh"
#include "kernels.h"

#include <stdlib.h>

namespace stk {

namespace {

using namespace hop;

constexpr int BM = 128, BN = 256, BK = 64, WK = 16;   // BK, WK: 16-bit elements (128 B / 32 B of a K row)
constexpr int BK8 = 128;                               // e4m3 elements per k-block (the same 128 B)
constexpr int A_TILE_BYTES = BM * BK * 2;      // 16 KiB
constexpr int B_TILE_BYTES = BN * BK * 2;      // 32 KiB
constexpr int CONSUMERS = 2;                   // warpgroups of 64 rows
constexpr int NUM_THREADS = CONSUMERS * 128 + 128;  // + one producer warpgroup (one thread of it issues the TMA loads)
// Register split (setmaxnreg): 2 x 128 x 232 + 128 x 40 = 64,512 of the 65,536 registers.  The consumers hold 128 fp32
// accumulators plus a batch of epilogue operands; at the 168 registers an even split leaves them, the epilogue spills.
constexpr int PRODUCER_REGS = 40, CONSUMER_REGS = 232;
constexpr int ACC = BN / 2;                    // fp32 accumulators per consumer thread
constexpr int kPrefetchKBlocks = 4;            // residual rows go to L2 this many k-blocks before the epilogue

template <int NSPLIT> struct Cfg {
  static constexpr int PLANES = NSPLIT == 3 ? 2 : 1;
  static constexpr int STAGE_BYTES = PLANES * (A_TILE_BYTES + B_TILE_BYTES);     // 48 KiB / 96 KiB
  static constexpr int STAGES = NSPLIT == 3 ? 2 : 4;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
};

__device__ __forceinline__ void wgmma_tile(float (&d)[ACC], uint64_t da, uint64_t db, uint32_t acc, bool fp16) {
  if (fp16) wgmma_m64n256k16_ss_f16(d, da, db, acc);
  else wgmma_m64n256k16_ss_bf16(d, da, db, acc);
}

__device__ __forceinline__ float2 ldg2(const float* p) { return *reinterpret_cast<const float2*>(p); }

// Rows of one consumer thread's accumulators (row0 and row0 + 8): output row (token-range plan, packed row_map or the plain
// [image][row] remap) and gate / addtab table row.  Resolved at tile start, so that the row_map / tab_rows reads and the L2
// prefetch of the residual rows (epilogue_prefetch) overlap the mainloop.
struct EpiRows {
  int orow[2], mrow[2];
  bool valid[2];
  float sa[2];                                         // e4m3: A row scales (GEMM rows, before any remap)
};

// m[r]: GEMM row of accumulator row r (a convolution's output pixel), valid[r]: m[r] < M and, for a convolution, inside the image
template <bool E4M3>
__device__ __forceinline__ EpiRows epilogue_rows(const Epilogue& e, const int64_t (&m)[2], const bool (&valid)[2]) {
  const bool per_row_gate = e.mode == EPI_RESID && e.gate && (e.gate_period > 1 || e.tab_rows);
  const bool per_row_add = e.mode == EPI_STORE && e.addtab;
  EpiRows rw;
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    rw.valid[r] = valid[r];
    const int mi = (int)m[r];
    rw.orow[r] = 0;
    if (e.row_map && rw.valid[r]) {
      rw.orow[r] = e.row_map[mi];
    } else if (e.plan && rw.valid[r]) {                 // token-range plan: image rows per slot = rpb_out - Kc
      const int b = mi / e.rpb_in;
      const int n_img = e.rpb_out - (e.plan_ctx ? e.rpb_in : e.row_off);
      rw.orow[r] = b * e.rpb_out + plan_slot_row(mi % e.rpb_in, e.plan[2 * b], e.plan[2 * b + 1], n_img, e.plan_ctx != 0);
    } else if (rw.valid[r]) {
      rw.orow[r] = e.rpb_in > 0 ? (mi / e.rpb_in) * e.rpb_out + e.row_off + (mi % e.rpb_in) : mi;
    }
    if (e.tab_rows && rw.valid[r]) rw.mrow[r] = e.tab_rows[mi];
    else rw.mrow[r] = per_row_gate ? mi % e.gate_period : (per_row_add ? mi % e.add_period : 0);
    rw.sa[r] = E4M3 && rw.valid[r] ? e.s_a[mi] : 0.f;
  }
  return rw;
}

// Residual rows of the tile into L2, a few k-blocks before the epilogue reads them: lane q of each quad takes 128 B lines
// 2q and 2q + 1 of the 1 KB row segment of both its rows.  Only rows < M and columns < N are touched.
__device__ __forceinline__ void epilogue_prefetch(const Epilogue& e, const EpiRows& rw, int col0, int N) {
  if (e.mode != EPI_RESID) return;
  const int c0 = col0 & ~(BN - 1);
  const int q = (col0 >> 1) & 3;
#pragma unroll
  for (int r = 0; r < 2; ++r) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int n = c0 + 32 * (2 * q + h);
      if (rw.valid[r] && n < N) prefetch_l2(e.resid + (int64_t)rw.orow[r] * e.ldo + n);
    }
  }
}

// Epilogue of one consumer thread's accumulators: rows rw.orow, column pairs col0 + 8 j (j < 32).  Every access of a quad of
// lanes covers 32 contiguous bytes of a row.  MODE / GELU are compile-time so that the per-element path carries no mode
// branches.  The columns go in batches of CH pairs: every load of a batch (bias, gate, residual, addtab) is issued before its
// first store.  The output may alias the residual (the in-place residual stream), so a load placed after a store could not be
// moved ahead of it and each pair would pay a full global round trip.  Per element the arithmetic is unchanged.
// E4M3: y = fma(acc, s_a[m] * s_w[n], bias); the W scales are loaded with the bias.
template <int MODE, bool GELU, bool E4M3>
__device__ __forceinline__ void epilogue_tile(const Epilogue& e, const float (&acc)[ACC], const EpiRows& rw, int col0, int N) {
  constexpr int CH = MODE == EPI_RESID ? 4 : 8;        // residual + gate of both rows: 8 registers per pair
  const bool per_row_gate = MODE == EPI_RESID && e.gate && (e.gate_period > 1 || e.tab_rows);
  const bool per_row_add = MODE == EPI_STORE && e.addtab;
  const bool fp16 = e.fp16 != 0;
  const float2 zero = make_float2(0.f, 0.f), one = make_float2(1.f, 1.f);
#pragma unroll
  for (int c = 0; c < BN / 8; c += CH) {
    float2 bias[CH], sw[CH], res[2][CH], gt[2][CH], add[2][CH];
#pragma unroll
    for (int i = 0; i < CH; ++i) {
      const int n = col0 + 8 * (c + i);
      const bool in = n < N;                             // N % 4 == 0 and n even: a pair is all in or all out
      bias[i] = e.bias && in ? ldg2(e.bias + n) : zero;
      if (E4M3) sw[i] = in ? ldg2(e.s_w + n) : zero;
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const bool v = in && rw.valid[r];
        const int64_t o = (int64_t)rw.orow[r] * e.ldo + n;
        if (MODE == EPI_RESID) {
          res[r][i] = v ? ldg2(e.resid + o) : zero;
          gt[r][i] = v && e.gate ? ldg2(per_row_gate ? e.gate + (int64_t)rw.mrow[r] * e.gate_ld + n : e.gate + n) : one;
        }
        if (MODE == EPI_STORE) add[r][i] = v && per_row_add ? ldg2(e.addtab + (int64_t)rw.mrow[r] * e.add_ld + n) : zero;
      }
    }
#pragma unroll
    for (int i = 0; i < CH; ++i) {
      const int j = c + i;
      const int n = col0 + 8 * j;
      if (n >= N) continue;
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        if (!rw.valid[r]) continue;
        float2 y;
        if (E4M3) {
          y = make_float2(fmaf(acc[4 * j + 2 * r], rw.sa[r] * sw[i].x, bias[i].x), fmaf(acc[4 * j + 2 * r + 1], rw.sa[r] * sw[i].y, bias[i].y));
        } else {
          y = make_float2(acc[4 * j + 2 * r] + bias[i].x, acc[4 * j + 2 * r + 1] + bias[i].y);
        }
        if (GELU) y = gelu_tanh_fast2(y);
        const int64_t o = (int64_t)rw.orow[r] * e.ldo + n;
        if (MODE == EPI_RESID) {
          y.x = fmaf(gt[r][i].x, y.x, res[r][i].x); y.y = fmaf(gt[r][i].y, y.y, res[r][i].y);
        }
        if (MODE == EPI_SPLIT) {
          const uint32_t hi = pack2_sat16(y.x, y.y, fp16);
          *reinterpret_cast<uint32_t*>(e.out_hi + o) = hi;
          if (e.out_lo) {                                // bf16x3: residual planes
            const float lx = y.x - __bfloat162float(__float2bfloat16_rn(y.x)), ly = y.y - __bfloat162float(__float2bfloat16_rn(y.y));
            *reinterpret_cast<uint32_t*>(e.out_lo + o) = pack2_sat16(lx, ly, false);
          }
        } else {
          if (per_row_add) { y.x += add[r][i].x; y.y += add[r][i].y; }
          *reinterpret_cast<float2*>(e.out + o) = y;
        }
      }
    }
  }
}

// mode / activation dispatch (uniform across the grid)
template <bool E4M3>
__device__ __forceinline__ void epilogue_dispatch(const Epilogue& e, const float (&acc)[ACC], const EpiRows& rw, int col0, int N) {
  if (e.mode == EPI_RESID) epilogue_tile<EPI_RESID, false, E4M3>(e, acc, rw, col0, N);
  else if (e.mode == EPI_SPLIT) {
    if (e.act == ACT_GELU) epilogue_tile<EPI_SPLIT, true, E4M3>(e, acc, rw, col0, N);
    else epilogue_tile<EPI_SPLIT, false, E4M3>(e, acc, rw, col0, N);
  } else {
    if (e.act == ACT_GELU) epilogue_tile<EPI_STORE, true, E4M3>(e, acc, rw, col0, N);
    else epilogue_tile<EPI_STORE, false, E4M3>(e, acc, rw, col0, N);
  }
}

struct TcMaps {
  CUtensorMap a_hi, a_lo, b_hi, b_lo;
};

struct GemmParams {
  int64_t M;
  int N, K;
  int fp16;
  Epilogue ep;
  // implicit-GEMM 3x3 convolution (stride 1, zero padding 1) over NHWC activations: A row m = output pixel (b, y, x), K index =
  // tap * C + c.  conv_C == 0: plain GEMM.  The A tile of k-block kb (tap = kb / (C / 64), channels chunk = kb % (C / 64)) is the
  // 4-D TMA box {64 channels, bw pixels, bh rows, bn images} (bw bh bn = 128) shifted by the tap offset; out-of-image elements
  // are zero-filled by the TMA unit -- exactly the padding.  The 128-row blocks tile each group of bn images as conv_ty x conv_tx
  // boxes (conv_origin); a box may overhang the right / bottom edge (conv_box), and its rows outside the image are dropped by the
  // epilogue: no store and no load of resid / gate / addtab.
  // conv_stride == 2 (Downsample, sd3_impls.py:287-298: zero pad right / bottom, 3x3 stride 2): the planes hold the four
  // polyphase components of the input, [image * 4 + (py * 2 + px)][H_out][W_out][C] with phase(py, px)[y][x] = in[2y + py][2x + px];
  // tap (dy, dx) reads phase (dy & 1, dx & 1) shifted by (dy >> 1, dx >> 1) -- unit-stride boxes again, the zero fill past the last
  // row / column is the one-sided padding.  conv_H / conv_W are the OUTPUT dims.
  int conv_C = 0, conv_H = 0, conv_W = 0, conv_stride = 1;
  int conv_bw = 0, conv_bh = 0, conv_bn = 1, conv_tx = 1, conv_ty = 1;
  int blocks = 0;        // 128-row A blocks: ceil(M / 128), or images / bn x conv_ty x conv_tx for a convolution
  int raster_gm = 4;     // cluster-rows per raster group (tile_coords)
};

// first output pixel (b, y, x) of 128-row block `blk` of a convolution
__device__ __forceinline__ void conv_origin(const GemmParams& p, int blk, int& b, int& y, int& x) {
  b = blk / (p.conv_tx * p.conv_ty) * p.conv_bn;
  y = blk / p.conv_tx % p.conv_ty * p.conv_bh;
  x = blk % p.conv_tx * p.conv_bw;
}

// Rows lrow and lrow + 8 of 128-row block blk, for one consumer thread's epilogue.  A convolution's row is the output pixel
// its box element lands on (the box is row-major: x fastest, then y, then image); pixels of an overhanging box that fall
// outside the image are invalid.  For the boxes that tile images exactly, m = 128 blk + row as in a plain GEMM.
template <bool E4M3>
__device__ __forceinline__ EpiRows tile_rows(const GemmParams& p, int blk, int lrow) {
  int64_t m[2];
  bool valid[2];
  if (!E4M3 && p.conv_C > 0) {
    int b, y, x;
    conv_origin(p, blk, b, y, x);
    const int per = p.conv_bw * p.conv_bh;
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int l = lrow + 8 * r;
      const int yy = y + l % per / p.conv_bw, xx = x + l % p.conv_bw;
      m[r] = ((int64_t)(b + l / per) * p.conv_H + yy) * p.conv_W + xx;
      valid[r] = yy < p.conv_H && xx < p.conv_W && m[r] < p.M;
    }
  } else {
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      m[r] = (int64_t)blk * BM + lrow + 8 * r;
      valid[r] = m[r] < p.M;
    }
  }
  return epilogue_rows<E4M3>(p.ep, m, valid);
}

// Cluster-row and column tile counts of both problems, problem 0's tile count and the total.  Each role derives them after its
// setmaxnreg: kept live across it, ptxas spills them.
struct TileCounts {
  int pm0, n0, pm1, n1, tiles0, total;
};
template <int CL>
__device__ __forceinline__ TileCounts tile_counts(const GemmParams& p0, const GemmParams& p1) {
  TileCounts c;
  c.pm0 = (p0.blocks + CL - 1) / CL; c.n0 = (p0.N + BN - 1) / BN;
  c.pm1 = (p1.blocks + CL - 1) / CL; c.n1 = (p1.N + BN - 1) / BN;
  c.tiles0 = c.pm0 * c.n0;
  c.total = c.tiles0 + c.pm1 * c.n1;
  return c;
}

__device__ __forceinline__ void tile_coords(int t, int pm_tiles, int n_tiles, int GM, int& pm, int& n_blk) {
  // GM cluster-rows share each W tile in L2; SELFTOK_GEMM_GM is a measurement knob (any value is a bijection of the tile
  // list, results never change)
  const int per_group = GM * n_tiles;
  const int group = t / per_group;
  const int first = group * GM;
  const int gm = min(GM, pm_tiles - first);
  const int local = t - group * per_group;
  pm = first + local % gm;
  n_blk = local / gm;
}

// ---------------------------------------------------------------------------------------------- kernel
// Up to two independent problems (same NSPLIT / operand type) share the launch: the context- and the image-stream GEMM of
// a layer.  Tiles of problem 0 come first; problem 1 may be empty (M == 0).  A tile is CL x 128 rows x 256 columns: CTA
// `rank` of the cluster computes rows [128 rank, 128 rank + 128) of it.
//   full[s]    per CTA: its own A box plus both halves of the W tile (one from each CTA of the cluster) complete_tx on it
//   empty[s]   per CTA: counts the two consumer warpgroups of EVERY CTA of the cluster, because the producer of this CTA
//              writes its half of the W tile into all of them
template <int NSPLIT, int CL, bool FP16, bool E4M3>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_tc_kernel(const __grid_constant__ TcMaps maps0, const __grid_constant__ TcMaps maps1, const GemmParams p0, const GemmParams p1) {
  static_assert(NSPLIT == 1 || !FP16, "the fp16 mode is single-pass");
  static_assert(!E4M3 || (NSPLIT == 1 && !FP16), "the e4m3 mode is single-pass on its own operand type");
  using C = Cfg<NSPLIT>;
  constexpr int KB = E4M3 ? BK8 : BK;                   // elements per k-block
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;           // SWIZZLE_128B tiles need 1024 B alignment
  const uint32_t bar_base = smem_base + C::STAGES * C::STAGE_BYTES;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (C::STAGES + s); };

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t rank = CL > 1 ? cluster_ctarank() : 0;
  const int cluster_id = blockIdx.x / CL, num_clusters = gridDim.x / CL;

  if (warp == CONSUMERS * 4 && lane == 0) {
    tma_prefetch_desc(&maps0.a_hi);
    tma_prefetch_desc(&maps0.b_hi);
    if (NSPLIT == 3) { tma_prefetch_desc(&maps0.a_lo); tma_prefetch_desc(&maps0.b_lo); }
    if (p1.M > 0) {
      tma_prefetch_desc(&maps1.a_hi);
      tma_prefetch_desc(&maps1.b_hi);
      if (NSPLIT == 3) { tma_prefetch_desc(&maps1.a_lo); tma_prefetch_desc(&maps1.b_lo); }
    }
    for (int s = 0; s < C::STAGES; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), CONSUMERS * CL); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (CL > 1) cluster_sync_all();                         // peer barriers initialised before any multicast / remote arrive

  if (warp >= CONSUMERS * 4) {
    // =========================================================== TMA producer
    setmaxnreg_dec<PRODUCER_REGS>();
    const auto [pm_tiles0, n_tiles0, pm_tiles1, n_tiles1, tiles0, num_tiles] = tile_counts<CL>(p0, p1);
    if (warp == CONSUMERS * 4 && lane == 0) {
      int stage = 0; uint32_t phase = 0;
      // The weight tile is re-read by every group of M tiles; without a hint the activation / residual / output streams of the
      // K = 6144 GEMM push it out of L2 between groups.  evict_last keeps it.
      const uint64_t w_policy = l2_policy_evict_last();
      for (int t = cluster_id; t < num_tiles; t += num_clusters) {
        const bool second = t >= tiles0;
        const TcMaps& mp = second ? maps1 : maps0;
        const GemmParams& pp = second ? p1 : p0;
        int pm, n_blk;
        if (second) tile_coords(t - tiles0, pm_tiles1, n_tiles1, p1.raster_gm, pm, n_blk);
        else tile_coords(t, pm_tiles0, n_tiles0, p0.raster_gm, pm, n_blk);
        const int nk = (pp.K + KB - 1) / KB;
        const int blk = pm * CL + (int)rank;                        // this CTA's 128 A rows
        const int m_row = blk * BM;
        const int n_row = n_blk * BN + (int)rank * (BN / CL);       // this CTA's share of the W tile
        // convolution: the 128 rows are the box of bh image rows of bw pixels (of bn images) starting at (cb, cy, cx)
        // (the e4m3 mode has no convolution: the host refuses it, and its instantiations carry no convolution code)
        const bool conv = !E4M3 && pp.conv_C > 0;
        const int chunks = conv ? pp.conv_C / BK : 1;
        int cx = 0, cy = 0, cb = 0;
        if (conv) conv_origin(pp, blk, cb, cy, cx);
        for (int kb = 0; kb < nk; ++kb) {
          mbar_wait(empty_bar(stage), phase ^ 1);
          const uint32_t sa = smem_base + stage * C::STAGE_BYTES;
          const uint32_t sb = sa + C::PLANES * A_TILE_BYTES + (uint32_t)rank * (B_TILE_BYTES / CL);
          const uint32_t fb = full_bar(stage);
          mbar_expect_tx(fb, C::STAGE_BYTES);
          if (conv) {
            const int tap = kb / chunks, c0 = (kb - tap * chunks) * BK;
            const int dy = tap / 3, dx = tap - dy * 3;
            int x0 = cx + dx - 1, y0 = cy + dy - 1, n0 = cb;
            if (pp.conv_stride == 2) { x0 = cx + (dx >> 1); y0 = cy + (dy >> 1); n0 = cb * 4 + (dy & 1) * 2 + (dx & 1); }
            tma_load_4d(sa, &mp.a_hi, fb, c0, x0, y0, n0);
            if (NSPLIT == 3) tma_load_4d(sa + A_TILE_BYTES, &mp.a_lo, fb, c0, x0, y0, n0);
          } else {
            tma_load_2d(sa, &mp.a_hi, fb, kb * KB, m_row);
            if (NSPLIT == 3) tma_load_2d(sa + A_TILE_BYTES, &mp.a_lo, fb, kb * BK, m_row);
          }
          if (CL > 1) {
            tma_load_2d_mc(sb, &mp.b_hi, fb, kb * KB, n_row, (uint16_t)((1u << CL) - 1), w_policy);
            if (NSPLIT == 3) tma_load_2d_mc(sb + B_TILE_BYTES, &mp.b_lo, fb, kb * BK, n_row, (uint16_t)((1u << CL) - 1), w_policy);
          } else {
            tma_load_2d_hint(sb, &mp.b_hi, fb, kb * KB, n_row, w_policy);
            if (NSPLIT == 3) tma_load_2d_hint(sb + B_TILE_BYTES, &mp.b_lo, fb, kb * BK, n_row, w_policy);
          }
          if (++stage == C::STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // =========================================================== consumer warpgroups: wgmma + epilogue
    setmaxnreg_inc<CONSUMER_REGS>();
    const auto [pm_tiles0, n_tiles0, pm_tiles1, n_tiles1, tiles0, num_tiles] = tile_counts<CL>(p0, p1);
    const int wg = warp >> 2;                                        // rows [64 wg, 64 wg + 64) of the CTA's 128
    const bool signaller = (threadIdx.x & 127) == 0;
    auto release = [&](int s) {                                      // the stage's wgmma reads have completed
      if (!signaller) return;
      if (CL == 1) mbar_arrive(empty_bar(s));
      else for (int r = 0; r < CL; ++r) mbar_arrive_cluster(empty_bar(s), (uint32_t)r);
    };
    int stage = 0; uint32_t phase = 0;
    for (int t = cluster_id; t < num_tiles; t += num_clusters) {
      const bool second = t >= tiles0;
      int pm, n_blk;
      if (second) tile_coords(t - tiles0, pm_tiles1, n_tiles1, p1.raster_gm, pm, n_blk);
      else tile_coords(t, pm_tiles0, n_tiles0, p0.raster_gm, pm, n_blk);
      const int nk = ((second ? p1.K : p0.K) + KB - 1) / KB;
      const int wl = threadIdx.x & 127;
      const int blk = pm * CL + (int)rank, lrow = wg * 64 + (wl >> 5) * 16 + ((wl & 31) >> 2);
      const int col0 = n_blk * BN + 2 * (wl & 3);
      // the two problems are handled by separate (statically addressed) copies of the epilogue
      const EpiRows rw = second ? tile_rows<E4M3>(p1, blk, lrow) : tile_rows<E4M3>(p0, blk, lrow);
      const int pf_kb = nk > kPrefetchKBlocks ? nk - kPrefetchKBlocks : 0;
      float acc[ACC];
#pragma unroll
      for (int i = 0; i < ACC; ++i) acc[i] = 0.f;
      int prev = -1;
      for (int kb = 0; kb < nk; ++kb) {
        mbar_wait(full_bar(stage), phase);
        const uint32_t sa_hi = smem_base + stage * C::STAGE_BYTES + wg * (64 * 128);
        const uint32_t sa_lo = sa_hi + A_TILE_BYTES;
        const uint32_t sb_hi = smem_base + stage * C::STAGE_BYTES + C::PLANES * A_TILE_BYTES;
        const uint32_t sb_lo = sb_hi + B_TILE_BYTES;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / WK; ++k) {
          const uint32_t koff = k * WK * 2;                          // bytes inside the 128 B swizzle row (e4m3: k32 steps)
          const uint64_t da_hi = make_smem_desc(sa_hi + koff), db_hi = make_smem_desc(sb_hi + koff);
          if (E4M3) wgmma_m64n256k32_ss_e4m3(acc, da_hi, db_hi, (kb > 0 || k > 0) ? 1u : 0u);
          else wgmma_tile(acc, da_hi, db_hi, (kb > 0 || k > 0) ? 1u : 0u, FP16);
          if (NSPLIT == 3) {
            const uint64_t da_lo = make_smem_desc(sa_lo + koff), db_lo = make_smem_desc(sb_lo + koff);
            wgmma_tile(acc, da_hi, db_lo, 1u, false);
            wgmma_tile(acc, da_lo, db_hi, 1u, false);
          }
        }
        wgmma_commit();
        if (kb == pf_kb) {
          if (!second) epilogue_prefetch(p0.ep, rw, col0, p0.N);
          else epilogue_prefetch(p1.ep, rw, col0, p1.N);
        }
        wgmma_wait<1>();                                             // the previous stage's MMAs have retired
        if (prev >= 0) release(prev);
        prev = stage;
        if (++stage == C::STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      fence_regs(acc);
      release(prev);
      if (!second) epilogue_dispatch<E4M3>(p0.ep, acc, rw, col0, p0.N);
      else epilogue_dispatch<E4M3>(p1.ep, acc, rw, col0, p1.N);
    }
  }
  // ---- teardown: nobody may exit while a peer can still multicast into its shared memory or arrive on its barriers
  if (CL > 1) cluster_sync_all();
}

// ---------------------------------------------------------------------------------------------- host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn g_encode = nullptr;
// per-device state: cudaFuncSetAttribute and the SM count belong to a device, and one process may hold a handle per GPU
constexpr int kMaxDev = 64;
int g_num_sms_dev[kMaxDev];
bool g_attr_dev[kMaxDev];
int g_raster_gm = 4;      // SELFTOK_GEMM_GM (measurement knob)
int g_gemm_ctas = 2;      // 2: two-CTA clusters sharing the W tile (default); 1: one CTA per tile (SELFTOK_GEMM_CTAS=1)

// e4m3: a UINT8 map, 128 elements (the same 128 B) per box row
int make_map(CUtensorMap* map, const __nv_bfloat16* ptr, int64_t rows, int K, int box_rows, int fp16, bool e4m3 = false) {
  cuuint64_t gdim[2] = {(cuuint64_t)K, (cuuint64_t)rows};
  cuuint64_t gstride[1] = {(cuuint64_t)K * (e4m3 ? 1 : 2)};
  cuuint32_t box[2] = {(cuuint32_t)(e4m3 ? BK8 : BK), (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  const CUtensorMapDataType dt =
      e4m3 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : fp16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  CUresult r = g_encode(map, dt, 2, const_cast<__nv_bfloat16*>(ptr), gdim, gstride, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed with CUresult " + std::to_string((int)r));
    return -5;
  }
  return 0;
}

// The A box {64 channels, bw pixels, bh rows, bn images} (bw bh bn = 128) of a convolution with output dims H x W, and the
// ty x tx boxes that cover one group of bn images.  It depends on the geometry alone, never on the batch, so an image's result
// does not depend on the images launched with it.  An exact box is part of an image row (W a multiple of 128), whole rows of one
// image, or whole images; stride 2 needs bn = 1, because consecutive planes are the phases of one image.  Without one, `edge`
// allows bn = 1 and the power-of-two bw x bh with the fewest boxes per image (the wider on a tie), overhanging the right and
// bottom edges; the TMA zero fill supplies the padding and the overhang alike.  Returns false when no box is allowed.
struct ConvBox {
  int bw, bh, bn, tx, ty;
};
bool conv_box(int H, int W, int stride, bool edge, ConvBox& bx) {
  const int64_t hw = (int64_t)H * W;
  const bool exact = (W % BM == 0 || BM % W == 0) && (hw % BM == 0 || BM % hw == 0) &&
                     (W >= BM || hw < BM || H % (BM / W) == 0) && (stride == 1 || hw % BM == 0);
  if (exact) {
    bx.bw = W < BM ? W : BM;
    bx.bh = (BM / bx.bw) < H ? (BM / bx.bw) : H;
    bx.bn = BM / (bx.bw * bx.bh);
  } else {
    if (!edge) return false;
    int64_t best = -1;
    for (int bw = BM; bw >= 1; bw /= 2) {
      const int bh = BM / bw;
      const int64_t n = (int64_t)((W + bw - 1) / bw) * ((H + bh - 1) / bh);
      if (best < 0 || n < best) { best = n; bx.bw = bw; bx.bh = bh; }
    }
    bx.bn = 1;
  }
  bx.tx = (W + bx.bw - 1) / bx.bw;
  bx.ty = (H + bx.bh - 1) / bx.bh;
  return true;
}

// 4-D map over NHWC 16-bit activations [B][H][W][C] with the box {64 channels, bw pixels, bh rows, bn images}
int make_map_nhwc(CUtensorMap* map, const __nv_bfloat16* ptr, int64_t B, int H, int W, int Cc, int fp16, const ConvBox& bx) {
  const int bw = bx.bw, bh = bx.bh, bn = bx.bn;
  cuuint64_t gdim[4] = {(cuuint64_t)Cc, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
  cuuint64_t gstride[3] = {(cuuint64_t)Cc * 2, (cuuint64_t)W * Cc * 2, (cuuint64_t)H * W * Cc * 2};
  cuuint32_t box[4] = {(cuuint32_t)BK, (cuuint32_t)bw, (cuuint32_t)bh, (cuuint32_t)bn};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = g_encode(map, fp16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<__nv_bfloat16*>(ptr), gdim, gstride,
                        box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled (NHWC) failed with CUresult " + std::to_string((int)r));
    return -5;
  }
  return 0;
}

}  // namespace

// Generic 2-D SWIZZLE_128B tensor map over a row-major 16-bit matrix [rows, cols] (box_cols * 2 bytes must be 128).
int make_tensor_map_2d(CUtensorMap* map, const void* ptr, uint64_t rows, uint64_t cols, uint32_t box_rows, uint32_t box_cols,
                       int fp16) {
  STK_CHECK(g_encode, -3, "gemm_tc_init has not been called");
  cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t gstride[1] = {(cuuint64_t)cols * 2};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = g_encode(map, fp16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), gdim,
                        gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                        CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed with CUresult " + std::to_string((int)r));
    return -5;
  }
  return 0;
}

void gemm_tc_set_ctas(int n) { g_gemm_ctas = n == 1 ? 1 : 2; }

// Idempotent per device (the current one): resolves cuTensorMapEncodeTiled once per process, opts the kernels into their
// dynamic shared memory and records the SM count once per device.
int gemm_tc_init() {
  int dev = 0;
  STK_CUDA(cudaGetDevice(&dev));
  STK_CHECK(dev >= 0 && dev < kMaxDev, -1, "gemm_tc: device ordinal out of range");
  if (g_encode && g_attr_dev[dev]) return 0;
  if (!g_encode) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    STK_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres));
    STK_CHECK(fn && qres == cudaDriverEntryPointSuccess, -5, "cuTensorMapEncodeTiled not available from the driver");
    const char* v = getenv("SELFTOK_GEMM_CTAS");
    if (v) g_gemm_ctas = atoi(v) == 1 ? 1 : 2;
    const char* gm = getenv("SELFTOK_GEMM_GM");
    if (gm && atoi(gm) >= 1 && atoi(gm) <= 1024) g_raster_gm = atoi(gm);
    g_encode = reinterpret_cast<EncodeTiledFn>(fn);
  }
  STK_CUDA(cudaDeviceGetAttribute(&g_num_sms_dev[dev], cudaDevAttrMultiProcessorCount, dev));
  STK_CUDA(cudaFuncSetAttribute(gemm_tc_kernel<1, 1, false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg<1>::SMEM_BYTES));
  STK_CUDA(cudaFuncSetAttribute(gemm_tc_kernel<1, 1, true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg<1>::SMEM_BYTES));
  STK_CUDA(cudaFuncSetAttribute(gemm_tc_kernel<3, 1, false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg<3>::SMEM_BYTES));
  STK_CUDA(cudaFuncSetAttribute(gemm_tc_kernel<1, 1, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg<1>::SMEM_BYTES));
  STK_CUDA(cudaFuncSetAttribute(gemm_tc_kernel<1, 2, false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg<1>::SMEM_BYTES));
  STK_CUDA(cudaFuncSetAttribute(gemm_tc_kernel<1, 2, true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg<1>::SMEM_BYTES));
  STK_CUDA(cudaFuncSetAttribute(gemm_tc_kernel<3, 2, false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg<3>::SMEM_BYTES));
  STK_CUDA(cudaFuncSetAttribute(gemm_tc_kernel<1, 2, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg<1>::SMEM_BYTES));
  g_attr_dev[dev] = true;
  return 0;
}

int check_gemm_tc_problem(const TcProblem& q, int nsplit, int fp16) {
  const Epilogue& ep = q.ep;
  const bool e4m3 = nsplit == NSPLIT_E4M3;
  STK_CHECK(q.A_hi && q.W_hi && q.M > 0 && q.N > 0 && q.K > 0, -1, "gemm_tc: bad arguments");
  STK_CHECK(nsplit == 1 || e4m3 || (nsplit == 3 && q.A_lo && q.W_lo), -1, "gemm_tc: nsplit must be 1, 3 with lo planes, or e4m3");
  STK_CHECK(!e4m3 || !fp16, -1, "gemm_tc: e4m3 operands are not IEEE half");
  STK_CHECK(e4m3 == (ep.s_a != nullptr) && e4m3 == (ep.s_w != nullptr), -1,
            "gemm_tc: e4m3 problems need both row-scale arrays and 16-bit problems take none (one launch, one operand type)");
  STK_CHECK(!e4m3 || q.conv_C == 0, -1, "gemm_tc: the e4m3 mode has no convolution");
  STK_CHECK(!e4m3 || q.K % 16 == 0, -2, "gemm_tc: e4m3 K must be a multiple of 16 (16-byte TMA row pitch)");
  STK_CHECK(reinterpret_cast<uintptr_t>(ep.s_a) % 4 == 0 && reinterpret_cast<uintptr_t>(ep.s_w) % 8 == 0, -1,
            "gemm_tc: s_a must be 4-byte and s_w 8-byte aligned");
  STK_CHECK(!fp16 || nsplit == 1, -1, "gemm_tc: the fp16 mode is single-pass");
  auto aligned16 = [](const void* p) { return reinterpret_cast<uintptr_t>(p) % 16 == 0; };
  STK_CHECK(aligned16(q.A_hi) && aligned16(q.A_lo) && aligned16(q.W_hi) && aligned16(q.W_lo), -1,
            "gemm_tc: operand planes must be 16-byte aligned (TMA)");
  STK_TRY(check_epilogue(ep, "gemm_tc"));
  STK_CHECK(ep.act == ACT_NONE || (ep.act == ACT_GELU && ep.mode != EPI_RESID), -2,
            "gemm_tc: epilogue activation must be none, or GELU-tanh with the store / split modes");
  STK_CHECK(ep.mode != EPI_STORE || ep.addtab == nullptr || ep.add_ld % 4 == 0, -2, "gemm_tc: addtab pitch must be a multiple of 4");
  STK_CHECK(q.K % 8 == 0, -2, "gemm_tc: K must be a multiple of 8 (16-byte TMA row pitch)");
  STK_CHECK(ep.ldo % 4 == 0 && q.N % 4 == 0, -2, "gemm_tc: N and the output pitch must be multiples of 4");
  STK_CHECK(ep.mode != EPI_RESID || ep.gate == nullptr || ep.gate_ld % 4 == 0, -2, "gemm_tc: gate pitch must be a multiple of 4");
  if (q.conv_C > 0) {                                      // implicit 3x3 convolution over NHWC planes
    STK_CHECK(q.conv_C % BK == 0 && q.K == 9 * q.conv_C, -2, "gemm_tc conv: channels must be a multiple of 64 and K = 9 C");
    STK_CHECK(q.conv_W > 0 && q.conv_H > 0 && (q.conv_stride == 1 || q.conv_stride == 2), -2, "gemm_tc conv: bad geometry or stride");
    STK_CHECK(q.M % ((int64_t)q.conv_H * q.conv_W) == 0, -2, "gemm_tc conv: M must be a whole number of images");
    ConvBox bx;
    STK_CHECK(conv_box(q.conv_H, q.conv_W, q.conv_stride, q.conv_edge != 0, bx), -2,
              "gemm_tc conv: without conv_edge, 128-pixel tiles must be part of a row, whole rows of one image, or whole images "
              "(stride 2: no whole images)");
  }
  return 0;
}

static int make_maps(TcMaps* m, const TcProblem& q, int nsplit, int fp16, int b_box) {
  const bool conv = q.conv_C > 0;
  if (nsplit == NSPLIT_E4M3) {
    STK_TRY(make_map(&m->a_hi, q.A_hi, q.M, q.K, BM, 0, true));
    STK_TRY(make_map(&m->b_hi, q.W_hi, q.N, q.K, b_box, 0, true));
    m->a_lo = m->a_hi; m->b_lo = m->b_hi;
    return 0;
  }
  const int64_t imgs = conv ? q.M / ((int64_t)q.conv_H * q.conv_W) * (q.conv_stride == 2 ? 4 : 1) : 0;   // stride 2: 4 phase planes per image
  ConvBox bx{};
  if (conv) conv_box(q.conv_H, q.conv_W, q.conv_stride, q.conv_edge != 0, bx);     // accepted by check_gemm_tc_problem
  if (conv) STK_TRY(make_map_nhwc(&m->a_hi, q.A_hi, imgs, q.conv_H, q.conv_W, q.conv_C, fp16, bx));
  else STK_TRY(make_map(&m->a_hi, q.A_hi, q.M, q.K, BM, fp16));
  STK_TRY(make_map(&m->b_hi, q.W_hi, q.N, q.K, b_box, fp16));
  if (nsplit == 3) {
    if (conv) STK_TRY(make_map_nhwc(&m->a_lo, q.A_lo, imgs, q.conv_H, q.conv_W, q.conv_C, fp16, bx));
    else STK_TRY(make_map(&m->a_lo, q.A_lo, q.M, q.K, BM, fp16));
    STK_TRY(make_map(&m->b_lo, q.W_lo, q.N, q.K, b_box, fp16));
  } else {
    m->a_lo = m->a_hi; m->b_lo = m->b_hi;
  }
  return 0;
}

template <int NSPLIT, int CL, bool FP16, bool E4M3>
static int launch_kernel(const TcMaps& m0, const TcMaps& m1, const GemmParams& p0, const GemmParams& p1, int clusters, cudaStream_t s) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(CL * clusters);
  cfg.blockDim = dim3(NUM_THREADS);
  cfg.dynamicSmemBytes = Cfg<NSPLIT>::SMEM_BYTES;
  cfg.stream = s;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = CL; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  STK_CUDA(cudaLaunchKernelEx(&cfg, gemm_tc_kernel<NSPLIT, CL, FP16, E4M3>, m0, m1, p0, p1));
  count_launch();
  return 0;
}

template <int CL>
static int launch_cl(const TcMaps& m0, const TcMaps& m1, const GemmParams& p0, const GemmParams& p1, int clusters, int nsplit, int fp16,
                     cudaStream_t s) {
  if (nsplit == NSPLIT_E4M3) return launch_kernel<1, CL, false, true>(m0, m1, p0, p1, clusters, s);
  if (nsplit == 3) return launch_kernel<3, CL, false, false>(m0, m1, p0, p1, clusters, s);
  if (fp16) return launch_kernel<1, CL, true, false>(m0, m1, p0, p1, clusters, s);
  return launch_kernel<1, CL, false, false>(m0, m1, p0, p1, clusters, s);
}

// One launch for up to two independent problems (the context- and the image-stream GEMM of an MMDiT layer): their tiles share
// the persistent grid, so the small N = 1536 GEMMs no longer pay a partially filled last wave each.
int launch_gemm_tc_grouped(const TcProblem* probs, int n, int nsplit, cudaStream_t s, int fp16) {
  STK_TRY(gemm_tc_init());                                // no-op after the first call on this device
  STK_CHECK(probs && (n == 1 || n == 2), -1, "gemm_tc: one or two problems per launch");
  int dev = 0;
  STK_CUDA(cudaGetDevice(&dev));
  const int g_num_sms = g_num_sms_dev[dev];
  for (int i = 0; i < n; ++i) STK_TRY(check_gemm_tc_problem(probs[i], nsplit, fp16));
  const int CL = g_gemm_ctas == 2 && g_num_sms >= 2 ? 2 : 1;
  TcMaps m0, m1;
  STK_TRY(make_maps(&m0, probs[0], nsplit, fp16, BN / CL));
  auto mk_params = [&](const TcProblem& q) {
    GemmParams g{q.M, q.N, q.K, fp16, q.ep};
    g.conv_C = q.conv_C; g.conv_H = q.conv_H; g.conv_W = q.conv_W; g.conv_stride = q.conv_stride;
    g.blocks = (int)((q.M + BM - 1) / BM);
    ConvBox bx;
    if (q.conv_C > 0 && conv_box(q.conv_H, q.conv_W, q.conv_stride, q.conv_edge != 0, bx)) {
      const int64_t imgs = q.M / ((int64_t)q.conv_H * q.conv_W);
      g.conv_bw = bx.bw; g.conv_bh = bx.bh; g.conv_bn = bx.bn; g.conv_tx = bx.tx; g.conv_ty = bx.ty;
      g.blocks = (int)((imgs + bx.bn - 1) / bx.bn * bx.ty * bx.tx);
    }
    g.raster_gm = g_raster_gm;
    return g;
  };
  auto tiles_of = [&](const GemmParams& g) { return (g.blocks + CL - 1) / CL * ((g.N + BN - 1) / BN); };
  GemmParams p0 = mk_params(probs[0]);
  GemmParams p1 = p0;
  p1.M = 0;
  p1.blocks = 0;
  m1 = m0;
  int tiles = tiles_of(p0);
  if (n == 2) {
    STK_TRY(make_maps(&m1, probs[1], nsplit, fp16, BN / CL));
    p1 = mk_params(probs[1]);
    tiles += tiles_of(p1);
  }
  const int clusters = tiles < g_num_sms / CL ? tiles : g_num_sms / CL;
  if (CL == 2) return launch_cl<2>(m0, m1, p0, p1, clusters, nsplit, fp16, s);
  return launch_cl<1>(m0, m1, p0, p1, clusters, nsplit, fp16, s);
}

int launch_gemm_tc(const __nv_bfloat16* A_hi, const __nv_bfloat16* A_lo, const __nv_bfloat16* W_hi,
                   const __nv_bfloat16* W_lo, int64_t M, int N, int K, int nsplit, const Epilogue& ep,
                   cudaStream_t s, int fp16) {
  TcProblem q{A_hi, A_lo, W_hi, W_lo, M, N, K, ep};
  return launch_gemm_tc_grouped(&q, 1, nsplit, s, fp16);
}

}  // namespace stk
