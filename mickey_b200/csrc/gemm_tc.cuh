// wgmma / TMA GEMM for sm_90a.
//
//   D[M,N] (fp32) = A[M,K] * B[N,K]^T,   A and B fp16, K-major, 128-byte swizzled tiles
//
// Output tiles are 128 x BN; every launch walks them in gemm_tile() order.  The persistent instantiations (PERSISTENT,
// large grids) have 640 threads (five warpgroups) in three roles:
//   warps 0-7  : MMA warpgroups 0 and 1 (wgmma m64nBNk16 on tile rows 0..63 / 64..127, fp32 accumulators in registers)
//   warps 8-15 : epilogue warps; warp 8 + w owns rows 32(w&3)..+31 and the column half w>>2 of the tile
//   warps 16-19: producer warpgroup; one elected lane of warp 16 issues cp.async.bulk.tensor.2d into the smem ring
// A grid of at most one CTA per SM strides through the tiles by gridDim.x.  The producer's ring stage and phase carry
// over from tile to tile, so the next tile's loads are in flight while the current one is still in its MMAs.  When a
// tile's K loop has drained, the MMA warpgroups park the accumulators in a staging buffer outside the ring, as eight
// 32 x (BN/2) blocks (the layout epilogue_rows reads), and go on to the next tile while the epilogue warps run
// tile_epilogue from the staged blocks.  The default persistent launch (PAIR) runs two-CTA clusters on M-adjacent tiles
// that share each B tile through TMA multicast (see the kernel), which cuts the L2-to-SM bytes per chunk from 32 KB to
// 24 KB (BN = 128).
//
// The other instantiations (!PERSISTENT) run one tile per CTA (grid = tiles, the same loop runs once) with 288 threads:
// the MMA warps park the accumulators in the idle ring and run the epilogue themselves, warp 8 is the producer.  They
// serve EPI_DUAL (its TMA-store staging takes the room of a second buffer), EPI_LN (its epilogue needs more registers
// than the persistent epilogue warps have) and grids too small to keep a persistent CTA per SM busy: a 3-stage ring (two
// CTAs per SM, one CTA's epilogue under the other's main loop, except for EPI_LN) or, for at most ~1.25 tiles per SM, a
// deep ring.
//
// The K loop walks `k_chunks` 64-element chunks.  For convolutions a chunk also selects a filter tap:
// the A tile of tap t is the same 2-D tensor read at row offset tap_shift[t] (negative / overflowing
// rows are zero-filled by TMA), which turns a 3x3 convolution over a zero-padded NHWC image into 9
// accumulated GEMMs without materialising im2col.
#pragma once
#include "common.cuh"
#include "epilogue.cuh"

namespace mk {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;        // 64 fp16 = 128 bytes = one swizzle row
constexpr int WGMMA_K = 16;
constexpr int GEMM_WARP_EPI = 8;

// Ring depths: the persistent kernel's ring shares shared memory with the accumulator staging buffer; the one-tile rings
// have the whole region to themselves.
template <int BN> constexpr int ring_stages() { return BN == 128 ? 4 : 6; }
template <int BN> constexpr int shallow_stages() { return BN == 128 ? 3 : 4; }
template <int BN> constexpr int deep_stages() { return BN == 128 ? 6 : 8; }
template <int EPI> constexpr bool persistent_epilogue() { return EPI != EPI_DUAL && EPI != EPI_LN; }
template <bool PERSISTENT> constexpr int gemm_threads() { return PERSISTENT ? 640 : 288; }
template <bool PERSISTENT> constexpr int gemm_warp_tma() { return PERSISTENT ? 16 : 8; }

// Per-warp staging of EPI_DUAL: three 32 x 32 fp32 boxes (1024-byte aligned) for the TMA stores + 64 floats of column
// operands (the st.global path uses the first box as its [32][33] transpose buffer)
constexpr int DUAL_STAGE_BYTES = 3 * 4096;
constexpr int DUAL_AUX_BYTES = 8 * 64 * 4;
constexpr int DUAL_BYTES = 8 * DUAL_STAGE_BYTES + DUAL_AUX_BYTES;

template <int BN> constexpr int acc_block_floats() { return 32 * (BN / 2); }   // one warp's 32 x (BN/2) block (acc_idx layout)
template <int BN> constexpr int acc_tile_bytes() { return 8 * acc_block_floats<BN>() * 4; }
template <int BN, int STAGES> constexpr int ring_bytes() { return STAGES * (BLOCK_M * BLOCK_K * 2 + BN * BLOCK_K * 2); }
// Persistent: the accumulator staging buffer follows the ring.  One tile per CTA: after the K loop the ring region
// holds [EPI_DUAL staging][accumulator tile].
template <int BN, int EPI, int STAGES, bool PERSISTENT> constexpr int acc_tile_offset() {
  return PERSISTENT ? ring_bytes<BN, STAGES>() : EPI == EPI_DUAL ? DUAL_BYTES : 0;
}
template <int BN, int EPI, int STAGES, bool PERSISTENT>
constexpr int region_bytes() {
  return ring_bytes<BN, STAGES>() > acc_tile_offset<BN, EPI, STAGES, PERSISTENT>() + acc_tile_bytes<BN>()
             ? ring_bytes<BN, STAGES>() : acc_tile_offset<BN, EPI, STAGES, PERSISTENT>() + acc_tile_bytes<BN>();
}
// + 1024 alignment slack + 256 barriers
template <int BN, int EPI, int STAGES, bool PERSISTENT> constexpr int gemm_smem_bytes() {
  return region_bytes<BN, EPI, STAGES, PERSISTENT>() + 1024 + 256;
}
// Two one-tile CTAs per SM when their shared memory allows it, except for EPI_LN: at two CTAs per SM a thread has 96
// registers, and its epilogue spills below about 140.
template <int BN, int EPI, int STAGES, bool PERSISTENT> constexpr int gemm_ctas_per_sm() {
  return !PERSISTENT && EPI != EPI_LN && gemm_smem_bytes<BN, EPI, STAGES, PERSISTENT>() <= 113 * 1024 ? 2 : 1;
}

// ---- tile order ----------------------------------------------------------------------------------------
// Linear tile index -> (group, m0, n0, n_tile).  N-tiles vary fastest, then the groups if they all read the same A
// rows and columns, then the M-tiles; groups with their own A (matcher pairs, heads with per-group input columns) are
// outermost, so a group's tiles stay together.  The ViT GEMMs have M in the ~1000 tiles and A far larger than the
// 50 MB L2 while all of B is a few MB: the ~132 tiles in flight at once then cover a few complete rows of tiles, every
// A row-panel is read from HBM about once and B stays resident in L2.  An M-fastest order would instead stream A once
// per column of N-tiles.
// MT = 2 (the paired persistent kernel) walks the same order over pairs of M-tiles 2 mp, 2 mp + 1: the CTA of cluster
// rank r takes M-tile 2 mp + r.  With an odd M-tile count the last pair's rank-1 tile starts at or beyond M.
struct GemmTile { int g, m0, n0, n_tile; };
template <int BN, int MT = 1>
__host__ __device__ __forceinline__ int gemm_tile_count(const GemmParams& p) {
  return ((p.M + MT * BLOCK_M - 1) / (MT * BLOCK_M)) * ((p.N + BN - 1) / BN) * p.groups;
}
template <int BN, int MT = 1>
__device__ __forceinline__ GemmTile gemm_tile(const GemmParams& p, int t, int rank = 0) {
  const int n_tiles = (p.N + BN - 1) / BN, m_units = (p.M + MT * BLOCK_M - 1) / (MT * BLOCK_M);
  const int n = t % n_tiles;
  t /= n_tiles;
  int g, m;
  if (p.a_row_group_off == 0 && p.a_col_group_off == 0) { g = t % p.groups; m = t / p.groups; }
  else { m = t % m_units; g = t / m_units; }
  return {g, (m * MT + rank) * BLOCK_M, n * BN, n};
}

// ---- PTX wrappers ------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred P1;\n\t"
      "WAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n\t"
      "@P1 bra DONE_%=;\n\t"
      "bra WAIT_%=;\n\t"
      "DONE_%=:\n\t"
      "}" ::"r"(bar), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1) : "memory");
}
// The same box written to offset `dst` of every CTA of the cluster in `cta_mask`; each destination's mbarrier at offset
// `bar` receives the box's bytes.
__device__ __forceinline__ void tma_load_2d_multicast(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1,
                                                      uint16_t cta_mask) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%3, %4}], [%2], %5;"
      ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "h"(cta_mask) : "memory");
}
// arrive on the mbarrier at offset `bar` of CTA `cta_rank` of the cluster (this CTA's own rank included).  The default
// .release.cta semantics: a .cluster-scoped release costs a MEMBAR.GPU per arrival (measured 3x slower GEMMs), and the
// only accesses it would order are the wgmma reads of the stage, which have retired (wgmma.wait_group) before the arrival.
__device__ __forceinline__ void mbar_arrive_cluster(uint32_t bar, uint32_t cta_rank) {
  asm volatile(
      "{\n\t.reg .b32 remote;\n\t"
      "mapa.shared::cluster.u32 remote, %0, %1;\n\t"
      "mbarrier.arrive.shared::cluster.b64 _, [remote];\n\t}"
      ::"r"(bar), "r"(cta_rank) : "memory");
}
__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t"
      ".reg .pred P1;\n\t"
      "elect.sync _|P1, 0xFFFFFFFF;\n\t"
      "selp.b32 %0, 1, 0, P1;\n\t"
      "}" : "=r"(pred));
  return pred != 0;
}
// Warpgroup register budgets of the persistent kernel (setmaxnreg): 640 threads start at 96 registers; the producer warpgroup drops to 40 so that
// the epilogue warpgroups can hold 120, the MMA warpgroups (64 accumulators) keep 96.  128 x 40 + 256 x 96 + 256 x 120
// <= 640 x 96.
constexpr int GEMM_REGS_PRODUCER = 40;
constexpr int GEMM_REGS_EPILOGUE = 120;
template <int R> __device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R> __device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
// named barrier of the 256 MMA threads (id 1; id 0 is __syncthreads)
__device__ __forceinline__ void consumer_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

// wgmma shared-memory descriptor: 128-byte swizzle, rows of 128 bytes, 8-row groups 1024 bytes apart
// (start>>4 [0,14), LBO>>4 [16,30), SBO>>4 [32,46), layout SWIZZLE_128B = 1 [62,64)).  K-major operands ignore LBO; for
// an MN-major operand of 64 elements along MN it is likewise unused.
__device__ __forceinline__ uint64_t gmma_desc_sw128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
template <int N> __device__ __forceinline__ void reg_fence(float (&d)[N]) {   // keep the compiler from touching d under an async wgmma
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

__device__ __forceinline__ void wgmma_m64n64k16(float (&d)[32], uint64_t desc_a, uint64_t desc_b, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(desc_a), "l"(desc_b), "r"(scale_d));
}

__device__ __forceinline__ void wgmma_m64n128k16(float (&d)[64], uint64_t desc_a, uint64_t desc_b, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(desc_a), "l"(desc_b), "r"(scale_d));
}

template <int BN>
__device__ __forceinline__ void wgmma_tile(float (&d)[BN / 2], uint64_t desc_a, uint64_t desc_b, uint32_t scale_d) {
  if constexpr (BN == 128) wgmma_m64n128k16(d, desc_a, desc_b, scale_d);
  else wgmma_m64n64k16(d, desc_a, desc_b, scale_d);
}

// ---- thread-block cluster barrier (PAIR) ---------------------------------------------------------------
__device__ __forceinline__ void cluster_sync_all() {     // every thread of every CTA of the cluster
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// ---- tile epilogue -----------------------------------------------------------------------------------
// One warp's share of the parked 128 x BN accumulator tile `acc`: rows 32q..32q+31 (quadrant q) and the column half
// `half`.  acc_chunk() gives lane l row 32q + l, 32 consecutive columns of any chunk (thread == row); `stage` is the
// warp's own 32 x W block, which the staged epilogues read in place.
template <int BN>
__device__ __forceinline__ void acc_chunk(const float* acc, int q, int lane, int c, float (&v)[32]) {
  constexpr int W = BN / 2;
  const float* blk = acc + (q + 4 * ((c * 32) / W)) * acc_block_floats<BN>();
#pragma unroll
  for (int k4 = 0; k4 < 8; ++k4) {
    const float4 t = *reinterpret_cast<const float4*>(blk + acc_idx<W>(lane, (c * 32) % W + 4 * k4));
    v[k4 * 4] = t.x; v[k4 * 4 + 1] = t.y; v[k4 * 4 + 2] = t.z; v[k4 * 4 + 3] = t.w;
  }
}

template <int BN, int EPI>
__device__ __forceinline__ void tile_epilogue(const GemmParams& p, const OutMaps& om, int g, int m0, int n0, int n_tile, int q, int half,
                                              int lane, float* acc, float* dual_stage, float* dual_aux) {
  constexpr int CHUNKS = BN / 32;
  constexpr int W = BN / 2;                             // columns owned by this warp
  constexpr int CPH = CHUNKS / 2;                       // chunks per half
  const int c_begin = half * CPH, c_end = c_begin + CPH;
  const int m = m0 + q * 32 + lane;
  float* stage = acc + (q + 4 * half) * acc_block_floats<BN>();
  float v[32];
  if constexpr (EPI == EPI_LN) {
    float sum = 0.f;
#pragma unroll
    for (int c = 0; c < CHUNKS; ++c) {
      acc_chunk<BN>(acc, q, lane, c, v);
#pragma unroll
      for (int j = 0; j < 32; ++j) sum += v[j];
    }
    const float mean = sum * (1.0f / BN);
    float sq = 0.f;
#pragma unroll
    for (int c = 0; c < CHUNKS; ++c) {
      acc_chunk<BN>(acc, q, lane, c, v);
#pragma unroll
      for (int j = 0; j < 32; ++j) { const float d = v[j] - mean; sq += d * d; }
    }
    const float rstd = rsqrtf(sq * (1.0f / BN) + p.eps);
    epilogue_rows<EPI_LN, W>(p, g, m0 + q * 32, lane, n0 + half * W, stage, mean, rstd);
  } else if constexpr (EPI == EPI_LSE) {
    static_assert(BN == 128, "matcher epilogues: 128-wide tiles");
    const bool row_ok = m < p.n_valid;
    float rmax = MK_NEG_INF, rsum = 0.f;
    if (p.lse_bound > 0.f) {
      rmax = p.lse_bound * p.inv_temp * 1.4426950408889634f;
      for (int c = c_begin; c < c_end; ++c) {
        if (n0 + c * 32 < p.n_valid) {
          acc_chunk<BN>(acc, q, lane, c, v);
          lse_chunk_bounded(p, g, n0 + c * 32, lane, (m0 / BLOCK_M) * 4 + q, row_ok, v, rsum);
        }
      }
    } else {
      for (int c = c_begin; c < c_end; ++c) {
        if (n0 + c * 32 < p.n_valid) {
          acc_chunk<BN>(acc, q, lane, c, v);
          lse_chunk(p, g, n0 + c * 32, lane, (m0 / BLOCK_M) * 4 + q, row_ok, v, rmax, rsum);
        }
      }
    }
    if (row_ok) p.part_row[((size_t)g * (p.part_ld / 64) + n_tile * 2 + half) * p.part_ld + m] = make_float2(rmax, rsum);
  } else if constexpr (EPI == EPI_DUAL) {
    static_assert(BN == 128, "matcher epilogues: 128-wide tiles");
    // per-row operands: lse of the row (+inf for rows beyond the valid range -> score 0) and its keypoint score
    const bool row_ok = m < p.n_valid;
    const float lr = row_ok ? __ldg(p.lse_r + (size_t)g * p.part_ld + m) : -MK_NEG_INF;
    const float s0 = row_ok ? __ldg(p.scr0 + (size_t)g * p.n_valid + m) : 0.0f;
    if (p.out_tma) {
      float lc_pre[CPH], s1_pre[CPH];
#pragma unroll
      for (int ci = 0; ci < CPH; ++ci) {
        const int col = n0 + (c_begin + ci) * 32 + lane;
        const bool ok = col < p.n_valid;
        lc_pre[ci] = ok ? __ldg(p.lse_c + (size_t)g * p.part_ld + col) : -MK_NEG_INF;
        s1_pre[ci] = ok ? __ldg(p.scr1 + (size_t)g * p.n_valid + col) : 0.0f;
      }
#pragma unroll
      for (int ci = 0; ci < CPH; ++ci) {
        const int c = c_begin + ci;
        if (n0 + c * 32 < p.n_valid && m0 + q * 32 < p.n_valid) {
          acc_chunk<BN>(acc, q, lane, c, v);
          dual_store_chunk_tma(p, om, g, m0 + q * 32, lane, n0 + c * 32, v, dual_stage, dual_aux, lr, s0, lc_pre[ci], s1_pre[ci]);
        }
      }
    } else {
      for (int c = c_begin; c < c_end; ++c) {
        if (n0 + c * 32 < p.n_valid) {
          acc_chunk<BN>(acc, q, lane, c, v);
          dual_store_chunk(p, g, m0 + q * 32, lane, n0 + c * 32, v, dual_stage, lr, s0);
        }
      }
    }
  } else {
    epilogue_rows<EPI, W>(p, g, m0 + q * 32, lane, n0 + half * W, stage, 0.f, 0.f);
  }
}

// ---- kernel ------------------------------------------------------------------------------------------
// PAIR (persistent only): the grid is made of two-CTA clusters.  Both CTAs of a cluster walk the same (group, N-tile)
// sequence on M-tiles 2 mp and 2 mp + 1 (gemm_tile<BN, 2>), so they read the same B tile in every K chunk.  Each
// CTA's producer loads its own A box and one half of the B box (BN/2 rows; tmB is encoded with that box), multicast
// into stage s of both CTAs; each CTA's full barrier still expects STAGE_BYTES.  A stage is refilled only when the
// MMA warps of both CTAs have released it: every MMA warp arrives on the empty barrier of both CTAs (16 arrivals per
// phase).  The MMAs, their operands and their K order are those of the unpaired kernel, so the outputs are identical.
template <int BN, int EPI, int STAGES, bool PERSISTENT, bool PAIR = false>
__global__ void __launch_bounds__((gemm_threads<PERSISTENT>()), (gemm_ctas_per_sm<BN, EPI, STAGES, PERSISTENT>()))
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmParams p,
               const __grid_constant__ OutMaps om) {
  static_assert(BN == 64 || BN == 128, "wgmma tiles: N = 64 or 128");
  static_assert(gemm_smem_bytes<BN, EPI, STAGES, PERSISTENT>() <= 227 * 1024, "GEMM: shared memory");
  extern __shared__ uint8_t smem_raw[];
  constexpr int A_BYTES = BLOCK_M * BLOCK_K * 2;
  constexpr int B_BYTES = BN * BLOCK_K * 2;
  constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  constexpr int W = BN / 2;
  static_assert(!PERSISTENT || persistent_epilogue<EPI>(), "this epilogue runs one tile per CTA");
  static_assert(!PAIR || PERSISTENT, "CTA pairs: persistent kernel only");
  constexpr bool ONE_TILE = !PERSISTENT;
  constexpr int WARP_TMA = gemm_warp_tma<PERSISTENT>();
  constexpr int MT = PAIR ? 2 : 1;                              // M-tiles per unit of work
  // a pair's two CTAs are blockIdx.x 2c and 2c + 1 (cluster c, rank blockIdx.x & 1)
  const int rank = PAIR ? (int)(blockIdx.x & 1) : 0;
  const int work0 = PAIR ? (int)(blockIdx.x >> 1) : (int)blockIdx.x;
  const int work_step = PAIR ? (int)(gridDim.x >> 1) : (int)gridDim.x;

  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;                 // swizzle-128B tiles need 1024-byte alignment
  // full[S], empty[S], acc_full, acc_empty
  const uint32_t bar_base = base + region_bytes<BN, EPI, STAGES, PERSISTENT>();
  const uint32_t full_bar0 = bar_base;
  const uint32_t empty_bar0 = bar_base + 8 * STAGES;
  const uint32_t acc_full_bar = bar_base + 16 * STAGES;         // staging buffer holds a tile (256 MMA threads arrive)
  const uint32_t acc_empty_bar = acc_full_bar + 8;              // the epilogue is done with it (256 epilogue threads)
  uint8_t* const gbase = smem_raw + (base - raw);
  float* const acc = reinterpret_cast<float*>(gbase + acc_tile_offset<BN, EPI, STAGES, PERSISTENT>());

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int n_work = gemm_tile_count<BN, MT>(p);

  if (warp == WARP_TMA && lane == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB) : "memory");
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full_bar0 + 8 * s, 1);
      mbar_init(empty_bar0 + 8 * s, 8 * MT);       // one arrive per MMA warp (of both CTAs of a pair)
    }
    mbar_init(acc_full_bar, 256);
    mbar_init(acc_empty_bar, 256);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  // a pair: the peer's barriers must be initialised before this CTA's multicasts or remote arrivals reach them
  if constexpr (PAIR) cluster_sync_all();
  else __syncthreads();
  pdl_wait();                    // everything above touched no global memory; operands of the previous kernel are now visible

  if (warp >= WARP_TMA) {
    // ===== TMA producer: the ring's stage and phase run on across tiles =====
    if constexpr (!ONE_TILE) setmaxnreg_dec<GEMM_REGS_PRODUCER>();
    if (warp == WARP_TMA && elect_one()) {
      int stage = 0;
      uint32_t phase = 0;
      for (int t = work0; t < n_work; t += work_step) {
        const GemmTile tile = gemm_tile<BN, MT>(p, t, rank);
        const int a_col0 = p.a_col_base + tile.g * p.a_col_group_off;
        const int a_row0 = tile.m0 + tile.g * p.a_row_group_off;
        const int b_row0 = tile.n0 + tile.g * p.b_row_group_off;
        for (int kc = 0; kc < p.k_chunks; ++kc) {
          const int tap = kc / p.chunks_per_tap;
          const int kin = kc - tap * p.chunks_per_tap;
          mbar_wait(empty_bar0 + 8 * stage, phase ^ 1);
          const uint32_t sa = base + stage * STAGE_BYTES;
          const uint32_t fb = full_bar0 + 8 * stage;
          mbar_expect_tx(fb, STAGE_BYTES);
          tma_load_2d(sa, &tmA, fb, a_col0 + kin * BLOCK_K, a_row0 + p.tap_shift[tap]);
          // B rows of a half box are a multiple of 8 (1024 bytes), so the halves keep the 128-byte swizzle pattern
          if constexpr (PAIR) tma_load_2d_multicast(sa + A_BYTES + rank * (B_BYTES / 2), &tmB, fb, kc * BLOCK_K, b_row0 + rank * (BN / 2), 0x3);
          else tma_load_2d(sa + A_BYTES, &tmB, fb, kc * BLOCK_K, b_row0);
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
    __syncwarp();
    pdl_trigger();
    // a pair: no CTA may exit while its peer can still multicast into its ring or arrive on its barriers
    if constexpr (PAIR) cluster_sync_all();
    return;
  }

  if (warp < GEMM_WARP_EPI) {
    // ===== MMA warpgroup wg computes tile rows 64 wg .. 64 wg + 63 =====
    const int wg = warp >> 2;
    int stage = 0;
    uint32_t phase = 0, acc_phase = 0;
    // release a ring stage to the producer(s) that fill it
    auto release = [&](int s) {
      if constexpr (PAIR) { mbar_arrive_cluster(empty_bar0 + 8 * s, 0); mbar_arrive_cluster(empty_bar0 + 8 * s, 1); }
      else mbar_arrive(empty_bar0 + 8 * s);
    };
    for (int t = work0; t < n_work; t += work_step) {
      float d[BN / 2];
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) d[i] = 0.f;
      for (int kc = 0; kc < p.k_chunks; ++kc) {
        mbar_wait(full_bar0 + 8 * stage, phase);
        const uint32_t sa = base + stage * STAGE_BYTES;
        const uint64_t da = gmma_desc_sw128(sa + wg * (64 * 128));
        const uint64_t db = gmma_desc_sw128(sa + A_BYTES);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BLOCK_K / WGMMA_K; ++k)
          // advance 32 bytes (16 fp16) along K inside the 128-byte swizzle row: +2 in the (addr>>4) field
          wgmma_tile<BN>(d, da + (uint64_t)(k * 2), db + (uint64_t)(k * 2), 1u);
        wgmma_commit();
        wgmma_wait<1>();                               // the previous chunk's MMAs have retired: release its stage
        reg_fence(d);
        if (kc > 0 && lane == 0) release(stage == 0 ? STAGES - 1 : stage - 1);
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      reg_fence(d);
      if (lane == 0) release(stage == 0 ? STAGES - 1 : stage - 1);
      if (t + work_step >= n_work) pdl_trigger();   // last K loop done: the next kernel may start its prologue

      // ===== hand the accumulators to the epilogue through the staging buffer =====
      if constexpr (ONE_TILE) consumer_sync();      // the staging buffer is the ring: both warpgroups are done reading it
      else mbar_wait(acc_empty_bar, acc_phase ^ 1);
      // fragment layout of wgmma m64nNk16: d[4j + 2h + e] = (row 16 (warp & 3) + lane / 4 + 8 h, column 8 j + 2 (lane & 3) + e)
      const int r_base = wg * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int r = r_base + 8 * h, c = 8 * j + 2 * (lane & 3);
          float* dst = acc + ((r >> 5) + 4 * (c / W)) * acc_block_floats<BN>() + acc_idx<W>(r & 31, c % W);
          *reinterpret_cast<float2*>(dst) = make_float2(d[4 * j + 2 * h], d[4 * j + 2 * h + 1]);
        }
      }
      if constexpr (ONE_TILE) {
        consumer_sync();
        const GemmTile tile = gemm_tile<BN>(p, t);
        tile_epilogue<BN, EPI>(p, om, tile.g, tile.m0, tile.n0, tile.n_tile, warp & 3, warp >> 2, lane, acc,
                               reinterpret_cast<float*>(gbase + warp * DUAL_STAGE_BYTES),
                               reinterpret_cast<float*>(gbase + 8 * DUAL_STAGE_BYTES) + warp * 64);
      } else {
        mbar_arrive(acc_full_bar);
        acc_phase ^= 1;
      }
    }
    if constexpr (EPI == EPI_DUAL) { if (p.out_tma && lane == 0) tma_store_wait_all(); }   // smem must outlive the bulk reads
    if constexpr (PAIR) cluster_sync_all();
    return;
  }

  // ===== epilogue warps (persistent instantiations only) =====
  if constexpr (ONE_TILE) return;
  setmaxnreg_inc<GEMM_REGS_EPILOGUE>();
  const int ew = warp - GEMM_WARP_EPI;
  uint32_t acc_phase = 0;
  for (int t = work0; t < n_work; t += work_step) {
    const GemmTile tile = gemm_tile<BN, MT>(p, t, rank);
    mbar_wait(acc_full_bar, acc_phase);
    if (t + work_step >= n_work) pdl_trigger();
    // the rank-1 tile of the last pair of an odd M-tile count lies wholly beyond M: it stores nothing
    if (tile.m0 < p.M)
      tile_epilogue<BN, EPI>(p, om, tile.g, tile.m0, tile.n0, tile.n_tile, ew & 3, ew >> 2, lane, acc,
                             reinterpret_cast<float*>(gbase + ew * DUAL_STAGE_BYTES),
                             reinterpret_cast<float*>(gbase + 8 * DUAL_STAGE_BYTES) + ew * 64);
    mbar_arrive(acc_empty_bar);
    acc_phase ^= 1;
  }
  if constexpr (PAIR) cluster_sync_all();
}

}  // namespace mk
