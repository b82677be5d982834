// Fused multi-head attention on wgmma / TMA (reference layers/attention.py:49-62).
//
//   out[img, q, head] = softmax(q k^T / 8) v          head_dim 64, T tokens per image (1939 at 720x540)
//
// A tile is 192 queries of one (image, head); KV is streamed in 128-key tiles.  Tiles are ordered (image, head)
// outermost and query tile fastest, so the query tiles of one (image, head) run at the same time and share its K and V
// in L2.  A grid of at most one CTA per SM strides through them.  512 threads in four warpgroups:
//   warps 0-11  : three consumer warpgroups, queries 0..63 / 64..127 / 128..191 of the tile (setmaxnreg 160)
//   warps 12-15 : producer warpgroup (setmaxnreg 32); one elected lane of warp 12 issues the TMA loads: Q into one of two
//                 buffers (the next tile's Q arrives while the current tile finishes), K and V through 4-stage rings of
//                 16 KB tiles, 128-byte swizzle.  The rings' stage and phase run on across tiles.
// Per key tile a warpgroup computes S = Q K^T (wgmma m64n128k16, both operands K-major in shared memory), runs the
// online softmax on the fragments in registers (a row's 128 logits are spread over the four lanes of a quad), rounds P
// to fp16 straight into wgmma's register A operand layout, and accumulates O += P V (wgmma m64n64k16, A from registers,
// V read MN-major from shared memory).  A warpgroup waits for each of its MMAs; the three warpgroups run independently,
// so one's softmax overlaps the others' MMAs.  The epilogue writes O / l in fp16 to a per-warpgroup staging buffer and
// leaves through a TMA tensor store over [n_img, T, D], which clips every image at T; the store drains under the next
// tile's main loop.
#include "gemm_tc.cuh"
#include "ops.h"
#include "gemm.h"
#include <algorithm>

namespace mk {

constexpr int FA_BQ = 192, FA_BK = 128, FA_D = 64, FA_KV_STAGES = 4;
constexpr int FA_CONSUMERS = 3, FA_THREADS = 128 * (FA_CONSUMERS + 1), FA_WARP_TMA = 4 * FA_CONSUMERS;
constexpr int FA_REGS_PRODUCER = 32, FA_REGS_CONSUMER = 160;
static_assert(FA_REGS_PRODUCER * 128 + FA_REGS_CONSUMER * 128 * FA_CONSUMERS <= 65536, "attention: register budget");
constexpr int FA_Q_BYTES = FA_BQ * 128;                                    // 192 rows x 64 fp16
constexpr int FA_KV_BYTES = FA_BK * 128;                                   // 128 rows x 64 fp16
constexpr int FA_O_BYTES = 64 * 128;                                       // one warpgroup's 64 rows x 64 fp16
constexpr int FA_REGION = 2 * FA_Q_BYTES + 2 * FA_KV_STAGES * FA_KV_BYTES + FA_CONSUMERS * FA_O_BYTES;
constexpr int FA_SMEM = FA_REGION + 1024 + 256;                            // + alignment slack + barriers
static_assert(FA_SMEM <= 227 * 1024, "attention: shared memory");

__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// D += A B with A (64 x 16 fp16) from registers in accumulator-fragment order and B from shared memory, MN-major
__device__ __forceinline__ void wgmma_m64n64k16_rs_tb(float (&d)[32], const uint32_t (&a)[4], uint64_t desc_b) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b), "r"(1u));
}

// named barrier of one consumer warpgroup (ids 2..4; 0 is __syncthreads)
__device__ __forceinline__ void warpgroup_sync(int wg) { asm volatile("bar.sync %0, 128;" ::"r"(2 + wg) : "memory"); }

struct AttnTile { int qt, head, im; };
__device__ __forceinline__ AttnTile attn_tile(int t, int q_tiles, int heads) {
  const int bh = t / q_tiles;
  return {t - bh * q_tiles, bh % heads, bh / heads};
}

// Online softmax of one key tile's S (fragment layout of wgmma m64nNk16: s[4c + 2h + e] = (row 16 (warp & 3) + lane / 4
// + 8 h, column 8 c + 2 (lane & 3) + e)).  P is rounded to fp16 here, once: the PV product and the row sum both use the
// rounded values, so the weights applied to V sum to exactly one after the final division.  The rounded pairs go straight
// into p, wgmma's register A operand: p[kk] = k-step kk (keys 16 kk .. 16 kk + 15 = column blocks 2 kk and 2 kk + 1).
__device__ __forceinline__ void softmax_tile(float (&s)[64], uint32_t (&p)[8][4], float (&m_run)[2], float (&l_run)[2],
                                             float (&alpha)[2], float scale_log2, int valid, int lane) {
  if (valid < FA_BK) {                                      // last key tile only (uniform branch)
#pragma unroll
    for (int i = 0; i < 64; ++i) {
      const int col = 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
      if (col >= valid) s[i] = -INFINITY;
    }
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float mx = -INFINITY;
#pragma unroll
    for (int c = 0; c < 16; ++c) mx = fmaxf(mx, fmaxf(s[4 * c + 2 * h], s[4 * c + 2 * h + 1]));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
    const float m_new = fmaxf(m_run[h], mx * scale_log2);  // finite: the tile holds at least one key
    alpha[h] = ex2_approx(m_run[h] - m_new);                // 0 on the first tile
    m_run[h] = m_new;
    float sum = 0.f;
#pragma unroll
    for (int c = 0; c < 16; ++c) {
      const float p0 = ex2_approx(fmaf(s[4 * c + 2 * h], scale_log2, -m_new));
      const float p1 = ex2_approx(fmaf(s[4 * c + 2 * h + 1], scale_log2, -m_new));
      const __half2 ph = __floats2half2_rn(p0, p1);
      const float2 r = __half22float2(ph);
      p[c >> 1][2 * (c & 1) + h] = *reinterpret_cast<const uint32_t*>(&ph);
      sum += r.x + r.y;
    }
    l_run[h] = l_run[h] * alpha[h] + sum;                   // this lane's columns only
  }
}

__global__ void __launch_bounds__(FA_THREADS, 1)
attention_tc_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmKV,
                    const __grid_constant__ CUtensorMap tmO, int T, int heads, int q_tiles, int n_tiles_total, float scale_log2) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  const uint32_t sQ = base;                                           // [2][192 x 64]
  const uint32_t sK = sQ + 2 * FA_Q_BYTES;                            // [stages][128 x 64]
  const uint32_t sV = sK + FA_KV_STAGES * FA_KV_BYTES;
  const uint32_t sO = sV + FA_KV_STAGES * FA_KV_BYTES;                // [3][64 x 64] output staging
  const uint32_t bars = base + FA_REGION;
  const uint32_t k_full = bars, k_empty = k_full + 8 * FA_KV_STAGES, v_full = k_empty + 8 * FA_KV_STAGES,
                 v_empty = v_full + 8 * FA_KV_STAGES, q_full = v_empty + 8 * FA_KV_STAGES, q_empty = q_full + 16;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int D = heads * FA_D;
  const int n_kv = (T + FA_BK - 1) / FA_BK;

  if (warp == FA_WARP_TMA && lane == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmQ) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmKV) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmO) : "memory");
    for (int s = 0; s < FA_KV_STAGES; ++s) {
      mbar_init(k_full + 8 * s, 1); mbar_init(k_empty + 8 * s, 4 * FA_CONSUMERS);   // one arrive per consumer warp
      mbar_init(v_full + 8 * s, 1); mbar_init(v_empty + 8 * s, 4 * FA_CONSUMERS);
    }
    for (int b = 0; b < 2; ++b) { mbar_init(q_full + 8 * b, 1); mbar_init(q_empty + 8 * b, 4 * FA_CONSUMERS); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  pdl_wait();

  if (warp >= FA_WARP_TMA) {
    // ===== TMA producer =====
    setmaxnreg_dec<FA_REGS_PRODUCER>();
    if (warp == FA_WARP_TMA && elect_one()) {
      int st = 0;
      uint32_t ph = 0;
      int it = 0;
      for (int t = blockIdx.x; t < n_tiles_total; t += gridDim.x, ++it) {
        const AttnTile tile = attn_tile(t, q_tiles, heads);
        const int row_base = tile.im * T;
        const int qb = it & 1;
        mbar_wait(q_empty + 8 * qb, ((it >> 1) & 1) ^ 1);      // the tile two back has released this Q buffer
        mbar_expect_tx(q_full + 8 * qb, FA_Q_BYTES);
        tma_load_2d(sQ + qb * FA_Q_BYTES, &tmQ, q_full + 8 * qb, tile.head * FA_D, row_base + tile.qt * FA_BQ);
        for (int j = 0; j < n_kv; ++j) {
          mbar_wait(k_empty + 8 * st, ph ^ 1);
          mbar_expect_tx(k_full + 8 * st, FA_KV_BYTES);
          tma_load_2d(sK + st * FA_KV_BYTES, &tmKV, k_full + 8 * st, D + tile.head * FA_D, row_base + j * FA_BK);
          mbar_wait(v_empty + 8 * st, ph ^ 1);
          mbar_expect_tx(v_full + 8 * st, FA_KV_BYTES);
          tma_load_2d(sV + st * FA_KV_BYTES, &tmKV, v_full + 8 * st, 2 * D + tile.head * FA_D, row_base + j * FA_BK);
          if (++st == FA_KV_STAGES) { st = 0; ph ^= 1; }
        }
      }
    }
    __syncwarp();
    pdl_trigger();
    return;
  }

  // ===== consumers =====
  setmaxnreg_inc<FA_REGS_CONSUMER>();
  const int wg = warp >> 2;
  const uint32_t stage_o = sO + wg * FA_O_BYTES;
  int ks = 0, vs = 0;                    // ring stages of the next K and the next V to consume
  uint32_t kph = 0, vph = 0;
  int it = 0;
  for (int t = blockIdx.x; t < n_tiles_total; t += gridDim.x, ++it) {
    const AttnTile tile = attn_tile(t, q_tiles, heads);
    const int qb = it & 1;
    const uint64_t dq = gmma_desc_sw128(sQ + qb * FA_Q_BYTES + wg * (64 * 128));
    float s[64], o[32];
    uint32_t p[8][4];
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] = 0.f;
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f}, alpha[2];
    mbar_wait(q_full + 8 * qb, (it >> 1) & 1);

    for (int j = 0; j < n_kv; ++j) {
      mbar_wait(k_full + 8 * ks, kph);
      const uint64_t dk = gmma_desc_sw128(sK + ks * FA_KV_BYTES);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < FA_D / WGMMA_K; ++k) wgmma_m64n128k16(s, dq + (uint64_t)(k * 2), dk + (uint64_t)(k * 2), k > 0 ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence(s);
      if (lane == 0) mbar_arrive(k_empty + 8 * ks);             // K tile consumed
      if (++ks == FA_KV_STAGES) { ks = 0; kph ^= 1; }
      softmax_tile(s, p, m_run, l_run, alpha, scale_log2, T - j * FA_BK, lane);
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        o[4 * c] *= alpha[0]; o[4 * c + 1] *= alpha[0];
        o[4 * c + 2] *= alpha[1]; o[4 * c + 3] *= alpha[1];
      }
      mbar_wait(v_full + 8 * vs, vph);
      const uint64_t dv = gmma_desc_sw128(sV + vs * FA_KV_BYTES);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < FA_BK / WGMMA_K; ++kk)   // 16 keys per MMA: 16 rows (2048 B) of V
        wgmma_m64n64k16_rs_tb(o, p[kk], dv + (uint64_t)(kk * 128));
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence(o);
      if (lane == 0) mbar_arrive(v_empty + 8 * vs);             // V tile consumed
      if (++vs == FA_KV_STAGES) { vs = 0; vph ^= 1; }
    }
    if (lane == 0) mbar_arrive(q_empty + 8 * qb);               // Q buffer free for the tile after next
    if (t + (int)gridDim.x >= n_tiles_total) pdl_trigger();   // last main loop done

    // ===== epilogue: O / l -> fp16 staging (128-byte swizzle) -> TMA tensor store =====
    const int row0 = tile.qt * FA_BQ + wg * 64;                 // first query of this warpgroup
    if (row0 >= T) continue;                                    // all 64 rows are padding
    if (threadIdx.x % 128 == 0) tma_store_wait_read();          // the previous tile's store has read the staging buffer
    warpgroup_sync(wg);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float l = l_run[h];
      l += __shfl_xor_sync(0xffffffffu, l, 1);
      l += __shfl_xor_sync(0xffffffffu, l, 2);
      const float inv = 1.0f / l;
      const int r = (warp & 3) * 16 + (lane >> 2) + 8 * h;
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        const __half2 v = __floats2half2_rn(o[4 * c + 2 * h] * inv, o[4 * c + 2 * h + 1] * inv);
        asm volatile("st.shared.b32 [%0], %1;" ::"r"(stage_o + r * 128 + ((c ^ (r & 7)) << 4) + 4 * (lane & 3)),
                     "r"(*reinterpret_cast<const uint32_t*>(&v)) : "memory");
      }
    }
    fence_async_smem();
    warpgroup_sync(wg);
    if (threadIdx.x % 128 == 0) {
      tma_store_3d(&tmO, stage_o, tile.head * FA_D, row0, tile.im);
      tma_store_commit();
    }
  }
  if (threadIdx.x % 128 == 0) tma_store_wait_all();             // shared memory must outlive the bulk reads
}

int attention_tc(const void* qkv, void* out, int n_img, int T, int D, int heads, cudaStream_t s) {
  if (D != heads * FA_D) { set_last_error("attention: head_dim must be 64 (D=%d heads=%d)", D, heads); return MK_ERR_UNSUPPORTED; }
  static unsigned long long attr_mask = 0;
  if (first_use_on_device(attr_mask)) {
    MK_CUDA_CHECK(cudaFuncSetAttribute(attention_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, FA_SMEM));
  }
  CUtensorMap tmQ, tmKV, tmO;
  int rc = make_tensor_map_f16(&tmQ, qkv, (long long)n_img * T, 3LL * D, 3LL * D, FA_BQ);
  if (!rc) rc = make_tensor_map_f16(&tmKV, qkv, (long long)n_img * T, 3LL * D, 3LL * D, FA_BK);
  if (!rc) rc = make_tensor_map_out_f16(&tmO, out, n_img, T, D, 64);
  if (rc) return rc;
  const int q_tiles = ceil_div(T, FA_BQ);
  const int tiles = q_tiles * heads * n_img;
  const float scale_log2 = 0.125f * 1.4426950408889634f;
  MK_CUDA_CHECK(launch_k(attention_tc_kernel, dim3(std::min(tiles, sm_count())), dim3(FA_THREADS), (size_t)FA_SMEM, s, tmQ, tmKV, tmO,
                         T, heads, q_tiles, tiles, scale_log2));
  return MK_OK;
}

// impl: 0 = default (wgmma), 1 = wgmma, 2 = mma.sync
int attention_dispatch(const void* qkv, void* out, int n_img, int T, int D, int heads, int impl, cudaStream_t s) {
  if (impl < 0 || impl > 2) { set_last_error("attention: unknown impl %d", impl); return MK_ERR_INVALID; }
  return impl == 2 ? attention(qkv, out, n_img, T, D, heads, s) : attention_tc(qkv, out, n_img, T, D, heads, s);
}

}  // namespace mk
