// Probabilistic Procrustes RANSAC (reference modules/utils/probabilisticProcrustes.py:183-348).
//
//  1. outer sampling  : IT_MATCHES x "2048 of N*N cells without replacement, prob ~ final_scores".
//                       ATen's multinomial is top-k of p / Exp(1) (an exponential race); we run the same race
//                       with a counter-based generator (Philox4x32-7) so that each pass can regenerate the
//                       noise instead of materialising the [B*IT_MATCHES, N*N] tile the reference allocates:
//                       pass A histograms the keys (8 exponent + 3 mantissa bits), a scan finds the bin holding
//                       the 2048-th largest key, pass B collects the <= ~2.3 k candidates at/above it, pass C
//                       sorts them (key desc, cell index as tie-break) and keeps the first 2048.
//  2. gather          : cell -> (keypoint i0, keypoint i1), back-projection X = d * K^-1 [u v 1]^T   (training_utils.py:7-22)
//  3. hypotheses      : IT_RANSAC x (3 of 2048 without replacement ~ weight; Kabsch via 3x3 one-sided Jacobi SVD;
//                       soft inlier score over the set's 2048 correspondences)                  (solvers.py:3-54, training_utils.py:55-61)
//  4. finalize        : argmax, <= NUM_REFINEMENTS masked-Kabsch refinements on hard inliers, final soft count.
#include "ops.h"
#include "ransac_dev.cuh"

namespace mk {


// Exp(1) variate with full relative precision near 0 (small E decides the race): E = -log1p(-u), u in (0,1)
__device__ __forceinline__ float exp1_from_u(float u) {
  u = fminf(u, 0.99999994f);
  return (u < 0.01f) ? u * (1.0f + u * (0.5f + u * (0.33333334f + 0.25f * u))) : -__logf(1.0f - u);
}

// 48-bit uniform of one (cell, stream): a 16-bit prefix (8 streams share one Philox call) refined by 32 more bits
// that are only generated for the few cells whose prefix does not already rule them out.
__device__ __forceinline__ float u_from_prefix(uint32_t prefix16, uint32_t low32) {
  return ((float)prefix16 + ((float)low32 + 0.5f) * 2.3283064365386963e-10f) * 1.52587890625e-5f;
}
__device__ __forceinline__ uint32_t race_key(float p, float u) { return __float_as_uint(__fdividef(p, exp1_from_u(u))); }

constexpr int HBINS = 2048;          // float bits >> 20 (sign is always 0): 8 exponent + 3 mantissa bits
constexpr int SAMP_THREADS = 256;
constexpr int SAMP_ELEMS_PER_BLOCK = 256 * 16;
constexpr uint32_t PHILOX_TAG_PREFIX = 0x5bd1e995u, PHILOX_TAG_LOW = 0x2545F491u;

// ---- pass A: histogram of the cell probabilities of one pair (no random numbers; shared by all its streams) -------
// A block covers SAMP_ELEMS_PER_BLOCK consecutive cells (or 4-cell slots).  final_scores is [N, N] per pair with row
// pitch `pitch` floats; the logical cell index e = i * N + j (what the generator's counters and the outputs use) does
// not depend on the pitch.  Addressing modes:
//   MODE_FLAT_VEC  contiguous rows (pitch == N) with N*N a multiple of 4: 16-byte loads over the flat array
//   MODE_ROW_VEC   padded rows (pitch % 4 == 0, as the matcher's TMA path writes them): 16-byte loads of 4-cell slots
//                  per row, slots beyond column N masked
//   MODE_SCALAR    anything else
// With the vector modes a thread issues its four float4 loads before touching any of them: with one scalar load in
// flight per thread these passes were latency-bound at ~1.5 TB/s out of L2.
enum { MODE_SCALAR = 0, MODE_FLAT_VEC = 1, MODE_ROW_VEC = 2 };

struct CellView {
  const float* p;          // pair base
  int N;
  long long pitch;
  __device__ __forceinline__ long long cells() const { return (long long)N * N; }
  // ROW_VEC: a block chunk is `rows_per_chunk` whole rows (no division in the cell loop); rows longer than a chunk
  // (N > 4096) are not vectorised (the host picks MODE_SCALAR)
  __device__ __forceinline__ int spr() const { return (N + 3) / 4; }                       // 4-cell slots per row
  __device__ __forceinline__ int rows_per_chunk() const { return (SAMP_ELEMS_PER_BLOCK / 4) / spr(); }
  __device__ __forceinline__ long long n_chunks(int mode) const {
    if (mode == MODE_ROW_VEC) { const int rpc = rows_per_chunk(); return (N + rpc - 1) / rpc; }
    return (cells() + SAMP_ELEMS_PER_BLOCK - 1) / SAMP_ELEMS_PER_BLOCK;
  }
};

// slot `sl` of chunk `chunk` in ROW_VEC mode -> (row, first column); false beyond the chunk's rows / the matrix
__device__ __forceinline__ bool row_vec_slot(const CellView& cv, long long chunk, int sl, int& row, int& c4) {
  const int spr = cv.spr(), rpc = cv.rows_per_chunk();
  int rr = 0;
  while (sl >= spr && rr < rpc) { sl -= spr; ++rr; }                                        // rpc is 2 for N = 1938
  row = (int)chunk * rpc + rr; c4 = sl * 4;
  return rr < rpc && row < cv.N;
}

template <int MODE, typename F>
__device__ __forceinline__ void for_each_cell(const CellView& cv, long long chunk, F&& f) {
  const long long e0 = chunk * SAMP_ELEMS_PER_BLOCK;
  if (MODE == MODE_FLAT_VEC) {
    const long long cells = cv.cells();
    float4 v[4];
    long long e[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      e[i] = e0 + 4LL * (threadIdx.x + SAMP_THREADS * i);
      v[i] = (e[i] < cells) ? __ldg(reinterpret_cast<const float4*>(cv.p + e[i])) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      f(e[i], v[i].x); f(e[i] + 1, v[i].y); f(e[i] + 2, v[i].z); f(e[i] + 3, v[i].w);
    }
  } else if (MODE == MODE_ROW_VEC) {
    float4 v[4];
    long long e[4];
    int rem[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      int row, c4;
      v[i] = make_float4(0.f, 0.f, 0.f, 0.f); e[i] = 0; rem[i] = 0;
      if (row_vec_slot(cv, chunk, threadIdx.x + SAMP_THREADS * i, row, c4)) {
        v[i] = __ldg(reinterpret_cast<const float4*>(cv.p + (long long)row * cv.pitch + c4));
        e[i] = (long long)row * cv.N + c4;
        rem[i] = cv.N - c4;                                          // valid cells in this slot (>= 4 except at the row end)
      }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      if (rem[i] > 0) f(e[i], v[i].x);
      if (rem[i] > 1) f(e[i] + 1, v[i].y);
      if (rem[i] > 2) f(e[i] + 2, v[i].z);
      if (rem[i] > 3) f(e[i] + 3, v[i].w);
    }
  } else {
    const long long cells = cv.cells();
    const long long e1 = min(cells, e0 + SAMP_ELEMS_PER_BLOCK);
    for (long long e = e0 + threadIdx.x; e < e1; e += SAMP_THREADS) {
      const int row = (int)(e / cv.N);
      f(e, cv.p[(long long)row * cv.pitch + (e - (long long)row * cv.N)]);
    }
  }
}

// p > 0 and finite, subnormals included (an integer test: it does not depend on how the compiler treats subnormals)
__device__ __forceinline__ bool positive_finite(float pv) { return __float_as_uint(pv) - 1u < 0x7f7fffffu; }

// Besides the histogram, pass A flags the cells torch.multinomial rejects: NaN (either sign bit), +-inf and p < 0
// (-0 is a zero), by OR-ing `invalid_bits` into the status: bit 0 for the solver, which then gives the reference's zero
// pose (probabilisticProcrustes.py:331-342); the training loss adds its own pre-check bit (loss.cu).
template <int MODE>
__global__ void __launch_bounds__(SAMP_THREADS)
sampler_phist_kernel(const float* __restrict__ fs, int N, long long pitch, unsigned int* __restrict__ hist, int* __restrict__ status,
                     int invalid_bits) {
  __shared__ unsigned int h[HBINS];
  for (int i = threadIdx.x; i < HBINS; i += SAMP_THREADS) h[i] = 0;
  __syncthreads();
  const int b = blockIdx.y;
  const CellView cv{fs + (long long)b * N * pitch, N, pitch};
  const long long n_chunks = cv.n_chunks(MODE);
  bool invalid = false;
  for (long long chunk = blockIdx.x; chunk < n_chunks; chunk += gridDim.x)      // grid = whole waves of resident blocks
    for_each_cell<MODE>(cv, chunk, [&](long long, float pv) {
      const uint32_t u = __float_as_uint(pv);
      if (positive_finite(pv)) atomicAdd(&h[u >> 20], 1u);
      else invalid |= (u & 0x7fffffffu) != 0u;
    });
  if (__syncthreads_or(invalid) && threadIdx.x == 0) atomicOr(status, invalid_bits);
  unsigned int* dst = hist + (long long)b * HBINS;
  for (int i = threadIdx.x; i < HBINS; i += SAMP_THREADS)
    if (h[i]) atomicAdd(dst + i, h[i]);
}

// ---- threshold ------------------------------------------------------------------------------------------------------
// A cell survives the cut "key >= tau" with probability 1 - exp(-p / tau).  From the histogram, a LOWER bound of the
// expected number of survivors f(tau) = sum_bins count * (1 - exp(-lower_edge / tau)) is evaluated on the grid of
// bin edges and the largest tau with f(tau) >= n_sample + 8 sqrt(n_sample) + 16 is taken (f decreases in tau).  The
// number of survivors of a stream is a sum of independent Bernoullis (variance <= mean), so fewer than n_sample
// survive with probability < 1e-13; pass C reports that event through status bit 1.
// One 1024-thread block per pair runs a 33-ary search: each round, warp w evaluates f at its own grid point (64 bins
// per lane, fixed-order shuffle reduction), so three rounds replace eleven bisection steps of block-wide reductions.
constexpr int TAU_THREADS = 1024;

__global__ void __launch_bounds__(TAU_THREADS)
sampler_tau_kernel(const unsigned int* __restrict__ hist, long long cells, int n_sample, int* __restrict__ thr,
                   float* __restrict__ inv_tau, int* __restrict__ status) {
  pdl_wait();        // launched with programmatic stream serialization: predecessors are complete past this point
  pdl_trigger();
  __shared__ float cc[HBINS], ee[HBINS];          // counts and lower edges of the occupied bins, in bin order
  __shared__ int wtot[32];
  __shared__ float fw[32];
  const int b = blockIdx.x, t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const unsigned int* h = hist + (long long)b * HBINS;
  // compact the occupied bins (a few hundred of the 2048): thread t owns bins 2t, 2t+1.  Pass A histograms positive
  // finite p only, so bin 0 holds 0 < p < 2^-129 (its lower edge 0 adds nothing to f) and the inf / nan bins >= 2040
  // stay empty.
  const int b0 = 2 * t, b1 = 2 * t + 1;
  const unsigned int c0 = (b0 < HBINS - 8) ? h[b0] : 0u, c1 = (b1 < HBINS - 8) ? h[b1] : 0u;
  const int k = (c0 > 0) + (c1 > 0);
  int incl = k;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const int x = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += x; }
  if (lane == 31) wtot[warp] = incl;
  __syncthreads();
  int off = incl - k, nnz = 0;
  for (int w = 0; w < 32; ++w) { const int x = wtot[w]; if (w < warp) off += x; nnz += x; }
  if (c0 > 0) { cc[off] = (float)c0; ee[off] = __uint_as_float((uint32_t)b0 << 20); ++off; }
  if (c1 > 0) { cc[off] = (float)c1; ee[off] = __uint_as_float((uint32_t)b1 << 20); }
  __syncthreads();
  auto warp_sum = [&](float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
  };
  float nz = 0.f;
  for (int i = lane; i < nnz; i += 32) nz += cc[i];
  const float nonzero = warp_sum(nz);             // every warp computes the same value in the same order
  const float target = (float)n_sample + 8.0f * sqrtf((float)n_sample) + 16.0f;
  // invariant: f(edge[lo]) >= target > f(edge[hi]).  lo == 7 stands for "tau below the normal floats": every nonzero
  // cell is a candidate (f = nonzero).
  int lo = 7, hi = HBINS - 9;
  if (nonzero < target) hi = 8;                   // few nonzero cells: keep them all
  while (hi - lo > 1) {
    const int mid = lo + (int)(((long long)(hi - lo) * (warp + 1)) / 33);   // lo <= mid < hi, non-decreasing in warp
    float f = target;                             // mid == lo: known to satisfy the invariant
    if (mid > lo) {
      const float it = 1.0f / __uint_as_float((uint32_t)mid << 20);
      f = 0.f;
      for (int i = lane; i < nnz; i += 32) {
        const float y = ee[i] * it;
        f += cc[i] * ((y < 0.01f) ? y * (1.0f - 0.5f * y) : 1.0f - __expf(-y));
      }
      f = warp_sum(f);
    }
    __syncthreads();
    if (lane == 0) fw[warp] = f;
    __syncthreads();
    // largest warp whose point still reaches the target -> new lo; the next warp's point (or hi) -> new hi
    int best = -1;
    for (int w = 0; w < 32; ++w) if (fw[w] >= target) best = w;
    const int span = hi - lo;
    const int new_lo = (best >= 0) ? lo + (int)(((long long)span * (best + 1)) / 33) : lo;
    const int new_hi = (best < 31) ? lo + (int)(((long long)span * (best + 2)) / 33) : hi;
    lo = new_lo; hi = (new_hi > new_lo) ? new_hi : new_lo + 1;
  }
  if (t == 0) {
    const float tau = __uint_as_float((uint32_t)lo << 20);
    const bool all = (lo < 8);
    thr[b] = all ? 1 : lo;
    inv_tau[b] = all ? __int_as_float(0x7f800000) : 1.0f / tau;
    // torch.multinomial without replacement raises on a row that sums to zero and when n_sample exceeds the row
    // length; the reference's try/except then returns the zero pose (probabilisticProcrustes.py:331-342).  With
    // 0 < positive cells < n_sample it does not raise: pass C draws every positive cell and fills with zero cells.
    if (nonzero == 0.f || cells < (long long)n_sample) atomicOr(status, 1);
  }
}

// ---- pass B: collect candidates (key bin >= threshold bin) -----------------------------------------------------------
// key >= tau  <=>  E <= p / tau  <=>  u <= 1 - exp(-p / tau): one MUFU.EX2 per cell gives the (slightly widened) bound
// that all IM streams of the pair share, one Philox call gives the 16-bit prefixes of 8 streams, and a stream's prefix
// above the bound rejects it without a log or a division.  The exact key is computed only for the ~0.06 % that pass,
// and its bin decides.
// rare path (a cell passes with probability ~8 p / tau): kept out of line so that the per-cell loop stays a few dozen
// instructions (inlined 16 times per thread it overflowed the instruction cache: 12 'no_instruction' stall cycles per issue)
__device__ __noinline__ void collect_refine(const Philox& rng, long long e, float pv, float uth, uint32_t pth, uint4 r, int sg, int b,
                                            int IM, int T, unsigned long long* __restrict__ cand, unsigned int* __restrict__ cnt, int cap) {
  const uint32_t w[4] = {r.x, r.y, r.z, r.w};
  for (int j = 0; j < 8; ++j) {
    const uint32_t prefix = (w[j >> 1] >> ((j & 1) * 16)) & 0xffffu;
    const int stream = sg * 8 + j;
    if (prefix <= pth && stream < IM) {
      const uint4 r2 = rng((uint32_t)e, (uint32_t)(e >> 32) ^ PHILOX_TAG_LOW, (uint32_t)stream, (uint32_t)b);
      const float u = u_from_prefix(prefix, r2.x);
      if (u <= uth) {
        const uint32_t k = race_key(pv, u);
        if (T <= 1 || (int)(k >> 20) >= T) {               // all-candidates mode: even a key that underflows to 0
          const long long s = (long long)b * IM + stream;
          const unsigned int slot = atomicAdd(cnt + s, 1u);
          if (slot < (unsigned)cap) cand[s * cap + slot] = ((unsigned long long)k << 32) | (uint32_t)e;
        }
      }
    }
  }
}

template <int MODE>
__global__ void __launch_bounds__(SAMP_THREADS, 3)       // three blocks per SM (<= 85 registers): the pitched mode compiled to 104 without the cap
sampler_collect_kernel(const float* __restrict__ fs, int N, long long pitch, int IM, const unsigned long long* __restrict__ seed_ptr,
                       const int* __restrict__ thr, const float* __restrict__ inv_tau_p, unsigned long long* __restrict__ cand,
                       unsigned int* __restrict__ cnt, int cap) {
  pdl_wait();        // launched with programmatic stream serialization: predecessors are complete past this point
  pdl_trigger();
  const int b = blockIdx.y;
  const Philox rng(*seed_ptr);
  const int T = thr[b];
  const float inv_tau = inv_tau_p[b];
  const CellView cv{fs + (long long)b * N * pitch, N, pitch};
  auto cell = [&](long long e, float pv) {
    if (!positive_finite(pv)) return;
    // u <= (1 - exp(-y)) * (1 + 2^-10) + 2^-30 with y = p / tau: a superset of the exact condition.  For small y
    // 1 - exp(-y) <= y is used instead (1 - q would cancel catastrophically in fp32).
    const float y = pv * inv_tau;
    float q;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(q) : "f"(-1.4426950408889634f * y));
    const float prob = (y < 0.01f) ? y : 1.0f - q;
    const float uth = fminf(fmaf(prob, 1.0009765625f, 9.3132257e-10f), 1.0f);
    const uint32_t pth = (uint32_t)(uth * 65536.0f);                 // prefix > pth  =>  u > uth
    for (int sg = 0; sg * 8 < IM; ++sg) {
      const uint4 r = rng((uint32_t)e, (uint32_t)(e >> 32) ^ PHILOX_TAG_PREFIX, (uint32_t)sg, (uint32_t)b);
      // any of the 8 16-bit prefixes at or below the bound?
      const bool any = ((r.x & 0xffffu) <= pth) | ((r.x >> 16) <= pth) | ((r.y & 0xffffu) <= pth) | ((r.y >> 16) <= pth) |
                       ((r.z & 0xffffu) <= pth) | ((r.z >> 16) <= pth) | ((r.w & 0xffffu) <= pth) | ((r.w >> 16) <= pth);
      if (any) collect_refine(rng, e, pv, uth, pth, r, sg, b, IM, T, cand, cnt, cap);
    }
  };
  const long long n_chunks = cv.n_chunks(MODE);
  for (long long chunk = blockIdx.x; chunk < n_chunks; chunk += gridDim.x) {    // grid = whole waves of resident blocks
    if (MODE != MODE_SCALAR) {
      // the four 16-byte loads first, then component-major processing: the loop body holds four (not sixteen)
      // copies of cell()
      const long long e0 = chunk * SAMP_ELEMS_PER_BLOCK;
      const long long cells = cv.cells();
      float4 v[4];
      long long eb[4];
      int rem[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        v[i] = make_float4(0.f, 0.f, 0.f, 0.f); eb[i] = 0; rem[i] = 0;
        if (MODE == MODE_FLAT_VEC) {
          const long long e = e0 + 4LL * (threadIdx.x + SAMP_THREADS * i);
          if (e < cells) { v[i] = __ldg(reinterpret_cast<const float4*>(cv.p + e)); eb[i] = e; rem[i] = 4; }
        } else {
          int row, c4;
          if (row_vec_slot(cv, chunk, threadIdx.x + SAMP_THREADS * i, row, c4)) {
            v[i] = __ldg(reinterpret_cast<const float4*>(cv.p + (long long)row * pitch + c4));
            eb[i] = (long long)row * N + c4; rem[i] = N - c4;
          }
        }
      }
#pragma unroll 1
      for (int c = 0; c < 4; ++c) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          // cells beyond the row end are fed as probability 0 (a select, not a branch: the four Philox evaluations of
          // this step stay interleaved); flat mode: out-of-range slots already hold zeros
          float pv = (c == 0) ? v[i].x : (c == 1) ? v[i].y : (c == 2) ? v[i].z : v[i].w;
          if (MODE != MODE_FLAT_VEC) pv = (rem[i] > c) ? pv : 0.f;
          cell(eb[i] + c, pv);
        }
      }
    } else {
      for_each_cell<MODE_SCALAR>(cv, chunk, cell);
    }
  }
}

// ---- pass C: keep the n_sample largest keys -------------------------------------------------------------------------
// One 512-thread block per stream; the candidates (key << 32 | cell, all distinct) sit in registers.
//   1. radix select, most significant byte first: a 256-bin histogram of the current byte among the elements that
//      still match the boundary prefix, a suffix scan, the bin where the running count crosses what is still needed.
//      It stops as soon as the boundary bin is taken whole (normally after the four key bytes).
//   2. the selected cells are compacted into shared memory and sorted ascending by cell index (32-bit bitonic network,
//      4 elements per thread: in-thread, shuffle and shared-memory stages), so the result does not depend on the order
//      in which pass B happened to append the candidates.  The order of a draw carries no information for the solver
//      (ATen's multinomial returns key order; the reference uses the draw as a set).
// Sorting the 64-bit candidates themselves was ALU-bound on the 8 active SMs (40 us for 8 streams).
constexpr int SEL_THREADS = 512;

template <int J>
__device__ __forceinline__ void sort4_local(uint32_t (&v)[4], int base, int k) {
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    if ((r & J) == 0) {
      const bool asc = (((base + r) & k) == 0);
      const uint32_t a = v[r], c = v[r | J];
      const uint32_t lo = min(a, c), hi = max(a, c);
      v[r] = asc ? lo : hi; v[r | J] = asc ? hi : lo;
    }
  }
}

// ascending bitonic sort of SZ = 2048 values, element i = 4 t + r
__device__ __forceinline__ void sort2048_u32(uint32_t (&v)[4], uint32_t* sh, int t) {
  constexpr int SZ = 4 * SEL_THREADS;
  const int base = t * 4;
#pragma unroll 1
  for (int k = 2; k <= SZ; k <<= 1) {
#pragma unroll 1
    for (int j = k >> 1; j > 0; j >>= 1) {
      const bool keep_min = (((base & j) == 0) == ((base & k) == 0));   // used when the partner is in another thread
      if (j >= 128) {
        __syncthreads();
#pragma unroll
        for (int r = 0; r < 4; ++r) sh[base + r] = v[r];
        __syncthreads();
        const int pbase = base ^ j;
#pragma unroll
        for (int r = 0; r < 4; ++r) { const uint32_t o = sh[pbase + r]; v[r] = keep_min ? min(v[r], o) : max(v[r], o); }
      } else if (j >= 4) {
#pragma unroll
        for (int r = 0; r < 4; ++r) { const uint32_t o = __shfl_xor_sync(0xffffffffu, v[r], j >> 2); v[r] = keep_min ? min(v[r], o) : max(v[r], o); }
      } else if (j == 2) {
        sort4_local<2>(v, base, k);
      } else {
        sort4_local<1>(v, base, k);
      }
    }
  }
}

template <int E>
__device__ __forceinline__ void select_run(const unsigned long long* __restrict__ src, int n, int n_sample, int* __restrict__ dst,
                                           unsigned int* hist, uint32_t* sel, int* ctrl) {
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  // padding is masked out rather than told apart by value: in all-candidates mode a real candidate can be 0
  // (cell 0 with a key that underflowed)
  unsigned long long v[E];
  auto valid = [&](int r) { return t + SEL_THREADS * r < n; };
#pragma unroll
  for (int r = 0; r < E; ++r) v[r] = valid(r) ? src[t + SEL_THREADS * r] : 0ull;
  // ---- 1. radix select of the n_sample-th largest
  unsigned long long prefix = 0;         // bytes already fixed (value of v >> (shift + 8) of the boundary element)
  int need = n_sample;                   // how many must still come out of the elements matching the prefix
  int shift = 56;
  bool whole = false;                    // boundary bin taken whole: selection = (v >> shift) >= boundary value
  unsigned long long bound = 0;
  while (true) {
    if (t < 256) hist[t] = 0;
    __syncthreads();
#pragma unroll
    for (int r = 0; r < E; ++r)
      if (valid(r) && (shift == 56 || (v[r] >> (shift + 8)) == prefix)) atomicAdd(&hist[(unsigned)(v[r] >> shift) & 0xffu], 1u);
    __syncthreads();
    if (warp == 0) {                     // suffix counts over the 256 bins: lane owns bins [8 lane, 8 lane + 8)
      unsigned int c[8], mine = 0;
#pragma unroll
      for (int i = 0; i < 8; ++i) { c[i] = hist[lane * 8 + i]; mine += c[i]; }
      unsigned int suf = mine;           // inclusive suffix sum over lanes
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const unsigned int x = __shfl_down_sync(0xffffffffu, suf, o); if (lane + o < 32) suf += x; }
      const unsigned int above = suf - mine;          // elements in bins of higher lanes
      if (above < (unsigned)need && suf >= (unsigned)need) {
        unsigned int run = above;
        for (int i = 7; i >= 0; --i) {
          if (run + c[i] >= (unsigned)need) { ctrl[0] = lane * 8 + i; ctrl[1] = need - (int)run; ctrl[2] = (int)c[i]; break; }
          run += c[i];
        }
      }
    }
    __syncthreads();
    const int digit = ctrl[0], need_in = ctrl[1], have_in = ctrl[2];
    __syncthreads();
    bound = (prefix << 8) | (unsigned)digit;
    if (have_in == need_in || shift == 0) { whole = true; break; }
    prefix = bound; need = need_in; shift -= 8;
  }
  (void)whole;
  // ---- 2. compact the selected cells, sort them by cell index
  if (t == 0) ctrl[3] = 0;
  __syncthreads();
#pragma unroll
  for (int r = 0; r < E; ++r)
    if (valid(r) && (v[r] >> shift) >= bound) { const int slot = atomicAdd(&ctrl[3], 1); if (slot < 4 * SEL_THREADS) sel[slot] = (uint32_t)v[r]; }
  __syncthreads();
  const int got = min(ctrl[3], 4 * SEL_THREADS);
  uint32_t c4[4];
#pragma unroll
  for (int r = 0; r < 4; ++r) c4[r] = (4 * t + r < got) ? sel[4 * t + r] : 0xffffffffu;
  __syncthreads();
  sort2048_u32(c4, sel, t);
#pragma unroll
  for (int r = 0; r < 4; ++r)
    if (4 * t + r < n_sample) dst[4 * t + r] = (4 * t + r < got) ? (int)c4[r] : 0;
}

// Fewer candidates than n_sample (n < n_sample <= 2048).  In all-candidates mode they are every positive cell, and
// torch.multinomial's draw is those cells plus n_sample - n zero-probability cells (keys 0 / Exp(1) = 0; which ones is
// implementation-defined).  The rule here: the lowest cell indices that are not candidates.  The first 2048 cells
// hold at least 2048 - n of them; with fewer than n_sample cells in the matrix (status bit 0) the rest is cell 0.
// The draw is sorted ascending by cell index like a full one.  Out of line: inlined, this rare path took the kernel
// from 64 to 87 registers (one 512-thread block per SM instead of two).
__device__ __noinline__ void select_fill(const unsigned long long* __restrict__ src, int n, int n_sample, long long cells,
                                         int* __restrict__ dst, unsigned int* taken, uint32_t* sel, int* ctrl) {
  constexpr int SZ = 4 * SEL_THREADS;
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  for (int i = t; i < SZ / 32; i += SEL_THREADS) taken[i] = 0u;
  __syncthreads();
  for (int i = t; i < n; i += SEL_THREADS) {
    const uint32_t c = (uint32_t)src[i];
    sel[i] = c;
    if (c < (uint32_t)SZ) atomicOr(&taken[c >> 5], 1u << (c & 31));
  }
  __syncthreads();
  // thread t looks at cells 4t .. 4t+3; the free ones get consecutive ranks in cell order (block-wide exclusive scan)
  bool fr[4];
  int k = 0;
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const uint32_t c = 4 * t + r;
    fr[r] = (long long)c < cells && !((taken[c >> 5] >> (c & 31)) & 1u);
    k += fr[r];
  }
  int incl = k;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const int x = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += x; }
  if (lane == 31) ctrl[warp] = incl;
  __syncthreads();
  int rank = n + incl - k;
  for (int w = 0; w < warp; ++w) rank += ctrl[w];
#pragma unroll
  for (int r = 0; r < 4; ++r)
    if (fr[r]) { if (rank < n_sample) sel[rank] = 4 * t + r; ++rank; }
  int got = n;
  for (int w = 0; w < SEL_THREADS / 32; ++w) got += ctrl[w];
  got = min(got, n_sample);
  __syncthreads();
  uint32_t c4[4];
#pragma unroll
  for (int r = 0; r < 4; ++r) c4[r] = (4 * t + r < got) ? sel[4 * t + r] : 0xffffffffu;
  __syncthreads();
  sort2048_u32(c4, sel, t);
#pragma unroll
  for (int r = 0; r < 4; ++r)
    if (4 * t + r < n_sample) dst[4 * t + r] = (4 * t + r < got) ? (int)c4[r] : 0;
}

template <int CAP>
__global__ void __launch_bounds__(SEL_THREADS)
sampler_select_kernel(const unsigned long long* __restrict__ cand, const unsigned int* __restrict__ cnt, int n_sample, int IM,
                      const int* __restrict__ thr, long long cells, int* __restrict__ idx_out, int* __restrict__ status) {
  pdl_wait();        // launched with programmatic stream serialization: predecessors are complete past this point
  pdl_trigger();
  __shared__ unsigned int hist[256];
  __shared__ uint32_t sel[4 * SEL_THREADS];
  __shared__ int ctrl[SEL_THREADS / 32];
  const long long s = blockIdx.x;
  const unsigned int n_raw = cnt[s];
  const int n = (int)min(n_raw, (unsigned)CAP);
  // bit 1: the candidate buffer overflowed (selection truncated), or a thresholded stream came short of n_sample
  // (probability < 1e-13, see sampler_tau_kernel)
  if (threadIdx.x == 0 && (n_raw > (unsigned)CAP || (n < n_sample && thr[s / IM] > 1))) atomicOr(status, 2);
  const unsigned long long* src = cand + s * CAP;
  int* dst = idx_out + s * n_sample;
  if (n < n_sample) { select_fill(src, n, n_sample, cells, dst, hist, sel, ctrl); return; }
  if (n <= 4 * SEL_THREADS) select_run<4>(src, n, n_sample, dst, hist, sel, ctrl);
  else if (n <= 8 * SEL_THREADS) select_run<8>(src, n, n_sample, dst, hist, sel, ctrl);
  else select_run<16>(src, n, n_sample, dst, hist, sel, ctrl);
}

constexpr int CAND_CAP = 8192;

size_t sampler_workspace_bytes(int B, int IM) {
  const size_t streams = (size_t)B * IM;
  return (size_t)B * HBINS * 4 + streams * 4 /*cnt*/ + (size_t)B * 8 /*thr, inv_tau*/ + streams * CAND_CAP * 8 + 512;
}

int sample_outer(const float* final_scores, int B, int N, long long pitch, int IM, int n_sample, const unsigned long long* seed,
                 void* ws, int* idx_out, int* status, cudaStream_t st, int invalid_bits) {
  if (n_sample > CAND_CAP / 2) { set_last_error("NUM_SAMPLED_MATCHES %d too large", n_sample); return MK_ERR_UNSUPPORTED; }
  const long long cells = (long long)N * N;
  const size_t streams = (size_t)B * IM;
  uint8_t* w = reinterpret_cast<uint8_t*>(ws);
  unsigned int* hist = reinterpret_cast<unsigned int*>(w); w += (size_t)B * HBINS * 4;
  unsigned int* cnt = reinterpret_cast<unsigned int*>(w); w += streams * 4;
  int* thr = reinterpret_cast<int*>(w); w += (size_t)B * 4;
  float* inv_tau = reinterpret_cast<float*>(w); w += (size_t)B * 4;
  w = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(w) + 255) & ~(uintptr_t)255);
  unsigned long long* cand = reinterpret_cast<unsigned long long*>(w);
  MK_CUDA_CHECK(cudaMemsetAsync(hist, 0, (size_t)B * HBINS * 4 + streams * 4, st));
  // one block per 4096-cell chunk (the hardware block scheduler balances the 1.5 waves at chunk granularity); the
  // kernels loop over chunks so that a smaller grid stays correct
  const bool aligned = reinterpret_cast<uintptr_t>(final_scores) % 16 == 0;
  const int spr = (N + 3) / 4, rpc = (SAMP_ELEMS_PER_BLOCK / 4) / spr;              // ROW_VEC: whole rows per block chunk
  const int mode = (pitch == N && cells % 4 == 0 && aligned) ? MODE_FLAT_VEC
                   : (pitch % 4 == 0 && pitch >= 4LL * spr && aligned && rpc >= 1) ? MODE_ROW_VEC : MODE_SCALAR;
  const long long chunks = (mode == MODE_ROW_VEC) ? (N + rpc - 1) / rpc : (cells + SAMP_ELEMS_PER_BLOCK - 1) / SAMP_ELEMS_PER_BLOCK;
  dim3 grid((unsigned)min(chunks, 65535LL * 16), B);
  if (mode == MODE_FLAT_VEC) sampler_phist_kernel<MODE_FLAT_VEC><<<grid, SAMP_THREADS, 0, st>>>(final_scores, N, pitch, hist, status, invalid_bits);
  else if (mode == MODE_ROW_VEC) sampler_phist_kernel<MODE_ROW_VEC><<<grid, SAMP_THREADS, 0, st>>>(final_scores, N, pitch, hist, status, invalid_bits);
  else sampler_phist_kernel<MODE_SCALAR><<<grid, SAMP_THREADS, 0, st>>>(final_scores, N, pitch, hist, status, invalid_bits);
  MK_CUDA_CHECK(cudaGetLastError());
  MK_CUDA_CHECK(launch_k(sampler_tau_kernel, dim3(B), dim3(TAU_THREADS), 0, st, hist, cells, n_sample, thr, inv_tau, status));
  MK_CUDA_CHECK(cudaGetLastError());
  if (mode == MODE_FLAT_VEC) MK_CUDA_CHECK(launch_k(sampler_collect_kernel<MODE_FLAT_VEC>, grid, dim3(SAMP_THREADS), 0, st, final_scores, N, pitch, IM, seed, thr, inv_tau, cand, cnt, CAND_CAP));
  else if (mode == MODE_ROW_VEC) MK_CUDA_CHECK(launch_k(sampler_collect_kernel<MODE_ROW_VEC>, grid, dim3(SAMP_THREADS), 0, st, final_scores, N, pitch, IM, seed, thr, inv_tau, cand, cnt, CAND_CAP));
  else MK_CUDA_CHECK(launch_k(sampler_collect_kernel<MODE_SCALAR>, grid, dim3(SAMP_THREADS), 0, st, final_scores, N, pitch, IM, seed, thr, inv_tau, cand, cnt, CAND_CAP));
  MK_CUDA_CHECK(cudaGetLastError());
  if (n_sample > 4 * SEL_THREADS) { set_last_error("NUM_SAMPLED_MATCHES %d too large", n_sample); return MK_ERR_UNSUPPORTED; }
  MK_CUDA_CHECK(launch_k(sampler_select_kernel<CAND_CAP>, dim3((unsigned)streams), dim3(SEL_THREADS), 0, st, cand, cnt, n_sample, IM,
                         (const int*)thr, cells, idx_out, status));
  MK_CUDA_CHECK(cudaGetLastError());
  return MK_OK;
}



// ---- hypotheses -------------------------------------------------------------------------------------------------------
constexpr int HYP_THREADS = 256;


// ONE launch per batch: grid (groups of hypotheses, IM, B), 256 threads.  Every block gathers its set of sampled matches
// into shared memory (X[3][n_s] Y[3][n_s] cdf[n_s]), draws and scores `hyp_per_block` 3-point hypotheses, and counts itself
// done on its pair; the LAST block of a pair (threadfence + atomic counter) takes the pair's argmax, re-gathers the winning
// set, runs the refinement and writes the pose; the last pair to finish applies the reference's batch-level zero fallback.
// `counters`: [0] = status bits, [1] = pairs finished, [4 + b] = blocks of pair b finished (zeroed by the caller).
constexpr int FIN_THREADS = HYP_THREADS;
__device__ void finalize_pair(const int* idx, const float* fs, const float* kps0, const float* d0, const float* kps1, const float* d1,
                              const float* Ki0, const float* Ki1, int N, long long pitch, const float* scores, const float* Rt,
                              int b, int IM, int IR, int n_s, int n_corr, int n_ref, float th_in, float* sm, float* pose,
                              int* best_set, float* inl_mask, int* best_hyp);

__global__ void __launch_bounds__(HYP_THREADS)
ransac_solve_kernel(const int* __restrict__ idx, const float* __restrict__ fs, const float* __restrict__ kps0,
                    const float* __restrict__ d0, const float* __restrict__ kps1, const float* __restrict__ d1,
                    const float* __restrict__ K0, const float* __restrict__ K1, int N, long long pitch,
                    const int* __restrict__ inner_idx, int IM, int IR, int n_s, int hyp_per_block, float th_soft,
                    const unsigned long long* __restrict__ seed_ptr, float* scores, float* Rt, int* counters,
                    int n_corr, int n_ref, float th_in, float* pose, int* best_set, float* inl_mask, int* best_hyp) {
  pdl_wait();        // launched with programmatic stream serialization: predecessors are complete past this point
  pdl_trigger();
  extern __shared__ float sm[];
  float* X = sm;                 // [3][n_s]
  float* Y = sm + 3 * n_s;       // [3][n_s]
  float* cdf = sm + 6 * n_s;     // [n_s] inclusive prefix sums of the weights
  __shared__ float warp_tot[HYP_THREADS / 32];
  __shared__ float Ki0[9], Ki1[9];
  __shared__ int last_flag;
  int* status = counters;
  const int s_in = blockIdx.y, b = blockIdx.z, s = b * IM + s_in;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if (tid == 0) { inv3x3(K0 + b * 9, Ki0); inv3x3(K1 + b * 9, Ki1); }
  __syncthreads();
  // block-wide inclusive scan of the weights (n_s is a multiple of HYP_THREADS)
  const int per = n_s / HYP_THREADS;
  float run;
  gather_set(idx, fs, kps0, d0, kps1, d1, Ki0, Ki1, N, pitch, b, s, n_s, HYP_THREADS, X, Y, cdf, run);
  float inc = run;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float v = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += v;
  }
  if (lane == 31) warp_tot[warp] = inc;
  __syncthreads();
  float base = inc - run;
  for (int w = 0; w < warp; ++w) base += warp_tot[w];
  for (int j = 0; j < per; ++j) cdf[tid * per + j] += base;
  __syncthreads();
  const float W = cdf[n_s - 1];
  const float beta = 5.0f / th_soft;
  const Philox rng(*seed_ptr ^ 0x9E3779B97F4A7C15ull);

  const int h0 = blockIdx.x * hyp_per_block;
  for (int hh = warp; hh < hyp_per_block; hh += HYP_THREADS / 32) {
    const int h = h0 + hh;
    if (h >= IR) break;
    const long long gh = (long long)s * IR + h;
    int id[3];
    if (inner_idx) {
      id[0] = inner_idx[gh * 3]; id[1] = inner_idx[gh * 3 + 1]; id[2] = inner_idx[gh * 3 + 2];
    } else {
      // successive sampling without replacement (== the exponential race in distribution)
      const uint4 r = rng((uint32_t)h, (uint32_t)s_in, (uint32_t)b, 0x3c6ef372u);
      const float u[3] = {u01_from_bits(r.x), u01_from_bits(r.y), u01_from_bits(r.z)};
      float removed = 0.f;
      for (int k = 0; k < 3; ++k) {
        float target = u[k] * (W - removed);
        // skip the mass of already drawn entries, in ascending index order
        int a = (k > 0) ? id[0] : -1, c = (k > 1) ? id[1] : -1;
        if (k > 1 && c < a) { const int t2 = a; a = c; c = t2; }
        if (a >= 0) { const float ex = cdf[a] - ((a > 0) ? cdf[a - 1] : 0.f); if (target >= cdf[a] - ex) target += ex; }
        if (c >= 0) { const float ex = cdf[c] - ((c > 0) ? cdf[c - 1] : 0.f); if (target >= cdf[c] - ex) target += ex; }
        int pick = cdf_search(cdf, n_s, fminf(target, W * 0.99999994f));
        // rounding may land on a removed entry: advance to the next free one
        for (int guard = 0; guard < 3; ++guard)
          if ((k > 0 && pick == id[0]) || (k > 1 && pick == id[1])) pick = (pick + 1) % n_s;
        id[k] = pick;
        removed += cdf[pick] - ((pick > 0) ? cdf[pick - 1] : 0.f);
      }
    }
    // Kabsch on the 3 sampled correspondences (unweighted branch, solvers.py:32-39), replicated on all lanes
    double xm[3] = {0, 0, 0}, ym[3] = {0, 0, 0};
    float xk[3][3], yk[3][3];
#pragma unroll
    for (int k = 0; k < 3; ++k)
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        xk[k][c] = X[c * n_s + id[k]]; yk[k][c] = Y[c * n_s + id[k]];
        xm[c] += xk[k][c]; ym[c] += yk[k][c];
      }
#pragma unroll
    for (int c = 0; c < 3; ++c) { xm[c] /= 3.0; ym[c] /= 3.0; }
    double H[9];
#pragma unroll
    for (int i = 0; i < 9; ++i) H[i] = 0.0;
#pragma unroll
    for (int k = 0; k < 3; ++k)
#pragma unroll
      for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) H[i * 3 + j] += ((double)xk[k][i] - xm[i]) * ((double)yk[k][j] - ym[j]);
    double Rd[9];
    kabsch_rotation(H, Rd);
    float R[9], t[3];
#pragma unroll
    for (int i = 0; i < 9; ++i) R[i] = (float)Rd[i];
#pragma unroll
    for (int i = 0; i < 3; ++i) t[i] = (float)(ym[i] - (Rd[i * 3] * xm[0] + Rd[i * 3 + 1] * xm[1] + Rd[i * 3 + 2] * xm[2]));
    // soft inlier count over the whole set (training_utils.py:55-61)
    float sc = 0.f;
    for (int i = lane; i < n_s; i += 32) {
      const float x0 = X[i], x1 = X[n_s + i], x2 = X[2 * n_s + i];
      const float r0 = R[0] * x0 + R[1] * x1 + R[2] * x2 + t[0] - Y[i];
      const float r1 = R[3] * x0 + R[4] * x1 + R[5] * x2 + t[1] - Y[n_s + i];
      const float r2 = R[6] * x0 + R[7] * x1 + R[8] * x2 + t[2] - Y[2 * n_s + i];
      const float dist = sqrtf(r0 * r0 + r1 * r1 + r2 * r2 + 1e-6f);
      sc += 1.0f / (1.0f + __expf(-beta * (th_soft - dist)));
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) sc += __shfl_xor_sync(0xffffffffu, sc, o);
    if (lane == 0) {
      scores[gh] = sc;
      bool bad = false;
#pragma unroll
      for (int i = 0; i < 9; ++i) { Rt[gh * 12 + i] = R[i]; bad |= !isfinite(R[i]); }
#pragma unroll
      for (int i = 0; i < 3; ++i) { Rt[gh * 12 + 9 + i] = t[i]; bad |= !isfinite(t[i]); }
      if (bad) atomicOr(status, 4);
    }
  }
  // ---- this block is done; the last block of the pair finalizes it ----
  __syncthreads();
  const int blocks_per_pair = gridDim.x * gridDim.y;
  if (tid == 0) {
    __threadfence();                                   // scores / Rt of this block before the count
    last_flag = (atomicAdd(&counters[4 + b], 1) == blocks_per_pair - 1) ? 1 : 0;
  }
  __syncthreads();
  if (!last_flag) return;
  __threadfence();                                     // the other blocks' scores / Rt after the count
  finalize_pair(idx, fs, kps0, d0, kps1, d1, Ki0, Ki1, N, pitch, scores, Rt, b, IM, IR, n_s, n_corr, n_ref, th_in, sm, pose,
                best_set, inl_mask, best_hyp);
  // ---- the last pair applies the batch-level zero fallback (probabilisticProcrustes.py:261-262,329-342): too few non-zero
  // cells (1), a non-finite hypothesis anywhere in the batch (4), and -- never silently -- a truncated candidate list (2)
  __syncthreads();
  if (tid == 0) {
    __threadfence();
    last_flag = (atomicAdd(&counters[1], 1) == (int)gridDim.z - 1) ? 1 : 0;
  }
  __syncthreads();
  if (!last_flag) return;
  __threadfence();
  if ((atomicOr(status, 0) & (1 | 2 | 4)) != 0)
    for (int i = tid; i < (int)gridDim.z * 13; i += HYP_THREADS) pose[i] = 0.f;
}

// ---- finalize: argmax + refinement + final score -------------------------------------------------------------------------

__device__ __forceinline__ void block_reduce_sum(double* vals, int nvals, double* scratch /*[nvals][FIN_THREADS/32]*/) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int k = 0; k < nvals; ++k) {
    double v = vals[k];
#pragma unroll
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) scratch[k * (FIN_THREADS / 32) + warp] = v;
  }
  __syncthreads();
  for (int k = 0; k < nvals; ++k) {
    double v = 0;
    for (int w = 0; w < FIN_THREADS / 32; ++w) v += scratch[k * (FIN_THREADS / 32) + w];
    vals[k] = v;
  }
  __syncthreads();
}

// out: pose [B,13] = R (9, row-major) | t (3) | inliers (1);  best_set [B];  inl_mask [B, n_s] (hard inliers @ final pose).
// Runs in the last block of pair b; `scores` / `Rt` were written by other blocks of this launch: L2 loads (__ldcg), never
// the read-only path.
__device__ void finalize_pair(const int* idx, const float* fs, const float* kps0, const float* d0, const float* kps1, const float* d1,
                              const float* Ki0, const float* Ki1, int N, long long pitch, const float* scores, const float* Rt,
                              int b, int IM, int IR, int n_s, int n_corr, int n_ref, float th_in, float* sm, float* pose,
                              int* best_set, float* inl_mask, int* best_hyp) {
  float* X = sm;
  float* Y = sm + 3 * n_s;
  __shared__ float red_v[FIN_THREADS];
  __shared__ int red_i[FIN_THREADS];
  __shared__ double scratch[12 * (FIN_THREADS / 32)];
  __shared__ float Rs[9], ts[3];
  const int tid = threadIdx.x;
  const int total = IM * IR;
  // argmax (first maximal index, like torch.argmax)
  float bv = -INFINITY; int bi = 0x7fffffff;
  for (int i = tid; i < total; i += FIN_THREADS) {
    const float v = __ldcg(scores + (long long)b * total + i);
    if (v > bv || (v == bv && i < bi)) { bv = v; bi = i; }
  }
  red_v[tid] = bv; red_i[tid] = bi;
  __syncthreads();
  for (int k = FIN_THREADS / 2; k; k >>= 1) {
    if (tid < k) {
      const float v = red_v[tid + k]; const int i = red_i[tid + k];
      if (v > red_v[tid] || (v == red_v[tid] && i < red_i[tid])) { red_v[tid] = v; red_i[tid] = i; }
    }
    __syncthreads();
  }
  int best = red_i[0];
  if (best < 0 || best >= total) best = 0;       // all-NaN scores
  const int sset = b * IM + best / IR;
  __syncthreads();                               // every thread has read red_i[0] / is done with the hypotheses' X, Y
  float unused;
  gather_set(idx, fs, kps0, d0, kps1, d1, Ki0, Ki1, N, pitch, b, sset, n_s, FIN_THREADS, X, Y, nullptr, unused);
  if (tid < 9) Rs[tid] = __ldcg(Rt + ((long long)b * total + best) * 12 + tid);
  if (tid < 3) ts[tid] = __ldcg(Rt + ((long long)b * total + best) * 12 + 9 + tid);
  __syncthreads();

  auto resid = [&](int i) {
    const float x0 = X[i], x1 = X[n_s + i], x2 = X[2 * n_s + i];
    const float r0 = Rs[0] * x0 + Rs[1] * x1 + Rs[2] * x2 + ts[0] - Y[i];
    const float r1 = Rs[3] * x0 + Rs[4] * x1 + Rs[5] * x2 + ts[1] - Y[n_s + i];
    const float r2 = Rs[6] * x0 + Rs[7] * x1 + Rs[8] * x2 + ts[2] - Y[2 * n_s + i];
    return sqrtf(r0 * r0 + r1 * r1 + r2 * r2 + 1e-6f);
  };

  double prev = (double)n_corr;
  for (int it = 0; it < n_ref; ++it) {
    // hard inliers at the current pose (training_utils.py:71-75) and their moments
    double m[7] = {0, 0, 0, 0, 0, 0, 0};          // count, sum x (3), sum y (3)
    for (int i = tid; i < n_s; i += FIN_THREADS) {
      if (th_in - resid(i) >= 0.f) {
        m[0] += 1.0;
        m[1] += X[i]; m[2] += X[n_s + i]; m[3] += X[2 * n_s + i];
        m[4] += Y[i]; m[5] += Y[n_s + i]; m[6] += Y[2 * n_s + i];
      }
    }
    block_reduce_sum(m, 7, scratch);
    const double cnt = m[0];
    if (!(cnt >= (double)n_corr && cnt > prev)) break;     // uniform across the block
    prev = cnt;
    const double wn = 1.0 / (cnt + 1e-16);                 // solvers.py:14-15 with a {0,1} mask
    const double xm[3] = {m[1] * wn, m[2] * wn, m[3] * wn}, ym[3] = {m[4] * wn, m[5] * wn, m[6] * wn};
    double H[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    for (int i = tid; i < n_s; i += FIN_THREADS) {
      if (th_in - resid(i) >= 0.f) {
        const double a[3] = {X[i] - xm[0], X[n_s + i] - xm[1], X[2 * n_s + i] - xm[2]};
        const double c[3] = {Y[i] - ym[0], Y[n_s + i] - ym[1], Y[2 * n_s + i] - ym[2]};
#pragma unroll
        for (int p = 0; p < 3; ++p)
#pragma unroll
          for (int q = 0; q < 3; ++q) H[p * 3 + q] += a[p] * c[q];
      }
    }
    block_reduce_sum(H, 9, scratch);
    if (tid == 0) {
      double Rd[9];
      kabsch_rotation(H, Rd);
      for (int i = 0; i < 9; ++i) Rs[i] = (float)Rd[i];
      for (int i = 0; i < 3; ++i) ts[i] = (float)(ym[i] - (Rd[i * 3] * xm[0] + Rd[i * 3 + 1] * xm[1] + Rd[i * 3 + 2] * xm[2]));
    }
    __syncthreads();
  }
  // final soft count at TH_INLIER (probabilisticProcrustes.py:303) + hard mask for the inlier list (:308)
  const float beta = 5.0f / th_in;
  double acc[1] = {0.0};
  for (int i = tid; i < n_s; i += FIN_THREADS) {
    const float d = resid(i);
    acc[0] += 1.0f / (1.0f + __expf(-beta * (th_in - d)));
    if (inl_mask) inl_mask[(long long)b * n_s + i] = (th_in - d >= 0.f) ? 1.0f : 0.0f;
  }
  block_reduce_sum(acc, 1, scratch);
  if (tid == 0) {
    float* o = pose + (long long)b * 13;           // the batch-level zero fallback is applied by the last pair to finish
    for (int i = 0; i < 9; ++i) o[i] = Rs[i];
    for (int i = 0; i < 3; ++i) o[9 + i] = ts[i];
    o[12] = (float)acc[0];
    best_set[b] = sset;
    if (best_hyp) best_hyp[b] = best;
  }
}

// seed state lives in device memory so that a captured CUDA graph draws fresh numbers on every replay
__global__ void seed_set_kernel(unsigned long long* s, unsigned long long v) { *s = v; }
__global__ void seed_advance_kernel(unsigned long long* s) {
  unsigned long long z = *s + 0x9E3779B97F4A7C15ull;          // splitmix64 step
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  *s = z ^ (z >> 31);
}
int seed_set(unsigned long long* s, unsigned long long v, cudaStream_t st) {
  seed_set_kernel<<<1, 1, 0, st>>>(s, v);
  MK_CUDA_CHECK(cudaGetLastError());
  return MK_OK;
}
int seed_advance(unsigned long long* s, cudaStream_t st) {
  seed_advance_kernel<<<1, 1, 0, st>>>(s);
  MK_CUDA_CHECK(cudaGetLastError());
  return MK_OK;
}

int ransac_solve(const float* final_scores, long long pitch, const float* kps0, const float* d0, const float* kps1, const float* d1,
                 const float* K0, const float* K1, int B, int N, const RansacParams& rp, const int* outer_idx,
                 const int* inner_idx, float* hyp_scores, float* hyp_Rt, int* counters, float* pose,
                 int* best_set, float* inl_mask, int* best_hyp, cudaStream_t st) {
  // counters: [0] status bits, [1] pairs finished, [4 + b] blocks of pair b finished; zeroed by the caller before the sampler
  const int IM = rp.it_matches, IR = rp.it_ransac, n_s = rp.n_sample;
  if (rp.n_corr != 3) { set_last_error("NUM_CORR_3D_3D must be 3 (got %d)", rp.n_corr); return MK_ERR_UNSUPPORTED; }
  if (n_s % HYP_THREADS) { set_last_error("NUM_SAMPLED_MATCHES must be a multiple of %d", HYP_THREADS); return MK_ERR_UNSUPPORTED; }
  const int hyp_per_block = 8;
  const size_t smem_h = (size_t)7 * n_s * 4;
  static unsigned long long attr_mask = 0;
  if (first_use_on_device(attr_mask)) {
    MK_CUDA_CHECK(cudaFuncSetAttribute(ransac_solve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
  }
  if (smem_h > 200 * 1024) { set_last_error("NUM_SAMPLED_MATCHES too large for shared memory"); return MK_ERR_UNSUPPORTED; }
  MK_CUDA_CHECK(launch_k(ransac_solve_kernel, dim3(ceil_div(IR, hyp_per_block), IM, B), dim3(HYP_THREADS), smem_h, st,
                         outer_idx, final_scores, kps0, d0, kps1, d1, K0, K1, N, pitch, inner_idx, IM, IR, n_s, hyp_per_block,
                         rp.th_soft, rp.seed, hyp_scores, hyp_Rt, counters, rp.n_corr, rp.n_refine, rp.th_inlier, pose, best_set,
                         inl_mask, best_hyp));
  MK_CUDA_CHECK(cudaGetLastError());
  return MK_OK;
}

// the Kabsch rotation alone, one 3x3 H per thread: the solver's and the loss's kabsch_rotation, exposed for tests
__global__ void kabsch_kernel(const double* __restrict__ H, double* __restrict__ R, int n) {
  pdl_wait();
  pdl_trigger();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  kabsch_rotation(H + (long long)i * 9, R + (long long)i * 9);
}

int kabsch_batch(const double* H, double* R, int n, cudaStream_t st) {
  if (n < 0 || !H || !R) { set_last_error("kabsch: n must be >= 0 and H, R non-null"); return MK_ERR_INVALID; }
  if (n == 0) return MK_OK;
  MK_CUDA_CHECK(launch_k(kabsch_kernel, dim3((unsigned)ceil_div(n, 128)), dim3(128), 0, st, H, R, n));
  return MK_OK;
}

}  // namespace mk
