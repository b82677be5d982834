// Non-GEMM kernels of the DINOv2 backbone: patch gathering, LayerNorm, fused multi-head attention.
#include "ops.h"

namespace mk {

// ------------------------------------------------------------------------------------------------------
// Patch gather (reference layers/patch_embed.py:66,76 conv k=s=14 == GEMM with K = 3*14*14 = 588).
// img fp32 [n_img, 3, H, W] -> P fp16 [n_img*gh*gw, kpad]  (k = c*196 + ky*14 + kx, zero-padded to kpad),
// rows beyond the crop (H, W not multiples of 14; mickey_extractor.py:46) are never read.
// Extra blocks write the cls rows of the token matrix: X[img*T] = cls + pos[0].
// ------------------------------------------------------------------------------------------------------
__global__ void patch_gather_kernel(const float* __restrict__ img, __half* __restrict__ P, int n_img, int H, int W,
                                    int gh, int gw, int kpad, float* __restrict__ X, const float* __restrict__ cls_pos,
                                    int D) {
  const int row = blockIdx.x;
  const int n_rows = n_img * gh * gw;
  if (row >= n_rows) {               // cls rows
    const int im = row - n_rows;
    float* x = X + (size_t)im * (gh * gw + 1) * D;
    for (int d = threadIdx.x; d < D; d += blockDim.x) x[d] = cls_pos[d];
    return;
  }
  const int im = row / (gh * gw), cell = row % (gh * gw), py = cell / gw, px = cell % gw;
  const float* src = img + (size_t)im * 3 * H * W;
  __half* dst = P + (size_t)row * kpad;
  for (int k = threadIdx.x; k < kpad; k += blockDim.x) {
    float v = 0.f;
    if (k < 588) {
      const int c = k / 196, r = (k % 196) / 14, q = k % 14;
      v = src[((size_t)c * H + py * 14 + r) * W + px * 14 + q];
    }
    dst[k] = __float2half_rn(v);
  }
}

int patch_gather(const float* img, void* P, int n_img, int H, int W, int kpad, float* X, const float* cls_pos, int D,
                 cudaStream_t s) {
  const int gh = H / 14, gw = W / 14;
  patch_gather_kernel<<<n_img * gh * gw + n_img, 128, 0, s>>>(img, (__half*)P, n_img, H, W, gh, gw, kpad, X, cls_pos, D);
  MK_CUDA_CHECK(cudaGetLastError());
  return MK_OK;
}

// ------------------------------------------------------------------------------------------------------
// LayerNorm over the last dim (eps 1e-6 in the ViT: dinov2.py:88; layers/block.py:105-106).
// One warp per row; fp32 in (the residual stream), fp16 out (the next GEMM's A operand).
// mode 0: out[row] = LN(x[row])                     (norm1 / norm2)
// mode 1: final norm (dinov2.py:230-233): drop the cls token and scatter patch tokens into the
//         zero-padded NHWC feature image that feeds the head convolutions:
//         out[(img*(gh+2) + y+1)*(gw+2) + x+1][:] = LN(x[img*T + 1 + y*gw + x])
// mode 2 (layernorm_cm_kernel): the same final norm written as the heads' fp32 input, channel-major [n_img, D, N]
//         (mickey_extractor.py:49-51: x_norm_patchtokens.permute(0, 2, 1).reshape(B, C, h, w).float()).
// All modes share ln_row_stats / ln_affine: one summation order, one expression, so mode 2's value rounded to fp16
// is mode 1's F interior bit for bit.
// ------------------------------------------------------------------------------------------------------
// One warp reads one row (lane holds float4s i*32 + lane) and reduces its mean and 1 / std.
template <int VEC>
__device__ __forceinline__ void ln_row_stats(const float* __restrict__ xrow, int lane, int D, float eps, float4 (&v)[VEC],
                                             float& mean, float& rstd) {
  const float4* xr = reinterpret_cast<const float4*>(xrow);
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < VEC; ++i) {
    v[i] = xr[i * 32 + lane];
    sum += v[i].x + v[i].y + v[i].z + v[i].w;
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  mean = sum / D;
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < VEC; ++i) {
    const float a = v[i].x - mean, c = v[i].y - mean, d = v[i].z - mean, e = v[i].w - mean;
    sq += a * a + c * c + d * d + e * e;
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
  rstd = rsqrtf(sq / D + eps);
}

__device__ __forceinline__ float ln_affine(float v, float mean, float rstd, float w, float b) { return (v - mean) * rstd * w + b; }

template <int VEC>   // D = 128 * VEC
__global__ void layernorm_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ b,
                                 __half* __restrict__ out, int rows, int D, float eps, int mode, int gh, int gw) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  pdl_wait();
  pdl_trigger();
  if (row >= rows) return;
  long long orow = row;
  if (mode == 1) {
    const int T = gh * gw + 1;
    const int im = row / T, t = row % T;
    if (t == 0) return;
    const int y = (t - 1) / gw, xx = (t - 1) % gw;
    orow = ((long long)im * (gh + 2) + y + 1) * (gw + 2) + xx + 1;
  }
  float4 v[VEC];
  float mean, rstd;
  ln_row_stats<VEC>(x + (size_t)row * D, lane, D, eps, v, mean, rstd);
  __half* orow_p = out + (size_t)orow * D;
#pragma unroll
  for (int i = 0; i < VEC; ++i) {
    const int c0 = (i * 32 + lane) * 4;
    const float4 ww = *reinterpret_cast<const float4*>(w + c0);
    const float4 bb = *reinterpret_cast<const float4*>(b + c0);
    __half2 h0 = __floats2half2_rn(ln_affine(v[i].x, mean, rstd, ww.x, bb.x), ln_affine(v[i].y, mean, rstd, ww.y, bb.y));
    __half2 h1 = __floats2half2_rn(ln_affine(v[i].z, mean, rstd, ww.z, bb.z), ln_affine(v[i].w, mean, rstd, ww.w, bb.w));
    uint2 u;
    u.x = *reinterpret_cast<uint32_t*>(&h0);
    u.y = *reinterpret_cast<uint32_t*>(&h1);
    *reinterpret_cast<uint2*>(orow_p + c0) = u;
  }
}

// Final norm into the channel-major [n_img, D, N] fp32 feature map.  A CTA takes LNCM_TOK consecutive patch tokens of
// one image (grid: ceil(N / LNCM_TOK) x n_img); each of its 16 warps normalises two of them with the row reads of
// layernorm_kernel (512-byte coalesced float4 loads).  The normalised tile leaves 128 channels at a time through a
// [128][LNCM_TOK + 1] shared-memory transpose: one warp stores 32 consecutive tokens of one channel (128 bytes).
constexpr int LNCM_TOK = 32, LNCM_WARPS = 16, LNCM_ROWS = LNCM_TOK / LNCM_WARPS;

template <int VEC>   // D = 128 * VEC
__global__ void __launch_bounds__(LNCM_WARPS * 32)
layernorm_cm_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ b,
                    float* __restrict__ out, int N, int D, float eps) {
  __shared__ float tile[128][LNCM_TOK + 1];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int im = blockIdx.y, t0 = blockIdx.x * LNCM_TOK;
  pdl_wait();
  pdl_trigger();
  float4 v[LNCM_ROWS][VEC];
  float mean[LNCM_ROWS], rstd[LNCM_ROWS];
#pragma unroll
  for (int r = 0; r < LNCM_ROWS; ++r) {
    const int t = min(t0 + warp * LNCM_ROWS + r, N - 1);        // rows past N repeat the last token; never stored
    ln_row_stats<VEC>(x + ((size_t)im * (N + 1) + 1 + t) * D, lane, D, eps, v[r], mean[r], rstd[r]);
  }
  float* obase = out + (size_t)im * D * N;
  const int t_out = t0 + lane;
#pragma unroll
  for (int i = 0; i < VEC; ++i) {
    const int c0 = (i * 32 + lane) * 4;
    const float4 ww = *reinterpret_cast<const float4*>(w + c0);
    const float4 bb = *reinterpret_cast<const float4*>(b + c0);
#pragma unroll
    for (int r = 0; r < LNCM_ROWS; ++r) {
      const int tt = warp * LNCM_ROWS + r;
      tile[lane * 4 + 0][tt] = ln_affine(v[r][i].x, mean[r], rstd[r], ww.x, bb.x);
      tile[lane * 4 + 1][tt] = ln_affine(v[r][i].y, mean[r], rstd[r], ww.y, bb.y);
      tile[lane * 4 + 2][tt] = ln_affine(v[r][i].z, mean[r], rstd[r], ww.z, bb.z);
      tile[lane * 4 + 3][tt] = ln_affine(v[r][i].w, mean[r], rstd[r], ww.w, bb.w);
    }
    __syncthreads();
    if (t_out < N) {
#pragma unroll
      for (int k = 0; k < 128 / LNCM_WARPS; ++k) {
        const int c = k * LNCM_WARPS + warp;
        obase[(size_t)(i * 128 + c) * N + t_out] = tile[c][lane];
      }
    }
    __syncthreads();
  }
}

int layernorm_channel_major(const float* x, const float* w, const float* b, float* out, int n_img, int N, int D, float eps,
                            cudaStream_t s) {
  dim3 grid(ceil_div(N, LNCM_TOK), n_img), block(LNCM_WARPS * 32);
  switch (D) {
    case 384:  MK_CUDA_CHECK(launch_k(layernorm_cm_kernel<3>, grid, block, 0, s, x, w, b, out, N, D, eps)); break;
    case 768:  MK_CUDA_CHECK(launch_k(layernorm_cm_kernel<6>, grid, block, 0, s, x, w, b, out, N, D, eps)); break;
    case 1024: MK_CUDA_CHECK(launch_k(layernorm_cm_kernel<8>, grid, block, 0, s, x, w, b, out, N, D, eps)); break;
    default: set_last_error("layernorm: unsupported width %d", D); return MK_ERR_UNSUPPORTED;
  }
  return MK_OK;
}

int layernorm(const float* x, const float* w, const float* b, void* out, int rows, int D, float eps, int mode, int gh,
              int gw, cudaStream_t s) {
  const int warps = 8;
  dim3 grid(ceil_div(rows, warps)), block(warps * 32);
  __half* o = (__half*)out;
  switch (D) {
    case 384:  MK_CUDA_CHECK(launch_k(layernorm_kernel<3>, grid, block, 0, s, x, w, b, o, rows, D, eps, mode, gh, gw)); break;
    case 768:  MK_CUDA_CHECK(launch_k(layernorm_kernel<6>, grid, block, 0, s, x, w, b, o, rows, D, eps, mode, gh, gw)); break;
    case 1024: MK_CUDA_CHECK(launch_k(layernorm_kernel<8>, grid, block, 0, s, x, w, b, o, rows, D, eps, mode, gh, gw)); break;
    default: set_last_error("layernorm: unsupported width %d", D); return MK_ERR_UNSUPPORTED;
  }
  return MK_OK;
}

// ------------------------------------------------------------------------------------------------------
// Fused attention (reference layers/attention.py:49-62): softmax(q k^T / 8) v per (image, head), head_dim 64.
// qkv fp16 [n_img*T, 3*D] (q | k | v, each [heads, 64]); out fp16 [n_img*T, D].
// Flash-style: one CTA = 64 queries of one (image, head); 4 warps x 16 query rows; K/V streamed in
// 64-key tiles through a double-buffered cp.async ring; S and PV on mma.sync.m16n8k16 with fp32
// accumulation and an online softmax in registers; the T x T logits are never materialised.
// ------------------------------------------------------------------------------------------------------
constexpr int ATT_BQ = 64, ATT_BK = 64, ATT_HD = 64, ATT_THREADS = 128;

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, bool valid) {
  const int sz = valid ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void mma_16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t pack_h2(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}

// tile [64 rows][64 halves] = 128 B per row, 16-byte chunks XOR-swizzled with (row & 7)
__device__ __forceinline__ uint32_t tile_off(int row, int chunk) { return (uint32_t)(row * 128 + ((chunk ^ (row & 7)) << 4)); }

__device__ __forceinline__ void load_tile(uint32_t smem_tile, const __half* gsrc, long long ld, int row0, int rows_valid,
                                          int tid) {
  // 64 rows x 8 chunks = 512 chunks over 128 threads
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int idx = tid + i * ATT_THREADS;
    const int r = idx >> 3, c = idx & 7;
    const bool ok = (row0 + r) < rows_valid;
    const __half* src = gsrc + (long long)(ok ? (row0 + r) : 0) * ld + c * 8;
    cp_async16(smem_tile + tile_off(r, c), src, ok);
  }
}

__global__ void __launch_bounds__(ATT_THREADS)
attention_kernel(const __half* __restrict__ qkv, __half* __restrict__ out, int T, int D, float scale_log2) {
  __shared__ __align__(128) uint8_t smem[ATT_BQ * 128 + 2 * ATT_BK * 128 + 2 * ATT_BK * 128];
  const uint32_t sQ = (uint32_t)__cvta_generic_to_shared(smem);
  const uint32_t sK = sQ + ATT_BQ * 128;
  const uint32_t sV = sK + 2 * ATT_BK * 128;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int q0 = blockIdx.x * ATT_BQ, head = blockIdx.y, im = blockIdx.z;
  const long long ld = 3LL * D;
  const __half* base = qkv + (long long)im * T * ld;
  const __half* gq = base + head * ATT_HD;
  const __half* gk = base + D + head * ATT_HD;
  const __half* gv = base + 2 * D + head * ATT_HD;

  load_tile(sQ, gq, ld, q0, T, tid);
  load_tile(sK, gk, ld, 0, T, tid);
  load_tile(sV, gv, ld, 0, T, tid);
  cp_async_commit();

  const int n_tiles = (T + ATT_BK - 1) / ATT_BK;
  float o[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i) { o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f; }
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  uint32_t qf[4][4];

  for (int kt = 0; kt < n_tiles; ++kt) {
    const int buf = kt & 1;
    if (kt + 1 < n_tiles) {
      load_tile(sK + (buf ^ 1) * ATT_BK * 128, gk, ld, (kt + 1) * ATT_BK, T, tid);
      load_tile(sV + (buf ^ 1) * ATT_BK * 128, gv, ld, (kt + 1) * ATT_BK, T, tid);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    if (kt == 0) {
      // Q fragments for this warp's 16 rows, 4 k-blocks of 16
      const int r = warp * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
#pragma unroll
      for (int kb = 0; kb < 4; ++kb) {
        const int chunk = kb * 2 + (lane >> 4);
        ldsm_x4(sQ + tile_off(r, chunk), qf[kb][0], qf[kb][1], qf[kb][2], qf[kb][3]);
      }
    }
    const uint32_t tK = sK + buf * ATT_BK * 128, tV = sV + buf * ATT_BK * 128;

    // S = Q K^T : 16 x 64 per warp -> 8 n-blocks of 8 keys
    float s[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) { s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f; }
#pragma unroll
    for (int kb = 0; kb < 4; ++kb) {
#pragma unroll
      for (int np = 0; np < 4; ++np) {        // pairs of n-blocks (16 keys)
        const int key = np * 16 + (lane & 7) + (lane >> 4) * 8;
        const int chunk = kb * 2 + ((lane >> 3) & 1);
        uint32_t b0, b1, b2, b3;
        ldsm_x4(tK + tile_off(key, chunk), b0, b1, b2, b3);
        mma_16816(s[np * 2], qf[kb], b0, b1);
        mma_16816(s[np * 2 + 1], qf[kb], b2, b3);
      }
    }
    // scale, mask the key tail, online softmax (rows g and g+8 of this warp's 16)
    const int key_base = kt * ATT_BK + (lane & 3) * 2;
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int nb = 0; nb < 8; ++nb) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int key = key_base + nb * 8 + (e & 1);
        const float val = (key < T) ? s[nb][e] * scale_log2 : -INFINITY;
        s[nb][e] = val;
        mx[e >> 1] = fmaxf(mx[e >> 1], val);
      }
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
      mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
    }
    float corr[2], m_new[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      m_new[h] = fmaxf(m_run[h], mx[h]);            // finite: every tile has at least one valid key
      corr[h] = exp2f(m_run[h] - m_new[h]);
      m_run[h] = m_new[h];
    }
    float rs[2] = {0.f, 0.f};
#pragma unroll
    for (int nb = 0; nb < 8; ++nb) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float pv = exp2f(s[nb][e] - m_new[e >> 1]);
        s[nb][e] = pv;
        rs[e >> 1] += pv;
      }
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) l_run[h] = l_run[h] * corr[h] + rs[h];
#pragma unroll
    for (int nb = 0; nb < 8; ++nb) {
      o[nb][0] *= corr[0]; o[nb][1] *= corr[0]; o[nb][2] *= corr[1]; o[nb][3] *= corr[1];
    }
    // O += P V : k-blocks of 16 keys, 8 n-blocks of 8 dims
#pragma unroll
    for (int kb = 0; kb < 4; ++kb) {
      uint32_t a[4];
      a[0] = pack_h2(s[kb * 2][0], s[kb * 2][1]);
      a[1] = pack_h2(s[kb * 2][2], s[kb * 2][3]);
      a[2] = pack_h2(s[kb * 2 + 1][0], s[kb * 2 + 1][1]);
      a[3] = pack_h2(s[kb * 2 + 1][2], s[kb * 2 + 1][3]);
#pragma unroll
      for (int dp = 0; dp < 4; ++dp) {        // pairs of d n-blocks (16 dims)
        const int key = kb * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
        const int chunk = dp * 2 + (lane >> 4);
        uint32_t b0, b1, b2, b3;
        ldsm_x4_t(tV + tile_off(key, chunk), b0, b1, b2, b3);
        mma_16816(o[dp * 2], a, b0, b1);
        mma_16816(o[dp * 2 + 1], a, b2, b3);
      }
    }
    __syncthreads();
  }

  // finalise: divide by the row sums (quad-reduced) and store fp16
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    l_run[h] += __shfl_xor_sync(0xffffffffu, l_run[h], 1);
    l_run[h] += __shfl_xor_sync(0xffffffffu, l_run[h], 2);
  }
  const int r0 = q0 + warp * 16 + (lane >> 2);
  __half* obase = out + (long long)im * T * D + head * ATT_HD + (lane & 3) * 2;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int r = r0 + h * 8;
    if (r < T) {
      const float inv = 1.0f / l_run[h];
#pragma unroll
      for (int nb = 0; nb < 8; ++nb) {
        const uint32_t pk = pack_h2(o[nb][h * 2] * inv, o[nb][h * 2 + 1] * inv);
        *reinterpret_cast<uint32_t*>(obase + (long long)r * D + nb * 8) = pk;
      }
    }
  }
}

int attention(const void* qkv, void* out, int n_img, int T, int D, int heads, cudaStream_t s) {
  if (D != heads * ATT_HD) { set_last_error("attention: head_dim must be 64 (D=%d heads=%d)", D, heads); return MK_ERR_UNSUPPORTED; }
  dim3 grid(ceil_div(T, ATT_BQ), heads, n_img);
  const float scale_log2 = 0.125f * 1.4426950408889634f;   // head_dim^-0.5 * log2(e)
  attention_kernel<<<grid, ATT_THREADS, 0, s>>>((const __half*)qkv, (__half*)out, T, D, scale_log2);
  MK_CUDA_CHECK(cudaGetLastError());
  return MK_OK;
}

}  // namespace mk
