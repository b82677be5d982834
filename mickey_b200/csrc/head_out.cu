// The heads' output layers (mickey_extractor.py:81-142, 160-178, 199-218, 246-249; extractor_utils.py:6-10) for
// training: forward and backward in fp32 on the CUDA cores (include/mickey_b200.h mk_head_out*, DESIGN.md §6i).
//
// x = rb4's output fp32 [B, C, h, w] with any element strides, W the 1x1 weight [k, C], r = W x per pixel (k = 1 or 2):
//   score softmax   p = e / (sum e + eps), e = exp((r - (mean r + eps)) / T) mask    one block per image
//   score sigmoid   p = sigmoid(r) mask
//   offset          o = sigmoid(r)                                                     k = 2
//   depth           r, or max_depth sigmoid(r)
//   descriptor      y = x / n, n = sqrt(sum_c x^2 + 1e-10)                              no weight; n is saved
// mask zeroes BORDER cells at each edge.  The backward forms dr from the saved output and the upstream gradient g:
//   softmax  dr = p (g - sum_i g_i p_i) / T  (the mean is detached, as in the reference)
//   sigmoid  dr = g p (1 - p) mask,  offset dr = g o (1 - o),  depth dr = g or g d (1 - d / max_depth)
//   descriptor dx = (g - y (y . g)) / n
// then dx = dr^T W and dW[j, c] = sum_{b,p} dr[j, b, p] x[b, c, p].  Every reduction (the per-image mean, sum e and
// sum g p, the per-pixel sums over channels, the dW pixel slots) accumulates in fp64 in a fixed order and rounds once;
// there are no atomics, so results are bit-identical run to run, and an image's output and dx do not depend on the other
// images of the batch.  A thread reads the channels of its pixel in index order whatever the strides, so NCHW, strided
// and channels_last inputs give the same bits.
#include "../../include/mickey_b200.h"
#include "common.cuh"

#include <algorithm>
#include <cmath>

namespace mk {

namespace {

constexpr int BORDER = 3;                 // remove_borders(..., borders=3), mickey_extractor.py:138, 140
constexpr float L2_EPS = 1e-10f;          // desc_l2norm, extractor_utils.py:8
constexpr int MAX_C = 4096;
constexpr long long MAX_PIXELS = 1LL << 26;
constexpr int PT = 256;                   // threads of the per-pixel kernels
constexpr int ST = 512;                   // threads of the per-image (softmax) kernels
constexpr int MAX_SLOTS = 1024;           // dW pixel slots

struct XView {                            // x [B, C, h, w] through its element strides
  const float* p;
  long long sb, sc, sy, sx;
  int hw, w;
  __device__ __forceinline__ long long base(long long q) const {      // q = b hw + y w + x
    const long long b = q / hw;
    const int r = (int)(q - b * hw);
    return b * sb + (long long)(r / w) * sy + (long long)(r % w) * sx;
  }
};

__device__ __forceinline__ bool interior(int r, int h, int w) {
  const int y = r / w, x = r % w;
  return y >= BORDER && y < h - BORDER && x >= BORDER && x < w - BORDER;
}

__device__ __forceinline__ float sigm(float t) { return 1.f / (1.f + expf(-t)); }

// Sum of v over the block in a fixed order: lanes by shuffle, then the warps' partials in warp order.
template <int NT>
__device__ double block_sum(double v, double* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();                        // red may still be read from the previous call
  if (lane == 0) red[warp] = v;
  __syncthreads();
  double s = 0.0;
  for (int i = 0; i < NT / 32; ++i) s += red[i];
  return s;
}

// kinds SCORE_SIGMOID, OFFSET, DEPTH, DEPTH_SIGMOID: one thread per pixel, out [B, k, hw]
__global__ void __launch_bounds__(PT) ho_conv_act_kernel(XView x, const float* wt, int C, int k, int kind, int h,
                                                         float max_depth, long long P, float* out) {
  pdl_wait();
  pdl_trigger();
  const long long q = (long long)blockIdx.x * PT + threadIdx.x;
  if (q >= P) return;
  const long long xb = x.base(q);
  float r0 = 0.f, r1 = 0.f;
  for (int c = 0; c < C; ++c) {
    const float v = x.p[xb + c * x.sc];
    r0 = fmaf(wt[c], v, r0);
    if (k == 2) r1 = fmaf(wt[C + c], v, r1);
  }
  const long long b = q / x.hw;
  const int r = (int)(q - b * x.hw);
  float* o = out + b * k * x.hw + r;
  if (kind == MK_HO_SCORE_SIGMOID) {
    o[0] = interior(r, h, x.w) ? sigm(r0) : 0.f;
  } else if (kind == MK_HO_OFFSET) {
    o[0] = sigm(r0);
    o[x.hw] = sigm(r1);
  } else if (kind == MK_HO_DEPTH_SIGMOID) {
    o[0] = max_depth * sigm(r0);
  } else {
    o[0] = r0;
  }
}

// SCORE_SOFTMAX: one block per image.  out holds r, then e, then p; each thread revisits only its own cells.
__global__ void __launch_bounds__(ST) ho_softmax_fwd_kernel(XView x, const float* wt, int C, int h, const float* eps_dev,
                                                            float temp, float* out) {
  __shared__ double red[ST / 32];
  pdl_wait();
  pdl_trigger();
  const int b = blockIdx.x, hw = x.hw;
  float* o = out + (long long)b * hw;
  double s = 0.0;
  for (int r = threadIdx.x; r < hw; r += ST) {
    const long long xb = x.base((long long)b * hw + r);
    float acc = 0.f;
    for (int c = 0; c < C; ++c) acc = fmaf(wt[c], x.p[xb + c * x.sc], acc);
    o[r] = acc;
    s += acc;
  }
  const float eps = *eps_dev;
  const float shift = (float)(block_sum<ST>(s, red) / hw) + eps;
  s = 0.0;
  for (int r = threadIdx.x; r < hw; r += ST) {
    const float e = interior(r, h, x.w) ? expf((o[r] - shift) / temp) : 0.f;
    o[r] = e;
    s += e;
  }
  const float denom = (float)block_sum<ST>(s, red) + eps;
  for (int r = threadIdx.x; r < hw; r += ST) o[r] = o[r] / denom;
}

// DESC_L2: one thread per pixel; out [B, C, hw] contiguous, norm [B, hw] (may be NULL)
__global__ void __launch_bounds__(PT) ho_l2_fwd_kernel(XView x, int C, long long P, float* out, float* norm) {
  pdl_wait();
  pdl_trigger();
  const long long q = (long long)blockIdx.x * PT + threadIdx.x;
  if (q >= P) return;
  const long long xb = x.base(q);
  double s = 0.0;
  for (int c = 0; c < C; ++c) {
    const double v = x.p[xb + c * x.sc];
    s += v * v;
  }
  const float n = (float)sqrt(s + (double)L2_EPS);
  const long long b = q / x.hw;
  const int r = (int)(q - b * x.hw);
  float* o = out + b * C * x.hw + r;
  for (int c = 0; c < C; ++c) o[(long long)c * x.hw] = x.p[xb + c * x.sc] / n;
  if (norm) norm[q] = n;
}

// dr of kinds SCORE_SIGMOID, OFFSET, DEPTH, DEPTH_SIGMOID: one thread per element of [B, k, hw]
__global__ void __launch_bounds__(PT) ho_act_bwd_kernel(const float* out, const float* g, int kind, int h, int w,
                                                        int hw, float max_depth, long long n, float* dr) {
  pdl_wait();
  pdl_trigger();
  const long long i = (long long)blockIdx.x * PT + threadIdx.x;
  if (i >= n) return;
  const float o = out[i], gi = g[i];
  const int r = (int)(i % hw);
  float d;
  if (kind == MK_HO_SCORE_SIGMOID) d = interior(r, h, w) ? gi * (o * (1.f - o)) : 0.f;
  else if (kind == MK_HO_OFFSET) d = gi * (o * (1.f - o));
  else if (kind == MK_HO_DEPTH_SIGMOID) d = gi * (o * (1.f - o / max_depth));
  else d = gi;
  dr[i] = d;
}

// dr of SCORE_SOFTMAX: one block per image
__global__ void __launch_bounds__(ST) ho_softmax_bwd_kernel(const float* out, const float* g, int hw, float temp,
                                                            float* dr) {
  __shared__ double red[ST / 32];
  pdl_wait();
  pdl_trigger();
  const long long off = (long long)blockIdx.x * hw;
  double s = 0.0;
  for (int r = threadIdx.x; r < hw; r += ST) s += (double)g[off + r] * out[off + r];
  const float gp = (float)block_sum<ST>(s, red);
  for (int r = threadIdx.x; r < hw; r += ST) dr[off + r] = out[off + r] * (g[off + r] - gp) / temp;
}

// DESC_L2 backward: one thread per pixel; y, g, dx [B, C, hw] contiguous
__global__ void __launch_bounds__(PT) ho_l2_bwd_kernel(const float* y, const float* norm, const float* g, int C, int hw,
                                                       long long P, float* dx) {
  pdl_wait();
  pdl_trigger();
  const long long q = (long long)blockIdx.x * PT + threadIdx.x;
  if (q >= P) return;
  const long long b = q / hw;
  const long long o = b * C * hw + (q - b * hw);
  double s = 0.0;
  for (int c = 0; c < C; ++c) s += (double)y[o + (long long)c * hw] * g[o + (long long)c * hw];
  const float yg = (float)s, n = norm[q];
  for (int c = 0; c < C; ++c) {
    const long long i = o + (long long)c * hw;
    dx[i] = (g[i] - y[i] * yg) / n;
  }
}

// dx [B, C, hw] = sum_j dr[b, j, p] W[j, c]: one thread per element of dx
__global__ void __launch_bounds__(PT) ho_dx_kernel(const float* dr, const float* wt, int C, int k, int hw, long long n,
                                                   float* dx) {
  pdl_wait();
  pdl_trigger();
  const long long i = (long long)blockIdx.x * PT + threadIdx.x;
  if (i >= n) return;
  const long long chw = (long long)C * hw;
  const long long b = i / chw;
  const long long rem = i - b * chw;
  const int c = (int)(rem / hw), r = (int)(rem % hw);
  const float* d = dr + b * k * hw + r;
  float v = d[0] * wt[c];
  if (k == 2) v = fmaf(d[hw], wt[C + c], v);
  dx[i] = v;
}

// dW slot partials: block s covers pixels [s slot_px, (s+1) slot_px) of all B hw; warp v takes channels v, v+8, ...
// part[(s k + j) C + c] = sum over the slot of dr[j] x[c], lanes over pixels, shuffle-folded in a fixed order.
__global__ void __launch_bounds__(PT) ho_dw_partial_kernel(XView x, const float* dr, int C, int k, long long P,
                                                           int slot_px, double* part) {
  pdl_wait();
  pdl_trigger();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long q0 = (long long)blockIdx.x * slot_px;
  const long long q1 = min(P, q0 + slot_px);
  for (int c = warp; c < C; c += PT / 32) {
    double a0 = 0.0, a1 = 0.0;
    for (long long q = q0 + lane; q < q1; q += 32) {
      const long long b = q / x.hw;
      const long long dro = b * k * x.hw + (q - b * x.hw);
      const double v = x.p[x.base(q) + c * x.sc];
      a0 += (double)dr[dro] * v;
      if (k == 2) a1 += (double)dr[dro + x.hw] * v;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      a0 += __shfl_down_sync(0xffffffffu, a0, o);
      a1 += __shfl_down_sync(0xffffffffu, a1, o);
    }
    if (lane == 0) {
      part[((long long)blockIdx.x * k) * C + c] = a0;
      if (k == 2) part[((long long)blockIdx.x * k + 1) * C + c] = a1;
    }
  }
}

// dW[j, c] = the slots' partials folded in slot order
__global__ void __launch_bounds__(PT) ho_dw_fold_kernel(const double* part, int n, int slots, float* dw) {
  pdl_wait();
  pdl_trigger();
  const int i = blockIdx.x * PT + threadIdx.x;
  if (i >= n) return;
  double s = 0.0;
  for (int t = 0; t < slots; ++t) s += part[(long long)t * n + i];
  dw[i] = (float)s;
}

int outputs_of(int kind, int C) {
  return kind == MK_HO_OFFSET ? 2 : kind == MK_HO_DESC_L2 ? C : 1;
}

bool geometry_ok(int kind, int B, int h, int w, int C) {
  return kind >= MK_HO_SCORE_SOFTMAX && kind <= MK_HO_DESC_L2 && B >= 1 && h >= 1 && w >= 1 && C >= 1 && C <= MAX_C &&
         (long long)B * h * w <= MAX_PIXELS;
}

#define HO_GEOM_MSG "kind in [0, 5], B, h, w >= 1, B h w <= 2^26 and 1 <= C <= 4096"

int dw_slot_px(long long P) {
  const long long per = (P + MAX_SLOTS - 1) / MAX_SLOTS;
  return (int)std::max(256LL, (per + 31) / 32 * 32);
}

struct BwdLayout { size_t dr, part, total; int slots, slot_px; };

size_t align256(size_t v) { return (v + 255) & ~(size_t)255; }

BwdLayout bwd_layout(int kind, int B, int h, int w, int C) {
  BwdLayout L{};
  const long long P = (long long)B * h * w;
  if (kind == MK_HO_DESC_L2) return L;
  const int k = outputs_of(kind, C);
  L.slot_px = dw_slot_px(P);
  L.slots = (int)((P + L.slot_px - 1) / L.slot_px);
  L.dr = 0;
  L.part = align256((size_t)P * k * sizeof(float));
  L.total = L.part + (size_t)L.slots * k * C * sizeof(double);
  return L;
}

XView xview(const float* x, const long long* s, int h, int w) {
  return XView{x, s[0], s[1], s[2], s[3], h * w, w};
}

unsigned grid_of(long long n, int threads) { return (unsigned)((n + threads - 1) / threads); }

}  // namespace

}  // namespace mk

using namespace mk;

long long mk_head_out_backward_ws_bytes(int kind, int B, int h, int w, int C) {
  if (!geometry_ok(kind, B, h, w, C)) return -1;
  return (long long)bwd_layout(kind, B, h, w, C).total;
}

int mk_head_out_forward(int kind, const float* x, const long long* x_strides, int B, int C, int h, int w,
                        const float* weight, const float* eps, float temperature, float max_depth, float* out,
                        float* norm, void* stream) {
  if (!geometry_ok(kind, B, h, w, C) || !x || !x_strides || !out) {
    set_last_error("mk_head_out_forward: need x, its strides and out, %s (got kind %d B %d C %d h %d w %d)", HO_GEOM_MSG, kind,
                   B, C, h, w);
    return MK_ERR_INVALID;
  }
  const bool desc = kind == MK_HO_DESC_L2;
  if (desc == (weight != nullptr) || (kind == MK_HO_SCORE_SOFTMAX && (!eps || !(temperature > 0.f) || std::isinf(temperature))) ||
      (kind == MK_HO_DEPTH_SIGMOID && !std::isfinite(max_depth))) {
    set_last_error("mk_head_out_forward: kind %d needs %s", kind,
                   desc ? "no weight" : kind == MK_HO_SCORE_SOFTMAX ? "the weight, eps and a finite temperature > 0"
                                      : kind == MK_HO_DEPTH_SIGMOID ? "the weight and a finite max_depth" : "the weight");
    return MK_ERR_INVALID;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const long long P = (long long)B * h * w;
  const XView xv = xview(x, x_strides, h, w);
  if (kind == MK_HO_SCORE_SOFTMAX)
    MK_CUDA_CHECK(launch_k(ho_softmax_fwd_kernel, dim3(B), dim3(ST), 0, st, xv, weight, C, h, eps, temperature, out));
  else if (desc)
    MK_CUDA_CHECK(launch_k(ho_l2_fwd_kernel, dim3(grid_of(P, PT)), dim3(PT), 0, st, xv, C, P, out, norm));
  else
    MK_CUDA_CHECK(launch_k(ho_conv_act_kernel, dim3(grid_of(P, PT)), dim3(PT), 0, st, xv, weight, C, outputs_of(kind, C),
                           kind, h, max_depth, P, out));
  return MK_OK;
}

int mk_head_out_backward(int kind, const float* x, const long long* x_strides, int B, int C, int h, int w,
                         const float* weight, float temperature, float max_depth, const float* out, const float* norm,
                         const float* grad_out, float* grad_x, float* grad_w, void* ws, long long ws_bytes, void* stream) {
  if (!geometry_ok(kind, B, h, w, C) || !out || !grad_out) {
    set_last_error("mk_head_out_backward: need out and grad_out, %s (got kind %d B %d C %d h %d w %d)", HO_GEOM_MSG, kind, B,
                   C, h, w);
    return MK_ERR_INVALID;
  }
  const bool desc = kind == MK_HO_DESC_L2;
  if (desc ? (!norm || grad_w || weight)
           : (!weight || (grad_w && (!x || !x_strides)) || (kind == MK_HO_SCORE_SOFTMAX && (!(temperature > 0.f) ||
                                                                                           std::isinf(temperature))) ||
              (kind == MK_HO_DEPTH_SIGMOID && !(std::isfinite(max_depth) && max_depth != 0.f)))) {
    set_last_error("mk_head_out_backward: kind %d needs %s", kind,
                   desc ? "the saved norm and no weight or weight gradient"
                        : "the weight, x and its strides for a weight gradient, a finite temperature > 0 (softmax) and a "
                          "finite non-zero max_depth (depth sigmoid)");
    return MK_ERR_INVALID;
  }
  const BwdLayout L = bwd_layout(kind, B, h, w, C);
  if (!desc && (!ws || ws_bytes < (long long)L.total || ((uintptr_t)ws & 255))) {
    set_last_error("mk_head_out_backward: workspace of %lld bytes (256-byte aligned), %lld needed", ws_bytes,
                   (long long)L.total);
    return MK_ERR_INVALID;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const long long P = (long long)B * h * w;
  if (desc) {
    if (grad_x) MK_CUDA_CHECK(launch_k(ho_l2_bwd_kernel, dim3(grid_of(P, PT)), dim3(PT), 0, st, out, norm, grad_out, C, h * w,
                                       P, grad_x));
    return MK_OK;
  }
  if (!grad_x && !grad_w) return MK_OK;
  const int k = outputs_of(kind, C);
  float* dr = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(ws) + L.dr);
  double* part = reinterpret_cast<double*>(reinterpret_cast<uint8_t*>(ws) + L.part);
  if (kind == MK_HO_SCORE_SOFTMAX)
    MK_CUDA_CHECK(launch_k(ho_softmax_bwd_kernel, dim3(B), dim3(ST), 0, st, out, grad_out, h * w, temperature, dr));
  else
    MK_CUDA_CHECK(launch_k(ho_act_bwd_kernel, dim3(grid_of(P * k, PT)), dim3(PT), 0, st, out, grad_out, kind, h, w, h * w,
                           max_depth, P * k, dr));
  if (grad_x)
    MK_CUDA_CHECK(launch_k(ho_dx_kernel, dim3(grid_of(P * C, PT)), dim3(PT), 0, st, (const float*)dr, weight, C, k, h * w,
                           P * C, grad_x));
  if (grad_w) {
    MK_CUDA_CHECK(launch_k(ho_dw_partial_kernel, dim3(L.slots), dim3(PT), 0, st, xview(x, x_strides, h, w),
                           (const float*)dr, C, k, P, L.slot_px, part));
    MK_CUDA_CHECK(launch_k(ho_dw_fold_kernel, dim3(grid_of(k * C, PT)), dim3(PT), 0, st, (const double*)part, k * C, L.slots,
                           grad_w));
  }
  return MK_OK;
}
