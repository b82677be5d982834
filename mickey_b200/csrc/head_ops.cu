// Non-GEMM kernels of the four MicKey heads: linear-attention reductions, output activations,
// descriptor normalisation / packing for the matcher.
//
// Token layout in the heads: every image is a zero-padded NHWC grid [(gh+2), (gw+2), C] flattened to rows
// ("padded positions"); R = n_img * (gh+2) * (gw+2) rows in total.  Pad rows are zero wherever a 3x3
// convolution reads them and are excluded from every reduction below.
#include "ops.h"

namespace mk {

__device__ __forceinline__ bool pos_valid(int pos, int h2, int w2, int& y, int& x) {
  y = pos / w2; x = pos % w2;
  return y >= 1 && y <= h2 - 2 && x >= 1 && x <= w2 - 2;
}
__device__ __forceinline__ float elu1(float v) { return v > 0.f ? v + 1.0f : expf(v); }   // elu(v) + 1

// ------------------------------------------------------------------------------------------------------
// Linear attention, reduction half (reference att_layers/attention.py:55-61):
//   K = elu(k)+1;  KV[h] = sum_s K[s,h,:]^T (v[s,h,:] / L);  Ksum[h] = sum_s K[s,h,:]
// qkv fp32 [R, G*384] (q|k|v per group, 8 heads x 16).  Each CTA writes the partial sums of its 32-row chunk to
// part[n_img, G, chunk, 8, 272]; linattn_kv_reduce_kernel adds the chunks in a fixed order (bit-reproducible,
// no float atomics) into out fp32 [n_img, G, 8, 272] (256 KV + 16 Ksum).
// grid (row chunks of 32, G, n_img), 256 threads: thread t owns head h = t/32, key dim d = (t%32)/2 and eight
// value dims; the chunk's k and v rows of all 8 heads are staged in shared memory once.
// ------------------------------------------------------------------------------------------------------
constexpr int KV_ROWS = 32;
__global__ void __launch_bounds__(256)
linattn_kv_kernel(const float* __restrict__ qkv, float* __restrict__ kvout, int G, int h2, int w2) {
  pdl_wait();        // launched with programmatic stream serialization: predecessors are complete past this point
  pdl_trigger();
  __shared__ float Ks[KV_ROWS][128 + 4];
  __shared__ float Vs[KV_ROWS][128 + 4];
  const int g = blockIdx.y, im = blockIdx.z;
  const int per_img = h2 * w2;
  const float inv_len = 1.0f / (float)((h2 - 2) * (w2 - 2));
  const int t = threadIdx.x;
  const long long ld = (long long)G * 384;
  const float* base = qkv + (long long)im * per_img * ld + g * 384;
  const int r0 = blockIdx.x * KV_ROWS;
  // 32 rows x (128 k + 128 v) floats = 2048 float4 over 256 threads
  for (int i = t; i < KV_ROWS * 64; i += 256) {
    const int r = i >> 6, c4 = i & 63;           // c4 < 32: k, else v
    const int pos = r0 + r;
    int y, x;
    float4 val = make_float4(0.f, 0.f, 0.f, 0.f);
    if (pos < per_img && pos_valid(pos, h2, w2, y, x)) {
      val = *reinterpret_cast<const float4*>(base + (long long)pos * ld + 128 + c4 * 4);
      if (c4 < 32) { val.x = elu1(val.x); val.y = elu1(val.y); val.z = elu1(val.z); val.w = elu1(val.w); }
      else { val.x *= inv_len; val.y *= inv_len; val.z *= inv_len; val.w *= inv_len; }
    }
    float* dst = (c4 < 32) ? &Ks[r][c4 * 4] : &Vs[r][(c4 - 32) * 4];
    dst[0] = val.x; dst[1] = val.y; dst[2] = val.z; dst[3] = val.w;
  }
  __syncthreads();
  const int head = t >> 5, d = (t & 31) >> 1, vh = (t & 1) * 8;
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  float ksum = 0.f;
#pragma unroll 4
  for (int r = 0; r < KV_ROWS; ++r) {
    const float kk = Ks[r][head * 16 + d];
    ksum += kk;
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = fmaf(kk, Vs[r][head * 16 + vh + j], acc[j]);
  }
  float* o = kvout + ((((long long)im * G + g) * gridDim.x + blockIdx.x) * 8 + head) * 272;
#pragma unroll
  for (int j = 0; j < 8; ++j) o[d * 16 + vh + j] = acc[j];
  if (vh == 0) o[256 + d] = ksum;
}

// out[i] = sum_c part[c][i] over the row chunks in a fixed order: four lanes per output element each add a contiguous
// quarter of the chunks (8 loads in flight), then the quarters are added in lane order -- the result depends only on
// `chunks`.  grid (ceil(2176/32), G, n_img), 128 threads.
__global__ void __launch_bounds__(128)
linattn_kv_reduce_kernel(const float* __restrict__ part, float* __restrict__ out, int G, int chunks) {
  pdl_wait();        // launched with programmatic stream serialization: predecessors are complete past this point
  pdl_trigger();
  const int g = blockIdx.y, im = blockIdx.z;
  const int i = blockIdx.x * 32 + (threadIdx.x >> 2), quarter = threadIdx.x & 3;
  const bool live = i < 8 * 272;
  const int per = (chunks + 3) >> 2;
  const int c0 = quarter * per, c1 = min(chunks, c0 + per);
  const float* src = part + ((long long)im * G + g) * chunks * (8 * 272) + (live ? i : 0);
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  int c = c0;
  if (live) {
    for (; c + 8 <= c1; c += 8) {
#pragma unroll
      for (int k = 0; k < 8; ++k) acc[k] += src[(long long)(c + k) * (8 * 272)];
    }
    for (; c < c1; ++c) acc[0] += src[(long long)c * (8 * 272)];
  }
  float v = ((acc[0] + acc[1]) + (acc[2] + acc[3])) + ((acc[4] + acc[5]) + (acc[6] + acc[7]));
  const float v1 = __shfl_down_sync(0xffffffffu, v, 1), v2 = __shfl_down_sync(0xffffffffu, v, 2), v3 = __shfl_down_sync(0xffffffffu, v, 3);
  if (live && quarter == 0) out[((long long)im * G + g) * (8 * 272) + i] = (v + v1) + (v2 + v3);
}

// Linear attention, query half (attention.py:52,60-61): msg = (Q KV) / (Q . Ksum + eps) * L, Q = elu(q)+1.
// msg fp16 [R, G*128].  grid (ceil(per_img/32), G, n_img), 256 threads = 32 rows x 8 heads.
__global__ void __launch_bounds__(256)
linattn_msg_kernel(const float* __restrict__ qkv, const float* __restrict__ kv, __half* __restrict__ msg, int G, int h2,
                   int w2, float eps) {
  pdl_wait();        // launched with programmatic stream serialization: predecessors are complete past this point
  pdl_trigger();
  // a warp reads KVs[head][..] for its 8 heads at once (4 positions share each address): a row stride of 272 floats
  // puts heads 0/2/4/6 in the same bank (4-way conflict on all 272 reads per thread); 276 = 4 mod 32 spreads them
  __shared__ float KVs[8][276];
  const int g = blockIdx.y, im = blockIdx.z, t = threadIdx.x;
  const int per_img = h2 * w2;
  const float len = (float)((h2 - 2) * (w2 - 2));
  const float* kvsrc = kv + ((long long)im * G + g) * 8 * 272;
  for (int i = t; i < 8 * 272; i += 256) KVs[i / 272][i % 272] = kvsrc[i];
  __syncthreads();
  const int pos = blockIdx.x * 32 + (t >> 3), head = t & 7;
  if (pos >= per_img) return;
  const long long row = (long long)im * per_img + pos;
  const float* q = qkv + row * ((long long)G * 384) + g * 384 + head * 16;
  float Q[16];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float4 f = reinterpret_cast<const float4*>(q)[i];
    Q[i * 4 + 0] = elu1(f.x); Q[i * 4 + 1] = elu1(f.y); Q[i * 4 + 2] = elu1(f.z); Q[i * 4 + 3] = elu1(f.w);
  }
  float den = eps;
#pragma unroll
  for (int dd = 0; dd < 16; ++dd) den = fmaf(Q[dd], KVs[head][256 + dd], den);
  const float z = len / den;
  float o[16];
#pragma unroll
  for (int v = 0; v < 16; ++v) {
    float a = 0.f;
#pragma unroll
    for (int dd = 0; dd < 16; ++dd) a = fmaf(Q[dd], KVs[head][dd * 16 + v], a);
    o[v] = a * z;
  }
  __half* dst = msg + row * ((long long)G * 128) + g * 128 + head * 16;
  uint4 u0, u1;
  __half2 h;
#define MK_PK(U, A, B) h = __floats2half2_rn(A, B); U = *reinterpret_cast<uint32_t*>(&h);
  MK_PK(u0.x, o[0], o[1]) MK_PK(u0.y, o[2], o[3]) MK_PK(u0.z, o[4], o[5]) MK_PK(u0.w, o[6], o[7])
  MK_PK(u1.x, o[8], o[9]) MK_PK(u1.y, o[10], o[11]) MK_PK(u1.z, o[12], o[13]) MK_PK(u1.w, o[14], o[15])
#undef MK_PK
  reinterpret_cast<uint4*>(dst)[0] = u0;
  reinterpret_cast<uint4*>(dst)[1] = u1;
}

int linattn_kv_chunks(int h2, int w2) { return ceil_div(h2 * w2, KV_ROWS); }

int linattn_kv(const float* qkv, float* kv_part, float* kv, int n_img, int G, int h2, int w2, cudaStream_t s) {
  const int chunks = linattn_kv_chunks(h2, w2);
  MK_CUDA_CHECK(launch_k(linattn_kv_kernel, dim3(chunks, G, n_img), dim3(256), 0, s, qkv, kv_part, G, h2, w2));
  MK_CUDA_CHECK(cudaGetLastError());
  MK_CUDA_CHECK(launch_k(linattn_kv_reduce_kernel, dim3(ceil_div(8 * 272, 32), G, n_img), dim3(128), 0, s, kv_part, kv, G, chunks));
  MK_CUDA_CHECK(cudaGetLastError());
  return MK_OK;
}
int linattn_msg(const float* qkv, const float* kv, void* msg, int n_img, int G, int h2, int w2, float eps, cudaStream_t s) {
  MK_CUDA_CHECK(launch_k(linattn_msg_kernel, dim3(ceil_div(h2 * w2, 32), G, n_img), dim3(256), 0, s, qkv, kv, (__half*)msg, G, h2, w2, eps));
  MK_CUDA_CHECK(cudaGetLastError());
  return MK_OK;
}

// ------------------------------------------------------------------------------------------------------
// Keypoint-head outputs (reference mickey_extractor.py:134,172-176,211-216 + compute_correspondences.py:20-31):
//   y fp32 [R, 3*64]  (resblock4 outputs of depth_head | det_offset | det_head)
//   depth[img, n]    = w_depth . y_depth            (or MAX_DEPTH * sigmoid(.))
//   kps[img, 0/1, n] = (sigmoid(w_xy . y_off) + (x, y)) * down_factor
//   score_raw[img, n] = w_score . y_det
// one warp per valid token.
// ------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
kp_head_out_kernel(const float* __restrict__ y, const float* __restrict__ w_depth, const float* __restrict__ w_xy,
                   const float* __restrict__ w_score, float* __restrict__ depth, float* __restrict__ kps,
                   float* __restrict__ score_raw, int n_img, int gh, int gw, int depth_sigmoid, float max_depth,
                   float down_factor) {
  pdl_wait();        // launched with programmatic stream serialization: predecessors are complete past this point
  pdl_trigger();
  const int tok = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  const int N = gh * gw;
  if (tok >= n_img * N) return;
  const int im = tok / N, n = tok % N, yy = n / gw, xx = n % gw;
  const long long row = ((long long)im * (gh + 2) + yy + 1) * (gw + 2) + xx + 1;
  const float* r = y + row * 192;
  float a_d = r[lane] * w_depth[lane] + r[lane + 32] * w_depth[lane + 32];
  float a_x = r[64 + lane] * w_xy[lane] + r[96 + lane] * w_xy[lane + 32];
  float a_y = r[64 + lane] * w_xy[64 + lane] + r[96 + lane] * w_xy[96 + lane];
  float a_s = r[128 + lane] * w_score[lane] + r[160 + lane] * w_score[lane + 32];
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    a_d += __shfl_xor_sync(0xffffffffu, a_d, o);
    a_x += __shfl_xor_sync(0xffffffffu, a_x, o);
    a_y += __shfl_xor_sync(0xffffffffu, a_y, o);
    a_s += __shfl_xor_sync(0xffffffffu, a_s, o);
  }
  if (lane == 0) {
    depth[(long long)im * N + n] = depth_sigmoid ? max_depth / (1.0f + expf(-a_d)) : a_d;
    kps[((long long)im * 2 + 0) * N + n] = (1.0f / (1.0f + expf(-a_x)) + (float)xx) * down_factor;
    kps[((long long)im * 2 + 1) * N + n] = (1.0f / (1.0f + expf(-a_y)) + (float)yy) * down_factor;
    score_raw[(long long)im * N + n] = a_s;
  }
}

// Score activation (mickey_extractor.py:98-124,137-142): spatial softmax with temperature 100 over the
// map minus its mean, 3-pixel border zeroed, normalised by (sum + 1e-16); or sigmoid * border mask.
// one block per image.
__global__ void __launch_bounds__(256)
score_activation_kernel(const float* __restrict__ raw, float* __restrict__ scr, int gh, int gw, int use_softmax,
                        int border, float temp, float eps) {
  pdl_wait();        // launched with programmatic stream serialization: predecessors are complete past this point
  pdl_trigger();
  __shared__ float red[256];
  const int im = blockIdx.x, N = gh * gw, t = threadIdx.x;
  const float* r = raw + (long long)im * N;
  float* o = scr + (long long)im * N;
  auto inside = [&](int n) {
    const int y = n / gw, x = n % gw;
    return y >= border && y < gh - border && x >= border && x < gw - border;
  };
  if (!use_softmax) {
    for (int n = t; n < N; n += 256) o[n] = inside(n) ? 1.0f / (1.0f + expf(-r[n])) : 0.0f;
    return;
  }
  float s = 0.f;
  for (int n = t; n < N; n += 256) s += r[n];
  red[t] = s;
  __syncthreads();
  for (int k = 128; k; k >>= 1) { if (t < k) red[t] += red[t + k]; __syncthreads(); }
  const float mean = red[0] / N + eps;
  __syncthreads();
  float e = 0.f;
  for (int n = t; n < N; n += 256) {
    const float v = inside(n) ? expf((r[n] - mean) / temp) : 0.0f;
    o[n] = v;
    e += v;
  }
  red[t] = e;
  __syncthreads();
  for (int k = 128; k; k >>= 1) { if (t < k) red[t] += red[t + k]; __syncthreads(); }
  const float inv = 1.0f / (red[0] + eps);
  for (int n = t; n < N; n += 256) o[n] *= inv;
}

int kp_head_out(const float* y, const float* w_depth, const float* w_xy, const float* w_score, float* depth, float* kps,
                float* score_raw, float* scr, int n_img, int gh, int gw, int depth_sigmoid, float max_depth,
                float down_factor, int use_softmax, cudaStream_t s) {
  MK_CUDA_CHECK(launch_k(kp_head_out_kernel, dim3(ceil_div(n_img * gh * gw, 8)), dim3(256), 0, s, y, w_depth, w_xy, w_score, depth, kps, score_raw, n_img,
                                                                    gh, gw, depth_sigmoid, max_depth, down_factor));
  MK_CUDA_CHECK(cudaGetLastError());
  MK_CUDA_CHECK(launch_k(score_activation_kernel, dim3(n_img), dim3(256), 0, s, score_raw, scr, gh, gw, use_softmax, 3, 100.0f, 1e-16f));
  MK_CUDA_CHECK(cudaGetLastError());
  return MK_OK;
}

// ------------------------------------------------------------------------------------------------------
// Descriptor output (mickey_extractor.py:246-249, extractor_utils.py:6-10): d / sqrt(sum d^2 + 1e-10).
//   y fp32 [R, 128] -> dsc_cm fp32 [n_img, 128, N]   (the data-dict layout of the reference)
//                   -> dsc_x  fp16 [n_img, N, 384]   (matcher operand: fp32 value split as hi + lo fp16;
//                      role 0 images store [hi | lo | hi], role 1 images [hi | hi | lo], so
//                      that one K=384 fp16 GEMM yields hi0.hi1 + lo0.hi1 + hi0.lo1 ~ fp32 dot product)
//                   -> nrm2 fp32 [n_img, N]  squared norm of the stored descriptor
// role < 0: an image's role is its half of the batch (img < n_img/2: role 0), as mk_forward extracts image0 then image1;
// role 0 / 1: every image takes that role (mk_localize extracts only queries).  dsc_cm == NULL: no fp32 copy.
// one warp per valid token, 4 channels per lane.
// ------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
desc_out_kernel(const float* __restrict__ y, float* __restrict__ dsc_cm, __half* __restrict__ dsc_x,
                float* __restrict__ nrm2, int n_img, int gh, int gw, int normalize, int role) {
  pdl_wait();        // launched with programmatic stream serialization: predecessors are complete past this point
  pdl_trigger();
  const int tok = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  const int N = gh * gw;
  if (tok >= n_img * N) return;
  const int im = tok / N, n = tok % N, yy = n / gw, xx = n % gw;
  const long long row = ((long long)im * (gh + 2) + yy + 1) * (gw + 2) + xx + 1;
  float4 v = reinterpret_cast<const float4*>(y + row * 128)[lane];
  float ss = v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
#pragma unroll
  for (int o = 16; o; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  float n2 = ss;
  if (normalize) {
    const float inv = 1.0f / sqrtf(ss + 1e-10f);
    v.x *= inv; v.y *= inv; v.z *= inv; v.w *= inv;
    n2 = ss * inv * inv;
  }
  if (lane == 0) nrm2[(long long)im * N + n] = n2;
  const float vals[4] = {v.x, v.y, v.z, v.w};
  __half hi[4], lo[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    if (dsc_cm) dsc_cm[((long long)im * 128 + lane * 4 + i) * N + n] = vals[i];
    hi[i] = __float2half_rn(vals[i]);
    lo[i] = __float2half_rn(vals[i] - __half2float(hi[i]));
  }
  const bool role1 = role < 0 ? im >= n_img / 2 : role == 1;
  __half* dst = dsc_x + ((long long)im * N + n) * 384 + lane * 4;
  uint2 uh, ul;
  uh.x = (uint32_t)__half_as_ushort(hi[0]) | ((uint32_t)__half_as_ushort(hi[1]) << 16);
  uh.y = (uint32_t)__half_as_ushort(hi[2]) | ((uint32_t)__half_as_ushort(hi[3]) << 16);
  ul.x = (uint32_t)__half_as_ushort(lo[0]) | ((uint32_t)__half_as_ushort(lo[1]) << 16);
  ul.y = (uint32_t)__half_as_ushort(lo[2]) | ((uint32_t)__half_as_ushort(lo[3]) << 16);
  *reinterpret_cast<uint2*>(dst) = uh;
  *reinterpret_cast<uint2*>(dst + 128) = role1 ? uh : ul;
  *reinterpret_cast<uint2*>(dst + 256) = role1 ? ul : uh;
}

int desc_out(const float* y, float* dsc_cm, void* dsc_x, float* nrm2, int n_img, int gh, int gw, int normalize, int role,
             cudaStream_t s) {
  MK_CUDA_CHECK(launch_k(desc_out_kernel, dim3(ceil_div(n_img * gh * gw, 8)), dim3(256), 0, s, y, dsc_cm, (__half*)dsc_x, nrm2, n_img, gh, gw,
                         normalize, role));
  MK_CUDA_CHECK(cudaGetLastError());
  return MK_OK;
}

// ------------------------------------------------------------------------------------------------------
// Feature-bank gather (mk_forward_pairs, mk_localize): the per-pair operands of the matcher and the solver, taken from
// banks of extracted images.  Block (x, p, r): tokens [32x, 32x + 32) of pair p in role r; its image is idx_r[p] of bank
// r.  mk_forward_pairs launches both roles; mk_localize only role 0 (grid z = 1), since it extracts the role-1 queries.
//   dsc  fp32 [n, 128, N] channel-major -> dsc_x fp16 [(r*P + p)*N + tok, 384], split exactly as desc_out_kernel does
//   kps [n,2,N], depth [n,1,N], scr [n,1,N] -> kps_out [2P,2,N], depth_out [2P,1,N], scr_out [2P,N]  (role-0 rows first)
// The descriptor tile is transposed through shared memory: each warp reads 128-byte runs of 32 tokens of one channel and
// writes 128-byte runs of 64 channels of one token.  An index outside [0, count) reads nothing from the bank and writes
// zeros (bank_index_check reports it after the solve).
// ------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
bank_gather_kernel(BankView b0, BankView b1, int P, int N, __half* __restrict__ dsc_x, float* __restrict__ kps_out,
                   float* __restrict__ depth_out, float* __restrict__ scr_out) {
  __shared__ float tile[128][33];
  pdl_wait();        // launched with programmatic stream serialization: predecessors are complete past this point
  pdl_trigger();
  const int r = blockIdx.z, p = blockIdx.y, n0 = blockIdx.x * 32, t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const BankView b = r ? b1 : b0;
  const int img = __ldg(b.idx + p);
  const bool ok = img >= 0 && img < b.count;
  const long long im = ok ? img : 0, orow = (long long)r * P + p;
  if (t < 128) {                                       // warp 0, 1: kps x, y; warp 2: depth; warp 3: scr
    const int n = n0 + lane;
    if (n < N) {
      const float* src = warp < 2 ? b.kps + (im * 2 + warp) * N : (warp == 2 ? b.depth : b.scr) + im * N;
      const float v = ok ? __ldg(src + n) : 0.f;
      float* dst = warp < 2 ? kps_out + (orow * 2 + warp) * N : (warp == 2 ? depth_out : scr_out) + orow * N;
      dst[n] = v;
    }
  }
  const float* src = b.dsc + im * 128 * N;
#pragma unroll
  for (int k = 0; k < 16; ++k) {
    const int c = warp + 8 * k, n = n0 + lane;
    tile[c][lane] = (ok && n < N) ? __ldg(src + (long long)c * N + n) : 0.f;
  }
  __syncthreads();
  for (int j = warp; j < 32 && n0 + j < N; j += 8) {
    __half* dst = dsc_x + (orow * N + n0 + j) * 384;
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      const int c = 64 * half + 2 * lane;
      const float v0 = tile[c][j], v1 = tile[c + 1][j];
      const __half h0 = __float2half_rn(v0), h1 = __float2half_rn(v1);
      const __half2 hi = __halves2half2(h0, h1);
      const __half2 lo = __halves2half2(__float2half_rn(v0 - __half2float(h0)), __float2half_rn(v1 - __half2float(h1)));
      *reinterpret_cast<__half2*>(dst + c) = hi;
      *reinterpret_cast<__half2*>(dst + 128 + c) = r ? hi : lo;      // role 0 [hi | lo | hi], role 1 [hi | hi | lo]
      *reinterpret_cast<__half2*>(dst + 256 + c) = r ? lo : hi;
    }
  }
}

int bank_gather(const BankView& b0, const BankView& b1, int P, int N, void* dsc_x, float* kps_out, float* depth_out, float* scr_out,
                int n_roles, cudaStream_t s) {
  MK_CUDA_CHECK(launch_k(bank_gather_kernel, dim3(ceil_div(N, 32), P, n_roles), dim3(256), 0, s, b0, b1, P, N, (__half*)dsc_x, kps_out,
                         depth_out, scr_out));
  MK_CUDA_CHECK(cudaGetLastError());
  return MK_OK;
}

// After the solve of mk_forward_pairs: an index outside its bank gives the batch the zero pose of the solver's status bits
// (R = 0, t = 0, inliers = 0) and sets status bit 3.  One block; it reads only the index vectors.
__global__ void __launch_bounds__(256)
bank_index_check_kernel(const int* __restrict__ idx0, int n0, const int* __restrict__ idx1, int n1, int P, float* __restrict__ pose,
                        int* __restrict__ status) {
  pdl_wait();
  pdl_trigger();
  int bad = 0;
  for (int p = threadIdx.x; p < P; p += blockDim.x) {
    const int a = __ldg(idx0 + p), b = __ldg(idx1 + p);
    bad |= (a < 0 || a >= n0 || b < 0 || b >= n1);
  }
  if (!__syncthreads_or(bad)) return;
  for (int i = threadIdx.x; i < P * 13; i += blockDim.x) pose[i] = 0.f;
  if (status && threadIdx.x == 0) *status |= 8;
}

int bank_index_check(const BankView& b0, const BankView& b1, int P, float* pose, int* status, cudaStream_t s) {
  MK_CUDA_CHECK(launch_k(bank_index_check_kernel, dim3(1), dim3(256), 0, s, b0.idx, b0.count, b1.idx, b1.count, P, pose, status));
  MK_CUDA_CHECK(cudaGetLastError());
  return MK_OK;
}

// Fold the online-softmax partials of matcher pass 1 (EPI_LSE: float2 (max, sum) per slot, slot-major) and the dustbin
// logit into the log2-domain log-sum-exp of every row and column of the dustbin-augmented S/T
// (feature_matcher.py:70-77: the dustbin score is appended AFTER the division by the temperature).
// grid = (ceil(N / 256), B, 2): z = 0 rows, z = 1 columns.  One thread per row/column; consecutive threads read
// consecutive float2 of a slot (coalesced); the slots are combined in index order (bit-reproducible).
__global__ void __launch_bounds__(256)
matcher_lse_reduce_kernel(const float2* __restrict__ part_row, const float2* __restrict__ part_col, const float* __restrict__ dustbin,
                          int N, int part_ld, float* __restrict__ lse_r, float* __restrict__ lse_c) {
  pdl_wait();        // launched with programmatic stream serialization: predecessors are complete past this point
  pdl_trigger();
  const int i = blockIdx.x * 256 + threadIdx.x, b = blockIdx.y, which = blockIdx.z;
  if (i >= N) return;
  const int slots = which ? part_ld / 32 : part_ld / 64;
  const float2* src = (which ? part_col : part_row) + (size_t)b * slots * part_ld + i;
  const float NEG_INF = __int_as_float(0xff800000);
  float M = dustbin ? __ldg(dustbin) * 1.4426950408889634f : NEG_INF;
  float S = dustbin ? 1.0f : 0.0f;
  for (int s0 = 0; s0 < slots; s0 += 8) {
    float2 v[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) v[k] = (s0 + k < slots) ? __ldg(src + (size_t)(s0 + k) * part_ld) : make_float2(NEG_INF, 0.f);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      if (v[k].x == NEG_INF) continue;               // a slot without a valid cell
      const float nm = fmaxf(M, v[k].x);
      S = S * exp2f(M - nm) + v[k].y * exp2f(v[k].x - nm);
      M = nm;
    }
  }
  (which ? lse_c : lse_r)[(size_t)b * part_ld + i] = M + log2f(S);
}

int matcher_lse_reduce(const void* part_row, const void* part_col, const float* dustbin, int B, int N, int part_ld, float* lse_r,
                       float* lse_c, cudaStream_t s) {
  MK_CUDA_CHECK(launch_k(matcher_lse_reduce_kernel, dim3((N + 255) / 256, B, 2), dim3(256), 0, s, reinterpret_cast<const float2*>(part_row),
                         reinterpret_cast<const float2*>(part_col), dustbin, N, part_ld, lse_r, lse_c));
  MK_CUDA_CHECK(cudaGetLastError());
  return MK_OK;
}

}  // namespace mk
