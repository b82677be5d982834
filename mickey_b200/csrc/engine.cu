// The C ABI (include/mickey_b200.h): handle, packed-weight registry, workspace carving and the kernel
// sequence of the three stages (extract -> match -> solve).
#include "../../include/mickey_b200.h"
#include "gemm.h"
#include "ops.h"

#include <algorithm>
#include <cfloat>
#include <cstring>
#include <string>
#include <unordered_map>
#include <vector>

using namespace mk;

struct Tensor { const void* ptr; int dtype; long long numel; };

struct mk_handle {
  int device;
  mk_config cfg;
  std::unordered_map<std::string, Tensor> tensors;
  int geo_h = 0, geo_w = 0;
  bool finalized = false;
  unsigned long long* seed_dev = nullptr;   // RNG state of the solver (device memory, advanced after every solve)
  long long launches = 0;
  // optional per-kernel-class timing with CUDA events on the launch stream (mk_profile_*)
  bool profiling = false;
  struct ProfRec { std::string tag; cudaEvent_t e0, e1; };
  std::vector<ProfRec> prof;
};

namespace {

// n_img: images one call extracts; n_pairs: pairs it matches and solves.  mk_forward and its stages: (2P, P);
// mk_extract_images: (n, 0); mk_forward_pairs: (0, P); mk_localize: (P, P), the P images being the role-1 queries.
struct Geo {
  int H, W, gh, gw, N, T, h2, w2, per_img, n_img, n_pairs;
  long long M, Mp, R;
};

Geo make_geo(int n_img, int n_pairs, int H, int W) {
  Geo g;
  g.H = H; g.W = W; g.gh = H / 14; g.gw = W / 14;
  g.N = g.gh * g.gw; g.T = g.N + 1; g.h2 = g.gh + 2; g.w2 = g.gw + 2; g.per_img = g.h2 * g.w2;
  g.n_img = n_img; g.n_pairs = n_pairs;
  g.M = (long long)g.n_img * g.T; g.Mp = (long long)g.n_img * g.N; g.R = (long long)g.n_img * g.per_img;
  return g;
}

constexpr int KPAD = 640;       // 3*14*14 = 588 padded to a multiple of 64
constexpr int G = 4;            // heads: depth_head, det_offset, det_head, dsc_head

// Bump allocator over the caller's workspace; with base == nullptr it only measures.
struct Carver {
  uint8_t* base; size_t off = 0;
  explicit Carver(void* b) : base(reinterpret_cast<uint8_t*>(b)) {}
  template <typename T> T* take(size_t count) {
    off = (off + 255) & ~(size_t)255;
    T* p = base ? reinterpret_cast<T*>(base + off) : nullptr;
    off += count * sizeof(T);
    return p;
  }
};

// The solver's scratch: the sampler's histogram and candidates, the drawn cells, every hypothesis's score and [R | t],
// the status word with the fused kernel's completion counters, and the winning hypothesis of each pair.
struct SolverWs { void* samp_ws; int* idx; float* hyp_scores; float* hyp_Rt; int* status; int* best_hyp; };

// Carved last in the handle's workspace (mk_solve_pose, mk_forward*) and alone in mk_procrustes_solve's.
void carve_solver(Carver& cv, int n_pairs, int it_matches, int it_ransac, int num_sampled, SolverWs& s) {
  const size_t streams = (size_t)n_pairs * it_matches;
  s.samp_ws = cv.take<uint8_t>(sampler_workspace_bytes(n_pairs, it_matches));
  s.idx = cv.take<int>(streams * num_sampled);
  s.hyp_scores = cv.take<float>(streams * it_ransac);
  s.hyp_Rt = cv.take<float>(streams * it_ransac * 12);
  s.status = cv.take<int>(SOLVER_COUNTER_BASE + n_pairs);     // status bits + the fused solver's completion counters
  s.best_hyp = cv.take<int>(n_pairs);
}

struct Workspace {
  // backbone
  __half* P; float* X; __half* XN; __half* QKV; __half* ATT; __half* H1;
  // heads
  __half* F; __half *T1, *S1, *O1, *T2, *S2, *O2, *T3, *S3, *CAT, *MSG, *HM, *T4k, *S4k, *T4d;
  float *X32, *QKV32, *KV, *KVP, *Y4k, *Y4d;
  // head outputs kept for the matcher
  float* score_raw; __half* DSCX; float* nrm2; float* scr_copy;
  // matcher
  float *part_row, *part_col, *lse_r, *lse_c;
  SolverWs sol;
  size_t bytes;
};

// The backbone's six buffers open every workspace, so a backbone-only call (mk_backbone_features) carves just them and
// they sit at the same offsets as in the full workspace of the same image count.
void carve_backbone(Carver& cv, const mk_config& c, const Geo& g, Workspace& w) {
  const size_t D = c.embed_dim, M = g.M;
  w.P = cv.take<__half>((size_t)g.Mp * KPAD);
  w.X = cv.take<float>(M * D);
  w.XN = cv.take<__half>(M * D);
  w.QKV = cv.take<__half>(M * 3 * D);
  w.ATT = cv.take<__half>(M * D);
  w.H1 = cv.take<__half>(M * 4 * D);
}

size_t backbone_ws_bytes(const mk_config& c, const Geo& g) {
  Carver cv(nullptr);
  Workspace w;
  carve_backbone(cv, c, g, w);
  return (cv.off + 255) & ~(size_t)255;
}

Workspace carve(void* base, const mk_config& c, const Geo& g) {
  Workspace w;
  Carver cv(base);
  const int n_pairs = g.n_pairs;
  const size_t D = c.embed_dim, R = g.R;
  // the matcher's operands: written by the extraction (n_img images), by the bank gather (2 * n_pairs role rows) or by
  // both (mk_localize: the gather fills the n_pairs role-0 rows, the extraction of n_img = n_pairs queries the role-1 rows)
  const size_t n_op = (size_t)std::max(g.n_img, 2 * g.n_pairs);
  const int* bd = c.block_dims;
  carve_backbone(cv, c, g, w);
  w.F = cv.take<__half>(R * D);
  w.T1 = cv.take<__half>(R * G * bd[0]); w.S1 = cv.take<__half>(R * G * bd[0]); w.O1 = cv.take<__half>(R * G * bd[0]);
  w.T2 = cv.take<__half>(R * G * bd[1]); w.S2 = cv.take<__half>(R * G * bd[1]); w.O2 = cv.take<__half>(R * G * bd[1]);
  w.T3 = cv.take<__half>(R * G * bd[2]); w.S3 = cv.take<__half>(R * G * bd[2]);
  w.CAT = cv.take<__half>(R * G * 256); w.MSG = cv.take<__half>(R * G * 128); w.HM = cv.take<__half>(R * G * 256);
  w.T4k = cv.take<__half>(R * 3 * bd[3]); w.S4k = cv.take<__half>(R * 3 * bd[3]); w.T4d = cv.take<__half>(R * c.desc_dim);
  w.X32 = cv.take<float>(R * G * 128); w.QKV32 = cv.take<float>(R * G * 384);
  w.KV = cv.take<float>((size_t)g.n_img * G * 8 * 272);
  w.KVP = cv.take<float>((size_t)g.n_img * G * linattn_kv_chunks(g.h2, g.w2) * 8 * 272);
  w.Y4k = cv.take<float>(R * 3 * bd[3]); w.Y4d = cv.take<float>(R * c.desc_dim);
  w.score_raw = cv.take<float>((size_t)g.n_img * g.N);
  w.DSCX = cv.take<__half>(n_op * g.N * 384);
  w.nrm2 = cv.take<float>((size_t)g.n_img * g.N);
  w.scr_copy = cv.take<float>(n_op * g.N);
  const size_t npad = (size_t)ceil_div(g.N, 128) * 128;          // matcher: float2 partials [pair][slot][npad], lse vectors [pair][npad]
  w.part_row = cv.take<float>((size_t)n_pairs * (npad / 64) * npad * 2); w.part_col = cv.take<float>((size_t)n_pairs * (npad / 32) * npad * 2);
  w.lse_r = cv.take<float>((size_t)n_pairs * npad); w.lse_c = cv.take<float>((size_t)n_pairs * npad);
  carve_solver(cv, n_pairs, c.it_matches, c.it_ransac, c.num_sampled, w.sol);
  w.bytes = cv.off + 256;
  return w;
}

// ---- weight lookup ---------------------------------------------------------------------------------------
struct Lookup {
  mk_handle* h; bool ok = true;
  const void* get(const std::string& name, int dtype, long long numel) {
    auto it = h->tensors.find(name);
    if (it == h->tensors.end()) { set_last_error("missing tensor '%s'", name.c_str()); ok = false; return nullptr; }
    if (it->second.dtype != dtype || it->second.numel != numel) {
      set_last_error("tensor '%s': expected dtype %d numel %lld, got dtype %d numel %lld", name.c_str(), dtype, numel,
                     it->second.dtype, it->second.numel);
      ok = false; return nullptr;
    }
    return it->second.ptr;
  }
  const float* f(const std::string& n, long long numel) { return reinterpret_cast<const float*>(get(n, 0, numel)); }
  const __half* hh(const std::string& n, long long numel) { return reinterpret_cast<const __half*>(get(n, 1, numel)); }
};

GemmParams base_params(long long M, int N, int K) {
  GemmParams p;
  memset(&p, 0, sizeof(p));
  p.M = (int)M; p.N = N; p.k_chunks = K / 64; p.chunks_per_tap = p.k_chunks; p.num_taps = 1; p.groups = 1;
  return p;
}

void set_conv_taps(GemmParams& p, int cin, int w2, bool three) {
  p.chunks_per_tap = cin / 64;
  if (three) {
    p.num_taps = 9;
    for (int ky = 0; ky < 3; ++ky)
      for (int kx = 0; kx < 3; ++kx) p.tap_shift[ky * 3 + kx] = (ky - 1) * w2 + (kx - 1);
  } else {
    p.num_taps = 1; p.tap_shift[0] = 0;
  }
  p.k_chunks = p.num_taps * p.chunks_per_tap;
}

// h == NULL (the handle-free solver) records nothing
struct ProfScope {
  mk_handle* h; cudaStream_t st; int slot = -1;
  ProfScope(mk_handle* h_, const char* tag, cudaStream_t st_) : h(h_), st(st_) {
    if (!h || !h->profiling) return;
    mk_handle::ProfRec r;
    r.tag = tag;
    if (cudaEventCreate(&r.e0) != cudaSuccess || cudaEventCreate(&r.e1) != cudaSuccess) return;
    cudaEventRecord(r.e0, st);
    h->prof.push_back(r);
    slot = (int)h->prof.size() - 1;
  }
  ~ProfScope() { if (slot >= 0) cudaEventRecord(h->prof[slot].e1, st); }
};

int gemm(mk_handle* h, const char* tag, int epi, const void* a, long long a_rows, long long a_cols, const void* b,
         long long b_rows, long long b_cols, const GemmParams& p, cudaStream_t st) {
  GemmOperand A{a, a_rows, a_cols, a_cols}, B{b, b_rows, b_cols, b_cols};
  h->launches++;
  ProfScope ps(h, tag, st);
  return launch_gemm(epi, A, B, p, st);
}
#define MK_KERNEL(tag, call) do { ProfScope ps_(h, tag, st); h->launches++; MK_TRY(call); } while (0)

// ---- stage 1 ----------------------------------------------------------------------------------------------
// The DINOv2 backbone up to (not including) the final norm: the residual stream of every token ends in w.X.
// img_fmt 0: fp32 NCHW in [0,1] (the reference's tensors); 1: uint8 NHWC RGB as cv2 delivers it (mk_*_u8, SURVEY.md §8 f1)
int run_backbone(mk_handle* h, const void* images, int img_fmt, const Geo& g, Workspace& w, cudaStream_t st) {
  const mk_config& c = h->cfg;
  const int H = g.H, W = g.W;
  const int D = c.embed_dim;
  Lookup L{h};
  // -- tokens: patch embedding + cls + position embedding (dinov2.py:191-200)
  if (img_fmt == 1)
    MK_KERNEL("vit.ingest_u8", ingest_u8(reinterpret_cast<const uint8_t*>(images), w.P, g.n_img, H, W, KPAD, w.X, L.f("patch.clspos", D), D, st));
  else
    MK_KERNEL("vit.patch_gather", patch_gather(reinterpret_cast<const float*>(images), w.P, g.n_img, H, W, KPAD, w.X, L.f("patch.clspos", D), D, st));
  {
    GemmParams p = base_params(g.Mp, D, KPAD);
    p.aux = L.f("patch.posb", (long long)g.N * D); p.tok_per_img = g.N; p.out_f = w.X; p.out_f_ld = D;
    const __half* wt = L.hh("patch.w", (long long)D * KPAD);
    if (!L.ok) return MK_ERR_MISSING_TENSOR;
    MK_TRY(gemm(h, "vit.patch_embed", EPI_PATCH, w.P, g.Mp, KPAD, wt, D, KPAD, p, st));
  }
  // -- transformer blocks (layers/block.py:105-106)
  for (int i = 0; i < c.depth; ++i) {
    const std::string b = "blk" + std::to_string(i) + ".";
    const float *ln1w = L.f(b + "ln1.w", D), *ln1b = L.f(b + "ln1.b", D), *ln2w = L.f(b + "ln2.w", D), *ln2b = L.f(b + "ln2.b", D);
    const __half *wqkv = L.hh(b + "qkv.w", 3LL * D * D), *wproj = L.hh(b + "proj.w", (long long)D * D);
    const __half *wfc1 = L.hh(b + "fc1.w", 4LL * D * D), *wfc2 = L.hh(b + "fc2.w", 4LL * D * D);
    const float *bqkv = L.f(b + "qkv.b", 3 * D), *bproj = L.f(b + "proj.b", D), *bfc1 = L.f(b + "fc1.b", 4 * D), *bfc2 = L.f(b + "fc2.b", D);
    const float *ls1 = L.f(b + "ls1", D), *ls2 = L.f(b + "ls2", D);
    if (!L.ok) return MK_ERR_MISSING_TENSOR;
    MK_KERNEL("vit.layernorm", layernorm(w.X, ln1w, ln1b, w.XN, (int)g.M, D, 1e-6f, 0, 0, 0, st));
    { GemmParams p = base_params(g.M, 3 * D, D); p.bias = bqkv; p.out_h = w.QKV; p.out_h_ld = 3 * D;
      MK_TRY(gemm(h, "vit.qkv", EPI_STORE_H, w.XN, g.M, D, wqkv, 3 * D, D, p, st)); }
    MK_KERNEL("vit.attention", attention_dispatch(w.QKV, w.ATT, g.n_img, g.T, D, c.heads, 0, st));
    { GemmParams p = base_params(g.M, D, D); p.bias = bproj; p.gamma = ls1; p.out_f = w.X; p.out_f_ld = D;
      MK_TRY(gemm(h, "vit.proj", EPI_RESID_F, w.ATT, g.M, D, wproj, D, D, p, st)); }
    MK_KERNEL("vit.layernorm", layernorm(w.X, ln2w, ln2b, w.XN, (int)g.M, D, 1e-6f, 0, 0, 0, st));
    { GemmParams p = base_params(g.M, 4 * D, D); p.bias = bfc1; p.act = ACT_GELU; p.out_h = w.H1; p.out_h_ld = 4 * D;
      MK_TRY(gemm(h, "vit.fc1", EPI_STORE_H, w.XN, g.M, D, wfc1, 4 * D, D, p, st)); }
    { GemmParams p = base_params(g.M, D, 4 * D); p.bias = bfc2; p.gamma = ls2; p.out_f = w.X; p.out_f_ld = D;
      MK_TRY(gemm(h, "vit.fc2", EPI_RESID_F, w.H1, g.M, 4 * D, wfc2, D, 4 * D, p, st)); }
  }
  return MK_OK;
}

// role < 0: images [0, n_img/2) take role 0 in the matcher and the rest role 1 (mk_forward; mk_extract_images leaves
// operands no matcher reads).  role 1: all n_img images are the queries of g.n_pairs = n_img pairs (mk_localize); their
// operands and score copy go to the role-1 halves of DSCX and scr_copy.  dsc may be NULL (no fp32 descriptors).
int run_extract(mk_handle* h, const void* images, int img_fmt, const Geo& g, float* kps, float* depth, float* scr,
                float* dsc, Workspace& w, cudaStream_t st, int role = -1) {
  const mk_config& c = h->cfg;
  const int D = c.embed_dim;
  Lookup L{h};
  MK_TRY(run_backbone(h, images, img_fmt, g, w, st));
  // -- final norm, drop cls, scatter into the zero-padded NHWC feature image (dinov2.py:230-233, mickey_extractor.py:49-51)
  MK_CUDA_CHECK(cudaMemsetAsync(w.F, 0, (size_t)g.R * D * sizeof(__half), st));
  MK_KERNEL("vit.layernorm", layernorm(w.X, L.f("norm.w", D), L.f("norm.b", D), w.F, (int)g.M, D, 1e-6f, 1, g.gh, g.gw, st));
  if (!L.ok) return MK_ERR_MISSING_TENSOR;

  // -- heads: three grouped residual blocks (extractor_utils.py:28-35; G = 4 heads side by side in channels)
  const int* bd = c.block_dims;
  struct Rb { const char* name; const __half* in; int cin; int in_goff; __half *T, *S, *O; int cout; };
  const Rb rbs[3] = {{"rb1", w.F, D, 0, w.T1, w.S1, w.O1, bd[0]},
                     {"rb2", w.O1, bd[0], bd[0], w.T2, w.S2, w.O2, bd[1]},
                     {"rb3", w.O2, bd[1], bd[1], w.T3, w.S3, nullptr, bd[2]}};
  if (bd[2] != 128) { set_last_error("KP_HEADS.BLOCKS_DIM[2] must be 128 (transformer width)"); return MK_ERR_UNSUPPORTED; }
  for (int r = 0; r < 3; ++r) {
    const Rb& rb = rbs[r];
    const std::string n = std::string(rb.name) + ".";
    const long long in_cols = (r == 0) ? D : (long long)G * rb.cin;
    const __half *wc1 = L.hh(n + "c1.w", (long long)G * rb.cout * 9 * rb.cin), *wsc = L.hh(n + "sc.w", (long long)G * rb.cout * rb.cin);
    const __half* wc2 = L.hh(n + "c2.w", (long long)G * rb.cout * 9 * rb.cout);
    const float *b1 = L.f(n + "c1.b", G * rb.cout), *b2 = L.f(n + "c2.b", G * rb.cout);
    if (!L.ok) return MK_ERR_MISSING_TENSOR;
    {  // conv1 + bn1 + relu
      GemmParams p = base_params(g.R, rb.cout, 64); set_conv_taps(p, rb.cin, g.w2, true);
      p.groups = G; p.a_col_group_off = rb.in_goff; p.b_row_group_off = rb.cout; p.bias = b1; p.bias_group_off = rb.cout;
      p.act = ACT_RELU; p.pad_h2 = g.h2; p.pad_w2 = g.w2; p.out_h = rb.T; p.out_h_ld = (long long)G * rb.cout; p.out_h_group_off = rb.cout;
      MK_TRY(gemm(h, "head.conv3x3", EPI_CONV, rb.in, g.R, in_cols, wc1, (long long)G * rb.cout, 9LL * rb.cin, p, st));
    }
    {  // 1x1 shortcut
      GemmParams p = base_params(g.R, rb.cout, 64); set_conv_taps(p, rb.cin, g.w2, false);
      p.groups = G; p.a_col_group_off = rb.in_goff; p.b_row_group_off = rb.cout;
      p.out_h = rb.S; p.out_h_ld = (long long)G * rb.cout; p.out_h_group_off = rb.cout;
      MK_TRY(gemm(h, "head.conv1x1", EPI_CONV, rb.in, g.R, in_cols, wsc, (long long)G * rb.cout, rb.cin, p, st));
    }
    {  // conv2 + bn2 + shortcut + relu (+ sine position encoding and fp32 copy after block 3)
      GemmParams p = base_params(g.R, rb.cout, 64); set_conv_taps(p, rb.cout, g.w2, true);
      p.groups = G; p.a_col_group_off = rb.cout; p.b_row_group_off = rb.cout; p.bias = b2; p.bias_group_off = rb.cout;
      p.res_h = rb.S; p.res_h_ld = (long long)G * rb.cout; p.res_h_group_off = rb.cout;
      p.act = ACT_RELU; p.pad_h2 = g.h2; p.pad_w2 = g.w2;
      if (r < 2) { p.out_h = rb.O; p.out_h_ld = (long long)G * rb.cout; p.out_h_group_off = rb.cout; }
      else {
        p.out_h = w.CAT; p.out_h_ld = G * 256; p.out_h_group_off = 256;
        p.out_f = w.X32; p.out_f_ld = G * 128; p.out_f_group_off = 128;
        p.aux = L.f("head.pe", (long long)g.per_img * 128);
        p.aux_group_mask = (c.kp_pos_enc ? 0x7 : 0) | (c.dsc_pos_enc ? 0x8 : 0);
        if (!L.ok) return MK_ERR_MISSING_TENSOR;
      }
      MK_TRY(gemm(h, "head.conv3x3", EPI_CONV, rb.T, g.R, (long long)G * rb.cout, wc2, (long long)G * rb.cout, 9LL * rb.cout, p, st));
    }
  }
  // -- linear-attention transformer, 3 layers (att_layers/transformer_utils.py:40-66)
  for (int l = 0; l < 3; ++l) {
    const std::string n = "att" + std::to_string(l) + ".";
    const __half *wqkv = L.hh(n + "qkv.w", (long long)G * 384 * 128), *wmerge = L.hh(n + "merge.w", (long long)G * 128 * 128);
    const __half *wm0 = L.hh(n + "mlp0.w", (long long)G * 256 * 256), *wm2 = L.hh(n + "mlp2.w", (long long)G * 128 * 256);
    const float *n1w = L.f(n + "n1.w", G * 128), *n1b = L.f(n + "n1.b", G * 128), *n2w = L.f(n + "n2.w", G * 128), *n2b = L.f(n + "n2.b", G * 128);
    if (!L.ok) return MK_ERR_MISSING_TENSOR;
    { GemmParams p = base_params(g.R, 384, 128); p.groups = G; p.a_col_group_off = 256; p.b_row_group_off = 384;
      p.out_f = w.QKV32; p.out_f_ld = G * 384; p.out_f_group_off = 384;
      MK_TRY(gemm(h, "head.att.qkv", EPI_STORE_F, w.CAT, g.R, G * 256, wqkv, G * 384, 128, p, st)); }
    { ProfScope ps_(h, "head.att.kv", st); h->launches += 2; MK_TRY(linattn_kv(w.QKV32, w.KVP, w.KV, g.n_img, G, g.h2, g.w2, st)); }
    MK_KERNEL("head.att.msg", linattn_msg(w.QKV32, w.KV, w.MSG, g.n_img, G, g.h2, g.w2, 1e-6f, st));
    { GemmParams p = base_params(g.R, 128, 128); p.groups = G; p.a_col_group_off = 128; p.b_row_group_off = 128;
      p.gamma = n1w; p.beta = n1b; p.ln_group_off = 128; p.eps = 1e-5f;
      p.out_h = w.CAT + 128; p.out_h_ld = G * 256; p.out_h_group_off = 256;
      MK_TRY(gemm(h, "head.att.merge_ln", EPI_LN, w.MSG, g.R, G * 128, wmerge, G * 128, 128, p, st)); }
    { GemmParams p = base_params(g.R, 256, 256); p.groups = G; p.a_col_group_off = 256; p.b_row_group_off = 256; p.act = ACT_RELU;
      p.out_h = w.HM; p.out_h_ld = G * 256; p.out_h_group_off = 256;
      MK_TRY(gemm(h, "head.att.mlp0", EPI_STORE_H, w.CAT, g.R, G * 256, wm0, G * 256, 256, p, st)); }
    { GemmParams p = base_params(g.R, 128, 256); p.groups = G; p.a_col_group_off = 256; p.b_row_group_off = 128;
      p.gamma = n2w; p.beta = n2b; p.ln_group_off = 128; p.eps = 1e-5f;
      p.out_f = w.X32; p.out_f_ld = G * 128; p.out_f_group_off = 128;
      p.out_h = w.CAT; p.out_h_ld = G * 256; p.out_h_group_off = 256;
      if (l == 2) { p.pad_h2 = g.h2; p.pad_w2 = g.w2; }       // zero the pad rows again before the next 3x3 conv
      MK_TRY(gemm(h, "head.att.mlp2_ln", EPI_LN, w.HM, g.R, G * 256, wm2, G * 128, 256, p, st)); }
  }
  // -- residual block 4: three keypoint heads (128 -> 64, with shortcut conv) and the descriptor head (128 -> desc_dim)
  {
    const int co = bd[3];
    const __half *wc1 = L.hh("rb4k.c1.w", 3LL * co * 9 * 128), *wsc = L.hh("rb4k.sc.w", 3LL * co * 128), *wc2 = L.hh("rb4k.c2.w", 3LL * co * 9 * co);
    const float *b1 = L.f("rb4k.c1.b", 3 * co), *b2 = L.f("rb4k.c2.b", 3 * co);
    if (!L.ok) return MK_ERR_MISSING_TENSOR;
    { GemmParams p = base_params(g.R, co, 64); set_conv_taps(p, 128, g.w2, true);
      p.groups = 3; p.a_col_group_off = 256; p.b_row_group_off = co; p.bias = b1; p.bias_group_off = co; p.act = ACT_RELU;
      p.pad_h2 = g.h2; p.pad_w2 = g.w2; p.out_h = w.T4k; p.out_h_ld = 3 * co; p.out_h_group_off = co;
      MK_TRY(gemm(h, "head.conv3x3", EPI_CONV, w.CAT, g.R, G * 256, wc1, 3 * co, 9 * 128, p, st)); }
    { GemmParams p = base_params(g.R, co, 64); set_conv_taps(p, 128, g.w2, false);
      p.groups = 3; p.a_col_group_off = 256; p.b_row_group_off = co; p.out_h = w.S4k; p.out_h_ld = 3 * co; p.out_h_group_off = co;
      MK_TRY(gemm(h, "head.conv1x1", EPI_CONV, w.CAT, g.R, G * 256, wsc, 3 * co, 128, p, st)); }
    { GemmParams p = base_params(g.R, co, 64); set_conv_taps(p, co, g.w2, true);
      p.groups = 3; p.a_col_group_off = co; p.b_row_group_off = co; p.bias = b2; p.bias_group_off = co; p.act = ACT_RELU;
      p.res_h = w.S4k; p.res_h_ld = 3 * co; p.res_h_group_off = co; p.pad_h2 = g.h2; p.pad_w2 = g.w2;
      p.out_f = w.Y4k; p.out_f_ld = 3 * co; p.out_f_group_off = co;
      MK_TRY(gemm(h, "head.conv3x3", EPI_CONV, w.T4k, g.R, 3 * co, wc2, 3 * co, 9 * co, p, st)); }
  }
  {
    const int co = c.desc_dim;
    const __half *wc1 = L.hh("rb4d.c1.w", (long long)co * 9 * 128), *wc2 = L.hh("rb4d.c2.w", (long long)co * 9 * co);
    const float *b1 = L.f("rb4d.c1.b", co), *b2 = L.f("rb4d.c2.b", co);
    if (co != 128) { set_last_error("DSC_HEAD.LAST_DIM must be 128"); return MK_ERR_UNSUPPORTED; }
    if (!L.ok) return MK_ERR_MISSING_TENSOR;
    { GemmParams p = base_params(g.R, co, 64); set_conv_taps(p, 128, g.w2, true);
      p.a_col_base = 3 * 256; p.bias = b1; p.act = ACT_RELU; p.pad_h2 = g.h2; p.pad_w2 = g.w2; p.out_h = w.T4d; p.out_h_ld = co;
      MK_TRY(gemm(h, "head.conv3x3", EPI_CONV, w.CAT, g.R, G * 256, wc1, co, 9 * 128, p, st)); }
    { GemmParams p = base_params(g.R, co, 64); set_conv_taps(p, co, g.w2, true);
      p.bias = b2; p.act = ACT_NONE; p.res_h = w.CAT + 3 * 256; p.res_h_ld = G * 256;   // identity shortcut (in == out planes)
      p.pad_h2 = g.h2; p.pad_w2 = g.w2; p.out_f = w.Y4d; p.out_f_ld = co;
      MK_TRY(gemm(h, "head.conv3x3", EPI_CONV, w.T4d, g.R, co, wc2, co, 9 * co, p, st)); }
  }
  // -- output layers and activations
  { ProfScope ps_(h, "head.kp_out", st); h->launches += 2;
    MK_TRY(kp_head_out(w.Y4k, L.f("out.depth.w", bd[3]), L.f("out.xy.w", 2 * bd[3]), L.f("out.score.w", bd[3]), depth, kps,
                       w.score_raw, scr, g.n_img, g.gh, g.gw, c.depth_sigmoid, c.max_depth, (float)c.down_factor, c.use_softmax, st)); }
  if (!L.ok) return MK_ERR_MISSING_TENSOR;
  if (bd[3] != 64) { set_last_error("KP_HEADS.BLOCKS_DIM[3] must be 64"); return MK_ERR_UNSUPPORTED; }
  const size_t op_row = role == 1 ? (size_t)g.n_pairs * g.N : 0;       // first operand row this extraction writes
  MK_KERNEL("head.desc_out", desc_out(w.Y4d, dsc, w.DSCX + op_row * 384, w.nrm2, g.n_img, g.gh, g.gw, c.norm_dsc, role, st));
  if (scr != w.scr_copy + op_row)
    MK_CUDA_CHECK(cudaMemcpyAsync(w.scr_copy + op_row, scr, (size_t)g.n_img * g.N * sizeof(float), cudaMemcpyDeviceToDevice, st));
  return MK_OK;
}

// ---- stage 2 ----------------------------------------------------------------------------------------------
// nn_pitch: row pitch (floats) of the three N x N outputs; N = the reference's contiguous layout.  With a pitch that is a
// multiple of 4 (16-byte rows) the outputs leave through TMA tensor stores; N = 1938 itself cannot (7752-byte rows).
int run_match(mk_handle* h, int n_pairs, int N, float* scores, float* kp_scores, float* final_scores, long long nn_pitch,
              Workspace& w, cudaStream_t st) {
  const mk_config& c = h->cfg;
  Lookup L{h};
  const float* dust = c.use_dustbin ? L.f("dustbin", 1) : nullptr;
  if (!L.ok) return MK_ERR_MISSING_TENSOR;
  if (!final_scores || ((scores == nullptr) != (kp_scores == nullptr))) {
    set_last_error("mk_match: final_scores is required; scores and kp_scores are given together or both NULL (lean mode)");
    return MK_ERR_INVALID;
  }
  MK_TRY(resolve_pitch(nn_pitch, N, "mk_match: nn_pitch"));
  const bool tma_ok = nn_pitch % 4 == 0 && reinterpret_cast<uintptr_t>(final_scores) % 16 == 0 &&
                      (!scores || (reinterpret_cast<uintptr_t>(scores) % 16 == 0 && reinterpret_cast<uintptr_t>(kp_scores) % 16 == 0));
  const float inv_t = 1.0f / c.temperature;
  const __half* A0 = w.DSCX;                                   // role-0 descriptors [n_pairs*N, 384]
  const __half* A1 = w.DSCX + (size_t)n_pairs * N * 384;       // role-1 descriptors
  const long long rows = (long long)n_pairs * N;
  const int npad = ceil_div(N, 128) * 128;
  auto mp = [&]() {
    GemmParams p = base_params(N, N, 384);
    p.groups = n_pairs; p.a_row_group_off = N; p.b_row_group_off = N; p.n_valid = N; p.inv_temp = inv_t; p.part_ld = npad;
    return p;
  };
  // pass 1: S once, row and column partials from the same tile; then the tiny fold (+ dustbin); pass 2: outputs
  { GemmParams p = mp(); p.part_row = reinterpret_cast<float2*>(w.part_row); p.part_col = reinterpret_cast<float2*>(w.part_col);
    // L2-normalised descriptors: |S| <= 1 (+ rounding), so 1.001 / T bounds every logit; used while 2 * 1.001 / T * log2(e)
    // stays far inside the fp32 exponent range (T >= 0.04); otherwise, and for un-normalised descriptors, true maxima
    p.lse_bound = (c.norm_dsc && inv_t <= 25.0f) ? 1.001f : 0.0f;
    MK_TRY(gemm(h, "match.lse", EPI_LSE, A0, rows, 384, A1, rows, 384, p, st)); }
  MK_KERNEL("match.reduce", matcher_lse_reduce(w.part_row, w.part_col, dust, n_pairs, N, npad, w.lse_r, w.lse_c, st));
  { GemmParams p = mp(); p.lse_r = w.lse_r; p.lse_c = w.lse_c; p.scr0 = w.scr_copy; p.scr1 = w.scr_copy + (size_t)n_pairs * N;
    p.scores = scores; p.kp_scores = kp_scores; p.final_scores = final_scores; p.out_pitch = nn_pitch; p.out_tma = tma_ok ? 1 : 0;
    MK_TRY(gemm(h, "match.dual_softmax", EPI_DUAL, A0, rows, 384, A1, rows, 384, p, st)); }
  return MK_OK;
}

// ---- stage 3 ----------------------------------------------------------------------------------------------
// The solve of one batch: the outer draw (unless outer_idx is given), the fused RANSAC kernel and the optional output
// copies, in the solver's scratch s.  rp holds the PROCRUSTES sizes and rp.seed the device word both draws read; nn_pitch
// is resolved.  h: the handle of mk_solve_pose / mk_forward*, whose profiling scopes and launch count this feeds, or NULL
// (mk_procrustes_solve).
int run_solve(mk_handle* h, const RansacParams& rp, const float* final_scores, long long nn_pitch, const float* kps,
              const float* depth, const float* K0, const float* K1, int n_pairs, int N, const int* outer_idx,
              const int* inner_idx, float* pose, int* best_set, float* inl_mask, int* sampled_out, float* hyp_scores_out,
              int* status_out, const SolverWs& s, cudaStream_t st) {
  MK_CUDA_CHECK(cudaMemsetAsync(s.status, 0, (size_t)(SOLVER_COUNTER_BASE + n_pairs) * sizeof(int), st));
  const size_t n_idx = (size_t)n_pairs * rp.it_matches * rp.n_sample;
  const int* idx = outer_idx;
  if (!idx) {
    { ProfScope ps_(h, "solve.sample_outer", st); if (h) h->launches += 4;
      MK_TRY(sample_outer(final_scores, n_pairs, N, nn_pitch, rp.it_matches, rp.n_sample, rp.seed, s.samp_ws, s.idx, s.status, st)); }
    idx = s.idx;
  }
  const float* kps0 = kps;
  const float* kps1 = kps + (size_t)n_pairs * 2 * N;
  const float* d0 = depth;
  const float* d1 = depth + (size_t)n_pairs * N;
  int* bs = best_set ? best_set : s.best_hyp;     // scratch when the caller does not want it
  { ProfScope ps_(h, "solve.ransac", st); if (h) h->launches += 1;
    MK_TRY(ransac_solve(final_scores, nn_pitch, kps0, d0, kps1, d1, K0, K1, n_pairs, N, rp, idx, inner_idx, s.hyp_scores,
                        s.hyp_Rt, s.status, pose, bs, inl_mask, best_set ? s.best_hyp : nullptr, st)); }
  if (sampled_out) MK_CUDA_CHECK(cudaMemcpyAsync(sampled_out, idx, n_idx * sizeof(int), cudaMemcpyDeviceToDevice, st));
  if (hyp_scores_out)
    MK_CUDA_CHECK(cudaMemcpyAsync(hyp_scores_out, s.hyp_scores, (size_t)n_pairs * rp.it_matches * rp.it_ransac * sizeof(float),
                                  cudaMemcpyDeviceToDevice, st));
  if (status_out) MK_CUDA_CHECK(cudaMemcpyAsync(status_out, s.status, sizeof(int), cudaMemcpyDeviceToDevice, st));
  return MK_OK;
}

// The handle's solve: its PROCRUSTES config and its device-side seed, which a non-zero seed resets and every solve advances.
int run_solve_handle(mk_handle* h, const float* final_scores, long long nn_pitch, const float* kps, const float* depth,
                     const float* K0, const float* K1, int n_pairs, int N, unsigned long long seed, const int* outer_idx,
                     const int* inner_idx, float* pose, int* best_set, float* inl_mask, int* sampled_out,
                     float* hyp_scores_out, int* status_out, Workspace& w, cudaStream_t st) {
  const mk_config& c = h->cfg;
  RansacParams rp{c.it_matches, c.it_ransac, c.num_sampled, c.num_corr, c.num_refine, c.th_inlier, c.th_soft_inlier, h->seed_dev};
  MK_TRY(resolve_pitch(nn_pitch, N, "mk_solve_pose: nn_pitch"));
  if (seed != 0) MK_TRY(seed_set(h->seed_dev, seed, st));      // seed == 0: continue the device-side sequence
  MK_TRY(run_solve(h, rp, final_scores, nn_pitch, kps, depth, K0, K1, n_pairs, N, outer_idx, inner_idx, pose, best_set,
                   inl_mask, sampled_out, hyp_scores_out, status_out, w.sol, st));
  return seed_advance(h->seed_dev, st);
}

// mk_procrustes_solve's sizes (include/mickey_b200.h): the sampler's selection sorts 2048 candidates per stream and the
// hypothesis kernel scans a set across its 256 threads; one grid dimension holds B, another IT_MATCHES; cells, hypotheses
// of a pair and streams are counted in int.
constexpr int PROC_MAX_SAMPLED = 2048, PROC_SAMPLED_STEP = 256, PROC_MAX_GRID = 65535;

bool procrustes_sizes_ok(int B, int N, int it_matches, int it_ransac, int num_sampled) {
  return B >= 1 && B <= PROC_MAX_GRID && N >= 1 && (long long)N * N <= 0x7fffffffLL && it_matches >= 1 &&
         it_matches <= PROC_MAX_GRID && it_ransac >= 1 && (long long)it_matches * it_ransac <= 0x7fffffffLL &&
         (long long)B * it_matches <= 0x7fffffffLL && num_sampled >= PROC_SAMPLED_STEP && num_sampled <= PROC_MAX_SAMPLED &&
         num_sampled % PROC_SAMPLED_STEP == 0;
}

// the solver's scratch, then the seed word
size_t procrustes_carve(void* ws, int B, int it_matches, int it_ransac, int num_sampled, SolverWs& s,
                        unsigned long long** seed_word) {
  Carver cv(ws);
  carve_solver(cv, B, it_matches, it_ransac, num_sampled, s);
  *seed_word = cv.take<unsigned long long>(1);
  return (cv.off + 255) & ~(size_t)255;
}

int check_ws(mk_handle* h, int n_img, int n_pairs, int H, int W, void* ws, long long ws_bytes, Workspace& out) {
  if (!h || !h->finalized) { set_last_error("handle not finalized"); return MK_ERR_INVALID; }
  MK_CUDA_CHECK(cudaSetDevice(h->device));        // one handle per device: every entry point runs on the handle's device
  if (H != h->geo_h || W != h->geo_w) {
    set_last_error("geometry %dx%d does not match the finalized geometry %dx%d", H, W, h->geo_h, h->geo_w);
    return MK_ERR_INVALID;
  }
  const Geo g = make_geo(n_img, n_pairs, H, W);
  out = carve(ws, h->cfg, g);
  if (!ws || (long long)out.bytes > ws_bytes) {
    set_last_error("workspace too small: need %zu bytes, got %lld", out.bytes, ws_bytes);
    return MK_ERR_INVALID;
  }
  return MK_OK;
}

}  // namespace

// ============================================================================================================
extern "C" {

const char* mk_last_error(void) { return mk::last_error(); }
const char* mk_version(void) { return "mickey_b200 0.1.0 (sm_90a)"; }
int mk_sizeof(const char* type) {
  const std::unordered_map<std::string, int> sizes = {
      {"mk_config", sizeof(mk_config)}, {"mk_gemm_args", sizeof(mk_gemm_args)}, {"mk_htr_layer", sizeof(mk_htr_layer)},
      {"mk_htr_layer_grads", sizeof(mk_htr_layer_grads)}, {"mk_resblock_params", sizeof(mk_resblock_params)},
      {"mk_resblock_grads", sizeof(mk_resblock_grads)}};
  const auto it = type ? sizes.find(type) : sizes.end();
  return it == sizes.end() ? -1 : it->second;
}

int mk_create(int device, const mk_config* cfg, mk_handle** out) {
  if (!cfg || !out) { set_last_error("null argument"); return MK_ERR_INVALID; }
  if (cfg->embed_dim != cfg->heads * 64 || cfg->embed_dim % 128) {
    set_last_error("unsupported backbone: embed_dim %d heads %d", cfg->embed_dim, cfg->heads);
    return MK_ERR_UNSUPPORTED;
  }
  int count = 0;
  if (cudaGetDeviceCount(&count) != cudaSuccess || device < 0 || device >= count) {
    set_last_error("CUDA device %d not available (an H100 is required; there is no CPU path)", device);
    return MK_ERR_CUDA;
  }
  cudaDeviceProp prop;
  MK_CUDA_CHECK(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0) {
    set_last_error("device %d is sm_%d%d; this library contains sm_90a code only", device, prop.major, prop.minor);
    return MK_ERR_UNSUPPORTED;
  }
  mk_handle* h = new mk_handle();
  h->device = device;
  h->cfg = *cfg;
  MK_CUDA_CHECK(cudaSetDevice(device));
  MK_CUDA_CHECK(cudaMalloc(&h->seed_dev, sizeof(unsigned long long)));
  const unsigned long long s0 = 0x243F6A8885A308D3ull;
  MK_CUDA_CHECK(cudaMemcpy(h->seed_dev, &s0, sizeof(s0), cudaMemcpyHostToDevice));
  *out = h;
  return MK_OK;
}

int mk_destroy(mk_handle* h) {
  if (h) {
    if (h->seed_dev) cudaFree(h->seed_dev);
    for (auto& r : h->prof) { cudaEventDestroy(r.e0); cudaEventDestroy(r.e1); }
    delete h;
  }
  return MK_OK;
}

int mk_set_tensor(mk_handle* h, const char* name, const void* ptr, int dtype, long long numel) {
  if (!h || !name || !ptr) { set_last_error("null argument"); return MK_ERR_INVALID; }
  h->tensors[name] = Tensor{ptr, dtype, numel};
  return MK_OK;
}

int mk_finalize(mk_handle* h, int H, int W) {
  if (!h) return MK_ERR_INVALID;
  if (H < 14 * 7 || W < 14 * 7) { set_last_error("image %dx%d too small (3-px border mask needs >= 7 cells)", H, W); return MK_ERR_INVALID; }
  h->geo_h = H; h->geo_w = W; h->finalized = true;
  return MK_OK;
}

long long mk_workspace_bytes(mk_handle* h, int n_pairs, int H, int W) {
  if (!h) return -1;
  return (long long)carve(nullptr, h->cfg, make_geo(2 * n_pairs, n_pairs, H, W)).bytes;
}

long long mk_workspace_bytes_for(mk_handle* h, int n_img, int n_pairs, int H, int W) {
  if (!h || n_img < 0 || n_pairs < 0) return -1;
  const Geo g = make_geo(n_img, n_pairs, H, W);
  return (long long)carve(nullptr, h->cfg, g).bytes;
}

int mk_extract(mk_handle* h, const float* images, int n_pairs, int H, int W, float* kps, float* depth, float* scr,
               float* dsc, void* ws, long long ws_bytes, void* stream) {
  Workspace w;
  MK_TRY(check_ws(h, 2 * n_pairs, n_pairs, H, W, ws, ws_bytes, w));
  return run_extract(h, images, 0, make_geo(2 * n_pairs, n_pairs, H, W), kps, depth, scr, dsc, w, (cudaStream_t)stream);
}

int mk_extract_u8(mk_handle* h, const unsigned char* images, int n_pairs, int H, int W, float* kps, float* depth, float* scr,
                  float* dsc, void* ws, long long ws_bytes, void* stream) {
  Workspace w;
  MK_TRY(check_ws(h, 2 * n_pairs, n_pairs, H, W, ws, ws_bytes, w));
  return run_extract(h, images, 1, make_geo(2 * n_pairs, n_pairs, H, W), kps, depth, scr, dsc, w, (cudaStream_t)stream);
}

static int extract_images_any(mk_handle* h, const void* images, int img_fmt, int n_img, int H, int W, float* kps, float* depth,
                              float* scr, float* dsc, void* ws, long long ws_bytes, void* stream) {
  if (n_img <= 0 || !images || !kps || !depth || !scr || !dsc) {
    set_last_error("mk_extract_images: n_img %d must be positive and every pointer non-NULL", n_img);
    return MK_ERR_INVALID;
  }
  Workspace w;
  MK_TRY(check_ws(h, n_img, 0, H, W, ws, ws_bytes, w));
  return run_extract(h, images, img_fmt, make_geo(n_img, 0, H, W), kps, depth, scr, dsc, w, (cudaStream_t)stream);
}

int mk_extract_images(mk_handle* h, const float* images, int n_img, int H, int W, float* kps, float* depth, float* scr,
                      float* dsc, void* ws, long long ws_bytes, void* stream) {
  return extract_images_any(h, images, 0, n_img, H, W, kps, depth, scr, dsc, ws, ws_bytes, stream);
}

int mk_extract_images_u8(mk_handle* h, const unsigned char* images, int n_img, int H, int W, float* kps, float* depth, float* scr,
                         float* dsc, void* ws, long long ws_bytes, void* stream) {
  return extract_images_any(h, images, 1, n_img, H, W, kps, depth, scr, dsc, ws, ws_bytes, stream);
}

long long mk_backbone_ws_bytes(mk_handle* h, int n_img, int H, int W) {
  if (!h || n_img < 1 || H < 98 || W < 98 || H % 14 || W % 14) return -1;
  return (long long)backbone_ws_bytes(h->cfg, make_geo(n_img, 0, H, W));
}

int mk_backbone_features(mk_handle* h, const float* images, int n_img, int H, int W, float* out, void* ws, long long ws_bytes,
                         void* stream) {
  // every argument is checked before the handle is read and before anything is launched
  if (!h || !images || !out || !ws) { set_last_error("mk_backbone_features: null argument"); return MK_ERR_INVALID; }
  if (n_img < 1) { set_last_error("mk_backbone_features: n_img %d must be positive", n_img); return MK_ERR_INVALID; }
  if (H < 98 || W < 98 || H % 14 || W % 14) {
    set_last_error("mk_backbone_features: image %dx%d must be multiples of 14 and at least 98", H, W);
    return MK_ERR_INVALID;
  }
  if (!h->finalized) { set_last_error("mk_backbone_features: handle not finalized"); return MK_ERR_INVALID; }
  if (H != h->geo_h || W != h->geo_w) {
    set_last_error("mk_backbone_features: geometry %dx%d does not match the finalized geometry %dx%d", H, W, h->geo_h, h->geo_w);
    return MK_ERR_INVALID;
  }
  const Geo g = make_geo(n_img, 0, H, W);
  const size_t need = backbone_ws_bytes(h->cfg, g);
  if ((long long)need > ws_bytes) {
    set_last_error("mk_backbone_features: workspace too small: need %zu bytes, got %lld", need, ws_bytes);
    return MK_ERR_INVALID;
  }
  MK_CUDA_CHECK(cudaSetDevice(h->device));
  const int D = h->cfg.embed_dim;
  Lookup L{h};
  const float *nw = L.f("norm.w", D), *nb = L.f("norm.b", D);
  if (!L.ok) return MK_ERR_MISSING_TENSOR;
  Workspace w;
  Carver cv(ws);
  carve_backbone(cv, h->cfg, g, w);
  cudaStream_t st = (cudaStream_t)stream;
  MK_TRY(run_backbone(h, images, 0, g, w, st));
  // -- final norm, drop cls, channel-major fp32 (dinov2.py:230-233, mickey_extractor.py:49-51)
  MK_KERNEL("vit.layernorm_cm", layernorm_channel_major(w.X, nw, nb, out, n_img, g.N, D, 1e-6f, st));
  return MK_OK;
}

int mk_match(mk_handle* h, int n_pairs, float* scores, float* kp_scores, float* final_scores, long long nn_pitch, void* ws,
             long long ws_bytes, void* stream) {
  Workspace w;
  MK_TRY(check_ws(h, 2 * n_pairs, n_pairs, h ? h->geo_h : 0, h ? h->geo_w : 0, ws, ws_bytes, w));
  const Geo g = make_geo(2 * n_pairs, n_pairs, h->geo_h, h->geo_w);
  return run_match(h, n_pairs, g.N, scores, kp_scores, final_scores, nn_pitch, w, (cudaStream_t)stream);
}

int mk_solve_pose(mk_handle* h, const float* final_scores, long long nn_pitch, const float* kps, const float* depth, const float* K0,
                  const float* K1, int n_pairs, int n_kpts, unsigned long long seed, const int* outer_idx,
                  const int* inner_idx, float* pose, int* best_set, float* inl_mask, int* sampled_out,
                  float* hyp_scores_out, int* status, void* ws, long long ws_bytes, void* stream) {
  Workspace w;
  MK_TRY(check_ws(h, 2 * n_pairs, n_pairs, h ? h->geo_h : 0, h ? h->geo_w : 0, ws, ws_bytes, w));
  const Geo g = make_geo(2 * n_pairs, n_pairs, h->geo_h, h->geo_w);
  if (n_kpts != g.N) { set_last_error("n_kpts %d does not match the geometry (%d)", n_kpts, g.N); return MK_ERR_INVALID; }
  return run_solve_handle(h, final_scores, nn_pitch, kps, depth, K0, K1, n_pairs, n_kpts, seed, outer_idx, inner_idx, pose,
                          best_set, inl_mask, sampled_out, hyp_scores_out, status, w, (cudaStream_t)stream);
}

long long mk_procrustes_ws_bytes(int B, int N, int it_matches, int it_ransac, int num_sampled) {
  if (!procrustes_sizes_ok(B, N, it_matches, it_ransac, num_sampled)) return -1;
  SolverWs s;
  unsigned long long* seed_word;
  return (long long)procrustes_carve(nullptr, B, it_matches, it_ransac, num_sampled, s, &seed_word);
}

int mk_procrustes_solve(const float* final_scores, long long nn_pitch, const float* kps, const float* depth, const float* K0,
                        const float* K1, int B, int N, int it_matches, int it_ransac, int num_sampled, int num_corr,
                        int num_refine, float th_inlier, float th_soft_inlier, unsigned long long seed, const int* outer_idx,
                        const int* inner_idx, float* pose, int* best_set, float* inl_mask, int* sampled_out,
                        float* hyp_scores_out, int* status, void* ws, long long ws_bytes, void* stream) {
  // every argument is checked before anything is launched
  if (!final_scores || !kps || !depth || !K0 || !K1 || !pose || !ws) {
    set_last_error("mk_procrustes_solve: final_scores, kps, depth, K0, K1, pose and the workspace must be non-NULL");
    return MK_ERR_INVALID;
  }
  if (!procrustes_sizes_ok(B, N, it_matches, it_ransac, num_sampled) || num_corr != 3 || num_refine < 0 ||
      !(th_inlier > 0.f && th_inlier <= FLT_MAX) || !(th_soft_inlier > 0.f && th_soft_inlier <= FLT_MAX)) {
    set_last_error("mk_procrustes_solve: need 1 <= B <= %d, N >= 1 with N*N < 2^31, 1 <= it_matches <= %d, it_ransac >= 1, "
                   "it_matches*it_ransac and B*it_matches < 2^31, num_sampled a multiple of %d up to %d, num_corr 3, "
                   "num_refine >= 0 and finite positive thresholds (got B %d N %d it_matches %d it_ransac %d num_sampled %d "
                   "num_corr %d num_refine %d th_inlier %g th_soft_inlier %g)", PROC_MAX_GRID, PROC_MAX_GRID,
                   PROC_SAMPLED_STEP, PROC_MAX_SAMPLED, B, N, it_matches, it_ransac, num_sampled, num_corr, num_refine,
                   (double)th_inlier, (double)th_soft_inlier);
    return MK_ERR_INVALID;
  }
  MK_TRY(resolve_pitch(nn_pitch, N, "mk_procrustes_solve: nn_pitch"));
  SolverWs s;
  unsigned long long* seed_word;
  const size_t need = procrustes_carve(ws, B, it_matches, it_ransac, num_sampled, s, &seed_word);
  if ((long long)need > ws_bytes) {
    set_last_error("mk_procrustes_solve: workspace of %lld bytes, %zu needed", ws_bytes, need);
    return MK_ERR_INVALID;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const RansacParams rp{it_matches, it_ransac, num_sampled, num_corr, num_refine, th_inlier, th_soft_inlier, seed_word};
  MK_TRY(seed_set(seed_word, seed, st));
  return run_solve(nullptr, rp, final_scores, nn_pitch, kps, depth, K0, K1, B, N, outer_idx, inner_idx, pose, best_set,
                   inl_mask, sampled_out, hyp_scores_out, status, s, st);
}

static int forward_any(mk_handle* h, const void* images, int img_fmt, const float* K0, const float* K1, int n_pairs, int H, int W,
                       unsigned long long seed, float* kps, float* depth, float* scr, float* dsc, float* scores,
                       float* kp_scores, float* final_scores, long long nn_pitch, float* pose, int* best_set, float* inl_mask,
                       int* sampled_out, int* status, void* ws, long long ws_bytes, void* stream) {
  Workspace w;
  MK_TRY(check_ws(h, 2 * n_pairs, n_pairs, H, W, ws, ws_bytes, w));
  const Geo g = make_geo(2 * n_pairs, n_pairs, H, W);
  cudaStream_t st = (cudaStream_t)stream;
  MK_TRY(run_extract(h, images, img_fmt, g, kps, depth, scr, dsc, w, st));
  MK_TRY(run_match(h, n_pairs, g.N, scores, kp_scores, final_scores, nn_pitch, w, st));
  return run_solve_handle(h, final_scores, nn_pitch, kps, depth, K0, K1, n_pairs, g.N, seed, nullptr, nullptr, pose, best_set,
                          inl_mask, sampled_out, nullptr, status, w, st);
}

int mk_forward(mk_handle* h, const float* images, const float* K0, const float* K1, int n_pairs, int H, int W,
               unsigned long long seed, float* kps, float* depth, float* scr, float* dsc, float* scores,
               float* kp_scores, float* final_scores, long long nn_pitch, float* pose, int* best_set, float* inl_mask,
               int* sampled_out, int* status, void* ws, long long ws_bytes, void* stream) {
  return forward_any(h, images, 0, K0, K1, n_pairs, H, W, seed, kps, depth, scr, dsc, scores, kp_scores, final_scores, nn_pitch,
                     pose, best_set, inl_mask, sampled_out, status, ws, ws_bytes, stream);
}

int mk_forward_u8(mk_handle* h, const unsigned char* images, const float* K0, const float* K1, int n_pairs, int H, int W,
                  unsigned long long seed, float* kps, float* depth, float* scr, float* dsc, float* scores,
                  float* kp_scores, float* final_scores, long long nn_pitch, float* pose, int* best_set, float* inl_mask,
                  int* sampled_out, int* status, void* ws, long long ws_bytes, void* stream) {
  return forward_any(h, images, 1, K0, K1, n_pairs, H, W, seed, kps, depth, scr, dsc, scores, kp_scores, final_scores, nn_pitch,
                     pose, best_set, inl_mask, sampled_out, status, ws, ws_bytes, stream);
}

int mk_forward_pairs(mk_handle* h, const float* kps0, const float* depth0, const float* scr0, const float* dsc0, int n0,
                     const float* kps1, const float* depth1, const float* scr1, const float* dsc1, int n1, const int* idx0,
                     const int* idx1, const float* K0, const float* K1, int n_pairs, unsigned long long seed, float* kps, float* depth,
                     float* scores, float* kp_scores, float* final_scores, long long nn_pitch, float* pose, int* best_set,
                     float* inl_mask, int* sampled_out, int* status, void* ws, long long ws_bytes, void* stream) {
  if (n_pairs <= 0 || n0 <= 0 || n1 <= 0 || !kps0 || !depth0 || !scr0 || !dsc0 || !kps1 || !depth1 || !scr1 || !dsc1 || !idx0 ||
      !idx1 || !K0 || !K1 || !kps || !depth || !pose) {
    set_last_error("mk_forward_pairs: n_pairs %d, bank sizes %d / %d must be positive; banks, indices, K, kps, depth and pose "
                   "must be non-NULL", n_pairs, n0, n1);
    return MK_ERR_INVALID;
  }
  Workspace w;
  MK_TRY(check_ws(h, 0, n_pairs, h ? h->geo_h : 0, h ? h->geo_w : 0, ws, ws_bytes, w));
  const Geo g = make_geo(0, n_pairs, h->geo_h, h->geo_w);
  cudaStream_t st = (cudaStream_t)stream;
  const BankView b0{kps0, depth0, scr0, dsc0, idx0, n0}, b1{kps1, depth1, scr1, dsc1, idx1, n1};
  MK_KERNEL("pairs.gather", bank_gather(b0, b1, n_pairs, g.N, w.DSCX, kps, depth, w.scr_copy, 2, st));
  MK_TRY(run_match(h, n_pairs, g.N, scores, kp_scores, final_scores, nn_pitch, w, st));
  MK_TRY(run_solve_handle(h, final_scores, nn_pitch, kps, depth, K0, K1, n_pairs, g.N, seed, nullptr, nullptr, pose, best_set,
                          inl_mask, sampled_out, nullptr, status, w, st));
  MK_KERNEL("pairs.index_check", bank_index_check(b0, b1, n_pairs, pose, status, st));
  return MK_OK;
}

// Pair p = (reference ref_idx[p] in role 0, query p in role 1).  The role-0 gather and the queries' extraction write
// disjoint halves of the operands, so the matcher and the solver then see exactly what mk_forward gives them.
static int localize_any(mk_handle* h, const float* ref_kps, const float* ref_depth, const float* ref_scr, const float* ref_dsc,
                        int n_ref, const int* ref_idx, const void* queries, int img_fmt, const float* K0, const float* K1,
                        int n_pairs, int H, int W, unsigned long long seed, float* kps, float* depth, float* scr, float* dsc,
                        float* scores, float* kp_scores, float* final_scores, long long nn_pitch, float* pose, int* best_set,
                        float* inl_mask, int* sampled_out, int* status, void* ws, long long ws_bytes, void* stream) {
  // every argument is checked before anything is launched
  if (!h || n_pairs < 1 || n_ref < 1 || !ref_kps || !ref_depth || !ref_scr || !ref_dsc || !ref_idx || !queries || !K0 || !K1 ||
      !kps || !depth || !final_scores || !pose) {
    set_last_error("mk_localize: n_pairs %d and n_ref %d must be positive; the handle, the reference bank, ref_idx, the "
                   "queries, K, kps, depth, final_scores and pose must be non-NULL", n_pairs, n_ref);
    return MK_ERR_INVALID;
  }
  if ((scores == nullptr) != (kp_scores == nullptr)) {
    set_last_error("mk_localize: scores and kp_scores are given together or both NULL (lean mode)");
    return MK_ERR_INVALID;
  }
  Workspace w;
  MK_TRY(check_ws(h, n_pairs, n_pairs, H, W, ws, ws_bytes, w));
  const Geo g = make_geo(n_pairs, n_pairs, H, W);
  long long pitch = nn_pitch;
  MK_TRY(resolve_pitch(pitch, g.N, "mk_localize: nn_pitch"));
  cudaStream_t st = (cudaStream_t)stream;
  const BankView ref{ref_kps, ref_depth, ref_scr, ref_dsc, ref_idx, n_ref};
  MK_KERNEL("localize.gather", bank_gather(ref, ref, n_pairs, g.N, w.DSCX, kps, depth, w.scr_copy, 1, st));
  float* q_scr = scr ? scr : w.scr_copy + (size_t)n_pairs * g.N;     // without scr_dev the scores go straight to the operand
  MK_TRY(run_extract(h, queries, img_fmt, g, kps + (size_t)n_pairs * 2 * g.N, depth + (size_t)n_pairs * g.N, q_scr, dsc, w, st, 1));
  MK_TRY(run_match(h, n_pairs, g.N, scores, kp_scores, final_scores, nn_pitch, w, st));
  MK_TRY(run_solve_handle(h, final_scores, nn_pitch, kps, depth, K0, K1, n_pairs, g.N, seed, nullptr, nullptr, pose, best_set,
                          inl_mask, sampled_out, nullptr, status, w, st));
  MK_KERNEL("localize.index_check", bank_index_check(ref, ref, n_pairs, pose, status, st));
  return MK_OK;
}

int mk_localize(mk_handle* h, const float* ref_kps, const float* ref_depth, const float* ref_scr, const float* ref_dsc, int n_ref,
                const int* ref_idx, const float* queries, const float* K0, const float* K1, int n_pairs, int H, int W,
                unsigned long long seed, float* kps, float* depth, float* scr, float* dsc, float* scores, float* kp_scores,
                float* final_scores, long long nn_pitch, float* pose, int* best_set, float* inl_mask, int* sampled_out,
                int* status, void* ws, long long ws_bytes, void* stream) {
  return localize_any(h, ref_kps, ref_depth, ref_scr, ref_dsc, n_ref, ref_idx, queries, 0, K0, K1, n_pairs, H, W, seed, kps, depth,
                      scr, dsc, scores, kp_scores, final_scores, nn_pitch, pose, best_set, inl_mask, sampled_out, status, ws,
                      ws_bytes, stream);
}

int mk_localize_u8(mk_handle* h, const float* ref_kps, const float* ref_depth, const float* ref_scr, const float* ref_dsc,
                   int n_ref, const int* ref_idx, const unsigned char* queries, const float* K0, const float* K1, int n_pairs,
                   int H, int W, unsigned long long seed, float* kps, float* depth, float* scr, float* dsc, float* scores,
                   float* kp_scores, float* final_scores, long long nn_pitch, float* pose, int* best_set, float* inl_mask,
                   int* sampled_out, int* status, void* ws, long long ws_bytes, void* stream) {
  return localize_any(h, ref_kps, ref_depth, ref_scr, ref_dsc, n_ref, ref_idx, queries, 1, K0, K1, n_pairs, H, W, seed, kps, depth,
                      scr, dsc, scores, kp_scores, final_scores, nn_pitch, pose, best_set, inl_mask, sampled_out, status, ws,
                      ws_bytes, stream);
}

int mk_pose_to_submission(const float* pose, int n_pairs, double* out, void* stream) {
  if (!pose || !out || n_pairs < 0) { set_last_error("null argument"); return MK_ERR_INVALID; }
  return pose_to_submission(pose, n_pairs, out, (cudaStream_t)stream);
}

long long mk_mutual_matches_ws_bytes(int B, int N) { return mutual_matches_ws_bytes(B, N); }
int mk_mutual_matches(const float* scores, long long nn_pitch, int B, int N, float min_conf, int* matches, float* match_scores,
                      int* count, void* ws, long long ws_bytes, void* stream) {
  return mutual_matches(scores, nn_pitch, B, N, min_conf, matches, match_scores, count, ws, ws_bytes, (cudaStream_t)stream);
}

long long mk_loss_search_ws_bytes(int B, int IM) { return (B > 0 && IM > 0) ? loss_search_ws_bytes(B, IM) : 0; }
int mk_loss_search(const float* final_scores, long long nn_pitch, const float* kps0, const float* depth0, const float* kps1,
                   const float* depth1, const float* K0, const float* K1, int B, int N, int it_matches, int it_ransac,
                   int n_sample, int n_corr, int n_ref, float th_ref, unsigned long long seed, const int* outer_idx,
                   const int* inner_idx, int* sampled_idx_out, int* inner_idx_out, unsigned int* inliers_out, int* status,
                   void* ws, long long ws_bytes, void* stream) {
  return loss_search(final_scores, nn_pitch, kps0, depth0, kps1, depth1, K0, K1, B, N, it_matches, it_ransac, n_sample, n_corr,
                     n_ref, th_ref, seed, outer_idx, inner_idx, sampled_idx_out, inner_idx_out, inliers_out, status, ws, ws_bytes,
                     (cudaStream_t)stream);
}
long long mk_loss_gradient_ws_bytes(int B, int it_matches, int n_sample) { return loss_gradient_ws_bytes(B, it_matches, n_sample); }
int mk_loss_gradient(const int* sampled_idx, const float* loss_value, const float* baseline, const float* mask_topk, int B, int N,
                     int it_matches, int n_sample, float* probs_grad, void* ws, long long ws_bytes, void* stream) {
  return loss_gradient(sampled_idx, loss_value, baseline, mask_topk, B, N, it_matches, n_sample, probs_grad, ws, ws_bytes,
                       (cudaStream_t)stream);
}

long long mk_launch_count(mk_handle* h) { return h ? h->launches : -1; }

int mk_pdl_enabled(void) { return pdl_enabled() ? 1 : 0; }

int mk_set_seed(mk_handle* h, unsigned long long seed, void* stream) {
  if (!h) return MK_ERR_INVALID;
  return seed_set(h->seed_dev, seed, (cudaStream_t)stream);
}

long long mk_workspace_offset(mk_handle* h, const char* name, int n_pairs, int H, int W) {
  if (!h || !name) return -1;
  const Geo g = make_geo(2 * n_pairs, n_pairs, H, W);
  uint8_t* base = reinterpret_cast<uint8_t*>(0x1000);     // fake base: only differences are used
  Workspace w = carve(base, h->cfg, g);
  const std::unordered_map<std::string, const void*> m = {
      {"P", w.P}, {"X", w.X}, {"XN", w.XN}, {"QKV", w.QKV}, {"ATT", w.ATT}, {"H1", w.H1}, {"F", w.F}, {"T1", w.T1},
      {"S1", w.S1}, {"O1", w.O1}, {"T2", w.T2}, {"S2", w.S2}, {"O2", w.O2}, {"T3", w.T3}, {"S3", w.S3}, {"CAT", w.CAT},
      {"MSG", w.MSG}, {"HM", w.HM}, {"T4k", w.T4k}, {"S4k", w.S4k}, {"T4d", w.T4d}, {"X32", w.X32}, {"QKV32", w.QKV32},
      {"KV", w.KV}, {"Y4k", w.Y4k}, {"Y4d", w.Y4d}, {"score_raw", w.score_raw}, {"DSCX", w.DSCX}, {"nrm2", w.nrm2},
      {"lse_r", w.lse_r}, {"lse_c", w.lse_c}, {"idx", w.sol.idx}, {"hyp_scores", w.sol.hyp_scores},
      {"hyp_Rt", w.sol.hyp_Rt}};
  auto it = m.find(name);
  if (it == m.end()) { set_last_error("unknown workspace buffer '%s'", name); return -1; }
  return (long long)(reinterpret_cast<const uint8_t*>(it->second) - base);
}

int mk_profile_enable(mk_handle* h, int enable) {
  if (!h) return MK_ERR_INVALID;
  for (auto& r : h->prof) { cudaEventDestroy(r.e0); cudaEventDestroy(r.e1); }
  h->prof.clear();
  h->profiling = enable != 0;
  return MK_OK;
}

// Synchronises the device and writes one line per kernel class: "<tag> <launch scopes> <total ms>\n".
int mk_profile_read(mk_handle* h, char* buf, int buf_bytes) {
  if (!h || !buf || buf_bytes <= 0) return MK_ERR_INVALID;
  MK_CUDA_CHECK(cudaDeviceSynchronize());
  std::vector<std::string> order;
  std::unordered_map<std::string, std::pair<int, double>> acc;
  for (auto& r : h->prof) {
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, r.e0, r.e1) != cudaSuccess) continue;
    if (!acc.count(r.tag)) order.push_back(r.tag);
    acc[r.tag].first += 1;
    acc[r.tag].second += ms;
  }
  std::string out;
  char line[256];
  for (auto& t : order) {
    snprintf(line, sizeof(line), "%s %d %.6f\n", t.c_str(), acc[t].first, acc[t].second);
    out += line;
  }
  if ((int)out.size() + 1 > buf_bytes) { set_last_error("profile buffer too small"); return MK_ERR_INVALID; }
  memcpy(buf, out.c_str(), out.size() + 1);
  return MK_OK;
}

// ---- operator-level entry points ---------------------------------------------------------------------------------
int mk_op_gemm(const mk_gemm_args* a, void* stream) {
  if (!a) return MK_ERR_INVALID;
  GemmParams p;
  memset(&p, 0, sizeof(p));
  p.M = a->M; p.N = a->N; p.k_chunks = a->k_chunks; p.chunks_per_tap = a->chunks_per_tap; p.num_taps = a->num_taps;
  for (int i = 0; i < 9; ++i) p.tap_shift[i] = a->tap_shift[i];
  p.groups = a->groups; p.a_row_group_off = a->a_row_group_off; p.a_col_group_off = a->a_col_group_off;
  p.a_col_base = a->a_col_base; p.b_row_group_off = a->b_row_group_off; p.act = a->act;
  p.bias = a->bias; p.bias_group_off = a->bias_group_off; p.gamma = a->gamma; p.beta = a->beta; p.ln_group_off = a->ln_group_off;
  p.out_f = a->out_f; p.out_f_ld = a->out_f_ld; p.out_f_group_off = a->out_f_group_off;
  p.out_h = (__half*)a->out_h; p.out_h_ld = a->out_h_ld; p.out_h_group_off = a->out_h_group_off;
  p.res_h = (const __half*)a->res_h; p.res_h_ld = a->res_h_ld; p.res_h_group_off = a->res_h_group_off;
  p.aux = a->aux; p.aux_group_mask = a->aux_group_mask; p.pad_h2 = a->pad_h2; p.pad_w2 = a->pad_w2; p.tok_per_img = a->tok_per_img;
  p.eps = a->eps; p.n_valid = a->n_valid; p.inv_temp = a->inv_temp; p.dustbin = a->dustbin;
  p.part_row = reinterpret_cast<float2*>(a->part_row); p.part_col = reinterpret_cast<float2*>(a->part_col); p.part_ld = a->part_ld;
  p.lse_r = a->lse_r; p.lse_c = a->lse_c; p.scr0 = a->scr0; p.scr1 = a->scr1; p.lse_bound = a->lse_bound;
  p.out_pitch = a->out_pitch > 0 ? a->out_pitch : a->n_valid;
  p.out_tma = (a->final_scores && p.out_pitch % 4 == 0 && reinterpret_cast<uintptr_t>(a->final_scores) % 16 == 0 &&
               (!a->scores || (reinterpret_cast<uintptr_t>(a->scores) % 16 == 0 && reinterpret_cast<uintptr_t>(a->kp_scores) % 16 == 0))) ? 1 : 0;
  p.scores = a->scores; p.kp_scores = a->kp_scores; p.final_scores = a->final_scores;
  GemmOperand A{a->a, a->a_rows, a->a_cols, a->a_ld}, B{a->b, a->b_rows, a->b_cols, a->b_ld};
  return launch_gemm(a->epi, A, B, p, (cudaStream_t)stream, a->impl);
}

int mk_op_patch_gather(const float* img, void* P, int n_img, int H, int W, int kpad, float* X, const float* cls_pos,
                       int D, void* stream) {
  return patch_gather(img, P, n_img, H, W, kpad, X, cls_pos, D, (cudaStream_t)stream);
}
int mk_op_ingest_u8(const unsigned char* img, void* P, int n_img, int H, int W, int kpad, float* X, const float* cls_pos,
                    int D, void* stream) {
  return ingest_u8(img, P, n_img, H, W, kpad, X, cls_pos, D, (cudaStream_t)stream);
}
int mk_op_layernorm(const float* x, const float* w, const float* b, void* out, int rows, int D, float eps, int mode,
                    int gh, int gw, void* stream) {
  return layernorm(x, w, b, out, rows, D, eps, mode, gh, gw, (cudaStream_t)stream);
}
int mk_op_attention(const void* qkv, void* out, int n_img, int T, int D, int heads, int impl, void* stream) {
  return attention_dispatch(qkv, out, n_img, T, D, heads, impl, (cudaStream_t)stream);
}
int mk_op_linattn(const float* qkv, float* kv_part, float* kv, void* msg, int n_img, int Gn, int h2, int w2, float eps,
                  void* stream) {
  MK_TRY(linattn_kv(qkv, kv_part, kv, n_img, Gn, h2, w2, (cudaStream_t)stream));
  return linattn_msg(qkv, kv, msg, n_img, Gn, h2, w2, eps, (cudaStream_t)stream);
}
int mk_op_matcher_reduce(const float* part_row, const float* part_col, const float* dustbin, int B, int N, int part_ld,
                         float* lse_r, float* lse_c, void* stream) {
  return matcher_lse_reduce(part_row, part_col, dustbin, B, N, part_ld, lse_r, lse_c, (cudaStream_t)stream);
}
long long mk_op_sample_workspace_bytes(int B, int IM) { return (long long)sampler_workspace_bytes(B, IM) + 512; }
int mk_op_sample(const float* fs, int B, int N, long long pitch, int IM, int n_sample, unsigned long long seed, void* ws,
                 long long ws_bytes, int* idx_out, int* status, void* stream) {
  MK_TRY(resolve_pitch(pitch, N, "mk_op_sample: pitch"));
  if ((long long)sampler_workspace_bytes(B, IM) + 256 > ws_bytes) { set_last_error("sampler workspace too small"); return MK_ERR_INVALID; }
  MK_CUDA_CHECK(cudaMemsetAsync(status, 0, sizeof(int), (cudaStream_t)stream));
  // the seed word lives at the (256-byte aligned) end of the caller's workspace
  const size_t off = ((size_t)sampler_workspace_bytes(B, IM) + 255) & ~(size_t)255;
  unsigned long long* sd = reinterpret_cast<unsigned long long*>(reinterpret_cast<uint8_t*>(ws) + off);
  MK_TRY(seed_set(sd, seed, (cudaStream_t)stream));
  return sample_outer(fs, B, N, pitch, IM, n_sample, sd, ws, idx_out, status, (cudaStream_t)stream);
}
int mk_op_kabsch(const double* H, double* R, int n, void* stream) { return kabsch_batch(H, R, n, (cudaStream_t)stream); }

}  // extern "C"
