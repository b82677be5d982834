// Host-callable launchers of the non-GEMM kernels.
#pragma once
#include "common.cuh"

namespace mk {

// vit_ops.cu
int patch_gather(const float* img, void* P, int n_img, int H, int W, int kpad, float* X, const float* cls_pos, int D, cudaStream_t s);
int layernorm(const float* x, const float* w, const float* b, void* out, int rows, int D, float eps, int mode, int gh, int gw, cudaStream_t s);
// the final norm as fp32 channel-major [n_img, D, N] from the residual [n_img * (N + 1), D] (cls row dropped)
int layernorm_channel_major(const float* x, const float* w, const float* b, float* out, int n_img, int N, int D, float eps,
                            cudaStream_t s);
int attention(const void* qkv, void* out, int n_img, int T, int D, int heads, cudaStream_t s);      // mma.sync version (v1, kept as a cross-check)
int attention_tc(const void* qkv, void* out, int n_img, int T, int D, int heads, cudaStream_t s);   // wgmma / TMA version
int attention_dispatch(const void* qkv, void* out, int n_img, int T, int D, int heads, int impl, cudaStream_t s);

// io_ops.cu (the steps either side of the path: image ingest, submission packing)
int ingest_u8(const uint8_t* img, void* P, int n_img, int H, int W, int kpad, float* X, const float* cls_pos, int D, cudaStream_t s);
int pose_to_submission(const float* pose, int n, double* out, cudaStream_t s);

// head_ops.cu
int linattn_kv_chunks(int h2, int w2);
int linattn_kv(const float* qkv, float* kv_part, float* kv, int n_img, int G, int h2, int w2, cudaStream_t s);
int linattn_msg(const float* qkv, const float* kv, void* msg, int n_img, int G, int h2, int w2, float eps, cudaStream_t s);
int kp_head_out(const float* y, const float* w_depth, const float* w_xy, const float* w_score, float* depth, float* kps,
                float* score_raw, float* scr, int n_img, int gh, int gw, int depth_sigmoid, float max_depth,
                float down_factor, int use_softmax, cudaStream_t s);
int desc_out(const float* y, float* dsc_cm, void* dsc_x, float* nrm2, int n_img, int gh, int gw, int normalize, cudaStream_t s);
int matcher_lse_reduce(const void* part_row, const void* part_col, const float* dustbin, int B, int N, int part_ld, float* lse_r,
                       float* lse_c, cudaStream_t s);
// one bank of extracted images (kps [n,2,N], depth [n,1,N], scr [n,1,N], dsc [n,128,N]) and the image index of every pair
struct BankView { const float *kps, *depth, *scr, *dsc; const int* idx; int count; };
int bank_gather(const BankView& b0, const BankView& b1, int P, int N, void* dsc_x, float* kps_out, float* depth_out, float* scr_out,
                cudaStream_t s);
int bank_index_check(const BankView& b0, const BankView& b1, int P, float* pose, int* status, cudaStream_t s);

// matches.cu: featureMatcher.get_matches_list, batched (include/mickey_b200.h mk_mutual_matches)
long long mutual_matches_ws_bytes(int B, int N);
int mutual_matches(const float* scores, long long pitch, int B, int N, float min_conf, int* matches, float* match_scores,
                   int* count, void* ws, long long ws_bytes, cudaStream_t s);

// ransac.cu
struct RansacParams {
  int it_matches, it_ransac, n_sample, n_corr, n_refine;
  float th_inlier, th_soft;
  const unsigned long long* seed;     // device pointer
};
int seed_set(unsigned long long* s, unsigned long long v, cudaStream_t st);
int seed_advance(unsigned long long* s, cudaStream_t st);
size_t sampler_workspace_bytes(int B, int IM);
// final_scores: [B][N][N] with row pitch `pitch` floats (N = contiguous)
int sample_outer(const float* final_scores, int B, int N, long long pitch, int IM, int n_sample, const unsigned long long* seed,
                 void* ws, int* idx_out, int* status, cudaStream_t st, int invalid_bits = 1);
int ransac_solve(const float* final_scores, long long pitch, const float* kps0, const float* d0, const float* kps1, const float* d1,
                 const float* K0, const float* K1, int B, int N, const RansacParams& rp, const int* outer_idx,
                 const int* inner_idx, float* hyp_scores, float* hyp_Rt, int* counters, float* pose,
                 int* best_set, float* inl_mask, int* best_hyp, cudaStream_t st);
// H [n][9], R [n][9] fp64 row-major, device: R = kabsch_rotation(H) per matrix (ransac_dev.cuh)
int kabsch_batch(const double* H, double* R, int n, cudaStream_t st);
constexpr int SOLVER_COUNTER_BASE = 4;      // counters: [0] status bits, [1] pairs finished, [4 + b] blocks of pair b finished

// loss.cu: MetricPoseLoss's draws, refinement search and REINFORCE gradient (include/mickey_b200.h mk_loss_search)
constexpr int LOSS_MAX_C = 16, LOSS_MAX_S = 2048;
long long loss_search_ws_bytes(int B, int IM);
int loss_search(const float* fs, long long pitch, const float* kps0, const float* d0, const float* kps1, const float* d1,
                const float* K0, const float* K1, int B, int N, int IM, int IR, int S, int C, int n_ref, float th_ref,
                unsigned long long seed, const int* outer_idx, const int* inner_idx, int* sampled_out, int* inner_out,
                uint32_t* inl_out, int* status, void* ws, long long ws_bytes, cudaStream_t st);
long long loss_gradient_ws_bytes(int B, int IM, int S);
int loss_gradient(const int* sampled, const float* loss_value, const float* baseline, const float* mask, int B, int N, int IM,
                  int S, float* grad, void* ws, long long ws_bytes, cudaStream_t st);

// loss_tail.cu: the loss's differentiable tail, forward and backward (include/mickey_b200.h mk_loss_tail_forward)
long long loss_tail_ws_bytes(int B, int N, int IM, int IR, int S);

}  // namespace mk
