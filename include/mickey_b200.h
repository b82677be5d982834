/* mickey_b200 — C ABI of the H100-native MicKey inference hot path.
 *
 * The reference (nianticlabs/mickey) has no native boundary: its hot path is the Python method
 * MickeyRelativePose.forward (lib/models/MicKey/compute_pose.py:20-37).  This library is what a
 * maintainer binds instead of the three Python stages that method calls; each entry point names the
 * reference interface it replaces.  INTEGRATION.md shows the ctypes stub.
 *
 * Conventions: extern "C", plain pointers and sizes, int status (0 = OK, < 0 = error, message via
 * mk_last_error()), no exceptions cross the ABI.  Every pointer named *_dev is a DEVICE pointer owned
 * by the caller (PyTorch on the Python side); kernels are enqueued asynchronously on `stream`
 * (a cudaStream_t passed as void*).  One handle per device; a handle is not re-entrant.
 */
#ifndef MICKEY_B200_H
#define MICKEY_B200_H

#ifdef __cplusplus
extern "C" {
#endif

typedef struct mk_handle mk_handle;

/* Mirrors the keys of the reference config that the hot path reads
 * (config/MicKey/curriculum_learning.yaml:4-32,89-96; config/default.py). */
typedef struct mk_config {
  int embed_dim, depth, heads;        /* DINOv2 variant (dinov2.py:306-342): 384/12/6, 768/12/12, 1024/24/16 */
  int down_factor;                    /* MICKEY.DINOV2.DOWN_FACTOR (14) */
  int block_dims[4];                  /* MICKEY.KP_HEADS.BLOCKS_DIM (512,256,128,64) */
  int desc_dim;                       /* MICKEY.DSC_HEAD.LAST_DIM (128) */
  int use_softmax;                    /* MICKEY.KP_HEADS.USE_SOFTMAX */
  int depth_sigmoid;                  /* MICKEY.KP_HEADS.USE_DEPTHSIGMOID */
  float max_depth;                    /* MICKEY.KP_HEADS.MAX_DEPTH */
  int kp_pos_enc, dsc_pos_enc;        /* *.POS_ENCODING */
  int norm_dsc;                       /* MICKEY.DSC_HEAD.NORM_DSC */
  float temperature;                  /* FEATURE_MATCHER.DUAL_SOFTMAX.TEMPERATURE */
  int use_dustbin;                    /* FEATURE_MATCHER.DUAL_SOFTMAX.USE_DUSTBIN */
  int it_matches, it_ransac;          /* PROCRUSTES.IT_MATCHES / IT_RANSAC */
  int num_sampled, num_corr, num_refine;   /* NUM_SAMPLED_MATCHES / NUM_CORR_3D_3D / NUM_REFINEMENTS */
  float th_inlier, th_soft_inlier;    /* TH_INLIER / TH_SOFT_INLIER */
} mk_config;

/* ---- lifecycle (replaces MickeyRelativePose.__init__, compute_pose.py:9-18, and builder.py:5-20) ---- */
int mk_create(int device, const mk_config* cfg, mk_handle** out);
int mk_destroy(mk_handle* h);
const char* mk_last_error(void);
const char* mk_version(void);
/* sizeof the struct named `type` ("mk_config", "mk_gemm_args", ...) as compiled into the library, or -1 for a name it
 * does not know (binding self-check). */
int mk_sizeof(const char* type);

/* Register a packed weight / table tensor that lives in device memory (replaces load_state_dict,
 * builder.py:11-13; the packing itself — fp16 cast, BatchNorm folding, per-head stacking — is done by
 * mickey_b200/engine.py and documented in DESIGN.md).  dtype: 0 = fp32, 1 = fp16. */
int mk_set_tensor(mk_handle* h, const char* name, const void* ptr_dev, int dtype, long long numel);
/* Declare the image geometry the size-dependent tables ("patch.posb", "patch.clspos", "head.pe") were
 * built for, and check that every tensor the pipeline needs has been registered. */
int mk_finalize(mk_handle* h, int img_h, int img_w);

long long mk_workspace_bytes(mk_handle* h, int n_pairs, int img_h, int img_w);
/* Workspace of a call that extracts n_img images and matches / solves n_pairs pairs: (n, 0) for mk_extract_images,
 * (0, P) for mk_forward_pairs; (2P, P) equals mk_workspace_bytes(P). */
long long mk_workspace_bytes_for(mk_handle* h, int n_img, int n_pairs, int img_h, int img_w);
/* Byte offset of a named intermediate buffer inside the workspace (debugging / stage-wise tests; names and
 * layouts are listed in DESIGN.md §3: "X", "F", "CAT", "Y4d", ...). */
long long mk_workspace_offset(mk_handle* h, const char* name, int n_pairs, int img_h, int img_w);

/* ---- stage 1: feature extraction for 2*n_pairs images
 * replaces MicKey_Extractor.forward (mickey_extractor.py:43-58) for image0 and image1 plus
 * get_abs_kpts_coordinates / prepare_kpts_dsc (compute_correspondences.py:20-43).
 * images_dev fp32 [2*n_pairs, 3, H, W] (all image0 first, then all image1), values in [0,1].
 * kps [2n,2,N] px coords, depth [2n,1,N], scr [2n,1,N], dsc [2n,128,N]  (N = (H/14)*(W/14)). */
int mk_extract(mk_handle* h, const float* images_dev, int n_pairs, int img_h, int img_w, float* kps_dev,
               float* depth_dev, float* scr_dev, float* dsc_dev, void* ws_dev, long long ws_bytes, void* stream);

/* Same stage fed by uint8 images straight from the decoder (SURVEY.md §8 f1): images_u8_dev uint8 [2*n_pairs, H, W, 3],
 * RGB, HWC — what lib/datasets/utils.py:61-71 (cv2.imread -> cvtColor -> resize) holds before `.float() / 255`
 * (:74); the division, the crop to multiples of 14 (mickey_extractor.py:46) and the patch gather happen in one kernel,
 * bit-identical to mk_extract on the reference's float tensor. */
int mk_extract_u8(mk_handle* h, const unsigned char* images_u8_dev, int n_pairs, int img_h, int img_w, float* kps_dev,
                  float* depth_dev, float* scr_dev, float* dsc_dev, void* ws_dev, long long ws_bytes, void* stream);

/* Stage 1 for any number of images (n_img >= 1, odd counts included), e.g. a feature bank for mk_forward_pairs: one
 * Map-free reference image and its queries are extracted once each instead of once per pair.  images_dev fp32
 * [n_img, 3, H, W] / images_u8_dev uint8 [n_img, H, W, 3]; kps [n_img,2,N], depth [n_img,1,N], scr [n_img,1,N],
 * dsc [n_img,128,N], bit-identical to what mk_extract writes for the same image.  Workspace:
 * mk_workspace_bytes_for(n_img, 0).  The matcher operands this leaves in the workspace are not meant for mk_match. */
int mk_extract_images(mk_handle* h, const float* images_dev, int n_img, int img_h, int img_w, float* kps_dev,
                      float* depth_dev, float* scr_dev, float* dsc_dev, void* ws_dev, long long ws_bytes, void* stream);
int mk_extract_images_u8(mk_handle* h, const unsigned char* images_u8_dev, int n_img, int img_h, int img_w, float* kps_dev,
                         float* depth_dev, float* scr_dev, float* dsc_dev, void* ws_dev, long long ws_bytes, void* stream);

/* ---- training: the frozen DINOv2 backbone alone (mickey_b200/dinov2.py wraps it as a drop-in module).  Replaces
 * DinoVisionTransformer.forward_features (dinov2.py:221-236) followed by the extractor's
 * x_norm_patchtokens.permute(0, 2, 1).reshape(B, C, h, w).float() (mickey_extractor.py:49-51), so that the heads can
 * run in torch in train mode.
 * images_dev fp32 [n_img, 3, H, W] (H, W multiples of 14, at least 98, equal to the finalized geometry); the patch
 * gather, the patch embedding and every block run exactly as in mk_extract, then the final LayerNorm writes out_dev fp32
 * [n_img, D, N] channel-major (cls token dropped).  out rounded to fp16 is bit for bit the feature image mk_extract
 * gives the heads.  Only the backbone's tensors need to be registered.  Workspace: mk_backbone_ws_bytes(n_img, H, W)
 * bytes; it holds the six backbone buffers ("P", "X", "XN", "QKV", "ATT", "H1") at the offsets mk_workspace_offset names
 * for n_img images.  Bad arguments (a NULL pointer, n_img < 1, a bad geometry, an unfinalized handle, a small workspace)
 * return MK_ERR_INVALID and launch nothing.  mk_backbone_ws_bytes returns -1 for a bad geometry or count. */
long long mk_backbone_ws_bytes(mk_handle* h, int n_img, int img_h, int img_w);
int mk_backbone_features(mk_handle* h, const float* images_dev, int n_img, int img_h, int img_w, float* out_dev,
                         void* ws_dev, long long ws_bytes, void* stream);

/* ---- stage 2: dual-softmax matcher
 * replaces featureMatcher/dualSoftmax.forward (feature_matcher.py:48-83), kp_matrix_scores
 * (compute_correspondences.py:46-50) and `final_scores = scores * kp_scores` (compute_pose.py:23).
 * Uses the descriptors/scores left in the workspace by mk_extract.  Outputs fp32 [n_pairs, N, N];
 * scores_dev AND kp_scores_dev may both be NULL ("lean" mode: only final_scores, the one matrix the solver reads, is
 * materialised: 17 instead of 47 MB per 720x540 pair); the same holds for mk_forward / mk_forward_u8.
 * nn_pitch: row pitch of the three outputs in floats.  N (or 0) = the reference's contiguous [n_pairs, N, N].  A pitch
 * that is a multiple of 4 (e.g. N rounded up to 32: 1952 for N = 1938) makes every row 16-byte aligned, which lets the
 * outputs leave through TMA tensor stores as full 128-byte lines; a caller then views the buffers as
 * [n_pairs, N, nn_pitch][:, :, :N].  N = 1938 itself cannot be described by a tensor map (7752-byte rows). */
int mk_match(mk_handle* h, int n_pairs, float* scores_dev, float* kp_scores_dev, float* final_scores_dev, long long nn_pitch,
             void* ws_dev, long long ws_bytes, void* stream);

/* ---- stage 3: probabilistic Procrustes RANSAC
 * replaces e2eProbabilisticProcrustesSolver.estimate_pose_vectorized (probabilisticProcrustes.py:183-348).
 * final_scores_dev fp32 [n_pairs, N, N] with row pitch nn_pitch floats (N or 0 = contiguous).
 * K0/K1 fp32 [n_pairs,3,3].  pose_dev fp32 [n_pairs,13] = R row-major (9) | t (3) | soft inlier count (1).
 * outer_idx_dev int32 [n_pairs*IT_MATCHES, NUM_SAMPLED] / inner_idx_dev int32 [n_pairs*IT_MATCHES*IT_RANSAC, 3]:
 * when non-NULL they replace the two random draws (:231, :251) — the parity tests inject the reference's.
 * seed: non-zero = (re)seed the solver's counter-based generator; 0 = continue the device-side sequence
 * (the state lives in device memory and advances after every solve, so a captured CUDA graph of this call
 * draws fresh numbers on every replay).
 * Optional outputs (NULL to skip): best_set_dev int32 [n_pairs] (index into the IT_MATCHES sampled sets),
 * inlier_mask_dev fp32 [n_pairs, NUM_SAMPLED] (hard inliers of the winning set at the final pose),
 * sampled_idx_out_dev int32 [n_pairs*IT_MATCHES, NUM_SAMPLED] (the cells that were drawn),
 * hyp_scores_out_dev fp32 [n_pairs, IT_MATCHES*IT_RANSAC].  status_dev int32[1]: bit0 = torch.multinomial would
 * raise on the outer draw (some pair's final_scores sums to zero, holds a NaN, an inf or a negative cell, or has
 * fewer than NUM_SAMPLED cells), bit1 = a stream's candidate list was truncated or came short (probability < 1e-13),
 * bit2 = non-finite hypothesis; any of these bits gives the reference's zero pose (R = 0, t = 0, inliers = 0 for the
 * whole batch, probabilisticProcrustes.py:331-342).  A pair with 0 < positive cells < NUM_SAMPLED is not a failure,
 * as in the reference: every positive cell is drawn and the lowest-index zero cells fill the set.  When such a set
 * holds fewer than 3 positive weights, the inner draw takes the positive ones and fills the triple with the entries
 * that follow them in the set, cyclically (ATen fills with zero-weight entries too, in an unspecified order). */
int mk_solve_pose(mk_handle* h, const float* final_scores_dev, long long nn_pitch, const float* kps_dev, const float* depth_dev,
                  const float* K0_dev, const float* K1_dev, int n_pairs, int n_kpts, unsigned long long seed,
                  const int* outer_idx_dev, const int* inner_idx_dev, float* pose_dev, int* best_set_dev,
                  float* inlier_mask_dev, int* sampled_idx_out_dev, float* hyp_scores_out_dev, int* status_dev,
                  void* ws_dev, long long ws_bytes, void* stream);

/* ---- stage 3 without a handle: the same solver for callers that have no finalized handle, e.g. the training model's
 * validation (mickey_b200/procrustes.py wraps it as a drop-in e2eProbabilisticProcrustesSolver).  Arguments, outputs and
 * the status bits are those of mk_solve_pose, with N and every PROCRUSTES value given by the caller: it_matches /
 * it_ransac / num_sampled / num_corr / num_refine / th_inlier / th_soft_inlier are IT_MATCHES / IT_RANSAC /
 * NUM_SAMPLED_MATCHES / NUM_CORR_3D_3D / NUM_REFINEMENTS / TH_INLIER / TH_SOFT_INLIER.  kps_dev [2B,2,N], depth_dev
 * [2B,1,N] (image-0 rows first), K0/K1 fp32 [B,3,3].  The seed is written into the workspace: there is no state across
 * calls, and a call with seed s draws what mk_solve_pose draws after being reseeded with s (so, with the handle's
 * PROCRUSTES values, every output is the same bits).
 * Sizes, from the kernels: 1 <= B <= 65535 and 1 <= it_matches <= 65535 (grid dimensions), N >= 1 with N*N < 2^31 (int32
 * cell indices), it_ransac >= 1 with it_matches*it_ransac < 2^31 and B*it_matches < 2^31, num_sampled a multiple of 256
 * (the hypothesis kernel scans a set across 256 threads) up to 2048 (the sampler's selection sorts 2048 candidates),
 * num_corr = 3 (the inner draw and the hypotheses' Kabsch take three correspondences), num_refine >= 0, both thresholds
 * finite and positive.  The shipped configurations use 2048 / 3 / 4.
 * Workspace: mk_procrustes_ws_bytes(B, N, it_matches, it_ransac, num_sampled) bytes, 256-byte aligned (-1 for
 * unsupported sizes).  Bad arguments (a NULL input, pose or workspace, an unsupported size, nn_pitch < N, a small
 * workspace) return MK_ERR_INVALID with a message and launch nothing. */
long long mk_procrustes_ws_bytes(int B, int N, int it_matches, int it_ransac, int num_sampled);
int mk_procrustes_solve(const float* final_scores_dev, long long nn_pitch, const float* kps_dev, const float* depth_dev,
                        const float* K0_dev, const float* K1_dev, int B, int N, int it_matches, int it_ransac,
                        int num_sampled, int num_corr, int num_refine, float th_inlier, float th_soft_inlier,
                        unsigned long long seed, const int* outer_idx_dev, const int* inner_idx_dev, float* pose_dev,
                        int* best_set_dev, float* inlier_mask_dev, int* sampled_idx_out_dev, float* hyp_scores_out_dev,
                        int* status_dev, void* ws_dev, long long ws_bytes, void* stream);

/* ---- grading a Map-free submission: the per-frame errors of the benchmark's MetricManager (benchmark/metrics.py:
 * trans_err, rot_err with the sin variant, reproj_err), fp64.  mickey_b200/mapfree_eval.py restates the benchmark's host
 * logic around it.  No handle, no workspace, no state between calls; enqueued on `stream`.  For P frames, row-major
 * device arrays:
 *   q_est_dev [P,4], t_est_dev [P,3]: each estimate as its submission line holds it (world-to-camera, qw qx qy qz tx ty tz);
 *   q_gt_dev [P,4], t_gt_dev [P,3]:   the ground truth of poses.txt, in the same convention;
 *   K_dev [P,3,3]:                    each frame's intrinsics;
 *   grid_dev [MK_VCRE_POINTS,3]:      the virtual points, mickey_b200.loss.vcre_grid();
 *   W, H:                             the image size both projections are clipped to (shared by the call's frames).
 * A quaternion need not be unit: as in the benchmark, its norm scales the camera centre (by 1/|q|^4) but not the rotation.
 * Out: err_dev fp64 [P,3] = trans_err (m), rot_err (deg), reproj_err (px); csrc/mapfree_eval.cu states each formula.
 * A frame's values are the same bits alone, inside any batch and on every run.
 * Bad arguments (a NULL pointer, P < 1 or P > MK_MAPFREE_MAX_FRAMES, W < 1 or H < 1) return MK_ERR_INVALID with a
 * message and launch nothing. */
#define MK_VCRE_POINTS 196
#define MK_MAPFREE_MAX_FRAMES 67108863   /* one warp per frame: 32 * P threads index in int32 */
int mk_mapfree_frame_metrics(const double* q_est_dev, const double* t_est_dev, const double* q_gt_dev,
                             const double* t_gt_dev, const double* K_dev, const double* grid_dev, int P, int W, int H,
                             double* err_dev, void* stream);

/* ---- whole path: replaces MickeyRelativePose.forward (compute_pose.py:20-37) ---- */
int mk_forward(mk_handle* h, const float* images_dev, const float* K0_dev, const float* K1_dev, int n_pairs,
               int img_h, int img_w, unsigned long long seed, float* kps_dev, float* depth_dev, float* scr_dev,
               float* dsc_dev, float* scores_dev, float* kp_scores_dev, float* final_scores_dev, long long nn_pitch,
               float* pose_dev, int* best_set_dev, float* inlier_mask_dev, int* sampled_idx_out_dev, int* status_dev,
               void* ws_dev, long long ws_bytes, void* stream);

int mk_forward_u8(mk_handle* h, const unsigned char* images_u8_dev, const float* K0_dev, const float* K1_dev, int n_pairs,
                  int img_h, int img_w, unsigned long long seed, float* kps_dev, float* depth_dev, float* scr_dev,
                  float* dsc_dev, float* scores_dev, float* kp_scores_dev, float* final_scores_dev, long long nn_pitch,
                  float* pose_dev, int* best_set_dev, float* inlier_mask_dev, int* sampled_idx_out_dev, int* status_dev,
                  void* ws_dev, long long ws_bytes, void* stream);

/* ---- stages 2 + 3 on pairs drawn from feature banks: replaces MickeyRelativePose.forward (compute_pose.py:20-37) for
 * pairs (bank0[idx0[p]], bank1[idx1[p]]) whose features mk_extract_images already computed.
 * bank b: kps [n_b,2,N], depth [n_b,1,N], scr [n_b,1,N], dsc [n_b,128,N] as mk_extract_images writes them, extracted at
 * the finalized geometry (so N x N stays square); bank0 and bank1 may be the same tensors.  idx0_dev / idx1_dev int32
 * [n_pairs] (device).  One gather kernel builds the matcher's role-0 / role-1 descriptor operands (the hi/lo fp16
 * split of mk_extract) and the solver's pair-major operands; the matcher and the solver then run as in mk_forward, so
 * the outputs are bit-identical to mk_forward on the same images with the same seed.
 * Out: kps_dev [2*n_pairs,2,N], depth_dev [2*n_pairs,1,N] (required: the solver reads them; role-0 rows first), and
 * scores / kp_scores / final_scores / nn_pitch / pose / best_set / inlier_mask / sampled_idx as in mk_forward.
 * status_dev bit3 = an index outside [0, n_b): nothing outside a bank is read, and the batch gets the zero pose of the
 * other status bits (R = 0, t = 0, inliers = 0).  Workspace: mk_workspace_bytes_for(0, n_pairs). */
int mk_forward_pairs(mk_handle* h, const float* kps0_dev, const float* depth0_dev, const float* scr0_dev, const float* dsc0_dev,
                     int n0, const float* kps1_dev, const float* depth1_dev, const float* scr1_dev, const float* dsc1_dev, int n1,
                     const int* idx0_dev, const int* idx1_dev, const float* K0_dev, const float* K1_dev, int n_pairs,
                     unsigned long long seed, float* kps_dev, float* depth_dev, float* scores_dev, float* kp_scores_dev,
                     float* final_scores_dev, long long nn_pitch, float* pose_dev, int* best_set_dev, float* inlier_mask_dev,
                     int* sampled_idx_out_dev, int* status_dev, void* ws_dev, long long ws_bytes, void* stream);

/* ---- after the path: submission records (replaces the per-pair loop of submission.py:43-59)
 * pose_dev fp32 [n_pairs,13] as written by mk_forward / mk_solve_pose -> out_dev fp64 [n_pairs, 9] =
 * qw qx qy qz | tx ty tz | inliers | valid.  Quaternion = transforms3d.quaternions.mat2quat(R) (principal eigenvector
 * of the symmetric 4x4 K(R), w >= 0) computed in fp64; valid = 0 where the reference skips the frame
 * (np.isnan(R).any() or np.isnan(t).any() or np.isinf(t).any(), submission.py:51-52).  One D2H copy per batch. */
int mk_pose_to_submission(const float* pose_dev, int n_pairs, double* out_dev, void* stream);

/* ---- correspondences: replaces featureMatcher.get_matches_list (lib/models/MicKey/modules/utils/feature_matcher.py:19-46),
 * batched.  scores_dev fp32 [B, N, N] with row pitch nn_pitch floats (N or 0 = contiguous; pairs N * nn_pitch floats
 * apart), e.g. the final_scores of mk_forward.  As in the reference the last row and column are dropped: (i, j), i, j < N-1,
 * is a match when j is the first argmax of row i, i the first argmax of column j (a NaN counts as maximal) and
 * exp(scores[i][j]) > min_conf (exp in double, rounded to fp32).  Per pair b, sorted by score descending and equal scores
 * by ascending i (the reference's sort leaves their order open):
 * matches_dev int32 [B, N-1, 2] = (i, j), match_scores_dev fp32 [B, N-1], count_dev int32 [B]; entries from count[b] on
 * are (-1, -1) / 0.  2 <= N <= 4097, finite min_conf.  ws_dev: mk_mutual_matches_ws_bytes(B, N) bytes, 8-byte aligned.
 * Bad arguments return MK_ERR_INVALID (message via mk_last_error) and launch nothing.  Deterministic (no atomics). */
int mk_mutual_matches(const float* scores_dev, long long nn_pitch, int B, int N, float min_conf, int* matches_dev,
                      float* match_scores_dev, int* count_dev, void* ws_dev, long long ws_bytes, void* stream);
long long mk_mutual_matches_ws_bytes(int B, int N);

/* ---- training loss: replaces the non-differentiated part of MetricPoseLoss.RANSAC_vectorized
 * (lib/models/MicKey/modules/loss/loss_class.py:79-329); mickey_b200/loss.py adds the differentiable tail in autograd.
 * No handle: the calls only need the caller's tensors and a workspace.
 *
 * mk_loss_search: the outer draw, the inner draws and the refinement search.
 * final_scores_dev fp32 [B, N, N] with row pitch nn_pitch floats (N or 0 = contiguous); kps0/kps1 [B,2,N] px coords,
 * depth0/depth1 [B,1,N], K0/K1 fp32 [B,3,3] (K_color0/1).  it_matches / it_ransac / n_sample / n_corr / n_ref / th_ref are
 * GENERATE_HYPOTHESES.IT_MATCHES / IT_RANSAC, SAMPLER.NUM_SAMPLES_MATCHES (S), NUM_CORR_3d3d (C), NUM_REF_STEPS and
 * INLIER_REF_TH; S a multiple of 256 up to 2048, 1 <= C <= 16.
 * outer_idx_dev int32 [B*IM, S] / inner_idx_dev int32 [B*IM*IR, C] (positions 0..S-1 in the set): when non-NULL they replace
 * the two random draws (:138, :159); they must hold valid indices.  seed: the draws' counter-based generator.
 * Out: sampled_idx_out_dev int32 [B*IM, S] (the drawn cells; the injected ones when given), inner_idx_out_dev int32
 * [B*IM*IR, C] (in draw order), inliers_out_dev uint32 [B*IM*IR, S/32]: inliers_final of every hypothesis (:168-191), bit
 * (i & 31) of word i / 32 for set position i.  status_dev int32[1]: bit0 = the outer torch.multinomial would raise (as
 * mk_solve_pose), bit1 = a candidate list was truncated (probability < 1e-13), MK_LOSS_STATUS_PRECHECK = the batch holds a
 * NaN, an inf or a negative cell (:126-131; the search is skipped, inliers 0, inner -1), MK_LOSS_STATUS_INNER = a set's
 * scores sum to zero, so the inner torch.multinomial would raise.  Any of these bits gives the reference's zero result
 * (num_valid_h = 0).  A set with fewer than C positive scores is not a failure, as in torch: the positive entries are drawn
 * first and the entries that follow the last pick, cyclically, fill the rest.  Workspace: mk_loss_search_ws_bytes(B, IM).
 * Sizes: S any multiple of 32 up to 2048 (64 and 512 in the reference's configs; the inlier masks are whole 32-bit words)
 * and 1 <= C <= min(16, S), S <= N*N; anything else is MK_ERR_INVALID.
 *
 * mk_loss_gradient: probs_grad_dev fp32 [B, N, N] contiguous = mask_b (sum_i [cell in S_i] loss_i - count baseline_b) / IM
 * (:251-261, :299-316) from sampled_idx_dev int32 [B*IM, S] (any order), loss_value_dev fp32 [B*IM], baseline_dev fp32 [B]
 * and mask_topk_dev fp32 [B].  Summed in iteration order without atomics (deterministic); cells never drawn are 0.
 * Workspace: mk_loss_gradient_ws_bytes(B, IM, S).
 * Both calls reject bad arguments with MK_ERR_INVALID (message via mk_last_error) before launching anything. */
#define MK_LOSS_STATUS_PRECHECK 16
#define MK_LOSS_STATUS_INNER 32
int mk_loss_search(const float* final_scores_dev, long long nn_pitch, const float* kps0_dev, const float* depth0_dev,
                   const float* kps1_dev, const float* depth1_dev, const float* K0_dev, const float* K1_dev, int B, int N,
                   int it_matches, int it_ransac, int n_sample, int n_corr, int n_ref, float th_ref, unsigned long long seed,
                   const int* outer_idx_dev, const int* inner_idx_dev, int* sampled_idx_out_dev, int* inner_idx_out_dev,
                   unsigned int* inliers_out_dev, int* status_dev, void* ws_dev, long long ws_bytes, void* stream);
long long mk_loss_search_ws_bytes(int B, int it_matches);
int mk_loss_gradient(const int* sampled_idx_dev, const float* loss_value_dev, const float* baseline_dev, const float* mask_topk_dev,
                     int B, int N, int it_matches, int n_sample, float* probs_grad_dev, void* ws_dev, long long ws_bytes,
                     void* stream);
long long mk_loss_gradient_ws_bytes(int B, int it_matches, int n_sample);

/* ---- training loss, the differentiable tail (loss_class.py:140-152, 199-248) in CUDA: mickey_b200/loss.py's opt-in
 * alternative to its autograd tail (MetricPoseLoss(cfg, cuda_tail=True)).  No handle.
 *
 * mk_loss_tail_forward: per hypothesis the weighted Procrustes on its inliers_final mask (fp64 Kabsch), the soft inlier
 * score over all S entries, and the VCRE (loss_type 0) or POSE_ERR (loss_type 1) loss; per outer iteration the score
 * softmax, with the null hypothesis (null_score = TH_OUTLIERS * S, null_loss = MAX_LOSS_SOFT/VALUE) when
 * null_hypothesis != 0.  Inputs: sampled_idx_dev int32 [B*IM, S] and inliers_dev uint32 [B*IM*IR, S/32] as mk_loss_search
 * writes them; kps0/kps1 [B,2,N], depth0/depth1 [B,1,N], K0/K1 (K_color), Kori0/Kori1 (Kori_color) fp32 [B,3,3], T_0to1
 * fp32 [B,4,4] and grid_dev fp32 [MK_VCRE_POINTS,3] (mickey_b200.loss.vcre_grid()).  Out: loss_value_dev, loss_rot_dev,
 * loss_trans_dev fp32 [B*IM]; status_dev int32[1] = MK_LOSS_TAIL_STATUS_NONFINITE when some hypothesis's R or t is not
 * finite (the reference's zero result, :213-223).  The workspace keeps the forward's state for the backward: pass the
 * same workspace, untouched, to mk_loss_tail_backward.
 *
 * mk_loss_tail_backward: from the upstream gradients of loss_value / loss_rot / loss_trans fp32 [B*IM] (the other
 * arguments as given to the forward), writes every entry of dkps0/dkps1 fp32 [B,2,N] and ddepth0/ddepth1 fp32 [B,1,N]
 * (0 at keypoints no set drew).  The rotation's backward needs no SVD (csrc/loss_tail.cu).  No float atomics: the
 * gradients are the same bits on every run.
 *
 * Workspace: mk_loss_tail_ws_bytes(B, N, IM, IR, S) bytes (-1 for unsupported sizes).  Sizes: 1 <= B <= 65535, N >= 1 with
 * N*N < 2^31, IM, IR >= 1 with B*IM*IR < 2^31, S a multiple of 32 up to 2048; inlier_3d_th finite and positive,
 * score_temperature finite and non-zero.  Bad arguments (a NULL pointer, an unsupported size or parameter, a small
 * workspace) return MK_ERR_INVALID with a message and launch nothing. */
#define MK_LOSS_TAIL_STATUS_NONFINITE 1
long long mk_loss_tail_ws_bytes(int B, int N, int it_matches, int it_ransac, int n_sample);
int mk_loss_tail_forward(const int* sampled_idx_dev, const unsigned int* inliers_dev, const float* kps0_dev,
                         const float* depth0_dev, const float* kps1_dev, const float* depth1_dev, const float* K0_dev,
                         const float* K1_dev, const float* Kori0_dev, const float* Kori1_dev, const float* T_0to1_dev,
                         const float* grid_dev, int B, int N, int it_matches, int it_ransac, int n_sample, int loss_type,
                         int soft_clipping, int null_hypothesis, float inlier_3d_th, float score_temperature,
                         float null_score, float null_loss, float* loss_value_dev, float* loss_rot_dev,
                         float* loss_trans_dev, int* status_dev, void* ws_dev, long long ws_bytes, void* stream);
int mk_loss_tail_backward(const int* sampled_idx_dev, const unsigned int* inliers_dev, const float* kps0_dev,
                          const float* depth0_dev, const float* kps1_dev, const float* depth1_dev, const float* K0_dev,
                          const float* K1_dev, const float* Kori0_dev, const float* Kori1_dev, const float* T_0to1_dev,
                          const float* grid_dev, int B, int N, int it_matches, int it_ransac, int n_sample, int loss_type,
                          int soft_clipping, int null_hypothesis, float inlier_3d_th, float score_temperature,
                          const float* grad_loss_value_dev, const float* grad_loss_rot_dev,
                          const float* grad_loss_trans_dev, float* dkps0_dev, float* dkps1_dev, float* ddepth0_dev,
                          float* ddepth1_dev, void* ws_dev, long long ws_bytes, void* stream);

/* ---- training: the dual-softmax matcher on the caller's descriptors and its backward (mickey_b200/dual_softmax.py wraps
 * both as a torch.autograd.Function).  Replaces dualSoftmax.forward (feature_matcher.py:64-83), kp_matrix_scores
 * (compute_correspondences.py:46-50) and scores * kp_scores (model.py:201), and autograd through them.  No handle.
 *
 * mk_dual_softmax: dsc0_dev / dsc1_dev fp32 [B, 128, N] channel-major (prepare_kpts_dsc's layout), scr0 / scr1 fp32 [B, N]
 * (both or neither), dustbin_dev a device fp32 scalar (USE_DUSTBIN) or NULL, temperature T > 0, 2 <= N <= 8192.
 * Writes scores, kp_scores and final_scores together (scr required), final_scores alone, or scores alone, fp32
 * [B, N, N] with row pitch nn_pitch floats (N or 0 = contiguous; a multiple of 4 lets them leave through TMA as in
 * mk_match); without scr, kp_scores = 1 and final_scores = scores.  lse_r_dev / lse_c_dev fp32 [B, npad] (npad = N
 * rounded up to 128): the log2-domain log-sum-exps of every row / column, which the backward reads.  unit_norm = 1 when
 * every descriptor has norm <= 1 (DSC_HEAD.NORM_DSC): it selects mk_match's fixed-shift row / column partials, and with
 * it the outputs are bit-identical to mk_match on the same descriptors (mk_match under NORM_DSC True for unit_norm = 1,
 * False for 0).  The descriptors enter the tensor cores as hi + lo fp16 pairs (as in mk_extract): |dsc| must stay below
 * 65504, and each value is carried to about 2^-22 relative plus 2^-25 absolute.
 *
 * mk_dual_softmax_backward: the forward's inputs and its lse_r / lse_c, plus the gradients of the three outputs,
 * grad_scores / grad_kp / grad_final fp32 [B, N, pitch] (pitch >= N floats, 0 = N; pairs N rows apart), any of which
 * may be NULL but not all; grad_kp needs scr.  Out: ddsc0 / ddsc1 fp32 [B, 128, N], dscr0 / dscr1 fp32 [B, N] (required
 * with scr, ignored without), ddustbin fp32 [1] (required with the dustbin; the sum over the batch).  The backward runs
 * in fp32 on the CUDA cores and writes no N x N intermediate; it is deterministic, and a pair's ddsc / dscr are the same
 * bits alone or inside a batch.
 *
 * Workspaces: mk_dual_softmax_ws_bytes(B, N) / mk_dual_softmax_backward_ws_bytes(B, N) bytes, 256-byte aligned (0 for
 * unsupported sizes).  Bad arguments return MK_ERR_INVALID and launch nothing.  Both calls always use the wgmma and
 * fp32 kernels.  Capturing them in a CUDA graph is not tested. */
long long mk_dual_softmax_ws_bytes(int B, int N);
long long mk_dual_softmax_backward_ws_bytes(int B, int N);
int mk_dual_softmax(const float* dsc0_dev, const float* dsc1_dev, const float* scr0_dev, const float* scr1_dev,
                    const float* dustbin_dev, float temperature, int B, int N, int unit_norm, float* scores_dev,
                    float* kp_scores_dev, float* final_scores_dev, long long nn_pitch, float* lse_r_dev, float* lse_c_dev,
                    void* ws_dev, long long ws_bytes, void* stream);
int mk_dual_softmax_backward(const float* dsc0_dev, const float* dsc1_dev, const float* scr0_dev, const float* scr1_dev,
                             const float* dustbin_dev, float temperature, int B, int N, const float* lse_r_dev,
                             const float* lse_c_dev, const float* grad_scores_dev, long long gs_pitch, const float* grad_kp_dev,
                             long long gk_pitch, const float* grad_final_dev, long long gf_pitch, float* ddsc0_dev,
                             float* ddsc1_dev, float* dscr0_dev, float* dscr1_dev, float* ddustbin_dev, void* ws_dev,
                             long long ws_bytes, void* stream);

/* ---- training: the heads' linear-attention transformer, Transformer_self_att (att_layers/transformer.py:75-103), forward
 * and backward (mickey_b200/head_transformer.py wraps both as a torch.autograd.Function).  No handle: the parameters change
 * at every optimizer step, so every call takes the caller's parameter pointers, one table per layer.
 *
 * Every parameter is an fp32 device pointer, contiguous and 16-byte aligned, in the reference's layout: q_proj, k_proj,
 * v_proj and merge [128, 128], mlp0 [256, 256] (mlp.0), mlp2 [128, 256] (mlp.2), norm1_w / norm1_b / norm2_w / norm2_b
 * [128].  In mk_htr_layer_grads the same names are the gradients to write (overwritten, not accumulated); NULL skips one.
 *
 * mk_head_transformer: x_dev fp32 [B, 128, h, w] contiguous, pe_dev the positional encoding [128, 256, 256] (posEnc.pe,
 * added as pe[:, :h, :w]) or NULL, out_dev fp32 [B, 128, h, w].  save = 1 keeps every layer's activations in the
 * workspace for mk_head_transformer_backward, which reads them from that workspace (saved_dev); save = 0 runs the forward
 * only, in a smaller workspace.  The output is the same bits either way.
 * mk_head_transformer_backward: grad_out_dev fp32 [B, 128, h, w] contiguous; grad_x_dev fp32 [B, 128, h, w] or NULL.
 * grads_host is an array of num_layers tables.  Only what a requested gradient needs is computed.
 *
 * All arithmetic is fp32 (FMA on the CUDA cores).  Both calls are deterministic, use no atomics, and an image's output and
 * input gradient are the same bits alone and inside a batch (weight gradients sum over the batch).  Workspaces:
 * mk_head_transformer_ws_bytes / mk_head_transformer_backward_ws_bytes bytes (-1 for a bad geometry: B, h, w >= 1,
 * 1 <= num_layers <= 1024, B <= 65535, B h w <= 4,194,240 = 65535 * 64).  Bad arguments return MK_ERR_INVALID and
 * launch nothing. */
typedef struct mk_htr_layer {
  const float* q_proj; const float* k_proj; const float* v_proj; const float* merge; const float* mlp0; const float* mlp2;
  const float* norm1_w; const float* norm1_b; const float* norm2_w; const float* norm2_b;
} mk_htr_layer;
typedef struct mk_htr_layer_grads {
  float* q_proj; float* k_proj; float* v_proj; float* merge; float* mlp0; float* mlp2;
  float* norm1_w; float* norm1_b; float* norm2_w; float* norm2_b;
} mk_htr_layer_grads;
long long mk_head_transformer_ws_bytes(int B, int h, int w, int num_layers, int save);
long long mk_head_transformer_backward_ws_bytes(int B, int h, int w, int num_layers);
int mk_head_transformer(const float* x_dev, const float* pe_dev, int B, int h, int w, const mk_htr_layer* layers_host,
                        int num_layers, float* out_dev, int save, void* ws_dev, long long ws_bytes, void* stream);
int mk_head_transformer_backward(const void* saved_dev, const float* grad_out_dev, int B, int h, int w,
                                 const mk_htr_layer* layers_host, int num_layers, float* grad_x_dev,
                                 mk_htr_layer_grads* grads_host, void* ws_dev, long long ws_bytes, void* stream);

/* ---- training: the heads' residual block, BasicBlock (extractor_utils.py:12-35), forward and backward with TF32 wgmma
 * convolutions and batch norm (mickey_b200/resblock.py wraps both as a torch.autograd.Function).  No handle: every call
 * takes the caller's parameter pointers, because the parameters change at every optimizer step.
 *
 * Parameters are fp32 device pointers, contiguous, in the torch layout: w1 [cout, cin, 3, 3], w2 [cout, cout, 3, 3], wsc
 * [cout, cin, 1, 1] (exactly when cin != cout; NULL for the identity shortcut), the BN weights, biases and running
 * statistics [cout].  momentum1 / momentum2 are the exponential-average factors of this call (the module's momentum, or
 * 1 / num_batches_tracked for the cumulative average); running_var receives the unbiased batch variance.
 *
 * mk_resblock_forward: x_dev fp32 [B, cin, h, w] with element strides x_strides_host[4] (any layout); out_dev fp32
 * [B, cout, h, w] contiguous.  flags: MK_RB_TRAIN (batch statistics, running statistics updated; otherwise the running
 * statistics normalise and nothing is updated), MK_RB_RELU (the final ReLU), MK_RB_BN (batch norm present; otherwise
 * both BN layers are identities), MK_RB_SAVE (also write the channel-major operand copies the backward needs).  saved_dev
 * (mk_resblock_saved_bytes) receives what mk_resblock_backward reads; ws_dev (mk_resblock_ws_bytes) is scratch that can
 * be freed when the forward has run.
 * mk_resblock_backward: grad_out_dev fp32 [B, cout, h, w] with element strides g_strides_host[4]; out_dev the forward's
 * output (its ReLU mask; may be NULL without MK_RB_RELU); flags as in the forward.  want is a mask of MK_RB_GRAD_* bits; a
 * requested gradient's pointer in grads_host must be set, and each is overwritten, not accumulated.  Contractions whose
 * results nobody wants are skipped: without MK_RB_GRAD_X there is no data gradient through conv1 or the shortcut.
 *
 * Channel counts are multiples of 32 in [32, 4096], B, h, w >= 1 and B (h+2)(w+2) <= 2^24; training-mode batch norm
 * needs B h w >= 2.  Workspace sizes: -1 for a bad geometry.  Bad arguments return MK_ERR_INVALID and launch nothing.
 * Deterministic: no atomics, bit-identical run to run. */
#define MK_RB_TRAIN 1
#define MK_RB_RELU 2
#define MK_RB_SAVE 4
#define MK_RB_BN 8
#define MK_RB_GRAD_X 1
#define MK_RB_GRAD_W1 2
#define MK_RB_GRAD_W2 4
#define MK_RB_GRAD_WSC 8
#define MK_RB_GRAD_BN1_W 16
#define MK_RB_GRAD_BN1_B 32
#define MK_RB_GRAD_BN2_W 64
#define MK_RB_GRAD_BN2_B 128
typedef struct mk_resblock_params {
  const float* w1; const float* w2; const float* wsc;
  const float* bn1_w; const float* bn1_b; float* bn1_mean; float* bn1_var;
  const float* bn2_w; const float* bn2_b; float* bn2_mean; float* bn2_var;
  float eps1, eps2, momentum1, momentum2;
} mk_resblock_params;
typedef struct mk_resblock_grads {
  float* dx; float* w1; float* w2; float* wsc; float* bn1_w; float* bn1_b; float* bn2_w; float* bn2_b;
} mk_resblock_grads;
long long mk_resblock_ws_bytes(int B, int h, int w, int cin, int cout);
long long mk_resblock_saved_bytes(int B, int h, int w, int cin, int cout);
long long mk_resblock_backward_ws_bytes(int B, int h, int w, int cin, int cout);
int mk_resblock_forward(const float* x_dev, const long long* x_strides_host, int B, int h, int w, int cin, int cout,
                        const mk_resblock_params* params_host, int flags, float* out_dev, void* saved_dev,
                        long long saved_bytes, void* ws_dev, long long ws_bytes, void* stream);
int mk_resblock_backward(const void* saved_dev, const float* grad_out_dev, const long long* g_strides_host,
                         const float* out_dev, int B, int h, int w, int cin, int cout, const mk_resblock_params* params_host,
                         int flags, int want, const mk_resblock_grads* grads_host, void* ws_dev, long long ws_bytes,
                         void* stream);

/* ---- training: the heads' output layers (mickey_extractor.py:81-142, 160-178, 199-218, 246-249), forward and backward
 * in fp32 (mickey_b200/heads.py wraps both as a torch.autograd.Function).  No handle.  x = rb4's output.
 *
 * kind                  weight   output [B, k, h, w]
 * MK_HO_SCORE_SOFTMAX   [1, C]   p = e / (sum e + eps), e = exp((r - (mean r + eps)) / temperature) mask, per image
 * MK_HO_SCORE_SIGMOID   [1, C]   sigmoid(r) mask
 * MK_HO_OFFSET          [2, C]   sigmoid(r)
 * MK_HO_DEPTH           [1, C]   r
 * MK_HO_DEPTH_SIGMOID   [1, C]   max_depth sigmoid(r)
 * MK_HO_DESC_L2         NULL     x / sqrt(sum_c x^2 + 1e-10)                                  (k = C)
 * with r = W x (the 1x1 convolution) and mask zeroing 3 cells at each border.  eps_dev is a device scalar (the det head's
 * `eps` Parameter), read by the kernel.
 *
 * mk_head_out_forward: x_dev fp32 [B, C, h, w] with element strides x_strides_host[4] (any layout); weight_dev fp32 [k, C]
 * contiguous; out_dev fp32 [B, k, h, w] contiguous.  norm_dev fp32 [B, h, w] receives the descriptor's per-pixel norm for
 * the backward (MK_HO_DESC_L2 only; NULL skips it).
 * mk_head_out_backward: out_dev and norm_dev as the forward wrote them, grad_out_dev fp32 [B, k, h, w] contiguous; grad_x_dev
 * fp32 [B, C, h, w] contiguous and grad_w_dev fp32 [k, C] (no weight gradient for MK_HO_DESC_L2), each NULL to skip, and
 * overwritten, not accumulated.  x_dev is read only for the weight gradient.  Workspace: mk_head_out_backward_ws_bytes
 * bytes, 256-byte aligned (0 for MK_HO_DESC_L2; -1 for a bad geometry).
 *
 * All arithmetic is fp32; the per-image and per-pixel reductions and the weight gradient's pixel slots accumulate in fp64 in
 * a fixed order.  No atomics: bit-identical run to run, an image's output and input gradient do not depend on the rest of
 * the batch, and every layout of x gives the same bits.  Limits: B, h, w >= 1, B h w <= 2^26, 1 <= C <= 4096.  Bad
 * arguments return MK_ERR_INVALID and launch nothing. */
#define MK_HO_SCORE_SOFTMAX 0
#define MK_HO_SCORE_SIGMOID 1
#define MK_HO_OFFSET 2
#define MK_HO_DEPTH 3
#define MK_HO_DEPTH_SIGMOID 4
#define MK_HO_DESC_L2 5
long long mk_head_out_backward_ws_bytes(int kind, int B, int h, int w, int C);
int mk_head_out_forward(int kind, const float* x_dev, const long long* x_strides_host, int B, int C, int h, int w,
                        const float* weight_dev, const float* eps_dev, float temperature, float max_depth, float* out_dev,
                        float* norm_dev, void* stream);
int mk_head_out_backward(int kind, const float* x_dev, const long long* x_strides_host, int B, int C, int h, int w,
                         const float* weight_dev, float temperature, float max_depth, const float* out_dev,
                         const float* norm_dev, const float* grad_out_dev, float* grad_x_dev, float* grad_w_dev, void* ws_dev,
                         long long ws_bytes, void* stream);

/* (Re)seed the solver's device-side generator on `stream` (used in front of a CUDA-graph replay of mk_forward
 * captured with seed = 0). */
int mk_set_seed(mk_handle* h, unsigned long long seed, void* stream);

/* Number of kernel launches issued by this library since the handle was created (for bench.py). */
long long mk_launch_count(mk_handle* h);
/* 1 when kernels are launched with programmatic dependent launch (the default), 0 under MICKEY_PDL=0.  The environment
 * is read once per process, at the first launch or the first call of this function. */
int mk_pdl_enabled(void);
/* Per-kernel-class device timing: while enabled every launch issued by the stages is bracketed by CUDA
 * events on the launch stream; mk_profile_read synchronises and writes "<class> <scopes> <total ms>" lines. */
int mk_profile_enable(mk_handle* h, int enable);
int mk_profile_read(mk_handle* h, char* buf, int buf_bytes);

/* ---- operator-level entry points (unit tests of single kernels; not needed by an integrator) ---- */
typedef struct mk_gemm_args {
  int epi;                 /* 0 STORE_H, 1 RESID_F, 2 PATCH, 3 CONV, 4 STORE_F, 5 LN, 6 LSE (row + column partials), 7 DUAL */
  int impl;                /* 0 default (wgmma), 1 wgmma, 2 SIMT debug kernel; 3 / 4: the persistent wgmma kernel with /
                              without two-CTA pairs sharing B, on any grid (the epilogues it does not serve run as 1) */
  const void* a; long long a_rows, a_cols, a_ld;
  const void* b; long long b_rows, b_cols, b_ld;
  int M, N, k_chunks, chunks_per_tap, num_taps;
  int tap_shift[9];
  int groups, a_row_group_off, a_col_group_off, a_col_base, b_row_group_off;
  int act;                 /* 0 none, 1 GELU(erf), 2 ReLU */
  const float* bias; int bias_group_off;
  const float* gamma; const float* beta; int ln_group_off;
  float* out_f; long long out_f_ld, out_f_group_off;
  void* out_h; long long out_h_ld, out_h_group_off;
  const void* res_h; long long res_h_ld, res_h_group_off;
  const float* aux; int aux_group_mask;
  int pad_h2, pad_w2, tok_per_img;
  float eps;
  int n_valid; float inv_temp;
  const float* dustbin;
  float* part_row; float* part_col; int part_ld;   /* LSE out: float2 (max, sum) partials, [groups][part_ld/64 | part_ld/32 slots][part_ld];
                                                      part_ld = n_valid rounded up to 128 */
  const float* lse_r; const float* lse_c;          /* DUAL in: log2-domain log-sum-exp per row / column, [groups, part_ld] (mk_op_matcher_reduce) */
  const float* scr0; const float* scr1;
  float* scores; float* kp_scores; float* final_scores;
  float lse_bound;         /* LSE: > 0 = every |A.B| <= lse_bound (normalised descriptors): fixed-shift partials; 0 = true maxima */
  long long out_pitch;     /* DUAL: row pitch of the outputs in floats (0 = n_valid); % 4 == 0 selects the TMA-store path */
} mk_gemm_args;

int mk_op_gemm(const mk_gemm_args* args, void* stream);
int mk_op_patch_gather(const float* img, void* patches_h, int n_img, int H, int W, int kpad, float* x_f,
                       const float* cls_pos, int D, void* stream);
int mk_op_ingest_u8(const unsigned char* img_u8, void* patches_h, int n_img, int H, int W, int kpad, float* x_f,
                    const float* cls_pos, int D, void* stream);
int mk_op_layernorm(const float* x, const float* w, const float* b, void* out_h, int rows, int D, float eps, int mode,
                    int gh, int gw, void* stream);
/* impl: 0 = default (wgmma), 1 = wgmma/TMA kernel, 2 = mma.sync kernel (cross-check) */
int mk_op_attention(const void* qkv_h, void* out_h, int n_img, int T, int D, int heads, int impl, void* stream);
/* kv_part_f: scratch [n_img, G, ceil(h2*w2/32), 8, 272] fp32 */
int mk_op_linattn(const float* qkv_f, float* kv_part_f, float* kv_f, void* msg_h, int n_img, int G, int h2, int w2, float eps,
                  void* stream);
int mk_op_matcher_reduce(const float* part_row, const float* part_col, const float* dustbin, int B, int N, int part_ld,
                         float* lse_r, float* lse_c, void* stream);
int mk_op_sample(const float* final_scores, int B, int N, long long pitch, int IM, int n_sample, unsigned long long seed, void* ws,
                 long long ws_bytes, int* idx_out, int* status, void* stream);
long long mk_op_sample_workspace_bytes(int B, int IM);
/* The solver's fp64 Kabsch rotation on n matrices, one per thread: H, R device [n, 9] row-major.  R is the rotation
   maximising tr(R H) (det R = +1); H == 0 gives the identity, a NaN or +-inf anywhere in H gives nine NaNs.
   MK_ERR_INVALID for n < 0 or a null pointer. */
int mk_op_kabsch(const double* H, double* R, int n, void* stream);

/* The residual block's TF32 wgmma convolution GEMM alone, on caller buffers (padded NHWC geometry of B, h, w as in
   mk_resblock_forward; R = B (h+2)(w+2), Rp = R rounded up to 4; taps 9 (3x3, padding 1) or 1 (1x1)):
     mode 0 forward: a = X [R, cin] padded NHWC, b = W [cout, cin, taps]           -> out [R, cout]
     mode 1 dgrad:   a = dZ [R, cout] padded NHWC, b = W [cout, cin, taps]         -> out [R, cin]
     mode 2 wgrad:   a = dZ^T [cout, Rp], b = X^T [cin, Rp] (channel-major)        -> out = dW [cout, cin, taps]
   W is rounded to TF32 on the way; a and b of mode 2 are used as given (the tensor core reads them as TF32).  Rows of the
   pad ring in out are unspecified.  Workspace: mk_op_conv_tf32_ws_bytes bytes (-1 for bad arguments). */
/* Byte offsets of the residual block's intermediates, for element-wise checks of each stage.  saved_off[6]: in the forward's
   saved region, z1, z2 (pre-BN conv outputs, fp32 padded NHWC [R, cout]), a1 (BN1-apply + ReLU, TF32 padded NHWC),
   a1^T (TF32 [cout, Rp]), x^T (TF32 [cin, Rp]), and the statistics mean1, rstd1, mean2, rstd2 (fp32 [4][cout]).  bwd_off[6]:
   in the backward's workspace after a call, g = grad_out * mask (fp32 [R, cout]), dz (TF32 padded NHWC [R, cout]: dz1 when
   the call computed dX or dW1/dBN1, else dz2), dz^T (TF32 [cout, Rp], the last BN backward's), dA1 (conv2's data gradient,
   fp32 [R, cout]), conv1's and the shortcut's data gradients (fp32 [R, cin]). */
int mk_resblock_layout(int B, int h, int w, int cin, int cout, long long* saved_off, long long* bwd_off);
long long mk_op_conv_tf32_ws_bytes(int mode, int B, int h, int w, int cin, int cout, int taps);
int mk_op_conv_tf32(int mode, const float* a, const float* b, float* out, int B, int h, int w, int cin, int cout, int taps,
                    void* ws, long long ws_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MICKEY_B200_H */
