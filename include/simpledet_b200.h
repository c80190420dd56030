/*
 * simpledet_b200 — C ABI of the H100-native (sm_90a) detection hot path.
 *
 * This header is the drop-in boundary (SURVEY.md §8b).  Every entry point replaces one MXNet
 * operator of tusen-ai/simpledet; the reference interface it replaces is cited as
 * `file:line` relative to the reference checkout.  Conventions (all entry points):
 *
 *   - plain pointers + sizes, no framework types.  Pointers named `d_*` or documented as
 *     "device" are CUDA device pointers on the current device; the caller owns every buffer,
 *     the library allocates nothing on the device and keeps no global state.
 *   - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream).  All work is
 *     stream-ordered on it; no entry point synchronises the device unless documented.
 *   - return value: SDET_OK (0) or an sdet_status error code; sdet_last_error() returns a
 *     thread-local human-readable message.  The library never aborts (the reference's
 *     CHECK / LOG(FATAL) macros become error codes).
 *   - fp32 tensors, dense row-major, shapes exactly as the reference operators define them.
 */
#ifndef SIMPLEDET_B200_H_
#define SIMPLEDET_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum sdet_status {
  SDET_OK = 0,
  SDET_ERR_INVALID_ARG = 1, /* bad shape / null pointer / parameter out of range */
  SDET_ERR_UNSUPPORTED = 2, /* valid for the reference, outside this build's limits */
  SDET_ERR_CUDA = 3,        /* a CUDA runtime call failed; message has cudaGetErrorString */
  SDET_ERR_WORKSPACE = 4    /* caller-provided workspace too small */
} sdet_status;

#define SDET_MAX_LEVELS 8
#define SDET_MAX_POOLED 32 /* max pooled_size per axis handled by the RoIAlign kernels */

/* ABI version of this header; bumped on any signature change. */
int sdet_abi_version(void);
/* sha256 prefix of the sources/headers/flags the library was built from; simpledet_b200.build.source_digest()
 * recomputes it from the tree, so a stale prebuilt binary is detected (__graft_entry__.smoke() checks it). */
const char* sdet_build_digest(void);
/* Thread-local message of the last failing call on this thread ("" if none). */
const char* sdet_last_error(void);
/* Number of kernels this library has launched in this process (all threads); used by bench.py's
 * `gpu_launches` claim. */
uint64_t sdet_launch_count(void);

/* ------------------------------------------------------------------------------------------
 * _contrib_ROIAlign_v2   (operator_cxx/contrib/roi_align_v2.cc:170-228, kernel
 *                         roi_align_v2-inl.h:61-153, driver :157-195)
 *   data  (B,C,H,W) device, rois (B,N,4) device [x1,y1,x2,y2] image px, image = n / N.
 *   out, argmax_x, argmax_y (B,N,C,PH,PW) device.  argmax_x/argmax_y may both be NULL
 *   (inference: they are hidden outputs, roi_align_v2.cc:175-178) — then they are not written.
 *   workspace: optional device scratch of sdet_roi_align_v2_workspace(B,N) bytes, 16B-aligned.
 *   With it the per-roi sample tables are computed once per roi by a small pre-kernel instead of
 *   once per (roi, channel group) CTA; NULL / 0 selects the inline path (identical results). */
size_t sdet_roi_align_v2_workspace(int B, int N);
int sdet_roi_align_v2_forward(const float* data, const float* rois, float* out, float* argmax_x,
                              float* argmax_y, int B, int N, int C, int H, int W, int pooled_h,
                              int pooled_w, float spatial_scale, void* workspace,
                              size_t workspace_bytes, void* stream);
/* Same operator with an explicit kernel choice (tests and A/B timing; results are bit-identical):
 *   path = 0  automatic;  1  per-roi kernel (roi_align.cu);  2  band-stationary kernel (bulk-TMA staged feature
 *   bands, roi_align_band.cu) for every roi it can take, per-roi kernel for the rest;  3  channels-last kernel
 *   (roi_align_cl.cu): the features are re-laid to NHWC in the scratch part of a workspace of
 *   sdet_fpn_roi_align_v2_workspace() bytes, then gathered with warp = 64 channels of one output bin.
 *   Automatic = 3 when the workspace is that large and no argmax planes are asked for, else 2, else 1.
 *   path_used (host int, may be NULL): 0 inline per-roi, 1 planned per-roi, 2 band-stationary, 3 channels-last.
 *   out (and argmax_x / argmax_y) need only 4-byte alignment; 16-byte stores are used only where the address allows. */
int sdet_roi_align_v2_forward_ex(const float* data, const float* rois, float* out, float* argmax_x,
                                 float* argmax_y, int B, int N, int C, int H, int W, int pooled_h,
                                 int pooled_w, float spatial_scale, void* workspace,
                                 size_t workspace_bytes, void* stream, int path, int* path_used);

/* _backward_ROIAlign_v2  (operator_cxx/contrib/roi_align_v2.cu:17-85 kernel, :88-143 driver).
 *   ograd, argmax_x, argmax_y (B,N,C,PH,PW); grad_data (B,C,H,W).
 *   accumulate = 0 -> kWriteTo (grad_data is zero-filled first, :130-133), 1 -> kAddTo.
 *   grad_rois (B,N,4) may be NULL; when given it is zero-filled (:139-141). */
int sdet_roi_align_v2_backward(const float* ograd, const float* argmax_x, const float* argmax_y,
                               float* grad_data, float* grad_rois, int B, int N, int C, int H,
                               int W, int pooled_h, int pooled_w, int accumulate, void* stream);

/* Deterministic backward, same arguments.  Returns bit for bit the reference's backward run serially: per gradient
 * plane, kWriteTo starts from +0.0 (kAddTo from the existing value) and the contributions are added with
 * round-to-nearest fadd in ascending index ((n*C + c)*PH + ph)*PW + pw, each index adding its corners TL, TR, BL, BR
 * as separate adds ((ograd * wy) * wx, rounded product by product); argmax -1 entries add nothing.  No global
 * atomics, no allocation, no host synchronisation.  Every check happens before the first launch or memset; on an
 * error nothing is launched and the outputs are untouched.  SDET_ERR_UNSUPPORTED: W > 12288 (a plane row must fit
 * one shared-memory band) or pooled_size > SDET_MAX_POOLED.  torch's deterministic mode selects it (ops.py). */
int sdet_roi_align_v2_backward_ordered(const float* ograd, const float* argmax_x, const float* argmax_y,
                                       float* grad_data, float* grad_rois, int B, int N, int C, int H,
                                       int W, int pooled_h, int pooled_w, int accumulate, void* stream);

/* Fused FPN RoIAlign: replaces  assign_layer_fpn (models/FPN/assign_layer_fpn.py:17-40) /
 * mxnext.tvm.fpn_roi_assign  +  num_levels x _contrib_ROIAlign_v2  +  add_n
 * (models/FPN/builder.py:573-605).  Each roi is sampled on its assigned level only; the result
 * equals the reference's sum over levels because a zeroed roi yields an all-zero output
 * (roi_align_v2-inl.h:111-117).
 *   feats[l]  device pointer to level l data (B,C,H[l],W[l]);  strides[l] the level's stride
 *   (spatial_scale = 1/stride, must be a power of two as in the reference's `2**lvl == s` test).
 *   feats/H/W/strides are HOST arrays of length num_levels (<= SDET_MAX_LEVELS).
 *   levels_out (B*N int32, device, may be NULL): assigned level index, -1 if no level matched.
 *   argmax_x/argmax_y and workspace as above (may be NULL). */
int sdet_fpn_roi_align_v2_forward(const float* const* feats, const int* H, const int* W,
                                  const int* strides, int num_levels, const float* rois,
                                  float* out, float* argmax_x, float* argmax_y,
                                  int32_t* levels_out, int B, int N, int C, int pooled_h,
                                  int pooled_w, int roi_canonical_scale, int roi_canonical_level,
                                  void* workspace, size_t workspace_bytes, void* stream);
/* Workspace including the NHWC scratch of the channels-last path (H, W: HOST arrays of num_levels entries; the
 * plain _contrib_ROIAlign_v2 is num_levels = 1). */
size_t sdet_fpn_roi_align_v2_workspace(int B, int N, int C, const int* H, const int* W, int num_levels);
/* Features already channels-last, feats_nhwc[l] = (B, H_l, W_l, C) device: no re-layout pass, inference only
 * (no argmax planes).  workspace: sdet_roi_align_v2_workspace(B, N) bytes, 16-byte aligned, required.  feats_nhwc[l]
 * must be 8-byte aligned and C even; out needs only 4-byte alignment (16-byte stores only where the address allows). */
int sdet_fpn_roi_align_v2_forward_nhwc(const float* const* feats_nhwc, const int* H, const int* W,
                                       const int* strides, int num_levels, const float* rois, float* out,
                                       int32_t* levels_out, int B, int N, int C, int pooled_h, int pooled_w,
                                       int roi_canonical_scale, int roi_canonical_level, void* workspace,
                                       size_t workspace_bytes, void* stream);
/* ... with the kernel choice of sdet_roi_align_v2_forward_ex. */
int sdet_fpn_roi_align_v2_forward_ex(const float* const* feats, const int* H, const int* W,
                                     const int* strides, int num_levels, const float* rois,
                                     float* out, float* argmax_x, float* argmax_y,
                                     int32_t* levels_out, int B, int N, int C, int pooled_h,
                                     int pooled_w, int roi_canonical_scale, int roi_canonical_level,
                                     void* workspace, size_t workspace_bytes, void* stream, int path,
                                     int* path_used);

/* assign_layer_fpn as a stand-alone operator (CustomOp 'assign_layer_fpn', models/FPN/assign_layer_fpn.py:17-40;
 * mxnext.tvm.fpn_roi_assign): rois (total_rois,4) device; strides HOST array; out_rois HOST array of num_levels
 * device pointers (total_rois,4) - the roi where it is assigned to that level, zeros elsewhere (may be NULL, or
 * hold NULL entries); levels_out (total_rois int32 device, may be NULL) index into strides, -1 if none. */
int sdet_fpn_assign(const float* rois, int total_rois, const int* strides, int num_levels,
                    int roi_canonical_scale, int roi_canonical_level, float* const* out_rois,
                    int32_t* levels_out, void* stream);

/* Backward of the fused op: scatters into the grad tensor of each roi's assigned level.
 *   grad_feats[l] device (B,C,H[l],W[l]); levels (B*N int32 device) as written by the forward. */
int sdet_fpn_roi_align_v2_backward(const float* ograd, const float* argmax_x,
                                   const float* argmax_y, const int32_t* levels,
                                   float* const* grad_feats, const int* H, const int* W,
                                   int num_levels, int B, int N, int C, int pooled_h, int pooled_w,
                                   int accumulate, void* stream);
/* Deterministic backward of the fused op, same arguments: per level l, the serial loop of
 * sdet_roi_align_v2_backward_ordered over the rois with levels[n] == l (rois with level -1 add nothing). */
int sdet_fpn_roi_align_v2_backward_ordered(const float* ograd, const float* argmax_x,
                                           const float* argmax_y, const int32_t* levels,
                                           float* const* grad_feats, const int* H, const int* W,
                                           int num_levels, int B, int N, int C, int pooled_h, int pooled_w,
                                           int accumulate, void* stream);

/* ------------------------------------------------------------------------------------------
 * ROIPooling_v1  (operator_cxx/roi_pooling_v1.cc:243, op roi_pooling_v1-inl.h:63-137,
 *                  kernels roi_pooling_v1.cu:49-113 / :116-152)
 *   data (B,C,H,W), rois (R,5) = [batch_index,x1,y1,x2,y2]; out, max_idx (R,C,PH,PW);
 *   max_idx holds the flat h*W+w index as float, -1 for empty bins.
 * ------------------------------------------------------------------------------------------ */
int sdet_roi_pooling_v1_forward(const float* data, const float* rois, float* out, float* max_idx,
                                int B, int R, int C, int H, int W, int pooled_h, int pooled_w,
                                float spatial_scale, void* stream);
/* Backward takes spatial_scale like ROIPoolBackwardAcc (roi_pooling_v1-inl.h:128-129): the bins are re-derived
 * from the rois so that gradients can be gathered per feature pixel. */
int sdet_roi_pooling_v1_backward(const float* ograd, const float* max_idx, const float* rois,
                                 float* grad_data, float* grad_rois, int B, int R, int C, int H,
                                 int W, int pooled_h, int pooled_w, float spatial_scale, int accumulate,
                                 void* stream);
/* Deterministic backward, same arguments: per gradient plane, ograd[index] is added at max_idx[index] of image
 * (int)rois[n*5] in ascending index ((n*C + c)*PH + ph)*PW + pw, from +0.0 on kWriteTo.  Entries with max_idx -1
 * (or outside [0, H*W)) or an image index outside [0, B) add nothing; spatial_scale is not used.  Checks, errors
 * and limits as sdet_roi_align_v2_backward_ordered. */
int sdet_roi_pooling_v1_backward_ordered(const float* ograd, const float* max_idx, const float* rois,
                                         float* grad_data, float* grad_rois, int B, int R, int C, int H,
                                         int W, int pooled_h, int pooled_w, float spatial_scale,
                                         int accumulate, void* stream);


/* ------------------------------------------------------------------------------------------
 * _contrib_DecodeBBox   (operator_cxx/contrib/decodebbox.cc:34-133 arithmetic, :150-209 op,
 *                        params decodebbox-inl.h:50-69)
 *   rois (B,N,4), bbox_pred (B,N,K4), im_info (B,3) [h,w,scale]  ->  out (B,N,4) when
 *   class_agnostic (reads class slot 1, decodebbox.cc:54) else (B,N,K4).
 *   bbox_mean / bbox_std: HOST float[4] (op defaults 0,0,0,0 / 0.1,0.1,0.2,0.2; class_agnostic
 *   defaults to TRUE).  decode_type 0 = "xywh", 1 = "xyxy".  All device pointers 16B-aligned.
 * ------------------------------------------------------------------------------------------ */
int sdet_decode_bbox(const float* rois, const float* bbox_pred, const float* im_info, float* out,
                     int B, int N, int K4, const float* bbox_mean, const float* bbox_std,
                     int class_agnostic, int decode_type, void* stream);

/* ------------------------------------------------------------------------------------------
 * _contrib_Proposal_v3  (GPU semantics: operator_cxx/contrib/proposal_v3.cu:435-638; params
 *                        proposal_v3-inl.h:141-183; anchors :280-318)
 *   cls_prob (B,2A,H,W) (fg = second half), bbox_pred (B,4A,H,W), im_info (B,3)
 *   -> out (B,post,4), out_score (B,post,1).  post = rpn_post_nms_top_n when !is_train, else
 *   min(post, pre); pre = min(rpn_pre_nms_top_n > 0 ? it : A*H*W, A*H*W).
 *   Padding beyond the kept boxes: zeros (is_train=0) or wrap keep[i % n_keep] (is_train=1).
 *   scales / ratios: HOST arrays.  workspace: device, >= sdet_proposal_v3_workspace() bytes.
 * ------------------------------------------------------------------------------------------ */
size_t sdet_proposal_v3_workspace(int B, int A, int H, int W, int rpn_pre_nms_top_n);
int sdet_proposal_v3(const float* cls_prob, const float* bbox_pred, const float* im_info, float* out,
                     float* out_score, int B, int A, int H, int W, int feature_stride,
                     const float* scales, int num_scales, const float* ratios, int num_ratios,
                     int rpn_pre_nms_top_n, int rpn_post_nms_top_n, float threshold,
                     int rpn_min_size, int iou_loss, int is_train, void* workspace,
                     size_t workspace_bytes, void* stream);

/* _contrib_Proposal (version 1: operator_cxx/contrib/proposal.cu:430-620; X.proposal at
 * symbol/builder.py:241-255) and _contrib_Proposal_v2 (version 2: proposal_v2.cu:405-600, TridentNet):
 * the legacy pipeline — floor(x+0.5) anchors, legacy decode without exp clip, padded-cell mask and
 * min-size (rpn_min_size * im_scale) filter BEFORE the sort, NMS removes IoU > threshold.
 * version 1 honours is_train (wrap padding, post = rpn_post_nms_top_n at test time); version 2
 * takes valid_ranges (B,2) device + filter_scales and always zero-pads with post = min(post, pre). */
size_t sdet_proposal_legacy_workspace(int B, int A, int H, int W, int rpn_pre_nms_top_n);
int sdet_proposal_legacy(const float* cls_prob, const float* bbox_pred, const float* im_info,
                         const float* valid_ranges, int version, float* out, float* out_score, int B,
                         int A, int H, int W, int feature_stride, const float* scales, int num_scales,
                         const float* ratios, int num_ratios, int rpn_pre_nms_top_n,
                         int rpn_post_nms_top_n, float threshold, int rpn_min_size, int iou_loss,
                         int is_train, int filter_scales, void* workspace, size_t workspace_bytes,
                         void* stream);

/* _contrib_GenProposal (generate_proposal.cu:289-430): the legacy decode + mask + min-size filter on
 * caller-supplied shifted anchors (H*W*A,4), stable sort, NO NMS.  out (B, rpn_pre_nms_top_n, 5) =
 * (x1,y1,x2,y2,score); rows past min(rpn_pre_nms_top_n, A*H*W) are zero. */
size_t sdet_gen_proposal_workspace(int B, int A, int H, int W, int rpn_pre_nms_top_n);
int sdet_gen_proposal(const float* cls_prob, const float* bbox_pred, const float* im_info,
                      const float* anchors, float* out, int B, int A, int H, int W, int feature_stride,
                      int rpn_pre_nms_top_n, int rpn_min_size, int iou_loss, void* workspace,
                      size_t workspace_bytes, void* stream);

/* _contrib_GenAnchor (generate_anchor.cu:62-140): out (H*W*A, 4) fp32 = float(double base anchor +
 * shift); scales/ratios are host doubles (GenAnchorParam keeps doubles "for consistency with python"). */
int sdet_gen_anchor(float* out, int H, int W, int feature_stride, const double* scales, int num_scales,
                    const double* ratios, int num_ratios, void* stream);

/* _contrib_GenProposalRetina (generate_proposal_retina.cu:307-469; models/retinanet/builder.py:374-387).
 * cls_prob (B, A*K, H, W) sigmoid probabilities, bbox_pred (B, A*4, H, W), anchors (H*W*A, 4).
 * out (B, rpn_pre_nms_top_n, 4), out_score (B, rpn_pre_nms_top_n, K+1 | 1): the top pairs by score
 * among those with score > thresh and both sides >= rpn_min_size*im_scale; every other row is zero.
 * anchor_mean/anchor_std: host float[4] (NULL = 0 / 1).  Unsupported (the reference reads out of
 * range there): iou_loss, batch_wise_anchor with K > 1; thresh must be >= 0. */
size_t sdet_gen_proposal_retina_workspace(int B, int AK, int H, int W);
int sdet_gen_proposal_retina(const float* cls_prob, const float* bbox_pred, const float* im_info,
                             const float* anchors, float* out, float* out_score, int B, int AK, int H,
                             int W, int num_anchors, int feature_stride, int rpn_pre_nms_top_n,
                             int rpn_min_size, float thresh, const float* anchor_mean,
                             const float* anchor_std, int iou_loss, int output_one_hot,
                             int batch_wise_anchor, void* workspace, size_t workspace_bytes,
                             void* stream);

/* All RPN levels of an FPN in one call: num_levels x _contrib_Proposal_v3 + Concat(dim=1)
 * (models/FPN/builder.py:267-317).  cls_prob[l] (B,2A,H[l],W[l]), bbox_pred[l] (B,4A,H[l],W[l]);
 * the pointer / H / W / feature_stride arrays are HOST arrays of length num_levels.
 * out (B, num_levels*post, 4), out_score (B, num_levels*post, 1): level-major per image, each
 * level's slice exactly what sdet_proposal_v3 writes for that level.
 * is_train: when every level has the same anchor count, post = min(rpn_post_nms_top_n, count) like sdet_proposal_v3.
 * When they differ and a level has fewer anchors than rpn_post_nms_top_n (P6 of an 800x1333 FPN: 819 < 2000), post
 * stays rpn_post_nms_top_n for every level; the small level writes min(post, its count) rows (kept boxes, then the
 * reference's wrap-around padding) and ZERO rows after them, which ProposalTarget drops (y2 > 0 test).  (The
 * reference leaves those rows unwritten and strides images by the shrunken count, proposal_v3.cu:471-476,:629-631.) */
size_t sdet_proposal_v3_fpn_workspace(int B, int A, const int* H, const int* W, int num_levels,
                                      int rpn_pre_nms_top_n);
int sdet_proposal_v3_fpn(const float* const* cls_prob, const float* const* bbox_pred,
                         const float* im_info, float* out, float* out_score, int B, int A,
                         const int* H, const int* W, const int* feature_stride, int num_levels,
                         const float* scales, int num_scales, const float* ratios, int num_ratios,
                         int rpn_pre_nms_top_n, int rpn_post_nms_top_n, float threshold,
                         int rpn_min_size, int iou_loss, int is_train, void* workspace,
                         size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------
 * _contrib_NMS   (operator_cxx/contrib/nms.cu:274-364; params nms-inl.h:49-70)
 *   proposals (B,count,5) [x1,y1,x2,y2,score] -> out (B,rpn_post_nms_top_n,4), out_score
 *   (B,rpn_post_nms_top_n,1).  Suppresses IoU > threshold; only the first min(post,pre) rows are
 *   written (zeros past the kept boxes), the rest are left untouched exactly like nms.cu:354-358.
 * ------------------------------------------------------------------------------------------ */
size_t sdet_contrib_nms_workspace(int B, int count, int rpn_pre_nms_top_n);
int sdet_contrib_nms(const float* proposals, float* out, float* out_score, int B, int count,
                     int rpn_pre_nms_top_n, int rpn_post_nms_top_n, float threshold,
                     int already_sorted, void* workspace, size_t workspace_bytes, void* stream);

/* Batched greedy NMS over boxes that are ALREADY in greedy (descending-score) order: the device
 * replacement of nms_kernel + the host scan in `_nms` (proposal_v3.cu:281-380,
 * operator_py/cython/nms_kernel.cu:34-144).
 *   dets (P,n,5) device; counts (P) device int32 or NULL (= n boxes everywhere); ge = 1 suppress
 *   IoU >= thresh (Proposal_v3, cpu_nms.greedy_nms), 0 suppress IoU > thresh (_contrib_NMS,
 *   gpu_nms).  keep (P,n) int32: kept positions in order, zero padded; nkeep (P) int32.
 *   n <= 12288. */
size_t sdet_nms_workspace(int problems, int n);
int sdet_nms_sorted(const float* dets, const int* counts, int problems, int n, float thresh, int ge,
                    int* keep, int* nkeep, void* workspace, size_t workspace_bytes, void* stream);

/* `_nms`: the reference's own C ABI (operator_py/cython/gpu_nms.hpp:1-2; implementation nms_kernel.cu:91-144,
 * bound by gpu_nms.pyx:13-14), kept under the exact symbol and signature so gpu_nms.pyx links against this
 * library unchanged.  HOST pointers in, blocking, allocates and frees its device buffers per call like the
 * reference; boxes_host (boxes_num, boxes_dim >= 4) must already be sorted by descending score (gpu_nms.pyx:25-29);
 * suppresses IoU > nms_overlap_thresh (nms_kernel.cu:71); keep_out (boxes_num ints) receives the kept positions,
 * *num_out their count.  Errors are printed to stderr (the reference's CUDA_CHECK only prints) and *num_out = 0. */
void _nms(int* keep_out, int* num_out, const float* boxes_host, int boxes_num, int boxes_dim,
          float nms_overlap_thresh, int device_id);

/* get_top_proposal  (CustomOp models/FPN/get_top_proposal.py:15-40; mxnext.tvm.get_top_proposal
 * at models/FPN/builder.py:319-321): per image keep the top_n rows by score, descending, ties by
 * lower row index (mx.nd.argsort(is_ascend=False) treated as stable).
 *   boxes (B,M,4), scores (B,M,1) -> out_boxes (B,top_n,4), out_scores (B,top_n,1). */
int sdet_get_top_proposal(const float* boxes, const float* scores, float* out_boxes,
                          float* out_scores, int B, int M, int top_n, void* stream);

/* Test-time per-class NMS, batched: replaces detection_test.py:233-260 `do_nms` (a Python loop
 * over classes inside multiprocessing.Pool) with operator_py/nms.py:41-75 semantics
 * (score > min_det_score; greedy by descending score; keep IoU <= nms_thresh).
 *   cls_score (B,N,K), bbox (B,N,4K) or (B,N,4); classes first_class..K-1 are processed
 *   (detection_test.py iterates all K columns of the score it is given).
 *   Problem p = b*(K-first_class) + (cid-first_class); n_pad = next_pow2(N) <= 4096.
 *   dets (P,n_pad,5): class candidates in descending-score order (zero padded);
 *   counts (P): candidates per problem; keep (P,n_pad): kept positions into dets; nkeep (P);
 *   src_index (P,n_pad) or NULL: roi index of each candidate (-1 padding). */
size_t sdet_multiclass_nms_workspace(int B, int N, int K, int first_class);
int sdet_multiclass_nms(const float* cls_score, const float* bbox, int B, int N, int K, int bbox_dim,
                        int first_class, float min_det_score, float nms_thresh, float* dets,
                        int* counts, int* keep, int* nkeep, int* src_index, void* workspace,
                        size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------
 * ProposalTarget   (operator_cxx/proposal_target-inl.h:81-114 params, :123-256 Forward;
 *                   operator_cxx/proposal_target.cc:22-227 SampleROI and helpers)
 *   rois (B,R,4) (padding rows have y2 <= 0), gt_boxes (B,G,5) [x1,y1,x2,y2,cls] (padding cls -1)
 *   -> rois_out (B,IR,4), labels (B,IR), bbox_targets / bbox_weights (B,IR,num_classes*4),
 *      match_gt_ious (B,IR); kept (B,IR) int32 or NULL: index of each output row in the image's
 *      compacted [valid rois ++ valid gt] list (-1 for a row the reference leaves zero).
 *   IR = image_rois (> 0), fg quota = (int)(image_rois * fg_fraction).  All outputs are fully
 *   written (zero-initialised like -inl.h:188-192).  bbox_mean/std/weight: HOST float[4].
 *   Sampling: each std::random_shuffle of the reference is "order by a 32-bit priority, ties by
 *   index".  priorities == NULL: cuRAND Philox4x32-10 keyed (seed, image*T+candidate, draw),
 *   T = R+G; else a DEVICE array (B, num_draws, T) uint32 supplied by the caller.  Draw 0 = fg,
 *   1 = bg, 2 + r % (num_draws-2) = r-th negative-padding shuffle; num_draws >= 3.
 *   priorities_used (B,num_draws,T) device or NULL receives the priorities of the draws executed.
 *   gt_index (B,IR) int32 or NULL: source row in gt_boxes of each output row's matched gt (-1: none);
 *   fg_count (B) int32 or NULL: foreground rows per image. */
int sdet_proposal_target(const float* rois, const float* gt_boxes, float* rois_out, float* labels,
                         float* bbox_targets, float* bbox_weights, float* match_gt_ious, int* kept,
                         int B, int R, int G, int num_classes, int image_rois, float fg_fraction,
                         float fg_thresh, float bg_thresh_hi, float bg_thresh_lo,
                         int proposal_without_gt, int class_agnostic, const float* bbox_mean,
                         const float* bbox_std, const float* bbox_weight, unsigned long long seed,
                         const uint32_t* priorities, int num_draws, uint32_t* priorities_used,
                         int* gt_index, int* fg_count, void* stream);

/* ProposalTarget_v2  (operator_cxx/proposal_target_v2-inl.h:145-270, proposal_target_v2.cc:22-175;
 * used by TridentNet, models/tridentnet/builder.py:281): ProposalTarget plus
 *   valid_ranges (B,2) device + filter_scales: gt boxes whose area is outside [min^2, max^2] are
 *   not appended to the proposals (they still take part in the IoU matching);
 *   image_rois == -1: every foreground roi is kept and each image yields R output rows. */
int sdet_proposal_target_v2(const float* rois, const float* gt_boxes, const float* valid_ranges,
                            float* rois_out, float* labels, float* bbox_targets, float* bbox_weights,
                            float* match_gt_ious, int* kept, int B, int R, int G, int num_classes,
                            int image_rois, float fg_fraction, float fg_thresh, float bg_thresh_hi,
                            float bg_thresh_lo, int proposal_without_gt, int class_agnostic,
                            int filter_scales, const float* bbox_mean, const float* bbox_std,
                            const float* bbox_weight, unsigned long long seed, const uint32_t* priorities,
                            int num_draws, uint32_t* priorities_used, int* gt_index, int* fg_count,
                            void* stream);

/* ------------------------------------------------------------------------------------------
 * ProposalMaskTarget  (operator_cxx/proposal_mask_target-inl.h:87-130 params, :139-337 Forward;
 *                      operator_cxx/proposal_mask_target.cc:155-213 convertPoly2Mask, :219-379
 *                      SampleROIMask) = sdet_proposal_target(..., gt_index, fg_count) followed by
 *   sdet_poly_mask_target: for image b and output row i < min(fg_count[b], num_mask_rows) the
 *   polygon gt_polys[b, gt_index[b,i]] ([category, n_seg, len_1..len_n, x,y,x,y,...], padded; see
 *   models/maskrcnn/input.py:166-175) is rasterised into mask_target[b,i] (mask_size^2, values
 *   0/1) in the roi-normalised frame; other rows are filled with -1 (ignored by
 *   SigmoidCrossEntropy).  num_mask_rows = (int)(image_rois * fg_fraction).  gt_index / fg_count
 *   are the optional outputs of sdet_proposal_target[_v2] (int32, device); filter_scales / valid_ranges
 *   (num_args = 4) is sdet_proposal_target_v2 in front of the same call.
 *   sdet_poly_mask_target_ratio = output_ratio=True (Mask Scoring R-CNN, models/msrcnn/builder.py:219-239;
 *   convertPoly2MaskWithRatio, proposal_mask_target.cc:20-152): the mask with the vertex transform carried out in
 *   double as that variant does, plus mask_ratio (B, num_mask_rows) = |polygon in the roi crop| / (|polygon| + 1e-4)
 *   counted on the reference's integer rasters, clamped from below at 1e-10; rows >= fg_count[b] are 0.  A roi whose
 *   polygon crosses more than 16384 pixel columns in one segment (32768 over all segments) gets NaN. */
int sdet_poly_mask_target(const float* rois_out, const float* gt_polys, const int* gt_index,
                          const int* fg_count, float* mask_target, int B, int image_rois, int G,
                          int poly_len, int num_mask_rows, int mask_size, void* stream);
int sdet_poly_mask_target_ratio(const float* rois_out, const float* gt_polys, const int* gt_index,
                                const int* fg_count, float* mask_target, float* mask_ratio, int B,
                                int image_rois, int G, int poly_len, int num_mask_rows, int mask_size,
                                void* stream);

/* ------------------------------------------------------------------------------------------
 * _contrib_FocalLoss  (operator_cxx/contrib/focal_loss-inl.h:52-79 params, :90-114 forward =
 *                      sigmoid, :116-231 backward).  data/out/gdata (B,N,K), label (B,N) with
 *                      -1 = ignore, 0 = background, k in 1..K = class k-1 (Appendix A.18).
 *   normalization: 0 "null", 1 "batch", 2 "valid" (divide by sum(label>=1)+1).  ograd may be
 *   NULL (out_grad=false).  workspace: >= 4 bytes of device memory.
 * _contrib_BBoxNorm   (bbox_norm-inl.h:99-129): forward is identity; backward divides the
 *                      incoming gradient by max(sum(label>=1)+1, 1).  n / n_label = element counts.
 * _contrib_SigmoidCrossEntropy (sigmoid_cross_entropy.cu:45-129): data,label (R,D); label -1 is
 *   ignored; out (R) = per-row sum(loss)/(count+1e-5); backward d = (sigmoid(x)-t)/(count+1e-5)*scale.
 *   workspace: >= 8*R bytes.
 * ------------------------------------------------------------------------------------------ */
int sdet_focal_loss_forward(const float* data, float* out, size_t n, void* stream);
int sdet_focal_loss_backward(const float* out, const float* label, const float* ograd, float* gdata,
                             int B, int N, int K, float alpha, float gamma, float grad_scale,
                             int normalization, void* workspace, size_t workspace_bytes, void* stream);
int sdet_bbox_norm_backward(const float* gout, const float* label, float* gdata, size_t n,
                            size_t n_label, void* workspace, size_t workspace_bytes, void* stream);
int sdet_sigmoid_ce_forward(const float* data, const float* label, float* out, int R, size_t D,
                            void* workspace, size_t workspace_bytes, void* stream);
int sdet_sigmoid_ce_backward(const float* data, const float* label, float* d_data, int R, size_t D,
                             float scale, void* workspace, size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------
 * soft_nms   (operator_py/cython/cpu_nms.pyx:98-203; wrapper operator_py/nms.py:5-16), batched:
 *   dets (P,m,5) device [x1,y1,x2,y2,score] in ANY order (the algorithm selects the max itself),
 *   counts (P) device int32 or NULL (= m boxes everywhere).
 *   method 0 hard, 1 linear, 2 gaussian; Nt = IoU threshold; boxes whose re-weighted score drops
 *   below `threshold` are removed.
 *   out_boxes (P,m,5): the surviving boxes with their final scores in the reference's output order
 *   (zero padded), out_inds (P,m): their original row indices (-1 padding), out_counts (P).
 * ------------------------------------------------------------------------------------------ */
int sdet_soft_nms(const float* dets, const int* counts, int problems, int m, float sigma, float Nt,
                  float threshold, int method, float* out_boxes, int* out_inds, int* out_counts,
                  void* stream);

/* ------------------------------------------------------------------------------------------
 * Deformable convolution v1 sampling  (mx.sym.contrib.DeformableConvolution — upstream
 * apache/incubator-mxnet src/operator/contrib/nn/deformable_im2col.cuh, NOT in the reference
 * tree; call sites models/dcn/builder.py:14-17; parity unpinned).
 *   data (B,C,H,W), offset (B, dg*2*KH*KW, Ho, Wo) [per tap: (dy, dx)],
 *   col (B, C*KH*KW, Ho*Wo): the sampled columns; the dense product with the (F, C/groups*KH*KW)
 *   weights is a library GEMM done by the caller.
 *   col2im: gradient of the gather w.r.t. data (grad_data, zero-filled first) and offset
 *   (grad_offset); either may be NULL.
 * ------------------------------------------------------------------------------------------ */
int sdet_deformable_im2col(const float* data, const float* offset, float* col, int B, int C, int H, int W,
                           int kernel_h, int kernel_w, int pad_h, int pad_w, int stride_h, int stride_w,
                           int dilate_h, int dilate_w, int num_deformable_group, void* stream);
/* The kernel sdet_deformable_im2col launches for this geometry (host only, no CUDA call): *tiled = 1 for the
 * shared-memory tiled kernel (9 taps) with *ct channels per stage and the channels of a group split over *slices
 * CTAs; *tiled = 0 for the generic kernel (*ct = *slices = 0).  Same argument checks as sdet_deformable_im2col. */
int sdet_deformable_im2col_plan(int B, int C, int H, int W, int kernel_h, int kernel_w, int pad_h, int pad_w,
                                int stride_h, int stride_w, int dilate_h, int dilate_w, int num_deformable_group,
                                int* tiled, int* ct, int* slices);
/* Channels-last sampling: data (B,H,W,C), same offset tensor, col_t (B, Ho*Wo, KH*KW, C) - the K index of the
 * following GEMM is (tap, channel), its output (B, Ho*Wo, F) is channels-last too.  Same values as
 * sdet_deformable_im2col, element for element.  C / num_deformable_group must be even, data and col_t 8-byte
 * aligned (SDET_ERR_INVALID_ARG otherwise). */
int sdet_deformable_im2col_nhwc(const float* data, const float* offset, float* col_t, int B, int C, int H, int W,
                                int kernel_h, int kernel_w, int pad_h, int pad_w, int stride_h, int stride_w,
                                int dilate_h, int dilate_w, int num_deformable_group, void* stream);
int sdet_deformable_col2im(const float* grad_col, const float* data, const float* offset, float* grad_data,
                           float* grad_offset, int B, int C, int H, int W, int kernel_h, int kernel_w,
                           int pad_h, int pad_w, int stride_h, int stride_w, int dilate_h, int dilate_w,
                           int num_deformable_group, void* stream);

/* DCNv2 (modulated) sampling, upstream MXNet `_contrib_ModulatedDeformableConvolution`
 * (modulated_deformable_im2col.cuh; not in the reference tree, restated from the published formulation):
 * like the v1 pair with an extra mask (B, num_deformable_group*KH*KW, Ho, Wo) multiplying every tap,
 * zero-padded (not clamped) corners and the sampling range -1 < h < H, -1 < w < W. */
int sdet_modulated_deformable_im2col(const float* data, const float* offset, const float* mask, float* col,
                                     int B, int C, int H, int W, int kernel_h, int kernel_w, int pad_h,
                                     int pad_w, int stride_h, int stride_w, int dilate_h, int dilate_w,
                                     int num_deformable_group, void* stream);
int sdet_modulated_deformable_col2im(const float* grad_col, const float* data, const float* offset,
                                     const float* mask, float* grad_data, float* grad_offset,
                                     float* grad_mask, int B, int C, int H, int W, int kernel_h,
                                     int kernel_w, int pad_h, int pad_w, int stride_h, int stride_w,
                                     int dilate_h, int dilate_w, int num_deformable_group, void* stream);

/* detection_test.py:268-291 after sdet_multiclass_nms: per image, the `max_det` highest-scoring kept
 * detections over all classes (ties: the later (class, rank) entry wins, as Python's stable ascending sort
 * followed by [-max_det:] does).  dets (B*num_classes, n_pad, 5), keep (B*num_classes, n_pad), nkeep
 * (B*num_classes) as written by sdet_multiclass_nms.  out (B, max_det, 6) rows [x, y, w, h, score,
 * class index] in ascending score order, unused rows zero with class -1; out_count (B). */
int sdet_final_detections(const float* dets, const int* keep, const int* nkeep, int B, int num_classes,
                          int n_pad, int max_det, float* out, int* out_count, void* stream);
/* Same selection with the row format of CustomOp 'BboxPostProcessing' (models/maskrcnn/bbox_post_processing.py:
 * 6-32): xyxy != 0 keeps [x1, y1, x2, y2, score, class]; descending != 0 lists the highest score first. */
int sdet_final_detections_ex(const float* dets, const int* keep, const int* nkeep, int B, int num_classes,
                             int n_pad, int max_det, float* out, int* out_count, int xyxy, int descending,
                             void* stream);

/* operator_py/nms.py:77-107 set_nms over boxes already sorted by descending score: like sdet_nms_sorted
 * with `>` (the reference keeps ovr <= thresh), but boxes whose `sets` value (P,n; column 5 of the
 * reference's dets) is equal never suppress each other. */
int sdet_set_nms_sorted(const float* dets, const float* sets, const int* counts, int problems, int n,
                        float thresh, int* keep, int* nkeep, void* workspace, size_t workspace_bytes,
                        void* stream);
/* operator_py/nms.py:110-157 py_weighted_nms over pre-sorted boxes: out (P,n,5) rows [score-weighted
 * mean box of the pool members with IoU > thresh_hi, score of the top box], nout (P) rows valid.  Sums
 * are float32 in warp order (numpy's pairwise order differs in the last bits). */
size_t sdet_weighted_nms_workspace(int problems, int n);
int sdet_weighted_nms_sorted(const float* dets, const int* counts, int problems, int n, float thresh_lo,
                             float thresh_hi, float* out, int* nout, void* workspace,
                             size_t workspace_bytes, void* stream);

/* operator_py/cython/bbox.pyx:32-73 (mode 0, IoU) and bbox_self.pyx:32-75 (mode 1, intersection over the
 * area of boxes[n]): boxes (N,4), query_boxes (K,4) -> overlaps (N,K), float32, bit-exact with the
 * compiled Cython (whose `+ 1` terms are evaluated in double). */
int sdet_bbox_overlaps(const float* boxes, const float* query_boxes, float* overlaps, int N, int K,
                       int mode, void* stream);
/* operator_py/bbox_transform.py:52-78 nonlinear_transform, float64: (N,4),(N,4) -> (N,4). */
int sdet_bbox_nonlinear_transform(const double* ex_rois, const double* gt_rois, double* targets, int N,
                                  void* stream);
/* bbox_transform.py:81-120 nonlinear_pred (iou = 0; dw, dh clipped at log(1000/16)) or :129-161 iou_pred
 * (iou = 1), optionally followed by clip_boxes(:34-49) to (im_h, im_w).  boxes (N,4) float32,
 * box_deltas / pred_boxes (N,4K) float64. */
int sdet_bbox_pred(const float* boxes, const double* box_deltas, double* pred_boxes, int N, int K,
                   int iou, int clip, double im_h, double im_w, void* stream);

/* bbox_transform.py:164-169 flip_boxes on (num_boxes,4) float32 (is_double = 0) or float64 boxes. */
int sdet_bbox_flip(const void* boxes, void* out, size_t num_boxes, double im_width, int is_double,
                   void* stream);
/* bbox_transform.py:172-221 box_voting: top_dets (T,5), all_dets (N,5) float32 -> out (T,5).
 * scoring_method: 0 ID, 1 TEMP_AVG, 2 AVG, 3 IOU_AVG, 4 GENERALIZED_AVG, 5 QUASI_SUM. */
int sdet_box_voting(const float* top_dets, const float* all_dets, float* out, int T, int N, float thresh,
                    int scoring_method, float beta, void* stream);

/* AnchorTarget2D (core/detection_input.py:353-565) and PyramidAnchorTarget2D (models/FPN/input.py:55-148)
 * for a batch, on the device.  gt_bbox (B,G,gt_stride) with gt_stride 4 or 5; rows whose x1 == -1 are
 * padding.  Level l has stride strides[l] and a (long x short) grid oriented by the image (h >= w puts
 * `long` on the height axis).  scales / aspects are host doubles (the reference computes base anchors in
 * float64).  Outputs, per image, in the pyramid layout: cls_label (A * S), reg_target and reg_weight
 * (4A, S) with S = sum_l short_l*long_l — for one level this is AnchorTarget2D's (A*fh*fw) / (4A,fh,fw).
 * fg_quota = int(pos_fraction * image_anchor), evaluated by the caller in double like the reference.
 * Sub-sampling disables the surplus anchors with the smallest 32-bit priority (ties: larger anchor
 * index first); priorities (B, A*S) device or NULL = Philox4x32-10(seed, image*A*S + anchor).
 * priorities[n] = n reproduces the reference's DEBUG mode. */
size_t sdet_anchor_target_workspace(int B, int total_anchors, int max_gt);
int sdet_anchor_target(const float* im_info, const float* gt_bbox, int gt_stride, float* cls_label,
                       float* reg_target, float* reg_weight, int B, int G, int num_levels,
                       const int* strides, const int* shorts, const int* longs, const double* scales,
                       int num_scales, const double* aspects, int num_aspects, float allowed_border,
                       float neg_thr, float pos_thr, float min_pos_thr, int image_anchor, int fg_quota,
                       const uint32_t* priorities, unsigned long long seed, void* workspace,
                       size_t workspace_bytes, void* stream);

/* Test-time mask paste: models/maskrcnn/utils.py:26-67 `segm_results` (expand_boxes :7-23, cv2.resize of the
 * zero-ringed mask to the expanded integer box, `> 0.5`, paste into an im_h x im_w image, pycocotools
 * `mask.encode` = column-major run lengths) without materialising the image.  boxes (N,4) float32 x1,y1,x2,y2 in
 * image coordinates, cls (N) int32 index into the K mask channels (the background channel already removed, as
 * mask_test.py:171 does), masks (N,K,M,M) float32 probabilities, M <= 62.
 *   sdet_mask_paste_count: col_counts (N, im_w) int32; entry (n, j) = number of value flips the pasted mask of
 *     detection n has in image column x_0(n) + j (x_0 = first pasted column; 0 for j past the pasted width), walking
 *     the image in column-major order.
 *   sdet_mask_paste_write: col_offsets (N, im_w) int64 = exclusive prefix sum of col_counts in row-major (n, j)
 *     order; positions[col_offsets[n][j] + k] = flat column-major index x*im_h + y of the k-th flip of that column.
 * The RLE counts of detection n are the differences of consecutive positions of rows (n, *), bracketed by 0 and
 * im_h*im_w (first count = run of zeros, as pycocotools).  A box with no pixel inside the image, an inverted box or
 * a class outside [0, K) pastes nothing (the reference raises on the first, pastes nothing on the second). */
int sdet_mask_paste_count(const float* boxes, const int* cls, const float* masks, int N, int K, int M, int im_h,
                          int im_w, int* col_counts, void* stream);
int sdet_mask_paste_write(const float* boxes, const int* cls, const float* masks, int N, int K, int M, int im_h,
                          int im_w, const long long* col_offsets, int* positions, void* stream);

/* _contrib_GroupNorm forward (operator_cxx/contrib/group_norm.cu:202-236, group_norm_helper.cu:36-147).  x, y
 * (N, C, HxW) fp32, NCHW-contiguous or, with channels_last, (N, HxW, C)-contiguous; gamma, beta (C).  Per (n, g),
 * D = C/G: mu = sum(x)*(1/(D*HxW)), var = sum(x*x)*(1/(D*HxW)) - mu*mu, rsig = rsqrtf(var + eps),
 * y = ((gamma[c]*(x - mu))*rsig) + beta[c], then max(y, 0) with NaN kept when relu != 0.  mean, rsig (N, G).
 * The statistics are summed in a fixed order (bit-identical from run to run; not the reference's cub order).
 * SDET_ERR_INVALID_ARG: NULL pointer, non-positive size, C % G != 0, a float pointer not 4-byte aligned or a
 * workspace not 8-byte aligned; SDET_ERR_WORKSPACE: workspace_bytes < sdet_group_norm_workspace(...);
 * SDET_ERR_UNSUPPORTED: channels-last with C > 1024 (C > 256 when x / y are not 16-byte aligned or C % 4 != 0).
 * Nothing is launched on an error return. */
size_t sdet_group_norm_workspace(int N, int C, int HxW, int G);
int sdet_group_norm_forward(const float* x, const float* gamma, const float* beta, float* y, float* mean, float* rsig,
                            int N, int C, int HxW, int G, float eps, int channels_last, int relu, void* workspace,
                            size_t workspace_bytes, void* stream);

/* CustomOp get_proposal_single_stage (models/FCOS/utils.py:7-94), one FPN level.  centerness (B,1,H,W),
 * cls_prob (B,C,H,W), offset (B,4,H,W) post-sigmoid / post-exp fp32, cls_prob and offset NCHW-contiguous or, with
 * channels_last, (B,H,W,C) / (B,H,W,4)-contiguous; im_info (B,3).  out (B, top_n, 6) rows [cls+1, score, x1, y1,
 * x2, y2]: with at least top_n entries of cls_prob > pre_nms_thresh, the top_n of score = cls_prob*centerness over
 * all C*H*W entries (descending, ties to the lower flat (c,y,x) index), positions recovered by the reference's
 * float32 index arithmetic; otherwise every such entry in flat order.  Boxes loc -/+ offset clipped to [0, im_w] /
 * [0, im_h]; a row with cls >= x1 AND score >= y1 (utils.py:63's columns) is all -1, as is every row not kept.
 * SDET_ERR_INVALID_ARG: NULL pointer, non-positive size, top_n <= 0, stride <= 0; SDET_ERR_WORKSPACE: short
 * workspace; SDET_ERR_UNSUPPORTED: C*H*W >= 2^24 or top_n > 25600. */
size_t sdet_fcos_proposal_workspace(int B, int C, int H, int W);
int sdet_fcos_proposal(const float* centerness, const float* cls_prob, const float* offset, const float* im_info,
                       float* out, int B, int C, int H, int W, int top_n, int stride, float pre_nms_thresh,
                       int channels_last, void* workspace, size_t workspace_bytes, void* stream);

/* CustomOp get_batch_proposal (models/FCOS/utils.py:97-149).  bbox (B, K, 6) rows [cls, score, x1, y1, x2, y2];
 * per image the rows sorted by score, descending and stable: res_bbox (B, K, 4) (16-byte aligned), cls_id (B, K, 1),
 * score (B, K, 81) zero except sqrtf(clip(score, 1e-20, 1)) in column int(cls), a negative id counting from the end
 * as numpy does (a -1 row writes column 80).  K <= 25600. */
int sdet_fcos_batch_proposal(const float* bbox, float* res_bbox, float* score, float* cls_id, int B, int K,
                             void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SIMPLEDET_B200_H_ */
