/*
 * step_b200.h -- C ABI of libstep_b200.so: the sm_90a implementation of the STEP hot path.
 *
 * This is the drop-in boundary (SURVEY.md section 8b).  Every entry point takes raw device
 * pointers, plain sizes and an explicit cudaStream_t; none allocates, synchronises or touches
 * the default stream, so each is CUDA-graph capturable.  Every entry returns 0 on success or a
 * non-zero code (a cudaError_t, or STEP_E_* below); step_last_error() then describes it.
 *
 * Reference interface each group replaces (paths relative to the NVlabs/STEP tree):
 *   nms            external/maskrcnn_benchmark/csrc/vision.cpp:31  _C.nms  (nms.h:34-51,
 *                  cpu/nms_cpu.cpp:29-99, cuda/nms.cu:47-155)
 *   roi_align_*    vision.cpp:32-33  _C.roi_align_forward/backward  (ROIAlign.h:35-69,
 *                  cpu/ROIAlign_cpu.cpp:137-281, cuda/ROIAlign_cuda.cu:88-370)
 *   roi_pool_*     vision.cpp:34-35  _C.roi_pool_forward/backward   (ROIPool.h:35-71,
 *                  cuda/ROIPool_cuda.cu:40-226)
 *   tube_*         utils/tube_utils.py:10-27,59-92,127-189,214-266 and the per-step host loop of
 *                  utils/utils.py:61-129
 *   conv / pool / linear / head_*   the torch.nn calls of models/i3dpt.py:43-163,
 *                  models/networks.py:69-83, models/two_branch.py:60-111,132-138,223-274,337
 *   clip_*         the permute + (apex) cast at models/networks.py:77
 *
 * Tensor conventions: activations are channels-last -- [N, T, H, W, C] ("NDHWC") with an explicit
 * channel stride `ld` (elements) so a kernel can read or write a channel slice of a wider buffer
 * (this is how Mixed's concat, i3dpt.py:162, and the local-branch concat, two_branch.py:256,
 * disappear).  The *_nchw entry points take the reference's NCHW fp32 layout unchanged.
 */
#ifndef STEP_B200_H_
#define STEP_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct CUstream_st* step_stream_t; /* == cudaStream_t */

enum { STEP_F32 = 0, STEP_F16 = 1 };
enum { STEP_OK = 0, STEP_E_ARG = 10001, STEP_E_UNSUPPORTED = 10002, STEP_E_WORKSPACE = 10003,
       STEP_E_DRIVER = 10004 };

int step_version(void);
const char* step_last_error(void);
/* number of kernels this library has launched in this process (bench.py's gpu_launches) */
uint64_t step_launch_count(void);

/* ------------------------------------------------------------------ NMS ------------------ */
/* Greedy NMS, legacy "+1" areas, bit-exact with cpu/nms_cpu.cpp (ge=1: suppress when
 * IoU >= thr) or cuda/nms.cu (ge=0: IoU > thr).  Order: score descending, original index
 * ascending on ties.  keep_out receives the kept ORIGINAL indices in ascending order,
 * *n_keep (device int) their count.  Fully device-resident (no host scan, no D2H). */
size_t step_nms_workspace_bytes(int n);
int step_nms_f32(const float* boxes /*[n,4]*/, const float* scores /*[n]*/, int n, float thr, int ge,
                 int64_t* keep_out /*[n]*/, int* n_keep, void* workspace, size_t ws_bytes,
                 step_stream_t stream);
/* Many independent small problems in one launch (the per-clip x per-class loop of test.py:178-201):
 * segment s = rows [seg_offsets[s], seg_offsets[s+1]); at most 1024 rows per segment.
 * keep_mask[i] = 1 if row i survives NMS inside its segment.  Rows with score < min_score are
 * dropped before NMS (test.py:183 confidence threshold; pass -INF to disable). */
int step_nms_segmented_f32(const float* boxes, const float* scores, const int* seg_offsets, int n_seg,
                           float thr, int ge, float min_score, uint8_t* keep_mask, step_stream_t stream);
/* Rows one segment may hold (shared-memory resident problem); a longer segment traps instead of overrunning. */
int step_nms_segmented_max_rows(void);

/* Detection post-processing of the reference drivers (test.py:156-218, demo.py:121-198) in two launches, no host
 * round trip: for every (clip, class) keep the tubes whose class score > conf_thresh (scores.gt, test.py:183), clamp
 * their box with valid_tubes(valid_w, valid_h) (the drivers use its 400x400 defaults, test.py:191), greedy NMS with the
 * cpu/nms_cpu.cpp predicate, divide by (norm_w, norm_h) (test.py:197-198); then per clip either all survivors in file
 * order (class, tube) when topk <= 0, or the topk best in the order of the tuple sort of test.py:205-208.
 *   prob [n_rows, prob_ld >= ncls]  class scores of the centre frame;  loc: centre-frame box of row r at loc + r*loc_ld
 *   clip_offsets [n_clips+1] (device int32): rows of clip b = [clip_offsets[b], clip_offsets[b+1]), at most
 *   step_nms_segmented_max_rows() of them (max_per_clip is the caller's host-side bound, checked here).
 * Candidate arrays (index clip_start*ncls + class*n_clip + tube): keep [n_rows*ncls] u8, score [n_rows*ncls],
 * box [n_rows*ncls, 4] normalised.  Compact result: det [n_clips, cap, 8] = {x1, y1, x2, y2, score, class, tube, 0},
 * det_count [n_clips] (int32, <= cap). */
int step_detect_f32(const float* prob, int prob_ld, const float* loc, int loc_ld, const int* clip_offsets,
                    int n_clips, int n_rows, int max_per_clip, int ncls, float conf_thresh, float nms_thresh,
                    int ge, float valid_w, float valid_h, float norm_w, float norm_h, int topk, int cap,
                    uint8_t* keep, float* score, float* box, float* det, int* det_count, step_stream_t stream);
/* Class-only detections of the classification pre-training stage's validation (train_cls.py:505-543) in one launch: for
 * every clip, class and row of the clip, in that order (the reference's file order), the row's class score when it is
 * > conf_thresh (scores.gt), with the row's box divided by (norm_w, norm_h) in float32.  No valid_tubes clamp, no NMS, no
 * top-k.  prob [n_rows, prob_ld >= ncls]; the box of row r at box + r*box_ld (the centre frame of a flat tube, e.g.
 * flat_tubes[:, T/2, 1:5]); clip_offsets as for step_detect_f32, at most max_per_clip rows per clip.  det [n_clips, cap, 8]
 * = {x1, y1, x2, y2, score, class, row in clip, 0}, det_count [n_clips]; cap >= max_per_clip * ncls, so no row is cut. */
int step_detect_scores_f32(const float* prob, int prob_ld, const float* box, int box_ld, const int* clip_offsets,
                           int n_clips, int n_rows, int max_per_clip, int ncls, float conf_thresh, float norm_w,
                           float norm_h, int cap, float* det, int* det_count, step_stream_t stream);
/* The checks of step_detect_scores_f32, with no launch. */
int step_detect_scores_check(const float* prob, int prob_ld, const float* box, int box_ld, const int* clip_offsets,
                             int n_clips, int n_rows, int max_per_clip, int ncls, int cap, const float* det,
                             const int* det_count);

/* ------------------------------------------------------------------ ROI ops -------------- */
/* Reference layout (NCHW fp32 in, [R,C,ph,pw] fp32 out), arithmetic order of the reference. */
int step_roi_align_fwd_nchw_f32(const float* feat, int K, int C, int H, int W, const float* rois, int R,
                                float scale, int ph, int pw, int sampling_ratio, float* out,
                                step_stream_t stream);
int step_roi_align_bwd_nchw_f32(const float* grad_out, const float* rois, int R, float scale, int ph,
                                int pw, int K, int C, int H, int W, int sampling_ratio,
                                float* grad_in /* zero-filled by the call */, step_stream_t stream);
int step_roi_pool_fwd_nchw_f32(const float* feat, int K, int C, int H, int W, const float* rois, int R,
                               float scale, int ph, int pw, float* out, int32_t* argmax,
                               step_stream_t stream);
int step_roi_pool_bwd_nchw_f32(const float* grad_out, const int32_t* argmax, const float* rois, int R,
                               int ph, int pw, int K, int C, int H, int W,
                               float* grad_in /* zero-filled by the call */, step_stream_t stream);
/* Channels-last fast path: feat [K,H,W,C] (channel stride feat_ld), out [R,ph,pw,C] (channel
 * stride out_ld).  dtype STEP_F32 / STEP_F16 (fp32 accumulation, same operation order as the
 * reference; the fp32 variant is bit-identical to the NCHW one up to the permutation).
 * C must be a multiple of 8 (f16) / 4 (f32); feat_ld, out_ld likewise.
 * Frame map: ROI column 0 indexes frames of the slice conv_feat[:, t_start:t_start+roi_T]
 * (utils/utils.py:48); with roi_T > 0 the kernel reads frame (f / roi_T) * feat_T + t_start + f % roi_T
 * of the full map instead of needing the slice copied.  roi_T == 0: identity.
 * exact == 1: reference operation order, bit-identical (always used for f32).  f16 storage only: exact == 2:
 * 1/count folded into the tap weights, one fp32 FMA per tap (within one fp16 ulp of the exact result);
 * exact == 0: per-pixel merged weights + packed half2 FMAs (a convex combination: a few fp16 ulps). */
int step_roi_align_fwd_nhwc(const void* feat, int dtype, int K, int H, int W, int C, int feat_ld,
                            const float* rois, int R, float scale, int ph, int pw, int sampling_ratio,
                            void* out, int out_ld, int roi_T, int feat_T, int t_start, int exact,
                            step_stream_t stream);
int step_roi_pool_fwd_nhwc(const void* feat, int dtype, int K, int H, int W, int C, int feat_ld,
                           const float* rois, int R, float scale, int ph, int pw, void* out, int out_ld,
                           int roi_T, int feat_T, int t_start, step_stream_t stream);
/* step_roi_pool_fwd_nhwc for training: the same pooled values bit for bit, plus argmax [R,ph,pw,C] int32 (channel
 * stride C, 16-byte aligned) holding the frame-local pixel h*W + w of each maximum as cuda/ROIPool_cuda.cu:40-101 picks it
 * (strict `>` from -FLT_MAX, h outer, w inner: on ties the first pixel in scan order wins), -1 for an empty bin.
 * H*W must not exceed the 6400 pixels step_roi_pool_bwd_slice_nhwc accepts (STEP_E_ARG otherwise). */
int step_roi_pool_fwd_argmax_nhwc(const void* feat, int dtype, int K, int H, int W, int C, int feat_ld,
                                  const float* rois, int R, float scale, int ph, int pw, void* out, int out_ld,
                                  int roi_T, int feat_T, int t_start, int32_t* argmax, step_stream_t stream);

/* ------------------------------------------------------------------ tube arithmetic ------ */
/* boxes are rows of 4 floats with a row stride (in floats) so the [.,5] flat-tube layout
 * (frame index first, tube_utils.py:238) can be addressed in place. */
int step_tube_decode_f32(const float* anchors, int anchor_stride, const float* deltas, int n, float* out,
                         step_stream_t stream);                         /* tube_utils.py:165-189 */
int step_tube_encode_f32(const float* gt, const float* anchors, int anchor_stride, int n, float* out,
                         step_stream_t stream);                         /* tube_utils.py:143-163 */
int step_tube_valid_f32(float* boxes /*in place, [n,4]*/, int n, float width, float height,
                        step_stream_t stream);                          /* tube_utils.py:59-92 */
int step_tube_extrapolate_f32(const float* tubes /*[n,L,4]*/, int n, int L, int T, float width,
                              float height, float* out /*[n,L+2T,4]*/, step_stream_t stream); /* :10-27 */
int step_tube_extend_f32(const float* tubes /*[n,5]*/, int n, float ratio, float width, float height,
                         float* out /*[n,5]*/, step_stream_t stream);   /* tube_utils.py:248-266 */
/* One launch for the whole between-steps host loop of utils/utils.py:61-129:
 * decode (local, and first/last when mode==PREDICT) -> optional temporal extension
 * (concat / extrapolate / mean) -> valid_tubes -> re-flatten with new frame indices.
 * flat_in [R,L,5]; loc/first/last [R,L,4]/[R,T,4]/[R,T,4]; clip_of_tube [R] int32;
 * pred_* are the history tensors; flat_out [R,L_out,5] with L_out = extend ? L+2T : L. */
enum { STEP_EXT_NONE = 0, STEP_EXT_PREDICT = 1, STEP_EXT_EXTRAPOLATE = 2, STEP_EXT_MEAN = 3 };
int step_tube_update_f32(const float* flat_in, const float* loc, const float* first, const float* last,
                         const int32_t* clip_of_tube, int R, int L, int T, int decode_neighbors,
                         int ext_mode, float width, float height, float* pred_loc, float* pred_first,
                         float* pred_last, float* flat_out, step_stream_t stream);

/* ------------------------------------------------------------------ layout --------------- */
/* clip [N,T,Cc,H,W] fp32 (the layout BaseNet.forward receives, networks.py:69-76) ->
 * channels-last [N,T,H,W,ld] in `dtype`, channels >= Cc zero-filled. */
int step_clip_to_ndhwc(const float* clip, int N, int T, int Cc, int H, int W, void* out, int dtype, int ld,
                       step_stream_t stream);
/* Same input, space-to-depth by 2 in (T,H,W) for the stride-2 stem (i3dpt.py:184-189):
 * out [N,T/2,H/2,W/2,ld] f16 with channel = ((rt*2+rh)*2+rw)*Cc + c. T,H,W must be even. */
int step_clip_to_s2d_f16(const float* clip, int N, int T, int Cc, int H, int W, void* out, int ld,
                         step_stream_t stream);
/* channels-last [M, C] (stride ld) <-> planar [N, C, S] fp32, M = N*S (boundary conversions). */
int step_nhwc_to_nchw_f32(const void* in, int dtype, int N, int S, int C, int ld, float* out,
                          step_stream_t stream);
int step_nchw_to_nhwc(const float* in, int N, int S, int C, void* out, int dtype, int ld,
                      step_stream_t stream);

/* ------------------------------------------------------------------ input -------------- */
/* One source clip of step_frames_to_clip_u8: uint8 frames of H0 x W0 pixels, 3 channels, addressed as
 * data[t*stride_t + c*stride_c + y*stride_h + x*stride_w] (strides in elements; any sign).  A stacked [B,T,3,H0,W0]
 * tensor, a per-clip view and cv2's HWC-BGR frames (stride_c = -1 from the last channel) are all just strides. */
typedef struct {
  const uint8_t* data;
  int H0, W0;
  long long stride_t, stride_c, stride_h, stride_w;
} step_frame_src;
/* The reference's BaseTransform (data/augmentations.py:601-615: ConvertFromInts(scale), cv2.resize INTER_LINEAR on float32,
 * SubtractMeans, DivideStds) followed by its dataset's permute, for B clips of T frames in one launch:
 * out [B,T,3,H,W] fp32 contiguous, channel c of the output reading channel c of the source.
 *   scale_mode 2: u*2/255 - 1, 1: u/255, 0: u; each step rounded in fp32 and applied before interpolation.
 *   Resize: cv2 4.x's generic (non-IPP) INTER_LINEAR arithmetic bit for bit, including its unclamped row weights at the
 *   border rows and its switch to INTER_AREA for an exact 2x downscale in both axes.
 *   mean3 / std3: HOST arrays indexed by output channel; out = (resized - mean3[c]) / std3[c].
 * `table` is a DEVICE array of B entries, read by the kernel: it is not validated here.  Each entry needs H0, W0 > 0 and
 * W0 <= 48 * W (a tile's source columns must fit shared memory; tiles of an entry beyond that are written as NaN). */
int step_frames_to_clip_u8(const step_frame_src* table, int B, int T, int H, int W, int scale_mode, const float* mean3,
                           const float* std3, float* out, step_stream_t stream);

/* What the reference's TubeAugmentation (data/augmentations.py:540-589) drew for one clip, in source pixels.  The host
 * stage (step_b200.transforms.TubeAugmentation) fills it in the DataLoader workers. */
typedef struct {
  int x0, y0, w, h;          /* RandomSampleCrop's rect: source columns x0..x0+w-1, rows y0..y0+h-1 (the whole frame if none) */
  int flip;                  /* RandomMirror: the crop is mirrored horizontally */
  int photometric;           /* PhotometricDistort ran: the program below, with its HSV round trip, precedes the rest */
  int brightness, contrast, contrast_first, saturation, hue;  /* the ops' gates; contrast_first: before the HSV round trip */
  float brightness_delta, contrast_alpha, saturation_alpha, hue_delta;  /* fp32, as applied */
  int perm[3];               /* RandomLightingNoise: BGR channel k of the result is channel perm[k] (identity: 0,1,2) */
  int erase_begin, erase_count;  /* this clip's RandomErase regions: erase[erase_begin .. erase_begin+erase_count-1] */
} step_clip_aug;
/* One RandomErase region, in the coordinates of the mirrored crop; later regions of a clip cover earlier ones.  Its values
 * are noise[noise .. noise + (y2-y1)*(x2-x1)*3 - 1], fp32 [y2-y1, x2-x1, 3] in BGR order, the same for every frame. */
typedef struct {
  int x1, y1, x2, y2;
  long long noise;
} step_aug_erase;
/* The reference's TubeAugmentation followed by its dataset's swap to RGB and permute, for B clips of T frames in one launch:
 * out [B,T,3,H,W] fp32 contiguous.  Per pixel, in the reference's order: u8 BGR -> f32; PhotometricDistort (brightness,
 * contrast, cv2's float BGR2HSV, saturation, hue with its wrap, cv2's HSV2BGR, contrast; cv2 4.x's arithmetic bit for bit,
 * DESIGN.md); the channel permutation; ConvertFromInts(scale_mode) (np.clip to [0, 255] first when scale_mode
 * is 2 and the clip is distorted); the erase regions.  Then the crop, mirrored when flipped, is resized and normalised as
 * step_frames_to_clip_u8 resizes and normalises the whole frame.
 * `table`, `params` (B entries), `erase` and `noise` are DEVICE arrays read by the kernel and are not validated here; erase
 * and noise may both be NULL when no clip erases.  Each entry needs its crop inside the frame, w, h > 0 and w <= 48 * W. */
int step_frames_to_clip_aug_u8(const step_frame_src* table, const step_clip_aug* params, const step_aug_erase* erase,
                               const float* noise, int B, int T, int H, int W, int scale_mode, const float* mean3,
                               const float* std3, float* out, step_stream_t stream);

/* ------------------------------------------------------------------ conv / pool / linear - */
/* step_conv_params.a_mode, the addressing of the f16 path: auto (linear for 1x1x1, else box), linear (1x1x1 only), box
 * tiles, TMA im2col, halo (input patch staged in shared memory: stride 1, Cin in {16,32,64}, Cout <= 256; or the s2d
 * stem, see zero_cin_last_kt), best of im2col / halo per layer shape, SIMT (the kernel of the fp32 path). */
enum { STEP_A_AUTO = 0, STEP_A_LINEAR = 1, STEP_A_BOX = 2, STEP_A_IM2COL = 3, STEP_A_HALO = 4, STEP_A_BEST = 5,
       STEP_A_SIMT = 9 };
typedef struct {
  int dtype;                 /* STEP_F32: SIMT fp32 path.  STEP_F16: wgmma implicit GEMM, fp32 accumulate */
  int N, T, H, W;            /* input extent (pixels) */
  int Cin, in_ld;            /* input channels read, channel stride of x */
  int Cout, out_ld, out_coff;/* output channels, channel stride of y, first channel written in y */
  int KT, KH, KW;            /* filter taps */
  int ST, SH, SW;            /* strides (the f16 path supports stride 1 only; the stem uses s2d) */
  int PT, PH, PW;            /* low-side zero padding (TF "SAME": i3dpt.py:14-31) */
  int OT, OH, OW;            /* output extent */
  int relu;                  /* apply max(.,0) last */
  int w_ld;                  /* weight channel stride: w is [Cout, KT, KH, KW, w_ld] in `dtype` */
  const void* x;
  const void* w;
  const float* scale;        /* per-Cout multiplier (folded BatchNorm, i3dpt.py:107) or NULL (=1) */
  const float* shift;        /* per-Cout addend (folded BN shift / conv bias) or NULL (=0) */
  const void* residual;      /* optional tensor added before relu (two_branch.py:79-81), layout of y */
  int res_ld, res_coff;
  void* y;
  int a_mode;                /* STEP_A_* (f16 path) */
  /* Horizontally fused 1x1x1 layers that share an input (Mixed.branch_0 / branch_1[0] / branch_2[0],
   * i3dpt.py:133-147): output channels [0, split[0]) go to y, [split[0], split[1]) to y_extra[0],
   * [split[1], Cout) to y_extra[1], each with its own channel stride / offset.  n_splits = 0: plain conv.
   * f16 1x1x1 only; split points must be multiples of 16. */
  int n_splits;
  int split[2];
  void* y_extra[2];
  int ld_extra[2];
  int coff_extra[2];
  /* Structured zeros of the weights (STEP_A_HALO only): for the filter taps of the LAST t plane (kt == KT-1) the input
   * channels [zero_cin_last_kt, Cin) carry zero weights.  0 = no such structure.  The space-to-depth stem has it: tap plane
   * qt = 2 only holds the rt = 0 sub-position (k = 2(q+1)+r <= 6), engine.pack_stem_s2d.  The stem kernel (STEP_A_HALO,
   * Cin = 24, Cout = 64, 4x4x4, pad 1) is chosen only when 0 < zero_cin_last_kt <= 16 and skips channels 16..23 of that
   * plane; the generic patch kernel multiplies the zeros. */
  int zero_cin_last_kt;
} step_conv_params;
int step_conv3d_fwd(const step_conv_params* p, step_stream_t stream);
/* Test hook of the f16 path: the raw bytes of the A tile m_tile, tap (kt, kh, kw), channels from c0, as the TMA stages it
 * in shared memory -> out [128 * BK * 2]; *bk_out = BK, box_out [3] = the box tile's (w, h, t) extent. */
int step_debug_tma_tile(const step_conv_params* p, int m_tile, int kt, int kh, int kw, int c0, void* out, int* bk_out,
                        int* box_out, step_stream_t stream);

/* MaxPool3dTFPadding (i3dpt.py:114-126): zero pad (low PT/PH/PW, high implied), ceil_mode. */
int step_maxpool3d_fwd(const void* x, int dtype, int N, int T, int H, int W, int C, int in_ld, int KT,
                       int KH, int KW, int ST, int SH, int SW, int PT, int PH, int PW, int pad_hi_t,
                       int pad_hi_h, int pad_hi_w, int OT, int OH, int OW, void* y, int out_ld,
                       step_stream_t stream);
/* mean over axis B: x [A, B, P, C] (C contiguous, pixel stride ld) -> y [A, P*C] fp32/f16
 * (the temporal mean of two_branch.py:249 taken before the classifier, which is linear). */
int step_mean_mid(const void* x, int dtype, int A, int B, int P, int C, int ld, void* y, int out_dtype,
                  step_stream_t stream);
/* step_mean_mid with row a of x at a * a_stride elements (a_stride >= B * P * ld): the mean over a slice of axis B of a
 * wider tensor, e.g. ContextNet's [clips, T', 1024] output over one refinement step's frames (train.py:317-321). */
int step_mean_mid_strided(const void* x, int dtype, int A, int B, int P, int C, int ld, long long a_stride, void* y,
                          int out_dtype, step_stream_t stream);
/* y[m, n] = act(sum_k x[m,k] * w[n,k] + bias[n]); small-N GEMM (N <= 64) for global_cls,
 * local_reg, neighbor_reg (two_branch.py:246,261,269-270).  x [M,K] (row stride x_ld) in dtype,
 * w [N,K] in dtype, y fp32 [M, y_ld].  act: 0 none, 1 sigmoid (applied after accumulation).
 * accumulate != 0: y += result.  row_map (optional, device int32 [M]): x row read for output row m
 * (the per-tube context gather of utils/utils.py:54-57).
 * Split-K with a caller-provided fp32 workspace of step_linear_small_n_workspace_bytes(M,K,N). */
size_t step_linear_small_n_workspace_bytes(int M, int K, int N);
int step_linear_small_n(const void* x, int dtype, int M, int K, int x_ld, const void* w, const float* bias,
                        int N, float* y, int y_ld, int act, int accumulate, const int32_t* row_map,
                        void* workspace, size_t ws_bytes, step_stream_t stream);

/* local_reg + neighbor_reg1 + neighbor_reg2 of TwoBranchNet (two_branch.py:261-270) in one pass over the
 * [R*T, K] feature rows: w12 = [W_local | W_nb1 | W_nb2] (12 x K), bias12 likewise.  Writes
 * local_loc [R,T,4], first_loc [R,s1-s0,4] = (local + nb1)[:, s0:s1], last_loc [R,e1-e0,4] = (local + nb2)[:, e0:e1].
 * workspace: step_linear_small_n_workspace_bytes(R*T, K, 12). */
int step_head_regress(const void* x, int dtype, int R, int T, int K, int x_ld, const void* w12, const float* bias12,
                      int s0, int s1, int e0, int e1, float* local_loc, float* first, float* last, void* workspace,
                      size_t ws_bytes, step_stream_t stream);

/* Exit of a 2-D bottleneck of the local branch fused with the 1x1 convolution that consumes it, fp16, channels-last rows:
 *   y[M, inplanes] = relu(h[M, planes] * w3[inplanes, planes]^T + x[M, inplanes])      Bottleneck.forward, models/two_branch.py:79-83
 *                                                                                 (Bottleneck_resample.forward, :106-110)
 *   z[M, outplanes] = act(y * w1[outplanes, inplanes]^T + shift2)                   the next block's conv1 + ReLU (:68-69, relu2 = 1,
 *                                                                                 shift2 = NULL) or downsample2 (:259, relu2 = 0, bias)
 * in one launch; y may be NULL when nothing else reads it.  Bit-identical to step_conv3d_fwd called twice.  Built for the
 * reference's fixed head widths planes = 256, inplanes = 1024, outplanes = 256 (two_branch.py:190-192); other widths return
 * STEP_E_ARG and the caller launches the two convolutions.  Row pitches in elements. */
int step_bottleneck_exit_f16(const void* h, long long h_ld, const void* w3, const void* x, long long x_ld, const void* w1,
                             const float* shift2, int relu2, void* y, long long y_ld, void* z, long long z_ld, long long M,
                             int planes, int inplanes, int outplanes, step_stream_t stream);

/* ------------------------------------------------------------------ training (first pieces) ---- */
/* TwoBranchNet's losses (models/two_branch.py:276-333) and, when the d* pointers are given, the gradient of the training
 * objective mean(loss_cls) + w_loc * loss_loc + w_nb * loss_nb (train.py:323-347) with respect to the head outputs.
 *   logits [N,cls] (pre-sigmoid), local_loc [N,T_len,4], first_loc / last_loc [N,Tc,4], tubes [N,T_len,5],
 *   targets [N,3,6+cls] = (first, centre, last) x (box 4 | cls mask | loc mask | labels).
 * loss_cls [N*cls] holds the element-wise BCE (all zeros when no sample is positive: flags[0] = 0 and the reference then
 * returns the scalar 0), loss_loc / loss_nb [1]; flags [3] = {cls, loc, neighbour mask sums non-zero}.
 * dloc [N,T_len,4] already includes what flows back through the first / last slices.  scratch: N*12 floats. */
int step_head_losses_f32(const float* logits, const float* local_loc, const float* first_loc, const float* last_loc,
                         const float* tubes, const float* targets, int N, int cls, int T_len, int T, int Tc, float w_loc,
                         float w_nb, float* loss_cls, float* loss_loc, float* loss_nb, int* flags, float* dlogits,
                         float* dloc, float* dfirst, float* dlast, float* scratch, step_stream_t stream);
/* The loss of a class-only head (TwoBranchNet(cls_only=True), models/two_branch.py:291-297; train_cls.py:310-311) and, when
 * dlogits is given, d mean(loss_cls) / d logits, with the arithmetic of step_head_losses_f32's classification part (bit for
 * bit the same loss_cls and dlogits).  logits [N,cls] (pre-sigmoid), targets [N,3,6+cls] (only the centre row is read).
 * loss_cls [N*cls] is the element-wise BCE; flags[0] = 0 when the centre rows' classification masks sum to zero, and then
 * loss_cls and dlogits are zeros (the reference returns a [1] zero loss). */
int step_cls_loss_f32(const float* logits, const float* targets, int N, int cls, float* loss_cls, int* flags, float* dlogits,
                      step_stream_t stream);
/* Channels-last ROIAlign backward without atomics (replaces _C.roi_align_backward, vision.cpp:33 /
 * cuda/ROIAlign_cuda.cu:201-278, whose atomicAdd scatter is not repeatable): grad_out [R,ph,pw,C] (channel stride
 * out_ld, STEP_F32 / STEP_F16) -> grad_in [K,H,W,C] fp32 (channel stride in_ld), written completely by the call. */
int step_roi_align_bwd_nhwc(const void* grad_out, int dtype, int out_ld, const float* rois, int R, float scale, int ph,
                            int pw, int K, int H, int W, int C, int sampling_ratio, float* grad_in, int in_ld,
                            step_stream_t stream);
/* step_roi_align_bwd_nhwc for ROIs whose frame index f is relative to the slice conv_feat[:, t_start:t_start+roi_T] of a
 * [K = clips * feat_T, H, W, C] map (the frame map of step_roi_align_fwd_nhwc).  The contribution of each ROI frame is formed
 * completely, in the same order as step_roi_align_bwd_nhwc, in a workspace of
 * step_roi_align_bwd_slice_workspace_bytes(K, H, W, C, roi_T, feat_T) bytes and then ADDED to grad_in frame
 * (f / roi_T) * feat_T + t_start + f % roi_T; frames outside the slice are untouched.  Deterministic, no atomics: with
 * t_start = 0 and roi_T = feat_T, calls on a zeroed grad_in give bit for bit the sum of the step_roi_align_bwd_nhwc results. */
size_t step_roi_align_bwd_slice_workspace_bytes(int K, int H, int W, int C, int roi_T, int feat_T);
int step_roi_align_bwd_slice_nhwc(const void* grad_out, int dtype, int out_ld, const float* rois, int R, float scale, int ph,
                                  int pw, int K, int H, int W, int C, int sampling_ratio, int roi_T, int feat_T, int t_start,
                                  float* grad_in, int in_ld, void* workspace, size_t ws_bytes, step_stream_t stream);
/* Channels-last ROIPool backward without atomics (replaces _C.roi_pool_backward, vision.cpp:35 / cuda/ROIPool_cuda.cu:103-132,
 * whose atomicAdd scatter is not repeatable), with the frame contract of step_roi_align_bwd_slice_nhwc: grad_out [R,ph,pw,C]
 * (channel stride out_ld, STEP_F32 / STEP_F16) and argmax [R,ph,pw,C] of step_roi_pool_fwd_argmax_nhwc for ROIs whose frame
 * index f is relative to the slice conv_feat[:, t_start:t_start+roi_T] of a [K = clips * feat_T, H, W, C] map; the
 * contribution is ADDED to grad_in (fp32, channel stride in_ld) frame (f / roi_T) * feat_T + t_start + f % roi_T, frames
 * outside the slice are untouched.  Every element sums its contributions in ascending (ROI row, ph, pw) order, the loop order
 * of torchvision's CPU roi_pool backward: with fp32 grad_out on a zeroed grad_in the result is bit-identical to it.  The
 * per-frame accumulator lives in shared memory: H*W must not exceed 6400 (STEP_E_ARG otherwise). */
int step_roi_pool_bwd_slice_nhwc(const void* grad_out, int dtype, int out_ld, const int32_t* argmax, const float* rois, int R,
                                 int ph, int pw, int K, int H, int W, int C, int roi_T, int feat_T, int t_start,
                                 float* grad_in, int in_ld, step_stream_t stream);
/* Gradient of ContextNet's output from one refinement step (train.py:317-321): dctx [R, C] (row stride dctx_ld) is the
 * gradient of each tube's context input of the classifier, tubes [R, T_len, 5] the step's flat tubes (frame index first).
 * acc [B, feat_T, C] fp32 += (sum over the tubes of clip b = floor(frame / T_len), ascending tube order) / T_len on frames
 * [t_start, t_start + T_len) of clip b.  Deterministic, no atomics. */
int step_ctx_grad_reduce_f32(const float* dctx, int dctx_ld, const float* tubes, int R, int T_len, int B, int feat_T,
                             int t_start, int C, float* acc, step_stream_t stream);
/* Backward of y = x W^T + b for the small-N linears of the head (nn.Linear / global_cls, two_branch.py:246-270):
 * dx [M,K] (+)= dy W, dw [Nn,K] = dy^T x, db [Nn] = column sums of dy; any of dx / dw may be NULL.  Fixed summation order. */
int step_linear_small_n_bwd(const void* x, int dtype, int M, int K, int x_ld, const float* w, const float* dy, int Nn,
                            float* dx, int dx_accumulate, float* dw, float* db, step_stream_t stream);
/* Weight gradient of a 1x1(x1) convolution: dw[Cout,Cin] (+)= scale * sum_m dz[m,co] x[m,ci]; fp16 operands, fp32
 * tensor-core accumulation, pixel chunks reduced in a fixed order (deterministic). */
size_t step_conv1x1_wgrad_workspace_bytes(int M, int Cout, int Cin);
int step_conv1x1_wgrad_f16(const void* dz, int dz_ld, const void* x, int x_ld, int M, int Cout, int Cin, float scale,
                           float* dw, int dw_ld, int accumulate, void* workspace, size_t ws_bytes, step_stream_t stream);

/* Weight gradient of a stride-1 convolution with KT x KH x KW taps and low padding (PT, PH, PW) (zero outside the map):
 * dw[Cout, taps, dw_ld >= Cin] (+)= scale * sum_m dz[m, co] x[shift_tap(m), ci], x and dz on the same [N,T,H,W] pixel grid. */
size_t step_conv_wgrad_workspace_bytes(int M, int Cout, int Cin, int taps);
int step_conv_wgrad_f16(const void* dz, int dz_ld, const void* x, int x_ld, int N, int T, int H, int W, int Cout, int Cin,
                        int KT, int KH, int KW, int PT, int PH, int PW, float scale, float* dw, int dw_ld, int accumulate,
                        void* workspace, size_t ws_bytes, step_stream_t stream);
/* y = relu(scale * conv + shift (+ residual)): dz = dy * [y > 0] * scale (dense [M, C] at dz_ld), and, when dres is given,
 * dres += dy * [y > 0] (the residual input's gradient, accumulated in place).  fp16, channel slices via the ld arguments. */
int step_act_bwd_f16(const void* dy, int dy_ld, const void* y, int y_ld, const float* scale, int relu, long long M, int C,
                     void* dz, int dz_ld, void* dres, int dres_ld, step_stream_t stream);
/* out[c] = scale * sum_m x[m, c] (bias gradients); workspace >= 64 * C floats; fixed summation order. */
int step_colsum_f16(const void* x, int ld, long long M, int C, float scale, float* out, float* workspace, step_stream_t stream);
/* Backward of step_mean_mid: dx[a, b, p, c] += gscale * g[a, p*C + c] / B (fp16 dx, channel stride ld). */
int step_mean_mid_bwd(const float* g, int A, int B, int P, int C, float gscale, void* dx, int ld, step_stream_t stream);
/* dst[m, c] (fp16, channel stride ld) += gscale * src[m, c] (fp32 [M, C]). */
int step_f32_accum_f16(const float* src, long long M, int C, float gscale, void* dst, int ld, step_stream_t stream);
/* Backward of step_maxpool3d_fwd (zero padding takes part in the maximum, first maximum in scan order wins as in ATen):
 * dx += scatter(dy) without atomics; argmax_ws: N*OT*OH*OW*C bytes of scratch. */
int step_maxpool3d_bwd_f16(const void* x, int x_ld, const void* dy, int dy_ld, int N, int T, int H, int W, int C, int KT,
                           int KH, int KW, int ST, int SH, int SW, int PT, int PH, int PW, int pad_hi_t, int pad_hi_h,
                           int pad_hi_w, int OT, int OH, int OW, void* dx, int dx_ld, uint8_t* argmax_ws, step_stream_t stream);

/* The fp32 training path (cfg.fp16 = False: fp32 activations and activation gradients).
 * Weight gradient of a convolution with any filter, stride and low padding on the CUDA cores (fp32 FFMA, no TF32):
 * dw[Cout, taps, dw_ld >= Cin] (+)= scale * sum_m dz[m, co] x[src(m, tap), ci] over the N*OT*OH*OW output pixels m, where
 * tap (kt, kh, kw) of output pixel (n, ot, oh, ow) reads input pixel (n, ot*ST + kt - PT, oh*SH + kh - PH, ow*SW + kw - PW)
 * of x [N, T, H, W] (zero outside).  dz [M, dz_ld], x [N*T*H*W, x_ld]; Cout, Cin and the strides multiples of 4; 16-byte
 * aligned operands.  The pixel chunks' partial sums are added in a fixed order: bit-identical from run to run. */
size_t step_conv_wgrad_f32_workspace_bytes(long long M, int Cout, int Cin, int taps);
int step_conv_wgrad_f32(const float* dz, int dz_ld, const float* x, int x_ld, int N, int T, int H, int W, int OT, int OH,
                        int OW, int Cout, int Cin, int KT, int KH, int KW, int ST, int SH, int SW, int PT, int PH, int PW,
                        float scale, float* dw, int dw_ld, int accumulate, void* workspace, size_t ws_bytes,
                        step_stream_t stream);
/* fp32 storage siblings of step_act_bwd_f16 (C and the ld arguments multiples of 4), step_colsum_f16, step_mean_mid_bwd,
 * step_f32_accum_f16 and step_maxpool3d_bwd_f16, with the same arithmetic in fp32 and no rounding to fp16. */
int step_act_bwd_f32(const float* dy, int dy_ld, const float* y, int y_ld, const float* scale, int relu, long long M, int C,
                     float* dz, int dz_ld, float* dres, int dres_ld, step_stream_t stream);
int step_colsum_f32(const float* x, int ld, long long M, int C, float scale, float* out, float* workspace, step_stream_t stream);
int step_mean_mid_bwd_f32(const float* g, int A, int B, int P, int C, float gscale, float* dx, int ld, step_stream_t stream);
int step_f32_accum_f32(const float* src, long long M, int C, float gscale, float* dst, int ld, step_stream_t stream);
int step_maxpool3d_bwd_f32(const float* x, int x_ld, const float* dy, int dy_ld, int N, int T, int H, int W, int C, int KT,
                           int KH, int KW, int ST, int SH, int SW, int PT, int PH, int PW, int pad_hi_t, int pad_hi_h,
                           int pad_hi_w, int OT, int OH, int OW, float* dx, int dx_ld, uint8_t* argmax_ws, step_stream_t stream);

/* BatchNorm affine gradients of y = relu(BN_eval(z)) = relu(scale * z + shift), scale = gamma / sqrt(running_var + eps), for a
 * Unit3Dpy whose gamma / beta train (freeze_affine=False).  Writes dz and dres exactly as step_act_bwd_f16 / _f32 (the same
 * arguments, bit for bit) and, from the same read of dy and y, with g = dy * [y > 0] (g = dy without relu):
 *   dbeta[c]  = gscale * sum_m g[m, c]
 *   dgamma[c] = gscale * (sum_m g[m, c] * (y[m, c] - beta[c])) / gamma[c]
 * because wherever g != 0, y = gamma * xhat + beta.  beta, gamma: fp32 [C], the BatchNorm's own parameters for the C channels
 * of the slice; gscale: 1 / loss_scale.  dgamma or dbeta may be NULL (not both).  gamma[c] == 0 gives dgamma[c] = 0, which
 * is exact when the channel's g is all zero (relu and beta[c] <= 0); with beta[c] > 0, xhat cannot be recovered from y and
 * the caller must refuse the channel.  Per-chunk partials go to the workspace (step_act_bn_bwd_workspace_bytes) and are added
 * in chunk order by a second kernel: no atomics, bit-identical from run to run.  C and the ld arguments multiples of the
 * 16-byte vector (8 fp16, 4 fp32), 16-byte aligned dy / y / dz / dres. */
size_t step_act_bn_bwd_workspace_bytes(long long M, int C);
int step_act_bn_bwd_f16(const void* dy, int dy_ld, const void* y, int y_ld, const float* scale, int relu, long long M, int C,
                        void* dz, int dz_ld, void* dres, int dres_ld, const float* beta, const float* gamma, float gscale,
                        float* dgamma, float* dbeta, void* workspace, size_t ws_bytes, step_stream_t stream);
int step_act_bn_bwd_f32(const float* dy, int dy_ld, const float* y, int y_ld, const float* scale, int relu, long long M, int C,
                        float* dz, int dz_ld, float* dres, int dres_ld, const float* beta, const float* gamma, float gscale,
                        float* dgamma, float* dbeta, void* workspace, size_t ws_bytes, step_stream_t stream);

/* BatchNorm with batch statistics (freeze_stats=False: BatchNorm3d in training mode, models/networks.py:85-99).  The
 * convolution writes z with the identity epilogue (no scale, shift or ReLU); these entries normalise it.  z, y, dy, dz are
 * channel slices of fp16 (_f16) or fp32 (_f32) buffers: C, every split and every ld a multiple of the 16-byte vector (8 fp16,
 * 4 fp32) and the pointers 16-byte aligned.  Statistics, parameters and sums are fp32.  Each reduction forms per-chunk
 * partials in the workspace that a second kernel combines in a fixed order: no atomics, bit-identical from run to run.
 *
 * step_bn_stats: per channel of z [M, C], mean and biased variance var (per-chunk Welford, chunks merged by Chan's formula) ->
 *   mean, rstd = 1 / sqrt(var + eps), scale = gamma * rstd, shift = beta - mean * scale.  With running_mean and running_var
 *   (both or neither): running = (1 - momentum) * running + momentum * batch, the unbiased variance M / (M - 1) * var for
 *   running_var (torch.nn.functional.batch_norm, training=True).  M < 2 is STEP_E_ARG, as torch refuses it. */
size_t step_bn_stats_workspace_bytes(long long M, int C);
int step_bn_stats_f16(const void* z, int z_ld, long long M, int C, const float* gamma, const float* beta, float eps, float momentum,
                      float* running_mean, float* running_var, float* mean, float* rstd, float* scale, float* shift,
                      void* workspace, size_t ws_bytes, step_stream_t stream);
int step_bn_stats_f32(const float* z, int z_ld, long long M, int C, const float* gamma, const float* beta, float eps, float momentum,
                      float* running_mean, float* running_var, float* mean, float* rstd, float* scale, float* shift,
                      void* workspace, size_t ws_bytes, step_stream_t stream);
/* y = relu(scale * z + shift) (relu = 0: no ReLU) for z [M, C]: columns [0, split1) go to y, [split1, split2) to y1 and
 * [split2, C) to y2, each range from its destination's column 0 (the three outputs of Mixed's fused 1x1 branches).  One
 * destination: split1 = split2 = C, y1 = y2 = NULL. */
int step_bn_apply_f16(const void* z, int z_ld, long long M, int C, const float* scale, const float* shift, int relu, void* y,
                      int y_ld, int split1, void* y1, int y1_ld, int split2, void* y2, int y2_ld, step_stream_t stream);
int step_bn_apply_f32(const float* z, int z_ld, long long M, int C, const float* scale, const float* shift, int relu, float* y,
                      int y_ld, int split1, float* y1, int y1_ld, int split2, float* y2, int y2_ld, step_stream_t stream);
/* Backward of y = relu(BN_train(z)) with g = dy * [y > 0] (g = dy without relu; y may then be NULL) and
 * xhat = (z - mean) * rstd, from step_bn_stats' mean and rstd:
 *   dz = gamma * rstd * (g - sum(g) / M - xhat * sum(g xhat) / M)     (in the storage type, at dz_ld; keeps dy's loss scale)
 *   dbeta = gscale * sum g,  dgamma = gscale * sum g xhat              (either may be NULL)
 * gscale: 1 / loss_scale.  Three launches: per-chunk partials, their sums in chunk order, the dz pass. */
size_t step_bn_bwd_workspace_bytes(long long M, int C);
int step_bn_bwd_f16(const void* dy, int dy_ld, const void* y, int y_ld, const void* z, int z_ld, long long M, int C,
                    const float* mean, const float* rstd, const float* gamma, int relu, float gscale, void* dz, int dz_ld,
                    float* dgamma, float* dbeta, void* workspace, size_t ws_bytes, step_stream_t stream);
int step_bn_bwd_f32(const float* dy, int dy_ld, const float* y, int y_ld, const float* z, int z_ld, long long M, int C,
                    const float* mean, const float* rstd, const float* gamma, int relu, float gscale, float* dz, int dz_ld,
                    float* dgamma, float* dbeta, void* workspace, size_t ws_bytes, step_stream_t stream);
/* The same statistics and backward split around a cross-rank exchange (synchronised BatchNorm: several ranks, each holding
 * some rows of one batch, normalise with the statistics of all of them).  Each rank runs the local entry on its own z, the
 * caller gathers every rank's output into one [ranks, ...] array in rank order, and each rank runs the merge on that array.
 * The merges combine the ranks in a fixed order, so every rank computes identical statistics and coefficients from the same
 * gathered array; with ranks = 1 local + merge give the fused entries' outputs bit for bit.  A rank may hold M = 1 pixel;
 * the merges refuse a total M < 2, as torch does.
 * step_bn_stats_local: this rank's (count, mean, M2) of every channel of z [M, C] -> stats [3, stats_ld] fp32 (columns
 *   [0, C)); workspace step_bn_stats_workspace_bytes(M, C).
 * step_bn_stats_merge: stats [ranks, 3, stats_ld] (every rank's step_bn_stats_local, columns [0, C)) merged by Chan's formula
 *   -> mean, rstd, scale, shift and the running-statistic update of step_bn_stats, with M the total count over the ranks.
 * step_bn_bwd_sums: this rank's sums (sum g, sum g xhat) -> sums [2, sums_ld] fp32 (columns [0, C)), and its own
 *   dbeta = gscale * sum g, dgamma = gscale * sum g xhat (either may be NULL); workspace step_bn_bwd_sums_workspace_bytes.
 * step_bn_bwd_merge_dz: sums [ranks, 2, sums_ld] added in rank order, then dz of this rank's M rows as step_bn_bwd forms it,
 *   with the total count M_total over the ranks; workspace step_bn_bwd_merge_dz_workspace_bytes(C). */
int step_bn_stats_local_f16(const void* z, int z_ld, long long M, int C, float* stats, int stats_ld, void* workspace, size_t ws_bytes,
                            step_stream_t stream);
int step_bn_stats_local_f32(const float* z, int z_ld, long long M, int C, float* stats, int stats_ld, void* workspace, size_t ws_bytes,
                            step_stream_t stream);
int step_bn_stats_merge(const float* stats, int ranks, int stats_ld, long long M, int C, const float* gamma, const float* beta, float eps,
                        float momentum, float* running_mean, float* running_var, float* mean, float* rstd, float* scale, float* shift,
                        step_stream_t stream);
size_t step_bn_bwd_sums_workspace_bytes(long long M, int C);
int step_bn_bwd_sums_f16(const void* dy, int dy_ld, const void* y, int y_ld, const void* z, int z_ld, long long M, int C,
                         const float* mean, const float* rstd, int relu, float gscale, float* sums, int sums_ld, float* dgamma,
                         float* dbeta, void* workspace, size_t ws_bytes, step_stream_t stream);
int step_bn_bwd_sums_f32(const float* dy, int dy_ld, const float* y, int y_ld, const float* z, int z_ld, long long M, int C,
                         const float* mean, const float* rstd, int relu, float gscale, float* sums, int sums_ld, float* dgamma,
                         float* dbeta, void* workspace, size_t ws_bytes, step_stream_t stream);
size_t step_bn_bwd_merge_dz_workspace_bytes(int C);
int step_bn_bwd_merge_dz_f16(const float* sums, int ranks, int sums_ld, long long M_total, const void* dy, int dy_ld, const void* y,
                             int y_ld, const void* z, int z_ld, long long M, int C, const float* mean, const float* rstd,
                             const float* gamma, int relu, void* dz, int dz_ld, void* workspace, size_t ws_bytes, step_stream_t stream);
int step_bn_bwd_merge_dz_f32(const float* sums, int ranks, int sums_ld, long long M_total, const float* dy, int dy_ld, const float* y,
                             int y_ld, const float* z, int z_ld, long long M, int C, const float* mean, const float* rstd,
                             const float* gamma, int relu, float* dz, int dz_ld, void* workspace, size_t ws_bytes, step_stream_t stream);

/* ------------------------------------------------------------------ the heads' dropout ---- */
/* One draw of torch.nn.functional.dropout(x, p, training=True) on a CUDA fp32 tensor of n elements (n % 4 == 0, n < 2^31,
 * 16-byte aligned and contiguous, as every dropout input of the heads is): seed and offset are the device generator's
 * initial_seed() and get_offset() before the draw, sm_count and threads_per_sm the device's multi_processor_count and
 * max_threads_per_multi_processor, which set torch's launch geometry and with it which random number every element takes.
 * The entries below reproduce that draw's keep mask bit for bit and regenerate it in the backward (nothing is stored); an
 * element is kept with factor (float)(1.0 / (double)(float)(1 - p)), dropped with factor 0.  The geometry is
 * step_b200/csrc/dropout.cuh's.  Every entry returns STEP_E_ARG for keep outside (0, 1) (torch draws nothing at p = 0 or 1),
 * non-positive sm_count or threads_per_sm < 256, and null pointers, and STEP_E_UNSUPPORTED for other n, before any launch.
 * The two draws of a head (two_branch.py:244, 261), each over the reference's tensor and element order:
 *   global  [R, C' = C*P + ctx_cols, T], element (r*C' + c')*T + t: c' = c*P + p is the downsample output's channel c at pixel
 *           p of frame t; c' = C*P + k is context column k (ctx_cols = 1024 with context, 0 without);
 *   local   [F = R*T, C, P], element (f*C + c)*P + p: downsample2's output, channel c at pixel p of frame row f.
 * Inputs and outputs stay in this library's channels-last layouts; the map to the reference's order is the entries' own. */
typedef struct {
  uint64_t seed, offset;
  float keep;                      /* (float)(1 - p), 1 - p formed in double from the drop probability p as torch does */
  int sm_count, threads_per_sm;
} step_dropout_draw;
/* The argument checks of a draw of n elements; *offset_step (may be NULL) receives what the draw advances the generator's
 * offset by, ((n - 1) / (4 * n_threads) + 1) * 4. */
int step_dropout_check(const step_dropout_draw* draw, long long n, uint64_t* offset_step);
/* mask[e] = 1 if element e of the draw is kept, else 0 (uint8 [n], the dropped tensor's element order). */
int step_dropout_mask_u8(const step_dropout_draw* draw, long long n, uint8_t* mask, step_stream_t stream);
/* The global draw's downsample part: y[r, t, p, c] = x[r, t, p, c] * factor (fp32 product rounded once to dtype) for the
 * channels-last slice x [R, T, P, C] (pixel stride x_ld; the downsample channels of the ROI concat buffer), y likewise. */
int step_dropout_global_fwd(const step_dropout_draw* draw, const void* x, int dtype, int x_ld, int R, int T, int P, int C,
                            int ctx_cols, void* y, int y_ld, step_stream_t stream);
/* The global draw's context part, reduced: out[r, k] = (sum over t ascending of ctx(r, t, k) * factor) / T, fp32 [R, K], for
 * ctx(r, t, k) = ctx[row * row_stride + t * t_stride + k * k_stride], row = row_map[r] (int32, may be NULL: row = r).
 * ContextNet's output [B, T', 1024] from frame t_start: ctx += t_start * 1024, row_stride = T' * 1024, t_stride = 1024,
 * k_stride = 1, row_map = each tube's clip; the per-tube [R, 1024, T]: row_stride = 1024 * T, t_stride = 1, k_stride = T.
 * P and C are the downsample part's pixels and channels (the draw is [R, C*P + K, T]). */
int step_dropout_ctx_mean_f32(const step_dropout_draw* draw, int P, int C, const float* ctx, const int32_t* row_map,
                              long long row_stride, int t_stride, int k_stride, int R, int T, int K, float* out,
                              step_stream_t stream);
/* The local draw: y[f, p, c] = x[f, p, c] * factor for x [F, P, C] channels-last (pixel stride x_ld), y likewise. */
int step_dropout_local_fwd(const step_dropout_draw* draw, const void* x, int dtype, int x_ld, int F, int P, int C, void* y,
                           int y_ld, step_stream_t stream);
/* step_mean_mid_bwd / step_mean_mid_bwd_f32 through the global draw (A = R tubes, B = T frames): dx[a, b, p, c] += gscale *
 * factor * g[a, p*C + c] / B; dx in dtype (STEP_F16 / STEP_F32), channel stride ld. */
int step_mean_mid_bwd_dropout(const step_dropout_draw* draw, int ctx_cols, const float* g, int A, int B, int P, int C,
                              float gscale, void* dx, int dtype, int ld, step_stream_t stream);
/* step_f32_accum_f16 / step_f32_accum_f32 through the local draw: dst[f, p, c] += gscale * factor * src[f, p, c], src fp32
 * [F*P, C] dense, dst in dtype with channel stride ld. */
int step_f32_accum_dropout(const step_dropout_draw* draw, const float* src, int F, int P, int C, float gscale, void* dst,
                           int dtype, int ld, step_stream_t stream);
/* step_ctx_grad_reduce_f32 through the global draw's context part, for the [R, 1024] gradient dctx of
 * step_dropout_ctx_mean_f32's output: acc[b, t_start + t, k] += (sum over the tubes r of clip b, ascending, of
 * factor(r, t, k) * dctx[r, k]) / T_len.  P, Cg: the downsample part's pixels and channels.  Deterministic, no atomics. */
int step_ctx_grad_reduce_dropout_f32(const step_dropout_draw* draw, int P, int Cg, const float* dctx, int dctx_ld,
                                     const float* tubes, int R, int T_len, int B, int feat_T, int t_start, int C, float* acc,
                                     step_stream_t stream);

/* ------------------------------------------------------------------ optimizer ------------ */
/* Multi-tensor parameter update (train.py:123-128, 345-348): one launch over every tensor of a parameter set, described by a
 * device table of step_optim_tensor rows and a device block map.  Row r describes one fp32 tensor of `numel` contiguous
 * elements; block b of a launch works on elements [chunk * step_multi_tensor_chunk(), + step_multi_tensor_chunk()) of row
 * blocks[b].tensor, so a tensor of n elements needs ceil(n / step_multi_tensor_chunk()) map entries.  The per-row scalars are
 * the ones torch's single-tensor optimizers pass to their kernels, computed on the host in double and rounded to float:
 *   Adam: step_size = lr / (1 - beta1^t), inv_bias_correction2_sqrt = 1 / sqrt(1 - beta2^t), one_minus_beta1 = 1 - beta1,
 *         one_minus_beta2 = 1 - beta2 (exp_avg_sq non-null);
 *   SGD:  step_size = lr, momentum (exp_avg = momentum buffer, NULL when momentum == 0), buf_uninit = 1 on the buffer's first
 *         step (the buffer is then set to the gradient, as torch.optim.SGD does).
 * Every tensor pointer that is 16-byte aligned together with the others of its row takes vector loads and stores. */
typedef struct {
  float* param;
  const float* grad;
  float* exp_avg;            /* Adam exp_avg | SGD momentum buffer (nullable for SGD) */
  float* exp_avg_sq;         /* Adam only */
  long long numel;
  float step_size;
  float inv_bias_correction2_sqrt;
  float weight_decay;        /* L2, added to the gradient (torch's weight_decay, not AdamW) */
  float one_minus_beta1;
  float beta2;
  float one_minus_beta2;
  float eps;
  float momentum;
  int buf_uninit;
} step_optim_tensor;
typedef struct {
  int tensor;                /* row of the table */
  int chunk;                 /* chunk of that tensor */
} step_optim_block;
/* Elements of one tensor one block map entry covers. */
int step_multi_tensor_chunk(void);
/* *flag (device int) = 1 if any gradient element of the table is inf or NaN, else 0 (the call clears it first).  Plain stores:
 * the result is deterministic. */
int step_multi_tensor_nonfinite_f32(const step_optim_tensor* table, int n_tensors, const step_optim_block* blocks, int n_blocks,
                                    int* flag, step_stream_t stream);
/* torch.optim.Adam (amsgrad=False, maximize=False), per element:  g += wd * p;  m = lerp(m, g, 1 - beta1);
 * v = v * beta2 + (1 - beta2) * g * g;  p -= step_size * m / (sqrt(v) * inv_bias_correction2_sqrt + eps). */
int step_multi_tensor_adam_f32(const step_optim_tensor* table, int n_tensors, const step_optim_block* blocks, int n_blocks,
                               step_stream_t stream);
/* torch.optim.SGD (dampening=0, nesterov=False), per element:  g += wd * p;  buf = buf_uninit ? g : buf * momentum + g;
 * p -= step_size * (momentum ? buf : g). */
int step_multi_tensor_sgd_f32(const step_optim_tensor* table, int n_tensors, const step_optim_block* blocks, int n_blocks,
                              step_stream_t stream);

/* ---- training-sample selection (select.cu): train_select, utils/utils.py:135-423, one refinement step per call ---- */
enum { STEP_SAMPLING_UNIFORM = 0, STEP_SAMPLING_RANDOM = 1, STEP_SAMPLING_SOFTMAX = 2 };
enum { STEP_SELECT_MT_WORDS = 625 };  /* one MT19937 state: 624 key words, then the position */
typedef struct {
  int step;                  /* 1-based refinement step; step 1 selects from the proposals, later steps from the history */
  int B;                     /* clips */
  int C;                     /* classes */
  int L;                     /* frames of the candidates (the proposals at step 1, the history's pred_loc after) */
  int T;                     /* frames per chunk */
  int Lout;                  /* frames of the selected tubes: L, or L + 2T when ext_mode extends them */
  int ext_mode;              /* STEP_EXT_*: how the selected tubes grow by one chunk on each side (utils.py:283-312) */
  int max_chunks;            /* chunks of the targets */
  int gt_mid;                /* chunk of the targets the IoU and the centre target use */
  int predict_nb;            /* write the neighbour targets of chunks nb_first / nb_last (utils.py:319-331) */
  int nb_first, nb_last;
  int topk;                  /* <= 0: every tube is a candidate */
  int max_pos, neg_ratio, sampling;
  int max_rows;              /* output rows per clip, >= max_pos * (1 + neg_ratio) */
  int n_max, g_max;          /* largest tube and ground-truth count of one clip */
  int prop_f64;              /* step 1: the proposals are float64 (the IoU then rounds as numpy does for mixed types) */
  float cls_thresh, reg_thresh, width, height;
  long long prob_sr, prob_sl, prob_sc;  /* element strides of pred_prob [R, L, C] */
  const int32_t* tube_off;   /* [B + 1] first tube of each clip */
  const int32_t* gt_off;     /* [B + 1] first ground truth of each clip */
  const float* prob;         /* step > 1 */
  const float* loc;          /* step > 1: [R, L, 4] */
  const float* first;        /* STEP_EXT_PREDICT: [R, T, 4] */
  const float* last;
  const double* props;       /* step 1: [R, L, 4] */
  const float* targets;      /* [sum G, max_chunks, 4 + C] */
  uint32_t* mt;              /* [2][STEP_SELECT_MT_WORDS]: numpy's, then Python's MT19937 state; advanced in place */
  float* out_tubes;          /* [B * max_rows, Lout, 5], rows packed clip after clip */
  float* out_targets;        /* [B * max_rows, 3, 6 + C] */
  int32_t* counts;           /* [B] rows of each clip */
  int target_mode;           /* STEP_TARGETS_*: the rows of train_select (0, the zero-initialised default) or train_cls.py */
} step_select_params;
/* step_select_params.target_mode.  STEP_TARGETS_CLS writes the rows of the classification pre-training stage
 * (train_cls.py:271-291): a positive carries its ground truth's box, classification flag 1 and labels, a negative only
 * classification flag 1; the regression flag stays 0 and the three rows of a sample are the same.  It needs step 1,
 * STEP_EXT_NONE and predict_nb 0. */
enum { STEP_TARGETS_SELECT = 0, STEP_TARGETS_CLS = 1 };
/* One CTA walks the clips in order: candidates, IoU, positive assignment, the draws from the two generators, and the
 * selected rows.  STEP_E_ARG before any launch when an argument is out of range. */
int step_select_step_f32(const step_select_params* p, step_stream_t stream);
/* The checks of step_select_step_f32 that need no pointer (every field, the shared memory the step needs), with no launch:
 * a caller validates every step before it uploads or launches anything. */
int step_select_check_f32(const step_select_params* p);

/* ---- frame-mAP (eval.cu): the AVA Pascal evaluator of get_ava_performance.run_evaluation, fed by step_detect_f32 ---- */
enum {
  STEP_EVAL_MAX_CLIPS = 64,              /* clips of one append call */
  STEP_EVAL_MAX_IMAGES = 1 << 20,        /* image ids are < this */
  STEP_EVAL_MAX_CLASSES = 128,           /* evaluator classes (the label map's largest id) */
  STEP_EVAL_MAX_GT_PER_IMAGE = 1024,     /* ground-truth rows of one image */
  STEP_EVAL_MAX_ROWS = 1 << 30           /* detection rows, and rows read (whitelisted rows, kept or not) */
};
/* The row store append and evaluate share: one row per kept detection, in the order the rows were read. */
typedef struct {
  long long capacity;        /* rows the arrays below hold */
  int32_t* counters;         /* [2] device: rows kept, rows read */
  int32_t* img_first;        /* [STEP_EVAL_MAX_IMAGES] first row read of each image (INT32_MAX: none yet) */
  double* box;               /* [capacity, 4] y1, x1, y2, x2 after the CSV rounding */
  double* score;             /* [capacity] score after the CSV rounding */
  int32_t* scode;            /* [capacity] order-preserving integer code of the rounded score */
  int32_t* img;              /* [capacity] image id */
  int32_t* cls;              /* [capacity] evaluator class index (label id - 1) */
} step_eval_rows;
typedef struct {
  const float* det;          /* [B, cap, 8] step_detect_f32's rows: x1, y1, x2, y2, score, class, tube, 0 */
  const int32_t* count;      /* [B] rows of each clip */
  int B, cap;
  int ncls;                  /* detector classes */
  const int32_t* class_of;   /* [ncls] evaluator class index of each detector class; -1 drops its rows (not whitelisted) */
  int32_t img[STEP_EVAL_MAX_CLIPS];  /* image id of each clip; -1 drops the clip (an excluded key) */
  step_eval_rows rows;
} step_eval_append_params;
/* Appends the clips' rows in order: every box coordinate and score rounded as '{:.4}' then float() round them, rows of
 * other classes dropped, rows with y1 >= y2, x1 >= x2 or score <= -10 dropped after they are counted as read.  One CTA,
 * no synchronisation.  Rows past rows.capacity are counted but not stored: the caller keeps room for B * cap more. */
int step_eval_append(const step_eval_append_params* p, step_stream_t stream);
/* The checks of step_eval_append, with no launch. */
int step_eval_append_check(const step_eval_append_params* p);
typedef struct {
  step_eval_rows rows;
  int n_rows;                /* rows kept (counters[0], read back by the caller) */
  int n_classes;             /* evaluator classes */
  int n_images;              /* image ids are < n_images */
  int n_gt;                  /* ground-truth rows */
  int max_gt_per_image;
  const double* gt_box;      /* [n_gt, 4] y1, x1, y2, x2, sorted by (image, class), row order kept within */
  const int32_t* gt_cls;     /* [n_gt] */
  const int32_t* gt_img_off; /* [n_images + 1] first ground-truth row of each image */
  const int32_t* num_gt;     /* [n_classes] ground-truth rows of each class */
  void* workspace;
  size_t workspace_bytes;    /* >= step_eval_workspace_bytes(n_rows, n_classes, n_gt) */
  double* ap;                /* [n_classes] per-class AP: NaN without ground truth */
} step_eval_params;
size_t step_eval_workspace_bytes(int n_rows, int n_classes, int n_gt);
/* Per-class AP of get_ava_performance.run_evaluation (PascalDetectionEvaluator, IoU 0.5).  Per image and class: the
 * rows by descending score (ties: later row first), the first 10,000, greedy matching on the float64 IoU of np_box_ops.iou.
 * Per class: the rows by descending score (ties: later image, then earlier row, first), precision and recall, the
 * precision made non-increasing, and the AP terms summed in numpy's pairwise order. */
int step_eval_run(const step_eval_params* p, step_stream_t stream);
/* The checks of step_eval_run, with no launch. */
int step_eval_check(const step_eval_params* p);

#ifdef __cplusplus
}
#endif
#endif /* STEP_B200_H_ */
