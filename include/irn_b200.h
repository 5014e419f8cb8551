/*
 * irn_b200.h -- C ABI of libirn_b200.so: the H100 (sm_90a) implementation of the IRN
 * pseudo-label hot path (jiwoon-ahn/irn).
 *
 * The reference has no FFI of its own (pure Python on torch); its seams are Python names
 * (SURVEY.md section 8(b)).  Each entry point below names the reference code it replaces
 * (file:line under the reference tree).  INTEGRATION.md shows the ctypes stub a reference
 * maintainer would add.
 *
 * Conventions
 *  - every function returns 0 on success, <0 on error; irn_last_error() (thread-local)
 *    describes the failure.  -1 = bad argument, -2 = CUDA error, -3 = workspace too small,
 *    -4 = unsupported configuration.
 *  - device pointers are BORROWED: the caller (PyTorch in this repo) owns every buffer.  The
 *    library allocates nothing on the device except inside plan objects (irn_net_*) which
 *    hold the repacked network weights.
 *  - all device work is enqueued asynchronously on the caller's stream, in call order: every
 *    launch, memset, CUB pass and copy of a call, including the uploads of its host
 *    descriptors (which are staged before the call returns, so the host arrays may be reused
 *    at once).  A call reads its device inputs only after the work enqueued before it on that
 *    stream.  The calls that return host values (the CRF's vertex counts) synchronise that
 *    stream only.  Workspaces and scratch buffers are the caller's: two calls in flight at once
 *    need two of them.
 *  - calls may come from several host threads at once, each on its own stream; the error text,
 *    launch counts, last-walk flags and timing switches are per thread.  A net plan (irn_net_*)
 *    or resize plan used by two threads at once is not covered by this promise.
 *  - no global mutable state except constant tables uploaded once per process per device, and
 *    the random walk's radius tables: a call at another radius than the resident one waits for
 *    every call still enqueueing at the old radius and for the whole device, then uploads
 *    (so a radius switch cannot happen inside CUDA graph capture).
 *  - tensors are dense row-major; "NCHW"/"NHWC" say which.
 */
#ifndef IRN_B200_H
#define IRN_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* irn_stream_t; /* a cudaStream_t / CUstream */

const char* irn_last_error(void);
int irn_version(void);

/* ------------------------------------------------------------------------------------
 * R1/R2  PathIndex tables (host, integer, bit-exact).
 * Replaces misc/indexing.py:6-88 (PathIndex.__init__, get_search_paths_dst,
 * get_path_indices).
 *
 * irn_path_index_shape: n_dst = number of half-plane offsets, n_groups = number of distinct
 *   path lengths; group_len[g] = path length L, group_paths[g] = paths of that length (both
 *   arrays sized >= 4*radius).
 * irn_path_index_fill : search_dst int64 [n_dst,2] (dy,dx); search_paths int64, groups
 *   concatenated, each [n_paths,L,2]; path_indices int64, groups concatenated, each
 *   [n_paths,L,n_src]; src_indices int64 [n_src]; dst_indices int64 [n_dst,n_src]; with
 *   n_src = (Hp-rf)*(Wp-2rf), rf = ceil(radius)-1.  Any output pointer may be NULL.
 */
int irn_path_index_shape(int radius, int* n_dst, int* n_groups, int* group_len, int* group_paths);
int irn_path_index_fill(int radius, int Hp, int Wp, int64_t* search_dst, int64_t* search_paths,
                        int64_t* path_indices, int64_t* src_indices, int64_t* dst_indices);

/* ------------------------------------------------------------------------------------
 * R3  edge -> affinity (device).  Replaces misc/indexing.py:91-109 (edge_to_affinity) on
 * the un-padded grid: aff[k,y,x] = 1 - max(edge over path k from (y,x)), 0 when the
 * destination leaves the image (the reference pads the edge map with 1.0,
 * misc/indexing.py:150).  edge fp32 [n_img,h,w]; aff fp32 [n_img,n_dst,h,w].
 */
int irn_edge_to_affinity(const float* edge, float* aff, int n_img, int h, int w, int radius,
                         irn_stream_t stream);

/* ------------------------------------------------------------------------------------
 * N4  training-side affinity.  Replaces net/resnet50_irn.py:162-175
 * (AffinityDisplacementLoss.to_affinity: index_select over PathIndex.path_indices +
 * max_pool2d over the path) and its autograd backward.  edge fp32 [n_img,h,w];
 * aff fp32 [n_img, n_dst, (h-rf)*(w-2rf)], rf = radius-1 (the source window of PathIndex);
 * arg int32, same shape: flat index h*w of the path point that held the maximum (first in
 * path order, as max_pool2d), NULL when no backward pass will follow.  backward: zeroes
 * grad_edge [n_img,h,w], then grad_edge[arg] -= grad_aff (atomic adds, like index_add_).
 */
int irn_to_affinity_forward(const float* edge, float* aff, int32_t* arg, int n_img, int h, int w,
                            int radius, irn_stream_t stream);
int irn_to_affinity_backward(const float* grad_aff, const int32_t* arg, float* grad_edge, int n_img,
                             int h, int w, int radius, irn_stream_t stream);

/* ------------------------------------------------------------------------------------
 * R3-R6  random walk.  Replaces misc/indexing.py:141-167 (propagate_to_edge) including
 * affinity_sparse2dense (:112-129) and to_transition_matrix (:132-139): instead of the
 * dense (hw)^2 matrix squared exp_times times it applies the 2*n_dst+1 tap stencil
 * y_j <- (sum_i a_ij^beta y_i)/s_j  n_iter = 2^exp_times times, fp64 state.
 *
 *  x    fp32 [total_channels,h,w]   seeds, images back to back
 *  edge fp32 [n_img,h,w]            sigmoid edge map in (0,1)
 *  out  fp32 [total_channels,h,w]
 *  chan_offsets  HOST int32 [n_img+1]: channels of image i are [off[i], off[i+1])
 *  workspace     device, >= irn_rw_workspace_bytes(...) bytes, 256-byte aligned
 */
size_t irn_rw_workspace_bytes(int n_img, int h, int w, int total_channels, int radius);
int irn_random_walk(const float* x, const float* edge, float* out, int n_img,
                    const int32_t* chan_offsets, int h, int w, int radius, double beta,
                    int n_iter, void* workspace, size_t workspace_bytes, irn_stream_t stream);

/* Same, selecting the kernel: variant 0 = production (radius 5: the fused cluster kernel -- all
 * n_iter steps in one launch, weights resident in shared memory -- or the per-step TMA kernel,
 * whichever a cost model expects to be faster; the fused kernel needs h, w <= 128; other radii:
 * the generic kernel), 1 = generic bounds-checked step kernel (any radius 2..10; validation /
 * radii the reference's hot path never uses), 2 = per-step TMA kernel (radius 5), 4 = fused
 * cluster kernel.  Variants 2 and 4 return -4 when they cannot run as asked; any other variant
 * returns -1.  Both are reported before anything is launched (except a device that cannot
 * co-schedule variant 4's cluster, which is found at launch time). */
int irn_random_walk_variant(const float* x, const float* edge, float* out, int n_img,
                            const int32_t* chan_offsets, int h, int w, int radius, double beta,
                            int n_iter, void* workspace, size_t workspace_bytes, int variant,
                            irn_stream_t stream);

/* Number of kernels the last API call on this thread launched; irn_total_launch_count: since process start
 * (bench.py's gpu_launches). */
int irn_rw_last_launch_count(void);
long long irn_total_launch_count(void);
/* Number of thread-block clusters the last walk on this thread ran on as the fused kernel; 0 when it ran step by step. */
int irn_rw_last_was_fused(void);

/* Device timing of the walk's step kernels for bench.py's roofline: when enabled, CUDA events are recorded on the
 * caller's stream around the n_iter step launches; irn_rw_last_step_ms waits for the last timed walk and returns
 * its mean step-kernel duration. */
int irn_rw_set_timing(int enable);
int irn_rw_last_step_ms(float* ms_per_step, int* n_steps);

/* ------------------------------------------------------------------------------------
 * S1  label map.  Replaces step/make_sem_seg_labels.py:43-49 (and the same tail at
 * step/make_ins_seg_labels.py:137-143): x4 bilinear (align_corners=False), crop to (H,W),
 * divide by the global max, prepend a constant background plane, argmax (ties -> lowest
 * index), map through keys.
 *
 *  rw   fp32 [C,h,w] one image;  keys_host HOST int32 [C+1] (entry 0 = background id, C+1 <= 129;
 *  passed to the kernel by value: no copy, no synchronisation) or NULL (identity);  outputs, each optional (NULL): labels uint8 [H,W] = keys[argmax];
 *  index_out int32 [H,W] = raw argmax (instance path: C may exceed 255);  up_norm fp32
 *  [C,H,W] = normalised upsampled scores (instance scoring).  scratch: device, >= 16 bytes.
 */
int irn_rw_labels(const float* rw, int C, int h, int w, int H, int W, float bg_thres,
                  const int32_t* keys_host, uint8_t* labels, int32_t* index_out, float* up_norm,
                  void* scratch, irn_stream_t stream);

/* ------------------------------------------------------------------------------------
 * S1b  background-threshold sweep: the confusion matrices of T background thresholds in one
 * pass over the scores.  At threshold t a pixel is labelled as by step/eval_cam.py:15-17 or
 * step/make_sem_seg_labels.py:43-49 with t as the background plane (float32 compare, ties ->
 * lowest index, the first NaN wins), and counted against its ground truth as
 * calc_semantic_segmentation_confusion does (255 = ignore).
 *
 *  irn_threshold_sweep_bytes: size of the accumulator `hist` for T thresholds (1..256) and
 *    n_class classes (1..129), 0 when out of range.  The caller zeroes it before the first
 *    accumulate; every accumulate of a run adds to it.
 *  irn_threshold_sweep_accumulate: one image.  source IRN_SWEEP_PLANES: scores fp32 [C,H,W]
 *    used as stored (eval_cam's high_res; h == H, w == W); IRN_SWEEP_WALK: the walk fp32
 *    [C,h,w], x4 bilinear, cropped to (H,W) and divided by its global max as irn_rw_labels
 *    does (H <= 4h, W <= 4w; scratch >= 16 bytes).  C = 0: background at every threshold.
 *    keys_host HOST int32 [C+1], entry 0 = 0 (background);  gt uint8 [H,W];  thresholds_host
 *    HOST fp32 [T], strictly ascending.  Both tables go to the kernel by value: no copy, no
 *    synchronisation.  A predicted label or a ground truth (other than 255) >= n_class is
 *    not counted; it is reported by irn_threshold_sweep_finalize.
 *  irn_threshold_sweep_finalize: conf int64 [T,n_class,n_class] (rows = ground truth,
 *    columns = prediction) from `hist`.  Synchronises the stream to read the error words, and
 *    returns -1 without writing conf if an accumulate met a label >= n_class.
 */
#define IRN_SWEEP_PLANES 0
#define IRN_SWEEP_WALK 1
size_t irn_threshold_sweep_bytes(int T, int n_class);
int irn_threshold_sweep_accumulate(int source, const float* scores, int C, int h, int w, int H, int W,
                                   const int32_t* keys_host, const uint8_t* gt,
                                   const float* thresholds_host, int T, int n_class, void* hist,
                                   void* scratch, irn_stream_t stream);
int irn_threshold_sweep_finalize(const void* hist, int T, int n_class, int64_t* conf,
                                 irn_stream_t stream);

/* ------------------------------------------------------------------------------------
 * C2/C3  ResNet-50 trunk + CAM head;  I1/I2  IRNet edge / displacement heads.
 * Replace net/resnet50.py:17-91, net/resnet50_cam.py:55-70 (CAM.forward) and
 * net/resnet50_irn.py:23-133,216-234 (Net.forward, MeanShift, EdgeDisplacement.forward).
 *
 * A plan (irn_net) owns the repacked weights on the current device.  `params` is a HOST fp32
 * blob holding the reference checkpoint's tensors in execution order (irn_b200/_pack.py):
 *   trunk: conv1.weight, bn1.{weight,bias,running_mean,running_var}; then per bottleneck
 *          conv1,bn1,conv2,bn2,conv3,bn3[,downsample.0,downsample.1] (weights OIHW);
 *   CAM  : + classifier.weight [C,2048], C the number of classes: 20 (PASCAL VOC) for irn_cam_net_create, n_classes
 *          (1..IRN_CAM_MAX_CLASSES; MS COCO has 80) for irn_cam_net_create_classes.  A C-class plan's CAMs are [.,C,.,.].
 *   IRN  : + fc_edge1..5 {conv.weight, gn.weight, gn.bias}, fc_edge6.{weight,bias},
 *          fc_dp1..7 {conv.weight, gn.weight, gn.bias}, fc_dp7.3.weight, mean_shift.running_mean.
 * FixedBatchNorm (eps 1e-5, inference statistics) is folded into the conv at creation.
 */
typedef struct irn_net irn_net;
#define IRN_CAM_MAX_CLASSES 128
int irn_cam_net_create(const float* params, size_t n_floats, irn_net** out);
int irn_cam_net_create_classes(const float* params, size_t n_floats, int n_classes, irn_net** out);
int irn_irn_net_create(const float* params, size_t n_floats, irn_net** out);
void irn_net_destroy(irn_net* net);
/* Convolution arithmetic: 2 (default) = wgmma tensor cores, f16x3 split (fp16 hi/lo operand parts, per-k-block fp32 partial
 * sums added in IEEE fp32: fp32-grade, ~22 bits per operand) for every conv with Cin % 64 == 0 and Cout % 64 == 0 and the stem,
 * SIMT fp32 for the rest; 1 = 3xTF32 split (Cin % 32 == 0) instead; 0 = SIMT IEEE fp32 everywhere (the on-device cross-check). */
int irn_net_set_conv_mode(irn_net* net, int mode);
int irn_net_get_conv_mode(const irn_net* net);

/* Layer taps (test instrumentation): a forward of `net` copies the named intermediate tensor into `dst` (device, at least the
 * tensor's bytes; NHWC fp32 with the shape irn_net_tap_shape gives) with a cudaMemcpyAsync on the forward's stream, issued
 * right after the kernel that produced it and before its arena buffer is reused.  dst = NULL clears the tap.  A forward with
 * no tap set launches exactly what it launches without this interface.  A tap whose buffer is too small fails the forward.
 *   trunk (both kinds)  IRN_TAP_STEM  stem conv + ReLU (after the ragged mask), before the max pool
 *                       IRN_TAP_POOL  max pool output
 *                       IRN_TAP_BLOCK0 + 3 j + {0, 1, 2}: bottleneck j = 0..15 (layer1.0 .. layer4.2): t1 = relu(bn1(conv1)),
 *                       t2 = relu(bn2(conv2)), the block output
 *   CAM                 IRN_TAP_CAM_CLS  relu(classifier) [B,h,w,64] (C <= 64) or [B,h,w,128] (channels C.. zero) in the
 *                       tensor-core modes 1 and 2; never written in mode 0, whose head kernel keeps it in registers
 *   IRN                 IRN_TAP_HEAD0 + i: head i's raw 1x1 conv output (i = 0..4 fc_edge1..5, 5..11 fc_dp1..7);
 *                       IRN_TAP_ECAT the 160-channel edge concat, IRN_TAP_DCAT3 dp3|dp4|dp5, IRN_TAP_DCAT2 dp1|dp2|dp6,
 *                       IRN_TAP_DP7A relu(gn(fc_dp7 conv)), IRN_TAP_ELOG the edge logits [B,h,w,1], IRN_TAP_DLOG dp [B,h,w,2]
 * irn_net_tap_shape (host only) gives tap `id`'s NHWC shape for a forward of B samples: kind 0 (CAM) on an H x W input, kind 1
 * (IRN) on the crop_size x crop_size canvas (H, W unused); it fails for an id the kind does not have.  Kind 0 is a 20-class
 * CAM plan; irn_cam_tap_shape gives the shapes of an n_classes CAM plan. */
enum {
    IRN_TAP_STEM = 0,
    IRN_TAP_POOL = 1,
    IRN_TAP_BLOCK0 = 2,
    IRN_TAP_CAM_CLS = 50,
    IRN_TAP_HEAD0 = 50,
    IRN_TAP_ECAT = 62,
    IRN_TAP_DCAT3 = 63,
    IRN_TAP_DCAT2 = 64,
    IRN_TAP_DP7A = 65,
    IRN_TAP_ELOG = 66,
    IRN_TAP_DLOG = 67,
    IRN_TAP_COUNT = 68
};
int irn_net_set_tap(irn_net* net, int id, float* dst, size_t bytes);
int irn_net_tap_shape(int kind, int id, int B, int H, int W, int crop_size, int shape[4]);
int irn_cam_tap_shape(int n_classes, int id, int B, int H, int W, int shape[4]);

/* One convolution (+ folded FixedBatchNorm, residual add, ReLU) as a plan of its own: the building block of
 * the two networks above (net/resnet50.py:34-54), exposed for unit tests and for wiring other topologies.
 *   weight_oihw HOST fp32 [cout,cin,k,k]; bn4 HOST fp32 [4,cout] = gamma,beta,running_mean,running_var or NULL.
 *   forward: in NHWC fp32 [B,H,W,cin] -> out NHWC [B,Ho,Wo,cout]; residual NHWC like out, or NULL. */
typedef struct irn_conv irn_conv;
int irn_conv_create(const float* weight_oihw, const float* bn4, int cin, int cout, int k, int stride,
                    int pad, irn_conv** out);
void irn_conv_destroy(irn_conv* conv);
int irn_conv_forward(irn_conv* conv, const float* in, int B, int H, int W, const float* residual,
                     float* out, int relu, int mode, irn_stream_t stream);

/* The networks' stem (conv 7x7/2 pad 3, 3 -> 64, + folded FixedBatchNorm, ReLU) as a plan of its own, run by the
 * same code as the trunk: input layout transform, then the SIMT (mode 0), 3xTF32 (mode 1) or f16x3 (mode 2) stem.
 *   weight_oihw HOST fp32 [64,3,7,7]; bn4 HOST fp32 [4,64] or NULL.  Free with irn_conv_destroy.
 *   forward: x_nchw fp32 [B,3,H,W] zero-padded on the right / bottom to Hin x Win (H <= Hin, W <= Win) ->
 *   out_nhwc [B,Ho,Wo,64], Ho = (Hin-1)/2+1, Wo = (Win-1)/2+1; workspace device, 256-byte aligned,
 *   >= irn_stem_workspace_bytes(B, Hin, Win). */
int irn_stem_create(const float* weight_oihw, const float* bn4, irn_conv** out);
size_t irn_stem_workspace_bytes(int B, int Hin, int Win);
int irn_stem_forward(irn_conv* stem, const float* x_nchw, int B, int H, int W, int Hin, int Win,
                     float* out_nhwc, int mode, void* workspace, size_t workspace_bytes, irn_stream_t stream);

/* conv3 and the projection shortcut of a ResNet-50 stage's first bottleneck as the f16x3 network runs them: one
 * K-concatenated 1x1 conv, out = relu(bn3(conv3(t2)) + bnds(ds(x sampled at `stride`))).
 *   w3 HOST fp32 [4 planes, planes]; wds HOST fp32 [4 planes, cin]; bn3, bnds HOST fp32 [4, 4 planes] (both required).
 *   Fails unless planes % 64 == 0 and cin % 64 == 0.  Free with irn_conv_destroy.
 *   forward: x NHWC fp32 [B,H,W,cin]; t2 NHWC [B,Ho,Wo,planes] and out NHWC [B,Ho,Wo,4 planes], Ho = (H-1)/stride+1. */
int irn_shortcut_conv_create(const float* w3, const float* bn3, const float* wds, const float* bnds, int planes,
                             int cin, int stride, irn_conv** out);
int irn_shortcut_conv_forward(irn_conv* conv, const float* t2, const float* x, int B, int H, int W, float* out,
                              irn_stream_t stream);

/* CAM.forward over B/2 (image, horizontally flipped image) pairs.
 *   x_nchw fp32 [B,3,H,W] (device), B even -> cam fp32 [B/2,C,ceil(H/16),ceil(W/16)], C the plan's classes:
 *   relu(classifier(trunk(x)))[2p] + relu(...)[2p+1].flip(-1)   (net/resnet50_cam.py:65-68)
 *   workspace: irn_cam_workspace_bytes for a 20-class plan, irn_cam_workspace_bytes_classes for any. */
size_t irn_cam_workspace_bytes(int B, int H, int W);
size_t irn_cam_workspace_bytes_classes(int B, int H, int W, int n_classes);
int irn_cam_forward(const irn_net* net, const float* x_nchw, int B, int H, int W, float* cam_out,
                    void* workspace, size_t workspace_bytes, irn_stream_t stream);

/* CAM.forward over B/2 pairs of different sizes on one canvas (irn_resize_ragged_forward lays it out).
 *   x_canvas fp32 [B,3,Hc,Wc] (device), B even: pair p (samples 2p, 2p+1) holds an image of hw[p] = (h_p, w_p) pixels at the
 *   top-left corner and +0.0 elsewhere; hw HOST int32 [B/2][2], 0 < h_p <= Hc, 0 < w_p <= Wc.
 *   -> cam fp32 [B/2,C,ceil(Hc/16),ceil(Wc/16)]: pair p's ceil(h_p/16) x ceil(w_p/16) corner is, bit for bit, what irn_cam_forward
 *   returns for that pair alone (the layers that read beyond an image's extent see zeros there, as they see padding alone); 0
 *   elsewhere.  workspace device, 256-byte aligned, >= irn_cam_workspace_bytes_classes(B, Hc, Wc, C). */
int irn_cam_forward_ragged(const irn_net* net, const float* x_canvas, int B, int Hc, int Wc, const int32_t* hw,
                           float* cam_out, void* workspace, size_t workspace_bytes, irn_stream_t stream);

/* EdgeDisplacement.forward for P (image, flipped image) pairs of equal size.
 *   x_nchw fp32 [2P,3,H,W]; zero-padded to crop_size (net/resnet50_irn.py:226) ->
 *   edge fp32 [P,1,fh,fw] = sigmoid(e[2p]/2 + e[2p+1].flip(-1)/2), dp fp32 [P,2,fh,fw] = dp[2p] - running_mean;
 *   fh = ceil(H/4), fw = ceil(W/4).  The reference runs P = 1. */
size_t irn_edge_displacement_workspace_bytes(int P, int H, int W, int crop_size);
int irn_edge_displacement_forward(const irn_net* net, const float* x_nchw, int P, int H, int W,
                                  int crop_size, float* edge_out, float* dp_out, void* workspace,
                                  size_t workspace_bytes, irn_stream_t stream);

/* EdgeDisplacement.forward for P images of any sizes (H_i, W_i <= crop_size) in one batch, from the decoded images.
 *   img_u8     device uint8, img_bytes long: image i is uint8 [H_i,W_i,3] (RGB, HWC) at byte img_offsets[i]
 *   img_offsets HOST int64 [P];  sizes_hw HOST int32 [P][2] = (H_i, W_i)
 *   lut768     device fp32 [3][256], irn_normalize_lut's table (the loader's normalisation)
 *   -> edge fp32 [P,1,fc,fc], dp fp32 [P,2,fc,fc], fc = (crop_size-1)/4+1.
 * Image i's ceil(H_i/4) x ceil(W_i/4) corner holds, bit for bit, what irn_edge_displacement_forward returns for its scale-1.0
 * (image, flipped image) pair alone (irn_resize_forward); outside it edge = 1 and dp = 0, which makes the edge map the padded
 * input of the random walk.  workspace device, 256-byte aligned, >= irn_edge_displacement_ragged_workspace_bytes(P, crop_size). */
size_t irn_edge_displacement_ragged_workspace_bytes(int P, int crop_size);
int irn_edge_displacement_forward_ragged(const irn_net* net, const uint8_t* img_u8, size_t img_bytes,
                                         const int64_t* img_offsets, const int32_t* sizes_hw, int P, int crop_size,
                                         const float* lut768, float* edge_out, float* dp_out, void* workspace,
                                         size_t workspace_bytes, irn_stream_t stream);

/* ------------------------------------------------------------------------------------
 * C4  multi-scale CAM merge.  Replaces step/make_cam.py:38-52.
 *   cams: HOST array of n_scales DEVICE pointers, each fp32 [C,hs[s],ws[s]] (CAM.forward outputs), C = 20 for
 *   irn_cam_merge, n_classes (1..IRN_CAM_MAX_CLASSES) for irn_cam_merge_classes;
 *   (H,W) original image size; keys_host HOST int32 [K] = classes present (torch.nonzero(label)), K <= C, ids in [0, C);
 *   strided_out fp32 [K,ceil(H/4),ceil(W/4)], highres_out fp32 [K,H,W] (either may be NULL):
 *   sum over scales of the bilinear (align_corners=False) resample, each kept class / (max + 1e-5).
 *   scratch: device, >= 2*K*4 bytes. */
int irn_cam_merge(const float* const* cams, const int* hs, const int* ws, int n_scales, int H, int W,
                  const int32_t* keys_host, int K, float* strided_out, float* highres_out,
                  void* scratch, irn_stream_t stream);
int irn_cam_merge_classes(const float* const* cams, const int* hs, const int* ws, int n_scales, int n_classes, int H,
                          int W, const int32_t* keys_host, int K, float* strided_out, float* highres_out,
                          void* scratch, irn_stream_t stream);

/* ------------------------------------------------------------------------------------
 * P1-P4  instance path.  Replaces step/make_ins_seg_labels.py:18-105.
 *
 * irn_find_centroids      P1 find_centroids_with_refinement (:18-56): dp fp32 [2,h,w] -> int32 [2,h,w] (y,x),
 *                         bit-exact with the numpy evaluation order (float64 update, float32 state).
 * irn_connected_components 4-connected components of equal non-zero values (skimage.measure.label(connectivity=1,
 *                         background=0) up to numbering): labels = 0 or 1 + smallest linear index of the component,
 *                         so ascending label order = raster order of first pixels.  scratch >= h*w*4 bytes.
 * irn_cluster_centroids   P2 cluster_centroids (:58-75) + compress_range: instance_map int32 [h,w] in 0..I-1
 *                         (one_hot(instance_map) is the reference's bool [I,h,w]), I -> *n_instances_dev.
 *                         scratch >= irn_cluster_scratch_bytes(h,w).
 * irn_instance_seeds      P3 separte_score_by_mask (:77-80): out[k*I+i] = cams[k] * (instance_map == i).
 * irn_segment_stats       P4 detect_instance (:82-105) statistics: per segment label l: area[l], max_bits[l] =
 *                         float bits of max(scores[index-1]) over the segment; arrays int32 [H*W+1].
 * irn_segment_masks       P4 detect_instance: the `pred_mask` planes (:96-101) -- masks[m] = (labels == seg_ids[m]) as
 *                         0/1 bytes (numpy bool layout) [M,H,W]; seg_ids device int32 [M].
 */
int irn_find_centroids(const float* dp, int32_t* centroids, int h, int w, int iterations, irn_stream_t stream);
int irn_connected_components(const int32_t* values, int32_t* labels, int h, int w, void* scratch, irn_stream_t stream);
size_t irn_cluster_scratch_bytes(int h, int w);
int irn_cluster_centroids(const float* dp, const int32_t* centroids, float thres, int32_t* instance_map,
                          int32_t* n_instances_dev, int h, int w, void* scratch, irn_stream_t stream);
int irn_instance_seeds(const float* cams, const int32_t* instance_map, int K, int I, int h, int w, float* out,
                       irn_stream_t stream);
int irn_segment_stats(const int32_t* labels, const int32_t* index, const float* scores, int H, int W,
                      int32_t* area, int32_t* max_bits, irn_stream_t stream);
int irn_segment_masks(const int32_t* labels, const int32_t* seg_ids, int M, int H, int W, uint8_t* masks,
                      irn_stream_t stream);

/* ------------------------------------------------------------------------------------
 * C1  multi-scale input preparation on the device.  Replaces, for a decoded uint8 image, the per-scale body of
 * VOC12ClassificationDatasetMSF.__getitem__ (voc12/dataloader.py:191-201): imutils.pil_rescale
 * (misc/imutils.py:8-22 -> Pillow BICUBIC resize of the uint8 image), TorchvisionNormalize
 * (voc12/dataloader.py:65-78), HWC->CHW and the stack with the W-flip.  Integer / table arithmetic: bit-exact
 * with Pillow's 8-bit resampler (two passes, horizontal first, 22-bit fixed-point coefficients) and numpy's
 * float64 normalisation rounded once to fp32.
 *
 * irn_resize_ksize / irn_resize_coeffs   (host) Pillow's coefficient table of one axis: bounds int32 [out,2]
 *                         (first source index, tap count), kk int32 [out, ksize] (2^22 fixed point).
 * irn_normalize_lut       (host) fp32 [3][256]: ((u/255 - mean[c]) / std[c]) evaluated in double.
 * irn_resize_plan_*       a plan owns the two coefficient tables and the normalisation table on the current device
 *                         for one (H, W) -> (out_h, out_w) pair (out == in on an axis skips that pass, like Pillow).
 * irn_resize_forward      img: device uint8 [B,H,W,3].  out (optional): device fp32 [2B,3,out_h,out_w], image b at
 *                         rows 2b (as is) and 2b+1 (W-flipped) = the [2,3,h,w] tensors the networks take.
 *                         out_u8 (optional): device uint8 [B,out_h,out_w,3], the resized image itself.
 *                         workspace >= irn_resize_workspace_bytes(plan, B) (the 8-bit intermediate image).
 */
typedef struct irn_resize_plan irn_resize_plan;
int irn_resize_ksize(int in_size, int out_size);
int irn_resize_coeffs(int in_size, int out_size, int32_t* bounds, int32_t* kk);
int irn_normalize_lut(const double* mean3, const double* std3, float* lut768);
int irn_resize_plan_create(int H, int W, int out_h, int out_w, const double* mean3, const double* std3,
                           irn_resize_plan** out);
int irn_resize_plan_destroy(irn_resize_plan* plan);
size_t irn_resize_workspace_bytes(const irn_resize_plan* plan, int B);
int irn_resize_forward(const irn_resize_plan* plan, const uint8_t* img, int B, float* out, uint8_t* out_u8,
                       void* workspace, size_t workspace_bytes, irn_stream_t stream);
/* irn_resize_ragged_forward   P images of different sizes resized in one call onto one canvas:
 *                         img_u8 device uint8, img_bytes long: image i is uint8 [H_i,W_i,3] at byte img_offsets[i] (HOST int64 [P]);
 *                         sizes_hw, out_hw HOST int32 [P][2] = (H_i, W_i), (out_h_i, out_w_i) with out_h_i <= Hc, out_w_i <= Wc;
 *                         lut768 device fp32 [3][256] (irn_normalize_lut).  out: device fp32 [2P,3,Hc,Wc], rows 2i and 2i+1 =
 *                         image i and its W-flip within out_w_i, each the out_h_i x out_w_i top-left corner holding what
 *                         irn_resize_forward writes for that image alone, +0.0 elsewhere.  P <= 65535.  workspace device, 256-byte
 *                         aligned, >= irn_resize_ragged_workspace_bytes (coefficient tables and the 8-bit intermediate images). */
size_t irn_resize_ragged_workspace_bytes(const int32_t* sizes_hw, const int32_t* out_hw, int P);
int irn_resize_ragged_forward(const uint8_t* img_u8, size_t img_bytes, const int64_t* img_offsets, const int32_t* sizes_hw,
                              const int32_t* out_hw, int P, int Hc, int Wc, const float* lut768, float* out,
                              void* workspace, size_t workspace_bytes, irn_stream_t stream);

/* ------------------------------------------------------------------------------------
 * N1  exact JPEG decode on the device: bit-identical to np.asarray(Image.open(f).convert("RGB")) (PIL on libjpeg-turbo:
 * islow IDCT, fancy chroma up-sampling), voc12/dataloader.py:101.  Our own kernels (csrc/jpeg_exact.cu); the arithmetic is
 * oracle/jpeg.py's.  Supported: SOF0/SOF1 8-bit Huffman, one interleaved scan, 1 component (decoded to R=G=B) or Y Cb Cr with
 * luma sampling 1x1 / 2x1 / 2x2 and chroma 1x1, optional DRI.  Anything else is -4 (unsupported); malformed or truncated
 * headers are -1, found on the host before any launch.
 *
 * irn_jpeg_exact_inspect: host only, no device needed.  info[6] = H, W, components, luma h / v sampling, restart interval.
 * irn_jpeg_exact_workspace_bytes: device workspace (256-byte aligned) and host staging bytes (pinned memory, so that the
 *   upload is asynchronous) for these n streams.
 * irn_jpeg_exact_decode: n host streams of any sizes; image i is written as uint8 RGB [H_i,W_i,3] at out_dev + out_offsets[i]
 *   (out_offsets a HOST int64 [n]).  status_dev (device int32 [n]) is zeroed and then receives error bits for image i's
 *   entropy-coded data (1 = stray marker, 2 = missing / surplus restart marker, 4 = invalid Huffman code, 8 = data ends early,
 *   16 = AC run past the block); read it after the stream has reached this call.  host_staging must stay untouched until then.
 * irn_jpeg_exact_set_timing / irn_jpeg_exact_last_ms: CUDA events between the stages of the next calls on this thread; last_ms
 *   waits and returns the four durations of the last timed call (ms): unstuff, entropy decode, IDCT, up-sampling + colour.
 */
int irn_jpeg_exact_inspect(const uint8_t* data, size_t length, int* info);
int irn_jpeg_exact_workspace_bytes(const uint8_t* const* data, const size_t* lengths, int n, size_t* device_bytes,
                                   size_t* host_bytes);
int irn_jpeg_exact_decode(const uint8_t* const* data, const size_t* lengths, int n, const int64_t* out_offsets, uint8_t* out_dev,
                          int32_t* status_dev, void* workspace, size_t workspace_bytes, void* host_staging, size_t host_bytes,
                          irn_stream_t stream);
int irn_jpeg_exact_set_timing(int enable);
int irn_jpeg_exact_last_ms(float* ms4);

/* ------------------------------------------------------------------------------------
 * N3  fully connected CRF and the cam_to_ir_label step.  Replaces misc/imutils.py:156-170 (crf_inference_label: pydensecrf's
 * DenseCRF2D with a Gaussian (sxy) and a bilateral (sxy, srgb) Potts term, mean-field inference on the permutohedral lattice)
 * and the body of step/cam_to_ir_label.py:19-41.  The arithmetic is oracle/crf.py's (float32, fixed evaluation order, no
 * floating-point atomics: bitwise reproducible).  A batch is n images of one size, images uint8 [n,H,W,3] (RGB, HWC), or, through
 * the _ragged entry points, n images of any sizes packed back to back.
 *
 * irn_crf_workspace_bytes  device workspace for n images with n_groups CRFs each (1: irn_dense_crf, 2: irn_ir_label) of at most
 *                         max_labels labels (<= irn_crf_max_labels()); 0 for arguments no call accepts.
 * irn_dense_crf           labels int32 [n,H,W] in [0, n_labels) -> labels_out int32 [n,H,W] = argmax of Q after t iterations,
 *                         q_out fp32 [n,n_labels,H,W] = Q (either may be NULL, not both); unary from the labels with gt_prob
 *                         (pydensecrf.utils.unary_from_labels, zero_unsure=False).  A label outside [0, n_labels) -> -1.
 * irn_ir_label            high_res fp32 [sum(counts),H,W] (make_cam's high_res planes, images back to back), keys_host HOST int32
 *                         [sum(counts)] (make_cam's keys), counts_host HOST int32 [n] -> out uint8 [n,H,W]: the conf map of the
 *                         step (fg / bg confident maps through the CRF, t=10, gt_prob=0.7, Gaussian (3, compat 3), bilateral
 *                         (50, 5, compat 10); 0 = bg, 255 = unsure, else class + 1).  An image with no class is all 0.
 * vertex_counts           optional HOST int32 [n,2]: lattice vertices per image (Gaussian, bilateral).
 * Both synchronise the stream once, after the lattice build (vertex counts and argument errors reach the host there).
 * irn_crf_set_timing / irn_crf_last_ms: CUDA events around the build, the iterations and the tail of the next calls on this
 * thread; last_ms waits and returns the three durations of the last timed call (ms).
 */
size_t irn_crf_workspace_bytes(int n, int H, int W, int n_groups, int max_labels);
int irn_crf_max_labels(void);
int irn_dense_crf(const uint8_t* img, const int32_t* labels, int n, int H, int W, int n_labels, int t, double gt_prob,
                  float gauss_sxy, float gauss_compat, float bil_sxy, float bil_srgb, float bil_compat, int32_t* labels_out,
                  float* q_out, int32_t* vertex_counts, void* workspace, size_t workspace_bytes, irn_stream_t stream);
int irn_ir_label(const uint8_t* img, const float* high_res, const int32_t* keys_host, const int32_t* counts_host, int n, int H,
                 int W, float conf_fg_thres, float conf_bg_thres, uint8_t* out, int32_t* vertex_counts, void* workspace,
                 size_t workspace_bytes, irn_stream_t stream);
/* Ragged batches: sizes_hw HOST int32 [n][2] = (H_i, W_i); every per-image array is image i's one-size array, the images back to back
 * in batch order (N_i = H_i*W_i; a batch of one size is laid out as above).  Image i's result is, bit for bit, the one-size entry
 * point's for that image, whatever its neighbours; a batch of equal sizes runs the same kernels as the one-size call.
 * irn_crf_ragged_workspace_bytes  as irn_crf_workspace_bytes for those sizes (0 for a size <= 0 or a batch too large for one call).
 * irn_dense_crf_ragged    img uint8 [sum N_i * 3] (img_bytes must be exactly that), labels int32 [sum N_i] -> labels_out int32
 *                         [sum N_i], q_out fp32 [n_labels * sum N_i] (image i's [n_labels,H_i,W_i] at n_labels * (N_0+..+N_{i-1})).
 * irn_ir_label_ragged     img as above, high_res fp32 [sum K_i*N_i] (image i's [K_i,H_i,W_i] planes; high_res_elems must be exactly
 *                         that), keys_host / counts_host as irn_ir_label -> out uint8 [sum N_i].
 */
size_t irn_crf_ragged_workspace_bytes(int n, const int32_t* sizes_hw, int n_groups, int max_labels);
int irn_dense_crf_ragged(const uint8_t* img, size_t img_bytes, const int32_t* sizes_hw, int n, const int32_t* labels, int n_labels,
                         int t, double gt_prob, float gauss_sxy, float gauss_compat, float bil_sxy, float bil_srgb, float bil_compat,
                         int32_t* labels_out, float* q_out, int32_t* vertex_counts, void* workspace, size_t workspace_bytes,
                         irn_stream_t stream);
int irn_ir_label_ragged(const uint8_t* img, size_t img_bytes, const int32_t* sizes_hw, int n, const float* high_res,
                        size_t high_res_elems, const int32_t* keys_host, const int32_t* counts_host, float conf_fg_thres,
                        float conf_bg_thres, uint8_t* out, int32_t* vertex_counts, void* workspace, size_t workspace_bytes,
                        irn_stream_t stream);
int irn_crf_set_timing(int enable);
int irn_crf_last_ms(float* ms3);

/* ---- MS COCO mask evaluation (irn_b200/csrc/coco_mask.cu) --------------------------------------------------------------------------
 * Every mask of an H x W image is a bit plane of irn_coco_plane_words(H, W) = W * ceil(H/32) uint32 words: column-major, bit b of word j
 * of column x = pixel (32j+b, x), the bits past row H-1 zero.  A call's planes lie back to back.  All sizes and descriptors are HOST
 * arrays, uploaded once per call into the workspace; every output is an exact integer.  Returns -1 for a bad size.
 *
 * irn_coco_rasterize   ground truth -> planes uint32 [plane_words], one plane per annotation (ann_hw HOST int32 [n_ann][2] = H, W).
 *                      An annotation is the union of its parts (part_ann HOST int32 [n_parts]: the part's annotation), each a polygon
 *                      or an uncompressed RLE.  edges HOST int32 [n_edges][4] = (part, first vertex, k, j): edge j -> j+1 mod k of the
 *                      part's polygon of k vertices at vertices[first..first+k) (HOST float64 [n_vertices][2] = x, y as in the JSON),
 *                      every edge of every polygon listed once; toggles HOST int32 [n_toggles][2] = (part, position in [0, H*W]): an
 *                      RLE's running count sums.  Polygons follow pycocotools' rleFrPoly (coco_mask.cu states the rule).
 * irn_coco_pack_masks  masks uint8 [sum M_i*H_i*W_i] (image i's bool [M_i,H_i,W_i] back to back, nonzero = inside), hwm HOST int32
 *                      [n_img][3] = H, W, M -> planes [sum M_i * plane_words(H_i, W_i)].
 * irn_coco_overlaps    pred / gt planes of n_img images (hwmg HOST int32 [n_img][4] = H, W, M, G; image i's M_i prediction planes and
 *                      G_i ground-truth planes back to back) -> inter int32 [sum M_i*G_i] (image i's [M_i][G_i] after the earlier
 *                      images'), area_pred int32 [sum M_i], area_gt int32 [sum G_i].  M_i = 0 or G_i = 0 is allowed.
 * The workspace queries return 0 for arguments the calls refuse.
 */
long long irn_coco_plane_words(int H, int W);
size_t irn_coco_raster_workspace_bytes(int n_parts, const int32_t* part_hw, int n_edges, int n_vertices, int n_toggles);
int irn_coco_rasterize(int n_ann, const int32_t* ann_hw, int n_parts, const int32_t* part_ann, int n_edges, const int32_t* edges,
                       int n_vertices, const double* vertices, int n_toggles, const int32_t* toggles, uint32_t* planes, size_t plane_words,
                       void* workspace, size_t workspace_bytes, irn_stream_t stream);
size_t irn_coco_pack_workspace_bytes(int n_img);
int irn_coco_pack_masks(const uint8_t* masks, size_t mask_bytes, int n_img, const int32_t* hwm, uint32_t* planes, size_t plane_words,
                        void* workspace, size_t workspace_bytes, irn_stream_t stream);
size_t irn_coco_overlap_workspace_bytes(int n_img, const int32_t* hwmg);
int irn_coco_overlaps(const uint32_t* pred_planes, size_t pred_words, const uint32_t* gt_planes, size_t gt_words, int n_img,
                      const int32_t* hwmg, int32_t* inter, int32_t* area_pred, int32_t* area_gt, void* workspace, size_t workspace_bytes,
                      irn_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* IRN_B200_H */
