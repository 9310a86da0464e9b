/* migan_b200.h -- C ABI of the H100-native MI-GAN generator forward.
 *
 * The shared library (mi-gan_b200/lib/libmigan_b200.so, built by __graft_entry__.build())
 * exports exactly the entry points declared here: plain pointers and sizes, no torch types.
 * Each one replaces a reference interface, cited as file:line in /root/reference:
 *
 *   migan_create / migan_destroy      Generator.__init__            lib/model_zoo/migan_inference.py:355-360
 *   migan_set_weight / _finalize      nn.Module.load_state_dict as used by scripts/demo.py:110
 *                                     (key names + shapes = the reference state_dict, SURVEY.md 8b)
 *   migan_forward                     Generator.forward(x)          lib/model_zoo/migan_inference.py:362-369
 *   migan_forward_host                scripts/demo.py:131-136 (x.to(device) -> model(x) -> .cpu())
 *   migan_forward_u8, b200_pre/postprocess_u8   scripts/demo.py:56-66 (preprocess) and :135-142 (uint8 + mask composite)
 *   b200_upfirdn2d                    _plugin.upfirdn2d(...)        torch_utils/ops/upfirdn2d.cpp:16-94
 *   b200_bias_act                     _plugin.bias_act(...)         torch_utils/ops/bias_act.cpp:32-90 (grad == 0)
 *   b200_conv1x1_nhwc                 the F.conv2d of conv2d_resample's 1x1 branches  torch_utils/ops/conv2d_resample.py:106-116
 *
 * Conventions: every function returns 0 on success and a non-zero code on failure, after
 * which migan_last_error() describes the failure (thread-local string).  All device pointers
 * are fp32, 16-byte aligned, on the device the context was created for; `stream` is a
 * cudaStream_t passed as void* (NULL = legacy default stream).  Nothing here falls back to
 * the CPU: without a CUDA device every compute entry point fails with MIGAN_ERR_CUDA.
 */
#ifndef MIGAN_B200_H_
#define MIGAN_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MIGAN_OK 0
#define MIGAN_ERR_INVALID 1   /* bad argument (shape, resolution, null pointer, unknown key) */
#define MIGAN_ERR_CUDA 2      /* a CUDA runtime/driver call or kernel launch failed */
#define MIGAN_ERR_STATE 3     /* call order (e.g. forward before weights are finalized) */
#define MIGAN_ERR_WORKSPACE 4 /* workspace too small or misaligned */

/* Contraction engine for the 1x1 pointwise convs. */
#define MIGAN_PATH_SIMT 0     /* fp32 CUDA-core FMA (bring-up / cross-check path) */
#define MIGAN_PATH_TC 1       /* wgmma tensor cores, fp16 hi/lo 3-pass split, fp32 accumulate (fp32-faithful) */
#define MIGAN_PATH_TC_FAST 2  /* wgmma, single fp16 pass (stated lower accuracy, see DESIGN.md) */

typedef struct migan_ctx migan_ctx;

const char* migan_last_error(void);
const char* migan_version(void);

/* Generator(resolution): resolution must be a power of two >= 8 (reference raises ValueError
 * otherwise, migan_inference.py:214-216).  `device` is a CUDA ordinal. */
int migan_create(int resolution, int device, migan_ctx** out);
int migan_destroy(migan_ctx* ctx);

/* Number of state_dict entries the context expects and their names/shapes, in the reference's
 * own state_dict order (154 keys @256, 177 @512). */
int migan_num_weights(const migan_ctx* ctx);
int migan_weight_info(const migan_ctx* ctx, int index, const char** name, int* ndim, int64_t shape[4]);

/* Copy one state_dict tensor (HOST pointer, fp32, contiguous, reference layout OIHW etc.).
 * Unknown names or wrong element counts fail with MIGAN_ERR_INVALID. */
int migan_set_weight(migan_ctx* ctx, const char* name, const float* host_data, int64_t numel);
/* Validate that every key was provided (and that filter_const is the zero-insertion pattern the
 * kernels implement), repack for the kernels (NHWC tap-major depthwise weights, K-major fp16
 * hi/lo pointwise weights, pre-multiplied noise) and upload.  Synchronous. */
int migan_finalize_weights(migan_ctx* ctx);

/* Scratch memory the caller must provide to migan_forward for a batch of n images. */
size_t migan_workspace_bytes(const migan_ctx* ctx, int n);

/* y[n,3,R,R] = Generator.forward(x[n,4,R,R]); x, y, workspace are DEVICE pointers (NCHW fp32,
 * contiguous).  Asynchronous on `stream`. */
int migan_forward(migan_ctx* ctx, const float* x, float* y, int n,
                  void* workspace, size_t workspace_bytes, int path, void* stream);

/* Fully convolutional forward: y[n,3,H,W] from x[n,4,H,W] for H, W >= R that are multiples of R/4 (need not be equal or
 * powers of two), with n*H*W*ch(R) < 2^31 (ch(R) = min(32768/R, 512): the largest activation).  Nominal level r keeps its
 * weights and channels and runs at the extent (H r/R, W r/R); each noise plane is its noise_const tiled,
 * noise[i][j] = noise_const[i mod r][j mod r] * noise_strength, and every up-sampling is zero insertion at its output extent.
 * At H = W = R this is migan_forward, byte for byte.
 * migan_workspace_bytes_hw returns 0 for a refused shape (the reason, with the nearest valid sizes, in migan_last_error());
 * migan_workspace_bytes(ctx, n) == migan_workspace_bytes_hw(ctx, n, R, R) for every n the latter accepts.
 * migan_forward_hw has migan_forward's contract and returns MIGAN_ERR_INVALID for a refused shape. */
size_t migan_workspace_bytes_hw(const migan_ctx* ctx, int n, int H, int W);
int migan_forward_hw(migan_ctx* ctx, const float* x, float* y, int n, int H, int W,
                     void* workspace, size_t workspace_bytes, int path, void* stream);

/* Latency form for small batches (the reference's primary caller runs batch 1: scripts/demo.py:125-142): the launch
 * sequence of one forward is captured ONCE into a CUDA graph that works on fixed staging buffers at the end of the
 * workspace, and replayed per call between two device-to-device copies (x in, y out) -- 3 submissions instead of ~50.
 * Same contract as migan_forward (DEVICE x / y, asynchronous on `stream`); the graph is rebuilt when n, path, the
 * workspace or the weights change.  workspace_bytes must be >= migan_workspace_bytes(n) + migan_graph_staging_bytes(n). */
size_t migan_graph_staging_bytes(const migan_ctx* ctx, int n);
int migan_forward_graph(migan_ctx* ctx, const float* x, float* y, int n,
                        void* workspace, size_t workspace_bytes, int path, void* stream);

/* Same with HOST x / y (pinned for full speed): H2D copy, forward, D2H copy; y_host is complete on return.
 * The batch is split into two micro-batches whose copies overlap the kernels (three streams).  The device
 * staging buffers (two slots) live at the end of the workspace:
 * workspace_bytes must be >= migan_workspace_bytes(n) + migan_host_staging_bytes(n). */
size_t migan_host_staging_bytes(const migan_ctx* ctx, int n);
int migan_forward_host(migan_ctx* ctx, const float* x_host, float* y_host, int n,
                       void* workspace, size_t workspace_bytes, int path, void* stream);
/* Serving form: enqueue only.  Consecutive calls alternate between the two staging slots, so the copies of
 * batch t+1 overlap the kernels and the copy-out of batch t (the batch is not split here: the overlap is across calls); migan_host_wait() blocks until every enqueued
 * batch has landed in its y_host.  x_host / y_host must stay valid (and unmodified) until then. */
int migan_forward_host_async(migan_ctx* ctx, const float* x_host, float* y_host, int n,
                             void* workspace, size_t workspace_bytes, int path, void* stream);
int migan_host_wait(migan_ctx* ctx);

/* uint8 request path (the callers' pre/post-processing fused around the forward, scripts/demo.py:56-66 and :135-142):
 * img_host u8 [n,R,R,3] (RGB, HWC), mask_host u8 [n,R,R] (255 = known pixel, anything else = hole) ->
 * out_host u8 [n,R,R,3] = known pixels of img, generated pixels elsewhere.  7 bytes per pixel cross PCIe instead of 28.
 * workspace_bytes must be >= migan_workspace_bytes(n) + migan_u8_staging_bytes(n) (two staging slots).
 * migan_forward_u8 is synchronous (out_host complete on return); migan_forward_u8_async only enqueues -- consecutive calls
 * alternate between the slots so that the copies of request t+1 / t-1 run under the kernels of request t, and
 * migan_host_wait() blocks until every enqueued request has landed (buffers must stay valid and unmodified until then). */
size_t migan_u8_staging_bytes(const migan_ctx* ctx, int n);
int migan_forward_u8(migan_ctx* ctx, const uint8_t* img_host, const uint8_t* mask_host, uint8_t* out_host, int n,
                     void* workspace, size_t workspace_bytes, int path, void* stream);
int migan_forward_u8_async(migan_ctx* ctx, const uint8_t* img_host, const uint8_t* mask_host, uint8_t* out_host, int n,
                           void* workspace, size_t workspace_bytes, int path, void* stream);
/* The two kernels on their own (DEVICE pointers): x[n,4,r,r] = cat([mask-0.5, img*mask]) and the composite of y[n,3,r,r]. */
int b200_preprocess_u8(const uint8_t* img_hwc, const uint8_t* mask_hw, float* x_nchw, int n, int r, void* stream);
int b200_postprocess_u8(const float* y_nchw, const uint8_t* img_hwc, const uint8_t* mask_hw, uint8_t* out_hwc, int n, int r,
                        void* stream);
/* The same at any H x W: img [n,H,W,3], mask [n,H,W] -> x [n,4,H,W]; y [n,3,H,W] -> out [n,H,W,3]. */
int b200_preprocess_u8_hw(const uint8_t* img_hwc, const uint8_t* mask_hw, float* x_nchw, int n, int H, int W, void* stream);
int b200_postprocess_u8_hw(const float* y_nchw, const uint8_t* img_hwc, const uint8_t* mask_hw, uint8_t* out_hwc, int n, int H,
                           int W, void* stream);

/* Feathered composite of the deployed (ONNX) pipeline, scripts/create_onnx_pipeline.py:233-245, for a crop at the model
 * resolution (DEVICE pointers, NCHW like the pipeline): blend weight = 5x5 smoothing (reflect border) of the 3x3 max-pooled
 * mask / 255; out = clamp(image * w + ((y*0.5+0.5)*255).clamp(0,255) * (1 - w), 0, 255) -> uint8.  k25 = the 25 smoothing
 * taps on the HOST (the GaussianSmoothing buffer of :66-88; migan_b200.ops.feather_kernel() builds it the same way). */
int b200_feather_composite(const float* y_nchw, const uint8_t* image_nchw, const uint8_t* mask_n1hw, uint8_t* out_nchw,
                           int n, int H, int W, const float* k25_host, void* stream);

/* Arbitrary-resolution crop pipeline of the deployed (ONNX) form, scripts/create_onnx_pipeline.py:121-264 (MIGAN_Pipeline):
 * the caller's image u8 [3,H,W] and mask u8 [H,W] (255 = known) stay at their own size; the hole's bounding box is padded,
 * squared and clipped into a crop window, the crop is resized to the model resolution for the generator and the result is
 * resized back and blended into the image with a feathered mask.  The stages (DEVICE pointers unless noted):
 *   b200_resize_nearest_u8    mask at another size -> image size (tvF.resize NEAREST, :255)
 *   b200_hole_flags           flags[x] / flags[W + y] = column x / row y contains a value < 255 (:144-149); copy them to the host
 *   migan_crop_box            HOST arithmetic of get_masked_bbox (:151-227) -> box = {x_min, x_max, y_min, y_max}
 *   b200_pipeline_preprocess  crop -> anti-aliased bilinear resize, round -> x[4,res,res] = cat([m/255-0.5, (v*2/255-1)*m/255]) (:229-236)
 *   b200_pipeline_postprocess y[3,res,res] -> [0,255] -> anti-aliased bilinear resize to the crop -> feathered blend (3x3 max-pool,
 *                             5x5 smoothing with the 25 HOST taps k25, reflect border) written into image[crop] in place (:238-262)
 * The resize reproduces what torchvision's tensor `resize` computes on the CPU (ATen's separable anti-aliased filter, fp32
 * fused multiply-adds, width pass first) bit for bit; a pass whose size does not change is the identity.
 * scratch: b200_pipeline_scratch_bytes(H, W, res) bytes of device memory, shared by the two stages. */
size_t b200_pipeline_scratch_bytes(int H, int W, int res);
int b200_resize_nearest_u8(const uint8_t* in_hw, int H, int W, uint8_t* out_hw, int out_h, int out_w, void* stream);
int b200_hole_flags(const uint8_t* mask_hw, int H, int W, uint8_t* flags_w_plus_h, void* stream);
int migan_crop_box(const uint8_t* flags_host, int H, int W, int resolution, int padding, int* box4_host);
int b200_pipeline_preprocess(const uint8_t* image_chw, const uint8_t* mask_hw, int H, int W, const int* box4_host, int resolution,
                             float* x_nchw, void* scratch, size_t scratch_bytes, void* stream);
int b200_pipeline_postprocess(const float* y_nchw, uint8_t* image_chw, const uint8_t* mask_hw, int H, int W, const int* box4_host,
                              int resolution, const float* k25_host, void* scratch, size_t scratch_bytes, void* stream);

/* The same stages for a batch of 1..MIGAN_PIPE_MAX_BATCH requests of any sizes, one launch per stage for the whole batch
 * (the request table is passed to the kernels by value).  reqs_host is a HOST array of n requests; every request must be
 * at least 3 x 3, and images must not overlap each other or any mask.  Request i's results equal the single-request
 * stages' bit for bit:
 *   b200_hole_flags_batch            request i's flags start at sum_{j<i} (W_j + H_j), laid out as b200_hole_flags;
 *                                    the boxes are not read
 *   b200_pipeline_batch_scratch_bytes  exact scratch size for these boxes (0 on a bad argument)
 *   b200_pipeline_preprocess_batch   request i -> x[i] of a contiguous x [n,4,res,res]
 *   b200_pipeline_postprocess_batch  y[i] of a contiguous y [n,3,res,res] -> request i's image[crop], in place
 * Fills the boxes with migan_crop_box (one call per request, on the host flags) between the flags and the pre-processing. */
#define MIGAN_PIPE_MAX_BATCH 32
typedef struct {
    uint8_t* image;        /* DEVICE u8 [3][H][W]; the post-processing writes image[crop] in place */
    const uint8_t* mask;   /* DEVICE u8 [H][W], 255 = known (already at the image size) */
    int H, W;
    int box[4];            /* x_min, x_max, y_min, y_max from migan_crop_box; not read by b200_hole_flags_batch */
} migan_pipe_request;
int b200_hole_flags_batch(const migan_pipe_request* reqs_host, int n, uint8_t* flags, void* stream);
size_t b200_pipeline_batch_scratch_bytes(const migan_pipe_request* reqs_host, int n, int resolution);
int b200_pipeline_preprocess_batch(const migan_pipe_request* reqs_host, int n, int resolution, float* x_n4rr,
                                   void* scratch, size_t scratch_bytes, void* stream);
int b200_pipeline_postprocess_batch(const float* y_n3rr, const migan_pipe_request* reqs_host, int n, int resolution,
                                    const float* k25_host, void* scratch, size_t scratch_bytes, void* stream);

/* The same batch with the crop windows planned on the DEVICE, so a whole pass is enqueued without a host round trip:
 *   b200_hole_flags_batch -> b200_pipeline_plan_batch -> b200_pipeline_preprocess_planned -> [generator]
 *   -> b200_pipeline_postprocess_planned
 * The boxes in reqs_host are not read.  Every call of a pass gets the same reqs_host (the same n, images, masks and sizes),
 * resolution and scratch; resolution must be at least 3.  Request i's boxes, x[i] and image[crop] equal the host-box
 * batched calls' on the windows migan_crop_box gives, bit for bit.
 *   b200_pipeline_batch_scratch_bound  scratch for every crop window the images allow, from the image sizes alone (0 on a
 *                                      bad argument); the phases' descriptors live there from the plan to the post-processing
 *   b200_pipeline_plan_batch           one launch: boxes_dev int32 [n][4] (DEVICE; x_min, x_max, y_min, y_max per request)
 *                                      and the descriptors of both phases, from the flags of b200_hole_flags_batch */
size_t b200_pipeline_batch_scratch_bound(const migan_pipe_request* reqs_host, int n, int resolution);
int b200_pipeline_plan_batch(const migan_pipe_request* reqs_host, int n, int resolution, int padding, const uint8_t* flags,
                             int* boxes_dev, void* scratch, size_t scratch_bytes, void* stream);
int b200_pipeline_preprocess_planned(const migan_pipe_request* reqs_host, int n, int resolution, float* x_n4rr,
                                     void* scratch, size_t scratch_bytes, void* stream);
int b200_pipeline_postprocess_planned(const float* y_n3rr, const migan_pipe_request* reqs_host, int n, int resolution,
                                      const float* k25_host, void* scratch, size_t scratch_bytes, void* stream);

/* The crop pipeline on decoded photos and raw masks.  The entry points above take image [3][H][W] (MIGAN_LAYOUT_CHW);
 * the *_layout forms take the layout of every image of the call: MIGAN_LAYOUT_CHW, or MIGAN_LAYOUT_HWC for image
 * [H][W][3] (a decoder's photo), with the same results bit for bit on the transposed image.  The planned descriptors
 * carry the layout, so a pass planned by b200_pipeline_plan_batch_layout runs b200_pipeline_preprocess_planned and
 * b200_pipeline_postprocess_planned as they are.
 *   b200_pipeline_mask_planes  one launch for 1..MIGAN_PIPE_MAX_BATCH raw masks (masks_host: HOST array): mask u8
 *                              [hm][wm][channels] as decoded -> out u8 [H][W] (DEVICE), 255 = known, 0 = hole, by
 *                              create_onnx_pipeline.py's read_mask (:27-45: alpha of LA / RGBA, R of RGB, L; 255 - v if
 *                              invert; v < 255 -> 0) and the NEAREST resize to H x W (:255), the plane the stages above read */
#define MIGAN_LAYOUT_CHW 0
#define MIGAN_LAYOUT_HWC 1
typedef struct {
    const uint8_t* mask;   /* DEVICE u8 [hm][wm][channels], channels 1..4 */
    uint8_t* out;          /* DEVICE u8 [H][W] */
    int hm, wm, channels, invert;
    int H, W;
} migan_raw_mask;
int b200_pipeline_mask_planes(const migan_raw_mask* masks_host, int n, void* stream);
int b200_pipeline_preprocess_batch_layout(const migan_pipe_request* reqs_host, int n, int resolution, int layout, float* x_n4rr,
                                          void* scratch, size_t scratch_bytes, void* stream);
int b200_pipeline_postprocess_batch_layout(const float* y_n3rr, const migan_pipe_request* reqs_host, int n, int resolution,
                                           int layout, const float* k25_host, void* scratch, size_t scratch_bytes, void* stream);
int b200_pipeline_plan_batch_layout(const migan_pipe_request* reqs_host, int n, int resolution, int padding, int layout,
                                    const uint8_t* flags, int* boxes_dev, void* scratch, size_t scratch_bytes, void* stream);

/* The reference demo's request path at any photo size (scripts/demo.py:26-66, :120-143), for a batch of
 * 1..MIGAN_PIPE_MAX_BATCH requests, one launch per stage:
 *   photo  -> PIL BICUBIC down-scale to at most R (only when W > R or H > R): img_resized, out_w x out_h
 *   mask   -> PIL NEAREST to at most 512 -> channel (alpha of LA / RGBA, R of RGB, L) -> 255 - v if invert -> v < 255 -> 0
 *             -> PIL NEAREST to at most R: mask_resized, which must come out at out_w x out_h
 *   b200_demo_preprocess   img_resized -> PIL BICUBIC R x R, mask_resized -> NEAREST R x R -> x[i] of x [n,4,R,R]
 *   [generator]
 *   b200_demo_postprocess  y[i] -> (y*0.5+0.5).clamp(0,1)*255 -> uint8 -> cv2.resize INTER_CUBIC to out_w x out_h ->
 *                          img_resized where mask_resized is 255, else the resized result -> out
 * Every resize reproduces its library's uint8 arithmetic bit for bit (OpenCV: the scalar path, cv2.setUseOptimized(False)).
 * The sizes follow demo.py's `resize`: (int(w * r), int(h * r)) with r = max_size / w if w > h else max_size / h;
 * migan_demo_resized_size computes them.  reqs_host is a HOST array; both calls of a pass get the same reqs_host,
 * resolution and scratch (b200_demo_scratch_bytes bytes of device memory; 0 on a bad argument). */
typedef struct {
    const uint8_t* img;    /* DEVICE u8 [H][W][3] */
    int H, W;
    const uint8_t* mask;   /* DEVICE u8 [Hm][Wm][mask_channels]: 1 (L), 2 (LA), 3 (RGB) or 4 (RGBA) */
    int Hm, Wm, mask_channels;
    int invert;            /* non-zero: 255 - v before the threshold */
    uint8_t* out;          /* DEVICE u8 [out_h][out_w][3], written by b200_demo_postprocess */
    int out_w, out_h;      /* the size of img_resized: migan_demo_resized_size(W, H, resolution) */
} migan_demo_request;
int migan_demo_resized_size(int w, int h, int max_size, int* out_w, int* out_h);
size_t b200_demo_scratch_bytes(const migan_demo_request* reqs_host, int n, int resolution);
int b200_demo_preprocess(const migan_demo_request* reqs_host, int n, int resolution, float* x_n4rr, void* scratch,
                         size_t scratch_bytes, void* stream);
int b200_demo_postprocess(const float* y_n3rr, const migan_demo_request* reqs_host, int n, int resolution, void* scratch,
                          size_t scratch_bytes, void* stream);

/* The evaluation batch of scripts/evaluate_fid_lpips.py (InferenceDataset and :246-249) on the demo path's stages, for
 * 1..MIGAN_PIPE_MAX_BATCH requests of migan_demo_request (out, out_w and out_h are not read):
 *   b200_eval_preprocess   photo -> PIL BICUBIC to R x R when it is not that size (one resize of both axes), mask ->
 *                          PIL NEAREST to R x R and the demo's per-pixel steps (L: 255 known) -> x[i] of x [n,4,R,R], and
 *                          the unmasked photo v * 2 / 255 - 1 -> img[i] of img [n,3,R,R].  Scratch:
 *                          b200_eval_scratch_bytes (0 on a bad argument).
 *   [generator]
 *   b200_eval_composite    composed = m * img + (1 - m) * y (m = x channel 0 + 0.5), then (v * 0.5 + 0.5).clamp(0, 1) of
 *                          img, in place (the script's `imgs`), and of composed, each product and sum rounded on its own. */
size_t b200_eval_scratch_bytes(const migan_demo_request* reqs_host, int n, int resolution);
int b200_eval_preprocess(const migan_demo_request* reqs_host, int n, int resolution, float* x_n4rr, float* img_n3rr,
                         void* scratch, size_t scratch_bytes, void* stream);
int b200_eval_composite(const float* x_n4rr, const float* y_n3rr, int n, int resolution, float* img_n3rr,
                        float* composed_n3rr, void* stream);

/* Full-resolution request path: a photo of ANY size (H, W >= 1) inpainted at its own resolution by migan_forward_hw.
 *   migan_fullres_extent   the padded extent Hp = max(R, q ceil(H / q)), Wp likewise (q = R / 4): the smallest size
 *                          migan_forward_hw accepts that holds the photo (a valid size is not padded), and the largest batch
 *                          migan_forward_hw accepts there.  MIGAN_ERR_INVALID when one photo alone is too large for a forward.
 *   b200_fullres_preprocess   photo + mask -> x of each request: the photo at the origin, padded on the bottom and right by
 *                          numpy's np.pad(mode="reflect") rule (no edge repeat, iterated when the pad is longer than the side;
 *                          a 1-pixel side replicates).  The mask's per-pixel steps are read_mask's without its resize (channel:
 *                          alpha of LA / RGBA, R of RGB, L; 255 - v if invert; v < 255 -> 0) and the known-mask is reflected
 *                          with the photo: x = cat([mask - 0.5, img * mask]) at Hp x Wp.
 *   [migan_forward_hw at Hp x Wp, one call per chunk of requests that share an extent]
 *   b200_fullres_postprocess  y -> (y*0.5+0.5).clamp(0,1)*255 -> uint8 on the top-left H x W; known pixels from the photo.
 * The result is byte for byte b200_preprocess_u8_hw -> migan_forward_hw -> b200_postprocess_u8_hw on the host-padded photo
 * and known-mask, cropped to H x W (at a valid size: on the photo itself).  reqs_host is a HOST array of 1..MIGAN_PIPE_MAX_BATCH
 * requests of any sizes and extents; each call is one launch. */
typedef struct {
    const uint8_t* img;    /* DEVICE u8 [H][W][3] */
    const uint8_t* mask;   /* DEVICE u8 [H][W][mask_channels]: 1 (L), 2 (LA), 3 (RGB) or 4 (RGBA) */
    int H, W, mask_channels;
    int invert;            /* non-zero: 255 - v before the threshold */
    float* x;              /* DEVICE, 16-byte aligned: the request's slot [4][Hp][Wp] of its chunk's x [n,4,Hp,Wp] */
    const float* y;        /* DEVICE: the request's slot [3][Hp][Wp] of its chunk's y [n,3,Hp,Wp] */
    int Hp, Wp;            /* migan_fullres_extent(H, W); at least H x W */
    uint8_t* out;          /* DEVICE u8 [H][W][3], written by b200_fullres_postprocess */
} migan_fullres_request;
int migan_fullres_extent(const migan_ctx* ctx, int H, int W, int* Hp, int* Wp, int* max_n);
int b200_fullres_preprocess(const migan_fullres_request* reqs_host, int n, void* stream);
int b200_fullres_postprocess(const migan_fullres_request* reqs_host, int n, void* stream);

/* Hole-window request path: only margin-padded windows around the holes of a photo of ANY size are inpainted, each at its
 * own resolution by the full-resolution path; every other pixel keeps the photo's value.  With q = R / 4:
 *   b200_hole_cells        the photo is split into q x q cells anchored at the origin (gh = ceil(H / q) rows by
 *                          gw = ceil(W / q) columns; the last ones may be partial).  cells[cy * gw + cx] = 1 when the cell
 *                          holds a hole pixel (not known by the full-resolution path's mask steps), else 0.  One launch for
 *                          1..MIGAN_PIPE_MAX_BATCH requests (reqs_host: HOST array); request i's cells follow request i - 1's;
 *                          b200_hole_cells_bytes gives the total (0 on a bad argument).  Each mask byte is read once.
 *   migan_hole_windows     HOST: the windows of one request from a HOST copy of its cells, sorted by (y0, x0), as
 *                          {y0, x0, h, w} quadruples in windows4 (room for max_windows).  On each axis (side n) a span of
 *                          cells [c0, c1] with a margin of m cells gives a = max(0, (c0 - m) q), b = min(n, (c1 + 1 + m) q),
 *                          L = min(n, max(R, q ceil((b - a) / q))), s = min(max(a - (L - (b - a)) / 2, 0), n - L) and the
 *                          window [s, s + L).  The hole cells are visited in row-major order; each starts as its own span,
 *                          and while its window overlaps (positive area) a window already listed, the first such window
 *                          is removed and the spans are united; the result is appended.  The windows are disjoint, cover
 *                          every hole pixel, and each side is a valid forward_fc size or the photo's side.
 *   migan_hole_windows_max the most windows an H x W photo can have: floor(H / min(R, H)) * floor(W / min(R, W)).
 *   b200_window_preprocess / b200_window_postprocess   the full-resolution pre- and post-processing of each window's crop
 *                          (reflect padding of the crop to Hp x Wp = migan_fullres_extent(h, w), composite); the
 *                          post-processing writes only the window's pixels of `out`, which holds a copy of the photo (it
 *                          may be the photo itself).  One launch for 1..MIGAN_PIPE_MAX_BATCH windows of any requests.
 * resolution: a power of two >= 8 (the generator's). */
typedef struct {
    const uint8_t* mask;   /* DEVICE u8 [H][W][mask_channels]: 1 (L), 2 (LA), 3 (RGB) or 4 (RGBA) */
    int H, W, mask_channels;
    int invert;            /* non-zero: 255 - v before the threshold */
} migan_cells_request;
size_t b200_hole_cells_bytes(const migan_cells_request* reqs_host, int n, int resolution);
int b200_hole_cells(const migan_cells_request* reqs_host, int n, int resolution, uint8_t* cells, void* stream);
int migan_hole_windows(const uint8_t* cells_host, int H, int W, int resolution, int margin, int* windows4, int max_windows,
                       int* count);
int migan_hole_windows_max(int H, int W, int resolution, int* max_windows);
typedef struct {
    const uint8_t* img;    /* DEVICE u8 [H][W][3]: the photo */
    const uint8_t* mask;   /* DEVICE u8 [H][W][mask_channels] */
    int H, W, mask_channels;
    int invert;            /* non-zero: 255 - v before the threshold */
    int y0, x0, h, w;      /* the window, inside the photo */
    float* x;              /* DEVICE, 16-byte aligned: the window's slot [4][Hp][Wp] of its chunk's x [n,4,Hp,Wp] */
    const float* y;        /* DEVICE: the window's slot [3][Hp][Wp] of its chunk's y [n,3,Hp,Wp] */
    int Hp, Wp;            /* migan_fullres_extent(h, w) */
    uint8_t* out;          /* DEVICE u8 [H][W][3]: a copy of the photo (or the photo); the window is written */
} migan_window_request;
int b200_window_preprocess(const migan_window_request* reqs_host, int n, void* stream);
int b200_window_postprocess(const migan_window_request* reqs_host, int n, void* stream);

/* Free-form masks of the evaluation protocol: RandomMask(s, hole_range) of scripts/generate_masks.py, byte for byte and
 * at the same position of numpy's legacy global stream.  One RandomMask result is the first *attempt* whose hole
 * count lies in (0, s^2) (hole_range [0, 1]; [h_min, h_max] of migan_mask_hole_bounds for another range); an attempt's
 * draws never depend on earlier results, so the stream is a fixed sequence of attempts:
 *   migan_np_seed            HOST: np.random.seed(seed) for an integer seed (MT19937 init_genrand, no cached gaussian).
 *   migan_mask_plan          HOST: the draws of the next n_attempts attempts of RandomMask(s), from *state (advanced):
 *                            one migan_mask_record each (records_host), and, when states_host is not NULL, the state
 *                            after each attempt (states_host[k]: after attempt k) so the caller can rewind to the last
 *                            attempt it uses.
 *   b200_mask_raster         DEVICE: paints every attempt into attempts [n_attempts][s][s] (16-byte aligned; 255 known, 0 hole; Pillow's
 *                            wide-line polygons and ellipse stamps, exact) and writes its hole count to holes[k].
 *   b200_mask_compact        DEVICE: copies the first min(n, accepted) accepted attempts (0 < holes < s^2), in attempt
 *                            order, to out [n][s][s].
 * s: MIGAN_MASK_MIN_SIZE..MIGAN_MASK_MAX_SIZE; n_attempts: 1..MIGAN_MASK_MAX_ATTEMPTS per call.
 * Another hole_range [lo, hi] (0 <= lo < hi <= 1, lo + hi >= 0.2: below that RandomMask draws numpy's refused
 * randint(0)):
 *   migan_mask_plan_range    HOST: migan_mask_plan with RandomMask's int(10 * coef), int(5 * coef) and int(20 * coef)
 *                            tries, coef = min(lo + hi, 1.0) in float64.  [0, 1] gives migan_mask_plan's records.
 *   migan_mask_hole_bounds   HOST: the hole counts RandomMask(s, [lo, hi]) keeps, [*h_min, *h_max] (empty when
 *                            *h_min > *h_max): hole_ratio = 1 - fl((s^2 - holes) / s^2) in float64, rejected when
 *                            hole_ratio <= lo or hole_ratio >= hi.  [0, 1] gives [1, s^2 - 1].
 *   b200_mask_compact_range  DEVICE: b200_mask_compact keeping the attempts with h_min <= holes <= h_max. */
#define MIGAN_MASK_MIN_SIZE 2
#define MIGAN_MASK_MAX_SIZE 4096
#define MIGAN_MASK_MAX_ATTEMPTS 65535
#define MIGAN_MASK_MAX_RECTS 13       /* randint(10) + randint(5) rectangles */
#define MIGAN_MASK_MAX_SEGMENTS 323   /* randint(20) brush tries x (randint(4, 18) segments) */
#define MIGAN_MASK_MAX_DISCS 342      /* the same tries x (segments + 1) vertex discs */
typedef struct {
    uint32_t key[624];     /* np.random.get_state()[1] */
    int pos;               /* [2] */
    int has_gauss;         /* [3] */
    double gauss;          /* [4] */
} migan_np_random;
typedef struct {
    int32_t n_rects, n_segments, n_discs;
    int32_t flips;                                  /* bit 0: brush rows flipped, bit 1: brush columns (not the rects) */
    int16_t rects[MIGAN_MASK_MAX_RECTS][4];         /* y0, y1, x0, x1: rows [y0, y1) x columns [x0, x1) become holes */
    int16_t quads[MIGAN_MASK_MAX_SEGMENTS][8];      /* Pillow's wide-line quad, (x, y) x 4; 4 equal vertices: one pixel */
    int16_t discs[MIGAN_MASK_MAX_DISCS][4];         /* x, y, r (6..23), 0 */
} migan_mask_record;
int migan_np_seed(migan_np_random* state, uint32_t seed);
int migan_mask_plan(migan_np_random* state, int s, int n_attempts, migan_mask_record* records_host,
                    migan_np_random* states_host);
int b200_mask_raster(const migan_mask_record* records, int n_attempts, int s, uint8_t* attempts, int* holes, void* stream);
int b200_mask_compact(const uint8_t* attempts, const int* holes, int n_attempts, int s, int n, uint8_t* out, void* stream);
int migan_mask_plan_range(migan_np_random* state, int s, double lo, double hi, int n_attempts,
                          migan_mask_record* records_host, migan_np_random* states_host);
int migan_mask_hole_bounds(int s, double lo, double hi, int* h_min, int* h_max);
int b200_mask_compact_range(const uint8_t* attempts, const int* holes, int n_attempts, int s, int h_min, int h_max, int n,
                            uint8_t* out, void* stream);

/* Training snapshot -> inference filter, scripts/export_inference_model.py:18-27 (`get_source_w`): out[cout][fan] =
 * v * rsqrt(sum_fan v^2 + 1e-8) with v = (w_0 + ... + w_{k-1}) / sqrt(k) for a re-parameterised layer (k tensors) or v = w_0
 * (k = 1).  w_dev: HOST array of k DEVICE pointers to [cout][fan] fp32 tensors (fan = cin/groups * kh * kw); out: device.
 * Agrees with the reference's CPU result to a few ulp (the sum of squares is accumulated in fp64). */
int b200_reparam_filter(const float* const* w_dev, int k, int cout, int64_t fan, float* out, void* stream);

/* Stream memory operations for multi-GPU signalling (mi-gan_b200/parallel.py): the stream waits until the 32-bit word at a
 * DEVICE address reaches `value` (cyclic comparison (int32)(*addr - value) >= 0), or writes `value` to it, in stream order.
 * Executed by the stream's front end: no kernel, no SM.  b200_stream_memops_available() is 1 when the driver offers them. */
int b200_stream_memops_available(void);
int b200_stream_wait_value32(void* stream, void* addr, uint32_t value);
int b200_stream_write_value32(void* stream, void* addr, uint32_t value);
/* cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDefault, stream): one copy-engine transfer between any two mapped device
 * addresses (local or a peer's), enqueued on `stream` of the CURRENT device and nothing else (no cross-device event exchange). */
int b200_memcpy_async(void* dst, const void* src, size_t bytes, void* stream);
/* cudaDeviceEnablePeerAccess(peer_device) for the CURRENT device (already enabled is not an error): copies between the two
 * devices' memory then go directly over NVLink instead of being staged. */
int b200_enable_peer_access(int peer_device);

/* Kernels launched by the most recent migan_forward on this context.
 * Execution plans (tensor maps, tile grids, noise-plane tables) are cached per (n, path, workspace, H, W), up to 8 of them,
 * least recently used first out; new weights clear the cache.  The profiling calls below report the plan of the last forward. */
int migan_last_launch_count(const migan_ctx* ctx);

/* Per-launch timing for roofline reports: when enabled, every kernel launch of subsequent
 * forwards is bracketed by cudaEvents on the launching stream.  migan_profile_step returns, for
 * step `index` of the current plan, its label ("<state_dict prefix><kernel>"), the duration of
 * its most recent launch (synchronizes on its end event), and its algorithmic bytes / flops
 * (own inputs read once + output written once; SURVEY.md section 8d). */
int migan_set_profiling(migan_ctx* ctx, int enable);
int migan_profile_num_steps(const migan_ctx* ctx);
int migan_profile_step(migan_ctx* ctx, int index, const char** label, float* ms, double* alg_bytes, double* flops);

/* Debug/test tap: during the next forwards, copy the named intermediate (converted to NCHW
 * fp32) into `dst` (device pointer, large enough).  name == NULL clears the tap.  Names follow
 * the oracle's tap names (oracle/migan_oracle.py), e.g. "encoder.b256.conv1.out". */
int migan_set_tap(migan_ctx* ctx, const char* name, float* dst);
/* Enumerate tap names produced by a forward on `path` (index from 0; returns MIGAN_ERR_INVALID
 * past the end).  shape = {C, H, W} of one image. */
int migan_tap_info(const migan_ctx* ctx, int path, int index, const char** name, int shape[3]);

/* Debug: every pipeline wait inside the wgmma kernel is bounded (seconds of wall-clock time); a wait that gives up records
 * (wait code | parity << 12 | block << 16) in a host-mapped word and traps.  Returns that record for `device` (0: none). */
int migan_debug_tc_timeout(int device);

/* Test hook: one launch of the tensor-core SeparableConv2d kernel on caller-provided operands, packed by the same
 * functions the weight loader uses.  Device pointers, reference layouts.  The package never calls it. */
typedef struct migan_sepconv_tc_io {
    int source;                 /* 0 NHWC, 1 SPLIT (pre-split fp16 A operand), 2 UP, 3 STEM */
    int n, h, w, cin, cout;
    int act, passes;            /* act: lrelu_agc in the epilogue; passes: 3 (fp16 hi/lo split) or 1 */
    const float* in;            /* NHWC [n,h,w,cin]; UP: the skip tensor */
    const float* up_t;          /* UP: [n,h/2,w/2,cin], the up-sampling layer's raw 1x1 output */
    const float* up_noise;      /* UP: [h][noise_pitch] added before the prologue's activation, or NULL */
    const float* up_fir;        /* UP: [4][4] channel-uniform FIR taps */
    const float* x;             /* STEM: NCHW [n,4,h,w] */
    const float* fromrgb_w;     /* STEM: [cin,4] */
    const float* fromrgb_b;     /* STEM: [cin] */
    const void* a_hi;           /* SPLIT: fp16 [n,h,w,cin], 64 * activation split into hi + lo */
    const void* a_lo;
    const float* dw_w;          /* depthwise [cin,1,3,3] */
    const float* dw_b;          /* [cin] */
    const float* pw_w;          /* pointwise [cout,cin]; NULL plans only (no device is touched; needs sms > 0) */
    const float* noise;         /* [h][noise_pitch] added before the epilogue's activation, or NULL */
    int noise_pitch;            /* floats, a multiple of 4, >= w */
    int torgb;                  /* fuse torgb + image into the epilogue */
    const float* rgb_w;         /* [3,cout] */
    const float* rgb_b;         /* [3] */
    const float* rgb_fir;       /* [3,4,4] image up-sampling taps (read if img_lo != NULL) */
    const float* img_lo;        /* [n,3,h/2,w/2] or NULL */
    float* img_out;             /* [n,3,h,w] */
    int store_out;              /* with torgb: 0 writes no feature map */
    float* out;                 /* NHWC [n,h,w,cout] */
} migan_sepconv_tc_io;

typedef struct migan_sepconv_tc_plan {
    int n_group, in_stages, a_stages, b_stages, b_resident, dw_global;
    int tile_w, tile_h, tile_n, n_tile, grid, num_tiles;
    int num_candidates;         /* length of the planner's candidate list for these shapes */
    int ep_stages;              /* stages of the epilogue's noise / image window ring (0: the epilogue reads global memory) */
    int ep_offset;              /* its byte offset and stage size in the 1024-aligned dynamic shared memory */
    int ep_stage_bytes;
    int smem_bytes;             /* dynamic shared memory of the launch (layout + 1024 bytes of alignment slack) */
} migan_sepconv_tc_plan;

/* Plans (and, unless io->pw_w is NULL, runs to completion on `stream`) one launch.  sms: SMs of the persistent grid
 * (0: what a forward uses, the device's minus MIGAN_TC_RESERVE_SMS).  candidate: -1 the planner's choice, i >= 0 the
 * i-th entry of its candidate list (MIGAN_ERR_INVALID if that layout does not fit).  `plan` receives the record. */
int migan_debug_sepconv_tc(const migan_sepconv_tc_io* io, int sms, int candidate, migan_sepconv_tc_plan* plan, void* stream);

/* Test hook: one launch of a CUDA-core stage kernel of the forward (elementwise.cu) on caller-provided operands, packed by
 * the same functions the weight loader uses.  Device pointers, reference layouts.  The package never calls it. */
enum { MIGAN_STAGE_STEM = 0, MIGAN_STAGE_DW = 1, MIGAN_STAGE_DOWN = 2, MIGAN_STAGE_UP2 = 3, MIGAN_STAGE_TORGB = 4,
       MIGAN_STAGE_NOISE_TILE = 5, MIGAN_STAGE_ADD = 6 };
/* The down-sampling kernel forms: fp32 output (CUDA-core path), or the tensor-core GEMM's pre-split fp16 operand from the
 * register-streaming or the TMA-staged kernel.  MIGAN_DOWN_AUTO: the form a forward picks for the layer. */
enum { MIGAN_DOWN_AUTO = -1, MIGAN_DOWN_F32 = 0, MIGAN_DOWN_SPLIT = 1, MIGAN_DOWN_TMA = 2 };

typedef struct migan_stage_io {
    int kind;                   /* MIGAN_STAGE_* */
    int n, h, w, c;             /* the kernel's input extent and channels (UP2: the low-resolution side; NOISE_TILE: the
                                   tiled plane, n and c unused; ADD: n * h * w * c elements) */
    int tc;                     /* DOWN with MIGAN_DOWN_AUTO: 1 the tensor-core path, 0 the CUDA-core path */
    int level;                  /* DOWN with MIGAN_DOWN_AUTO: the layer's nominal output side (R x R forward: h / 2) */
    int r;                      /* NOISE_TILE: side of the source plane */
    int noise_pitch;            /* UP2 / NOISE_TILE: floats between noise rows (>= 2w / w) */
    const float* in;            /* STEM: NCHW [n,4,h,w]; DW / DOWN / UP2 / TORGB: NHWC [n,h,w,c]; NOISE_TILE: [r][r];
                                   ADD: the addend */
    const float* dw_w;          /* DW / DOWN: depthwise [c,1,3,3] */
    const float* dw_b;          /* DW / DOWN: [c] */
    const float* fir;           /* DOWN / UP2: [c,1,4,4]; TORGB: [3,1,4,4] image up-sampling taps (read if img_lo) */
    const float* fromrgb_w;     /* STEM: [c,4] */
    const float* fromrgb_b;     /* STEM: [c] */
    const float* rgb_w;         /* TORGB: [3,c] */
    const float* rgb_b;         /* TORGB: [3] */
    const float* img_lo;        /* TORGB: [n,3,h/2,w/2] or NULL */
    const float* noise;         /* UP2: [2h][noise_pitch] or NULL */
    const float* skip;          /* UP2: NHWC [n,2h,2w,c] or NULL */
    float* out;                 /* STEM / DW: NHWC [n,h,w,c]; DOWN fp32: [n,h/2,w/2,c]; UP2: [n,2h,2w,c]; TORGB: NCHW
                                   [n,3,h,w]; NOISE_TILE: [h][noise_pitch]; ADD: the tensor added to in place */
    void* out_hi;               /* DW / DOWN split forms: fp16 hi / lo of the activation * 64 (DOWN: * 64 * 2^-fir_shift) */
    void* out_lo;
} migan_stage_io;

typedef struct migan_stage_plan {
    int kind;
    int down_form;              /* DOWN: the MIGAN_DOWN_* form that ran; -1 otherwise */
    int rs;                     /* rows per thread of the DW / DOWN kernels, 0 otherwise */
    int cg;                     /* DOWN split: the C template; TORGB: G lanes per pixel; 0 otherwise */
    int grid;                   /* blocks of the (first) launch */
    int groups;                 /* launches (image groups of < 2^31 work items) */
    int fir_shift;              /* DOWN tensor-core forms: m of the 2^-m folded into the taps (the GEMM undoes it) */
} migan_stage_plan;

/* Plans (and, when the kind's weights are given -- or, for NOISE_TILE / ADD, `in` -- runs to completion on `stream`) one
 * stage launch.  variant: the DOWN form, MIGAN_DOWN_AUTO for a forward's choice; ignored by the other kinds.  A form the
 * launcher refuses for the shape returns MIGAN_ERR_INVALID and launches nothing.  Plan-only calls touch no device. */
int migan_debug_stage(const migan_stage_io* io, int variant, migan_stage_plan* plan, void* stream);

/* upfirdn2d(x[n,c,h,w], f[fh,fw]) -> y[n,c,oh,ow], oh = (h*upy + pady0 + pady1 - fh + downy) / downy
 * (upfirdn2d.cpp:32-33).  f == NULL means the 1x1 identity filter.  Device pointers. */
int b200_upfirdn2d(const float* x, const float* f, float* y, int n, int c, int h, int w, int fh, int fw,
                   int upx, int upy, int downx, int downy, int padx0, int padx1, int pady0, int pady1,
                   int flip_filter, float gain, void* stream);

/* 1x1 convolution on channels-last data: y[p][o] = sum_i x[p][i] * w_t[i][o]  (fp32 CUDA-core GEMM;
 * the conv inside conv2d_resample's 1x1 branches, torch_utils/ops/conv2d_resample.py:106-116).
 * cin % 16 == 0, cout % 64 == 0. */
int b200_conv1x1_nhwc(const float* x, const float* w_t, float* y, int64_t pixels, int cin, int cout, void* stream);

/* bias_act forward: y = clamp(gain * act(x + b)), b indexed along the dimension whose stride is
 * step_b and size size_b (bias_act.cpp:72-73: (xi / stepB) % sizeB); b == NULL: no bias.
 * act: 1 linear 2 relu 3 lrelu 4 tanh 5 sigmoid 6 elu 7 selu 8 softplus 9 swish (bias_act.py:22-32);
 * clamp < 0 disables clamping. */
int b200_bias_act(const float* x, const float* b, float* y, int64_t numel, int64_t step_b, int size_b,
                  int act, float alpha, float gain, float clamp, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MIGAN_B200_H_ */
