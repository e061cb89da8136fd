/* pf_b200.h -- C ABI of the H100-native (sm_90a) PerspectiveFields inference engine (libpf_b200.so).
 *
 * The reference (jinlinyi/PerspectiveFields) is pure Python and has no FFI boundary of its own: the boundary it
 * offers is the class perspective2d.PerspectiveFields (perspective2d/perspectivefields.py:121-272).  This header is
 * what a maintainer binds (ctypes, see INTEGRATION.md) underneath that class to replace
 *
 *     PerspectiveFields.forward                 perspectivefields.py:223-272
 *       ResizeTransform.apply_image (uint8)     perspectivefields.py:38-46     (pf_forward, images_u8 path)
 *       (x - pixel_mean) / pixel_std, stack     perspectivefields.py:234-236
 *       backbone (MiT-B3), ll_enc               mix_transformers.py:449-485, perspectivefields.py:79-83
 *       persformer_heads.inference/postprocess  persformer_heads.py:73-101, gravity_head.py:139-197,237-261,
 *                                               latitude_head.py:138-219, utils/utils.py:114-162,483-507
 *       param_net                               param_network.py:46-69,193-221, convnext.py:140-152,
 *                                               utils/utils.py:47-91
 *
 * Conventions: plain pointers and sizes only; every DEVICE pointer refers to memory on the engine's device that the
 * caller owns (allocated e.g. through PyTorch); the engine owns nothing but small lookup tables.  All work is
 * enqueued on the caller's stream and the call returns without synchronising.  Functions return 0 on success and a
 * negative pf_status otherwise; pf_last_error() gives the message (thread-local).  A handle is not re-entrant.
 * There is no CPU fallback: without a CUDA device every compute entry point fails with PF_ERR_CUDA.
 */
#ifndef PF_B200_H_
#define PF_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PF_ABI_VERSION 3

typedef struct pf_engine* pf_handle;

enum pf_status { PF_OK = 0, PF_ERR_ARG = -1, PF_ERR_CUDA = -2, PF_ERR_WEIGHT = -3, PF_ERR_WORKSPACE = -4 };

enum pf_dtype { PF_F32 = 0, PF_BF16 = 1 };

enum pf_param_net { PF_PARAM_NONE = 0, PF_PARAM_CENTERED = 1 /* ParamNet @320x320 */, PF_PARAM_UNCENTERED = 2 /* ParamNetConvNextRegress @64x64 */ };

/* Model variant (the five yaml files of perspective2d/config/ reduce to these fields). */
typedef struct pf_model_desc {
  int gravity_classes;   /* 2 = regression (L2-normalised up-vector), 73 = classification logits            */
  int latitude_classes;  /* 1 = regression (clamped sin(latitude)),   180 = classification logits           */
  int param_net;         /* enum pf_param_net                                                               */
  int param_input_size;  /* MODEL.PARAM_DECODER.INPUT_SIZE for PF_PARAM_UNCENTERED (64)                     */
  float pixel_mean[3];   /* MODEL.PIXEL_MEAN, channel order of the input image (B, G, R)                    */
  float pixel_std[3];    /* MODEL.PIXEL_STD                                                                 */
} pf_model_desc;

/* One inference_batch call.  Exactly one of images_u8 / images_chw is non-NULL. */
typedef struct pf_batch {
  int n;                       /* number of images                                                          */
  /* uint8 path (PerspectiveFields.inference{,_batch}): DEVICE blob of tightly packed HWC uint8 BGR images   */
  const uint8_t* images_u8;
  const int64_t* image_offset; /* HOST [n] byte offset of each image in the blob                            */
  /* float path (PerspectiveFields.forward called directly): DEVICE fp32 [n,3,320,320], already resized      */
  const float* images_chw;
  const int32_t* height;       /* HOST [n] original heights ("height" key)                                  */
  const int32_t* width;        /* HOST [n] original widths  ("width" key)                                   */
  /* outputs, DEVICE, fp32 */
  float* pred_gravity;         /* [n, gravity_classes, 320, 320]                                            */
  float* pred_latitude;        /* [n, latitude_classes, 320, 320]                                           */
  float* gravity_original;     /* blob; image i occupies [2, H_i, W_i] at gravity_original_offset[i]        */
  const int64_t* gravity_original_offset;   /* HOST [n], in floats                                         */
  float* latitude_original;    /* blob; image i occupies [H_i, W_i] at latitude_original_offset[i]          */
  const int64_t* latitude_original_offset;  /* HOST [n], in floats                                         */
  float* params;               /* [n, 8]: roll, pitch, vfov|general_vfov (deg), rel_cx, rel_cy, rel_focal, raw x2, 0;
                                  may be NULL when param_net == PF_PARAM_NONE                               */
} pf_batch;

int pf_abi_version(void);
const char* pf_last_error(void);

/* Number of CUDA kernels launched by this library in the calling process so far (all handles). */
int64_t pf_kernel_launch_count(void);

/* Engine lifetime.  `device` is the CUDA ordinal; the engine makes it current for its own calls. */
int pf_create(int device, const pf_model_desc* desc, pf_handle* out);
/* The same at working size net_h x net_w (DATALOADER.RESIZE = [net_h, net_w]): multiples of 32 in [64, 640] with
 * (net_h/32) * (net_w/32) <= 256 (the attention key count of every MiT stage).  pf_forward then expects images_chw as
 * [n,3,net_h,net_w] and writes pred_gravity / pred_latitude as [n,C,net_h,net_w].  pf_create = pf_create_sized(.., 320, 320, ..). */
int pf_create_sized(int device, const pf_model_desc* desc, int net_h, int net_w, pf_handle* out);
int pf_destroy(pf_handle h);

/* Register one repacked weight tensor (DEVICE pointer, stays owned by the caller and must outlive the handle).
 * Names and layouts are listed in perspectivefields_b200/weights.py; pf_finalize checks that all are present. */
int pf_set_weight(pf_handle h, const char* name, const void* dev_ptr, int64_t numel, int dtype);
int pf_finalize(pf_handle h);

/* Bytes of DEVICE scratch pf_forward needs for a batch of n images whose largest member has max_h rows. */
int64_t pf_workspace_bytes(pf_handle h, int n, int max_h);

/* Whole forward of perspectivefields.py:223-272 for one batch, enqueued on `stream` (a cudaStream_t). */
int pf_forward(pf_handle h, const pf_batch* batch, void* workspace, int64_t workspace_bytes, void* stream);

/* ---- ParamNet on the caller's fields (param_network.py:46-69 ParamNet.forward, :193-221 ParamNetConvNextRegress.forward) -----
 * The ParamNet section of pf_forward (same kernels, same order, same results on the same fields) run on any fields at the
 * engine's working size net_h x net_w: gravity DEVICE float32 [n,2,net_h,net_w] up vectors, latitude [n,1,net_h,net_w]
 * sin(latitude), contiguous, used as given (no normalisation or clamp).  Outputs (DEVICE): params float32 [n,8] in the
 * pf_batch.params layout; raw float32 [n,5] (or NULL) = the ConvNeXt head's five outputs before any scaling, the prediction of
 * the reference's training branch (param_network.py:71-128, :223-241).  The option "bf16" applies as in pf_forward.  An engine
 * without a ParamNet, n < 1, NULL gravity / latitude / params / workspace, or a workspace smaller than
 * pf_param_workspace_bytes(h, n) is PF_ERR_ARG before anything is launched.  workspace: DEVICE, 256-byte aligned.  Enqueued on
 * `stream` without synchronisation. */
int64_t pf_param_workspace_bytes(pf_handle h, int n);
int pf_param_forward(pf_handle h, int n, const float* gravity, const float* latitude, float* params, float* raw, void* workspace,
                     int64_t workspace_bytes, void* stream);

/* ---- ParamNet training: gradients of a loss of the raw head outputs with respect to every ParamNet parameter --------------------
 * pf_param_train_forward is pf_param_forward's raw output (bit for bit) that also keeps, at the start of `workspace`, what the
 * backward needs: the packed input, the stem's output and the residual stream around every block (the rest is recomputed).
 * pf_param_backward then takes draw DEVICE float32 [n,5] = d loss / d raw and writes grads DEVICE float32 [pf_param_grad_numel()]
 * (overwritten, not accumulated): one tensor per parameter in the engine's weight layout, at the offsets pf_param_grad_entry
 * lists.  With grad_gravity [n,2,net_h,net_w] and grad_latitude [n,1,net_h,net_w] (both or neither) it also writes d loss / d
 * fields.  It must follow a pf_param_train_forward of the same engine, n and workspace on the same stream, with the workspace
 * untouched in between, and it needs the training weights registered with pf_set_weight (names "pn.ds<k>.t.whi/.wlo",
 * "pn.s<s>.b<j>.pw1t.whi/.wlo", ".pw2t.whi/.wlo" = the transposed weights, ".dw.wr" = the depthwise kernel rotated by 180 degrees,
 * "pn.zero" = 768 zeros), else PF_ERR_WEIGHT.  Parameter gradients are sums in a fixed order without atomics: repeated calls
 * are bit-identical.  The option "bf16" applies to every GEMM.  Bad arguments as for pf_param_forward (workspace: at least
 * pf_param_train_workspace_bytes(h, n)) are PF_ERR_ARG before anything is launched.  Enqueued on `stream` without
 * synchronisation. */
int64_t pf_param_train_workspace_bytes(pf_handle h, int n);
int pf_param_train_forward(pf_handle h, int n, const float* gravity, const float* latitude, float* raw, void* workspace,
                           int64_t workspace_bytes, void* stream);
int pf_param_backward(pf_handle h, int n, const float* draw, float* grads, float* grad_gravity, float* grad_latitude, void* workspace,
                      int64_t workspace_bytes, void* stream);
int64_t pf_param_grad_numel(void);
/* entry i of the gradient buffer: engine weight name ("pn.stem.w", "pn.s0.b0.pw1.w", ...), offset and length in floats */
int pf_param_grad_entry(int i, const char** name, int64_t* offset, int64_t* numel);

/* Per-launch timing of the GEMM engine with CUDA events on the launch stream (bench.py roofline leg).  pf_profile_read
 * fills out21[cfg*3 + {0,1,2}] = {milliseconds, algorithmic FLOPs (2*M*N*K), launches} per engine configuration (slots 0-4 are
 * unused since ABI 2 -- the earlier HMMA / register-staged engines were removed; 5: TMA+wgmma GEMM mode, 6: TMA+wgmma halo
 * 3x3 mode) accumulated since the previous read; synchronise the stream first. */
int pf_profile_enable(pf_handle h, int on /* 0 off, 1 on, n > 1: on + pre-create events for n GEMM launches */);
int pf_profile_read(pf_handle h, double* out21);
/* A CUDA-event pair around EVERY kernel launch of the forward graph: in-pipeline time per kernel (bench.py "per_kernel").
 * enable(max_launches > 0) pre-creates the events and starts recording, enable(0) stops.  read() writes a text table
 * "kernel,launches,ms\n..." (aggregated since the last read) into buf and returns its length; synchronise the stream first. */
int pf_profile_kernels_enable(pf_handle h, int max_launches);
int pf_profile_kernels_read(pf_handle h, char* buf, int cap);

/* Engine options (the whole graph runs on the persistent TMA -> wgmma engine with pre-split bf16 hi/lo activations,
 * gemm_tma.cuh); any other name is an error:
 * "pdl" (default 1): programmatic dependent launch of the graph's kernels (a kernel's prologue overlaps its predecessor's tail).
 * "decode_only" (default 0; classification heads, SURVEY.md 8f-3): the 73 / 180 logits are never written -- the 1x1 prediction
 *   conv, argmax and bin decode (gravity_head.py:243-244 + utils/utils.py:114-130, latitude_head.py:205-208 + utils.py:148-162)
 *   run in one kernel and pred_gravity / pred_latitude receive the decoded fields [n,2,320,320] / [n,1,320,320] (degrees).
 * "bf16" (default 0; NOT the reference's numerics, DESIGN.md section 3): every tensor-core product -- the TMA -> wgmma engine's
 *   GEMMs and 3x3 convolutions, the 7x7 stems and both products of the mma.sync attention core -- is one bf16 MMA of the
 *   operands' hi planes (bf16-rounded operands, fp32 accumulation) instead of the three of the split-precision scheme.  The
 *   CUDA-core kernels (LayerNorm, depthwise convolutions, resampling, softmax, prediction tails, the conv1 border ring, the
 *   ParamNet stem and tail) stay fp32.  Read at every launch: it can be switched between pf_forward calls on one handle. */
int pf_set_option(pf_handle h, const char* name, int value);

/* Debug taps (tests only): when enabled, intermediates of the next pf_forward (or pf_param_forward) are kept (never recycled) and can be
 * copied out by name (device-to-device, enqueued on `stream`).  Names are listed by pf_debug_name(i). */
int pf_debug_enable(pf_handle h, int on);
int pf_debug_count(pf_handle h);
const char* pf_debug_name(pf_handle h, int i);
int64_t pf_debug_numel(pf_handle h, const char* name);
int pf_debug_copy(pf_handle h, const char* name, float* dst_dev, int64_t numel, void* stream);

/* ---- camera parameters -> dense perspective fields (SURVEY.md 8f-1) -------------------------------------
 * Replaces PanoCam.get_up_general / PanoCam.get_lat_general (perspective2d/utils/panocam.py:451-513, :515-556), which callers
 * evaluate right after the inference path on ParamNet's output (utils/utils.py:367-385, demo/demo.py:69-78).  One launch per
 * 24 images; float64 arithmetic, float32 results.  No engine handle: the function has no weights. */
typedef struct pf_camera {
  int32_t height, width;        /* im_h, im_w */
  double focal_rel;             /* focal length / image height */
  double elevation, roll;       /* radians */
  double cx_rel, cy_rel;        /* principal point: pixel / size - 0.5 */
  int64_t up_offset;            /* float offset of this image's [H,W,2] (x,y) block in `up` */
  int64_t lat_offset;           /* float offset of this image's [H,W] block (degrees) in `lat` */
} pf_camera;
/* cams: HOST array of n descriptors; up / lat: DEVICE blobs (either may be NULL to skip that field). */
int pf_camera_fields(int device, const pf_camera* cams, int n, float* up, float* lat, void* stream);
/* The same, where vp (HOST [n][2] or NULL) may give image i a point (vp[2i], vp[2i+1]) in pixel-centre coordinates (pixel
 * (i, j) at (j + .5, i + .5)) that its up field points to instead of the one its elevation and roll imply: PanoCam.get_up
 * (panocam.py:385-448) at elevation 0, whose vanishing point lies 1e8 px away (:293-300).  NaN pairs keep the camera's own.
 * pf_camera_fields(..) = pf_camera_fields_vp(.., NULL, ..). */
int pf_camera_fields_vp(int device, const pf_camera* cams, const double* vp, int n, float* up, float* lat, void* stream);

/* ---- views of a panorama and their ground-truth fields -------------------------------------------------------------------
 * Replaces PanoCam.crop_distortion (perspective2d/utils/panocam.py:559-752) for a batch of views of ONE equirectangular panorama:
 * each view is a perspective (xi = 0) or Unified Spherical Model (xi > 0) camera of size H x W, focal length f (pixels) and
 * rotation rot_az * rot_roll^T * rot_el (degrees).  Geometry in float64 in the reference's order of operations, float32 fields.
 * The crop is a bilinear sample of the panorama (columns wrap, rows clamp, float64 weights, truncated to uint8; DESIGN.md
 * section 5), 0 outside the catadioptric disk when xi > 1 and f < fmin.  One launch per 12 views; no engine handle, no
 * synchronisation: offset / status are written on the device. */
typedef struct pf_pano_view {
  int32_t height, width;        /* H, W of the view */
  double f, xi;                 /* focal length in pixels (> 0), mirror parameter */
  double az, el, roll;          /* degrees */
  int64_t im_offset;            /* byte offset of this view's [H,W,3] crop in `im` (the layout of pf_batch.images_u8) */
  int64_t field_offset;         /* float offset of this view's [H,W] blocks in ntheta / nphi / lat; its [H,W,2] blocks in up / xy
                                   start at 2 * field_offset */
} pf_pano_view;
/* pano: DEVICE uint8 [pano_h, pano_w, 3] HWC (pano_h, pano_w >= 2); views: HOST array of n descriptors.  Outputs, DEVICE, each
 * may be NULL to skip it (at least one must be given):
 *   im uint8 crops (RGB order of the panorama);  ntheta, nphi, lat float32 [H,W] radians (lat == nphi);
 *   up float32 [H,W,2] normalised up-vector field;  xy float32 [H,W,2] (x, y) panorama pixel of every view pixel;
 *   offset double [n]: horizon row at column W / 2 (nan when nphi does not change sign there);
 *   status int32 [n]: 0 one zero crossing or none, 1 several (the reference prints a WARNING and uses the first), 2 one of the
 *   reference's assertions fails (e.g. an upside-down camera; offset is nan).
 * Every argument is checked before anything is launched (PF_ERR_ARG). */
int pf_pano_views(int device, const uint8_t* pano, int pano_h, int pano_w, const pf_pano_view* views, int n, uint8_t* im, float* ntheta,
                  float* nphi, float* up, float* lat, float* xy, double* offset, int32_t* status, void* stream);

/* ---- pinhole views of a panorama ----------------------------------------------------------------------------------------------
 * Replaces PanoCam.crop_equi and the crop of PanoCam(path).get_image (perspective2d/utils/panocam.py:121-249; equilib's equi2pers
 * there) for a batch of views of ONE equirectangular panorama.  A view of width W has fov_x = 2 atan(tan(vfov / 2) ar) and focal
 * length W / (2 tan(fov_x / 2)); it is rotated by roll, then elevation, then azimuth, and sampled by the rule of DESIGN.md
 * section 1 (float64 geometry; bilinear: columns wrap, rows clamp, float64 weights).  One launch per 24 views; no engine handle, no
 * synchronisation. */
typedef struct pf_equi_view {
  int32_t height, width;        /* im_h, im_w of the view */
  double vfov;                  /* vertical field of view, degrees, in (0, 180) */
  double azimuth, elevation, roll;   /* degrees */
  double ar;                    /* aspect ratio the field of view is widened by (> 0; fov_x must stay below 180 degrees) */
  int64_t offset;               /* byte offset of this view's [H,W,C] crop in `im` (a multiple of the element size) */
} pf_equi_view;
enum pf_equi_dtype { PF_EQUI_U8 = 0, PF_EQUI_F32 = 1 };
enum pf_equi_mode { PF_EQUI_BILINEAR = 0, PF_EQUI_NEAREST = 1 };
/* PF_EQUI_CAST: the sample rounded to float32, then cast to the panorama's dtype (uint8: truncated), crop_equi's
 * np.asarray(.., dtype=equi_img.dtype).  PF_EQUI_UNIT (uint8 panoramas only): get_image's path, the sample of p / 255 in float32
 * (ToTensor), rounded to float32, times 255 in float32 and truncated to uint8 (ToPILImage). */
enum pf_equi_out { PF_EQUI_CAST = 0, PF_EQUI_UNIT = 1 };
/* pano: DEVICE [pano_h, pano_w, channels] HWC (channels 1 or 3) of dtype enum pf_equi_dtype; views: HOST array of n descriptors;
 * mode: enum pf_equi_mode; out_kind: enum pf_equi_out; swap_rb: 1 writes channels in the order 2, 1, 0 (BGR from an RGB panorama,
 * 3 channels only); im: DEVICE blob of crops in the output dtype (float32 for a float32 panorama, uint8 otherwise).  Every
 * argument is checked before anything is launched (PF_ERR_ARG). */
int pf_equi_views(int device, const void* pano, int pano_h, int pano_w, int channels, int dtype, const pf_equi_view* views, int n, int mode,
                  int out_kind, int swap_rb, void* im, void* stream);

/* ---- perspective-field overlays (draw_perspective_fields / draw_up_field / draw_latitude_field, utils/utils.py:165-430) -----
 * Draws the latitude contours (18 filled bands and 19 lines of linspace(-pi/2, pi/2, 19), seismic colours) and the up-vector
 * arrows (quiver on the lattice arange(0, W, W // density) x arange(0, H, H // density), length up * (sqrt(W^2 + H^2) //
 * arrow_inv_len)) over an RGB image, 4 x 4 samples per pixel, by the rule of DESIGN.md section 1 (parity with matplotlib
 * unpinned).  Order: fill, arrows, lines.  One launch per 24 canvases; no engine handle, no synchronisation. */
typedef struct pf_draw_canvas {
  int32_t height, width;        /* H, W of the canvas (H * W < 2^31) */
  int64_t img_offset;           /* byte offset of the input uint8 [H,W,3] RGB canvas in `img` */
  int64_t out_offset;           /* byte offset of the output [H,W,3] in `out` (may be the input itself; no partial overlap) */
  int64_t lat_offset;           /* float offset of the [H,W] latitude map (radians, row-major) in `lat`; -1 when draw_lat is 0 */
  int64_t up_offset;            /* float offset of the up field's element (0, 0, x) in `up`; -1 when draw_up is 0 */
  int64_t up_stride[3];         /* element strides (>= 0) of the up field: row, column, component ([2,H,W]: W, 1, H*W;  [H,W,2]: 2W, 2, 1) */
  int32_t density;              /* arrows every W // density columns and H // density rows (both >= 1) */
  int32_t arrow_inv_len;        /* arrow length = up * (sqrt(W^2 + H^2) // arrow_inv_len), >= 1 */
  float arrow_rgb[3];           /* arrow colour, [0, 1] */
  float alpha_fill, alpha_line; /* contourf / contour alpha, [0, 1] */
  int32_t draw_lat, draw_up;    /* 0 / 1: draw the latitude fill and lines / the arrows */
} pf_draw_canvas;
/* canvases: HOST array of n descriptors; img / out: DEVICE uint8 blobs; lat / up: DEVICE float blobs (NULL when no canvas
 * draws them).  Every argument is checked before anything is launched (PF_ERR_ARG). */
int pf_draw_fields(int device, const pf_draw_canvas* canvases, int n, const uint8_t* img, uint8_t* out, const float* lat, const float* up,
                   void* stream);

/* ---- scoring against ground-truth perspective fields (csrc/metrics.cuh) -------------------------------------------------
 * Targets of the heads' losses from ground-truth fields at one size H x W, for n images.  up: DEVICE float32 (x, y) vectors
 * at up + b*s[0] + y*s[1] + x*s[2] (+ s[3] for y), up_stride = s (elements); lat: DEVICE float32 at lat + b*t[0] + y*t[1] + x*t[2],
 * degrees (lat_rad 0) or radians (1).  Either may be NULL (that output is skipped).
 *   gravity_classes 2: gt_gravity = float32 [n, 2, H, W] copy of the up field; >= 3: int64 [n, H, W] labels of
 *     encode_bin(up, gravity_classes) (utils/utils.py:94-111).
 *   latitude_classes 1: gt_latitude = float32 [n, 1, H, W] sin(latitude); >= 2: int64 [n, H, W] labels of
 *     encode_bin_latitude(latitude in degrees, latitude_classes) (utils/utils.py:133-146). */
int pf_encode_fields(int device, int n, int H, int W, const float* up, const int64_t* up_stride, const float* lat, const int64_t* lat_stride,
                     int lat_rad, int gravity_classes, int latitude_classes, void* gt_gravity, void* gt_latitude, void* stream);
/* The heads' losses dicts (persformer_heads.py:60-70) over a batch of n predictions at H x W, into DEVICE float32 losses:
 *   regression (2 / 1): pred_gravity / gt_gravity float32 [n, 2, H, W], pred_latitude / gt_latitude [n, 1, H, W] ->
 *     losses[4] = gravity-msg-normal-loss, gravity-l2-loss, latitude-msg-normal-loss, latitude-l2-loss (gravity_head.py:204-218,
 *     latitude_head.py:225-237);
 *   classification (>= 3 / >= 2): logits float32 [n, C, H, W] (16-byte aligned, H * W % 4 == 0), labels int64 [n, H, W] ->
 *     losses[2] = loss_gravity, loss_latitude (cross-entropy, mean over the labels that are not the head's ignore value).
 * Every value is multiplied by its head's weight.  A mean over no pixel is NaN, and so is a cross-entropy with a label outside
 * [0, C) that is not the ignore value.  workspace: DEVICE, 256-byte aligned, pf_head_losses_workspace bytes. */
int64_t pf_head_losses_workspace(int n, int H, int W, int gravity_classes, int latitude_classes);
int pf_head_losses(int device, int n, int H, int W, int gravity_classes, const float* pred_gravity, const void* gt_gravity, int latitude_classes,
                   const float* pred_latitude, const void* gt_latitude, int gravity_ignore, int latitude_ignore, float gravity_weight,
                   float latitude_weight, float* losses, void* workspace, int64_t workspace_bytes, void* stream);
/* Per-image errors of predicted fields at the original sizes (DESIGN.md section 1).  Offsets and strides are in elements
 * relative to the base pointers (mask: bytes; -1 = no mask); latitudes are [H, W] row-major, the mask uint8 [H, W]. */
typedef struct pf_field_image {
  int32_t height, width;
  int64_t pred_up_offset, pred_up_stride[3];   /* row, column, component */
  int64_t pred_lat_offset;                     /* degrees */
  int64_t gt_up_offset, gt_up_stride[3];
  int64_t gt_lat_offset;                       /* degrees or radians (lat_rad) */
  int64_t mask_offset;
} pf_field_image;
/* Outputs (DEVICE), field f = 0 (up, degrees between vectors) or 1 (latitude, absolute difference in degrees) of image i at
 * f * n + i: count int64, mean and median float64 (NaN for count 0), fraction float64 [2, n, n_thresholds] of valid pixels with
 * an error below each threshold (at most 8).  up_maps / lat_maps: DEVICE float32 blobs of the per-pixel errors (images one
 * after the other, NaN at invalid pixels), or both NULL.  workspace: DEVICE, 256-byte aligned, pf_field_errors_workspace bytes. */
int64_t pf_field_errors_workspace(const pf_field_image* images, int n, int with_maps);
int pf_field_errors(int device, const pf_field_image* images, int n, const float* pred_up, const float* pred_lat, const float* gt_up,
                    const float* gt_lat, const uint8_t* mask, int lat_rad, const double* thresholds, int n_thresholds, float* up_maps,
                    float* lat_maps, int64_t* count, double* mean, double* median, double* fraction, void* workspace,
                    int64_t workspace_bytes, void* stream);

/* ---- camera parameters from perspective fields (csrc/calib.cuh) ------------------------------------------------------------
 * A Levenberg-Marquardt fit of roll, pitch, f_rel and (principal_point != 0) cx_rel, cy_rel to predicted fields, one camera
 * per image (DESIGN.md section 1, "Camera fit").  Offsets and strides are in elements relative to the base pointers (mask:
 * bytes; -1 = no mask).  up: float32 (x, y) vectors at up_base + up_offset + y*s[0] + x*s[1] (+ s[2] for y), so [2, H, W]
 * predictions and [H, W, 2] camera fields are read in place; lat: float32 [H, W] row-major, degrees; mask: uint8 [H, W].
 * init: the start (roll, pitch in radians, f_rel > 0, cx_rel, cy_rel; the last two are ignored without principal_point), or a
 * NaN roll for the closed-form start from the fields. */
typedef struct pf_fit_image {
  int32_t height, width;                       /* >= 3 each */
  int64_t up_offset, up_stride[3];             /* row, column, component */
  int64_t lat_offset;
  int64_t mask_offset;
  double init[5];
} pf_fit_image;
/* Outputs (DEVICE), image i: params[5i .. 5i + 4] = roll (degrees, (-180, 180]), pitch (degrees, |pitch| <= 90), f_rel, cx_rel,
 * cy_rel (0 without principal_point); cost[i] = 1/2 sum delta^2 rho((r / delta)^2) at them (huber = delta > 0: Huber's rho;
 * huber = 0: least squares, rho(z) = z), with residuals in radians; iterations[i] = cost evaluations; status[i] = 0 converged,
 * 1 stopped at max_iterations (1 .. 1000) evaluations, 2 fewer valid residuals than parameters (params and cost NaN).
 * Enqueued on `stream` without synchronisation.  workspace: DEVICE, 256-byte aligned, pf_fit_camera_workspace bytes. */
int64_t pf_fit_camera_workspace(const pf_fit_image* images, int n);
int pf_fit_camera(int device, const pf_fit_image* images, int n, const float* up_base, const float* lat_base, const uint8_t* mask_base,
                  int principal_point, double huber, int max_iterations, double* params, double* cost, int32_t* iterations,
                  int32_t* status, void* workspace, int64_t workspace_bytes, void* stream);

/* ---- upright warp: straightened images from camera parameters (csrc/rectify.cuh) --------------------------------------------
 * Warps each uint8 image (1 or 3 channels, HWC) to a camera with roll 0, pitch 0 (or the input pitch with keep_pitch), a centred
 * principal point and the focal length of enum pf_rectify_focal, by the rule of DESIGN.md section 1 ("Upright warp").  Offsets are
 * relative to the base pointers: bytes for the images and the mask, floats for the map; -1 skips that image's mask / map. */
typedef struct pf_rectify_image {
  int32_t height, width;            /* input size */
  int32_t out_height, out_width;    /* output size */
  int64_t in_offset;                /* bytes of the [height, width, channels] input in in_base */
  int64_t out_offset;               /* bytes of the [out_height, out_width, channels] output in out_base */
  int64_t mask_offset;              /* bytes of the uint8 [out_height, out_width] mask (1: sampled, 0: fill) in mask_base, or -1 */
  int64_t map_offset;               /* floats of the float32 [out_height, out_width, 2] input positions in map_base, or -1 */
} pf_rectify_image;
/* PF_RECTIFY_SAME: f_rel * out_height; PF_RECTIFY_VFOV: out_height / (2 tan(vfov / 2)); PF_RECTIFY_FILL: the smallest focal length
 * >= the SAME one that keeps the four canvas corners inside the input (status 1 and the SAME focal length when none can). */
enum pf_rectify_focal { PF_RECTIFY_SAME = 0, PF_RECTIFY_VFOV = 1, PF_RECTIFY_FILL = 2 };
enum pf_rectify_sampler { PF_RECTIFY_BILINEAR = 0, PF_RECTIFY_NEAREST = 1 };
/* images: HOST array of n (1 .. 65535) descriptors.  params: DEVICE float64 [n, 5] = roll, pitch, general vfov (degrees),
 * cx_rel, cy_rel per image, read on the device (no synchronisation).  fill: HOST int32 [channels] in 0 .. 255, or NULL for 0.
 * Outputs (DEVICE): the images, the optional masks and maps (input pixel-centre positions (x, y), NaN where not sampled),
 * camera float64 [n, 5] (the output camera in the form of params) and status int32 [n] (0 ok, 1 PF_RECTIFY_FILL impossible, 2
 * unusable parameters: the image is all fill, mask 0, map and camera NaN).  workspace: DEVICE, 256-byte aligned,
 * pf_rectify_workspace bytes.  Every argument is checked before anything is launched (PF_ERR_ARG). */
int64_t pf_rectify_workspace(const pf_rectify_image* images, int n);
int pf_rectify_views(int device, const pf_rectify_image* images, int n, const uint8_t* in_base, uint8_t* out_base, uint8_t* mask_base,
                     float* map_base, int channels, const double* params, int keep_pitch, int focal_mode, double vfov, int sampler,
                     const int32_t* fill, double* camera, int32_t* status, void* workspace, int64_t workspace_bytes, void* stream);

/* ---- multi-GPU gather of results (SURVEY.md 8e: one process per GPU; NCCL point-to-point over NVLink) ---------------------
 * inference_batch shards its list over the ranks; the per-image results live on each rank's device and are gathered to ONE
 * rank with grouped ncclSend / ncclRecv enqueued on the caller's stream (so that the gather of micro-batch k overlaps the
 * forward of micro-batch k+1 when issued on a side stream).  NCCL is resolved at run time from the process
 * (libnccl.so.2 -- the one PyTorch ships); the 128-byte unique id is created on rank 0 and distributed by the caller
 * (torch.distributed / MPI / a file: plumbing). */
typedef struct pf_comm* pf_comm_handle;
int pf_comm_unique_id(void* id128);                                              /* rank 0: ncclGetUniqueId -> 128 bytes */
int pf_comm_create(int device, int rank, int nranks, const void* id128, pf_comm_handle* out);
int pf_comm_destroy(pf_comm_handle c);
/* One grouped exchange.  On every rank != root: send `count` segments (DEVICE pointer, bytes) to root.  On root: receive
 * `count` segments, segment i from rank peer[i].  All segments of one call travel in one ncclGroup on `stream`. */
int pf_gather(pf_comm_handle c, int root, int count, void* const* dev_ptrs, const int64_t* bytes, const int32_t* peer, void* stream);

/* ---- decode front-end (SURVEY.md 8f-2): JPEG bytes -> the device blob of BGR uint8 HWC images pf_forward reads ---------
 * Replaces `cv2.imread` in front of the path (demo/demo.py:151) with nvJPEG (bound at run time), the images of a batch fanned out
 * over worker threads / streams and joined into `stream`.  pf_jpeg_info parses the header only (sizes for the blob layout). */
typedef struct pf_jpeg* pf_jpeg_handle;
int pf_jpeg_create(int device, int max_threads /* 0 = half the host's hardware threads, at most 32 */, pf_jpeg_handle* out);
int pf_jpeg_destroy(pf_jpeg_handle j);
int pf_jpeg_info(pf_jpeg_handle j, const uint8_t* data, int64_t length, int32_t* height, int32_t* width);
/* data[i] / length[i]: HOST JPEG streams; blob: DEVICE; image i is written as [height[i], width[i], 3] BGR at byte offset[i]. */
int pf_jpeg_decode_batch(pf_jpeg_handle j, int n, const uint8_t* const* data, const int64_t* length, const int32_t* height,
                         const int32_t* width, uint8_t* blob, const int64_t* offset, void* stream);

/* ---- single-operator entry points (unit tests; the same kernels pf_forward launches) -------------------- */

/* Conv / linear on NHWC fp32 on the TMA -> wgmma engine, bf16x3 split precision (the input is split into hi/lo planes first,
 * as a producer kernel of the forward graph would; 3x3/s1/p1 with Cin % 64 == 0 -> halo mode, 1x1 -> GEMM mode, else patch gather).  x: [B,H,W,Cin]; whi/wlo: bf16 [N][KH*KW*Cin]
 * ordered (ky,kx,ci); bias: [N] or NULL; res: [B,OH,OW,N] or NULL; y: [B,OH,OW,N].
 * y = act(conv(relu_in?(x)) + bias) (+ relu_res?(res));  act: 0 none, 1 ReLU, 2 GELU. */
int pf_op_conv_gemm(const float* x, int B, int H, int W, int Cin, const void* whi, const void* wlo, const float* bias,
                    int N, int KH, int KW, int stride, int pad, int in_relu, int act, const float* res, int res_relu,
                    float* y, void* stream);
/* One launch of the TMA -> wgmma engine with every epilogue feature the forward graph uses, on operands the caller has already
 * split into bf16 hi/lo planes (DEVICE pointers).  Runs the forward's own helpers (map construction, tile dispatch, the
 * per-group launch split), so a test reaches exactly what pf_forward launches.  Enqueued on `stream`, no synchronisation.
 *   mode 0 (GEMM): C[M, N] = A[M, K] W[N, K]^T, one group; A rows of pitch lda, first column a_c0.
 *   mode 1 (halo): 3x3 / stride 1 / pad 1 convolution of NHWC [B, H, W, lda] planes, Cin (multiple of 64) channels per group
 *     starting at a_c0 + g * a_gc; with a2_hi / a2_lo, input channels >= c_split come from A2 (pitch lda2) at a2_c0 + (ci - c_split),
 *     the same for every group.  W: [groups * N][9 * Cin], K ordered (ky, kx, ci).
 * Epilogue per output row m and column n of group g:
 *   v = acc + bias[g * bias_gstride + cls * N + n]  (bias_mode 1: cls = 0; 2: border class (ry * 3 + rx), halo mode, H, W >= 2)
 *   v = act(v) (0 none, 1 ReLU, 2 GELU);  v *= gamma[n];  v += relu?(res[m * ldr + r_coff + g * r_gcoff + n]);
 *   v += res2[m * ldr2 + r2_coff + g * r2_gcoff + n]
 *   C[m * ldc + c_coff + g * c_gcoff + n] = v;  S planes at m * lds + s_coff + g * s_gcoff + n = split(relu?(v)) (split_relu).
 * phase4 (halo mode, N = 128): column 32 ph + c is channel c of output pixel (2y + ph / 2, 2x + ph % 2) of a 2H x 2W grid.
 * pred[g] (halo mode, npred = groups): fused 1x1 conv 32 -> nc + normalise (mode 1) / clamp (mode 2), NCHW into pred[g].out.
 * force_bn / force_kb: run this instantiation instead of the dispatcher's (0 = its choice); a pair the engine does not
 * instantiate, or cannot run this problem with, is PF_ERR_ARG before anything is launched.  picked_bn / picked_kb: what ran.
 * force_sched (GEMM mode): 0 = the dispatcher's schedule, 1 = cooperative (128-row tiles), 2 = ping-pong (64-row tiles, one
 * MMA warpgroup's epilogue overlapping the other's main loop); picked_sched: what ran (1 / 2; 0 in halo mode).  Every
 * schedule gives bit-identical results. */
typedef struct pf_tma_pred { const float* w; const float* b; float* out; int nc, mode; } pf_tma_pred;
typedef struct pf_tma_op {
  int mode;
  int64_t M; int K;
  int B, H, W, Cin;
  int N, groups;
  const void* a_hi; const void* a_lo; int lda, a_c0, a_gc;
  const void* a2_hi; const void* a2_lo; int lda2, c_split, a2_c0;
  const void* w_hi; const void* w_lo; const float* bias; int bias_mode, bias_gstride;
  int act; const float* gamma;
  const float* res; int ldr, r_coff, r_gcoff, res_relu;
  const float* res2; int ldr2, r2_coff, r2_gcoff;
  float* C; int ldc, c_coff, c_gcoff;
  void* s_hi; void* s_lo; int lds, s_coff, s_gcoff, split_relu;
  int phase4;
  int npred; pf_tma_pred pred[2];
  int force_bn, force_kb;
  int picked_bn, picked_kb;   /* out */
  int force_sched, picked_sched;
} pf_tma_op;
int pf_op_tma(pf_tma_op* op, void* stream);
/* pf_op_tma in the bf16 precision mode (option "bf16"): the same struct, semantics and tile override, with one bf16 MMA per
 * product (A_hi * W_hi^T; a_lo / w_lo must still be valid pointers and are not read).  Split outputs still get both planes. */
int pf_op_tma_bf16(pf_tma_op* op, void* stream);
/* The border ring of the phase-composed conv_fuse_conv1 (the two outermost rows / columns of the 2H x 2W output, H, W >= 2),
 * recomputed in fp32 as pf_forward does after the phase4 launch: c_hi / c_lo: split planes [B, H, W, 128] (head 0 channels
 * 0-63, head 1 64-127); wf: fp32 [2][9 taps][64 ci][32 o]; bias [2][32]; out: NHWC [B, 2H, 2W, 64] or NULL; with pg_w the
 * prediction tails of both heads (pg_*: gravity, 2 channels, normalised; pl_*: latitude, 1 channel, clamped; NCHW). */
int pf_op_conv1_ring(const void* c_hi, const void* c_lo, int B, int H, int W, const float* wf, const float* bias, float* out,
                     const float* pg_w, const float* pg_b, float* pg_out, const float* pl_w, const float* pl_b, float* pl_out, void* stream);
/* Host only, no device needed: the (bn, kb) the engine's dispatcher picks for a launch (mode 0 GEMM with M rows; mode 1 halo:
 * K = 9 * Cin) on a device with sm_count SMs. */
int pf_tma_pick_tile(int mode, int64_t M, int N, int K, int sm_count, int* bn, int* kb);
/* ParamNet training's backward, one piece at a time, through the host helper pf_param_backward runs it with (same partition,
 * same reduction order).  DEVICE pointers; scratch is allocated, sized by a dry run and filled with NaN bytes, inside the call,
 * which ends with a stream synchronisation.  Every argument is checked before anything is launched (PF_ERR_ARG).
 *   pn_wgrad: out[N][K] = sum over r < R of dy[r * ldy + n] * X[r][k], X = x (fp32, row pitch ldx; op 1: GELU(x)) or
 *     x_hi + x_lo (split planes, pitch ldx, op 0), on the GEMM engine as S grouped row chunks of `chunk` rows; S and chunk out.
 *   pn_colsum: out[c] = sum over r of src[r * C + c].
 *   pn_ln_bwd: LayerNorm (eps 1e-6) backward over rows of C channels (a multiple of 32, <= 768): dx written, d weight at g,
 *     d bias at g + C.
 *   pn_dw7_bwd: depthwise 7x7 (pad 3) on NHWC [B, H, W, C] (C a multiple of 32): dw [50][C] (49 taps (ky, kx), then the bias)
 *     from x and dt = d output; dx = d input (the forward kernel with w_rot, the kernel rotated by 180 degrees, [49][C]).
 *   pn_stem_bwd: 4x4 / stride 4 stem on pin [B, 4 OH, 4 OW, 4] (channel 3 unused) from dS [B, OH, OW, 96]: dw [49][96]
 *     ((ky, kx, ci) rows, then the bias); dpin channels 0-2 from w [48][96] (channel 3 is not written).
 *   rows_per_block (may be NULL): image rows per partial sum of the weight-gradient kernel.
 *   pn_fields_grad: backward of the nearest resize [B, 3, IH, IW] -> dpin [B, OH, OW, 4]: dgrav [B, 2, IH, IW], dlat [B, 1, IH, IW].
 *   pn_tail_bwd: mean pool -> LayerNorm(768) -> Linear 768 -> 5 of feat [n, HW, 768] from draw [n, 5]: dx [n, HW, 768];
 *     grads: norm.w (768), norm.b (768), head.w (5 x 768), head.b (5).
 *   pn_pw2_grads: from G [C][K], sdy [C], gamma [C], W = w_hi + w_lo [C][K], b [C]: dW = gamma G, db = gamma sdy,
 *     dgamma = sum_k W G + b sdy.
 *   pn_gelu_bwd: u[i] = dh[i] * GELU'(u[i]) in place (exact erf), and its split planes when hi / lo are given.
 *   pn_scale_split: split planes of src [n / C][C] (times scale[c] when scale is not NULL).
 *   pn_col2im2: the 2 x 2 / stride 2 patch matrix dP [B * H/2 * W/2][4 C] back to [B, H, W, C] (H, W even). */
int pf_op_pn_wgrad(const float* dy, int ldy, const float* x, const void* x_hi, const void* x_lo, int op, int ldx, int64_t R, int N, int K,
                   float* out, int* S, int* chunk, void* stream);
int pf_op_pn_colsum(const float* src, int64_t R, int C, float* out, void* stream);
int pf_op_pn_ln_bwd(const float* x, const float* dy, int64_t R, int C, const float* w, float* dx, float* g, void* stream);
int pf_op_pn_dw7_bwd(const float* x, const float* dt, int B, int H, int W, int C, const float* w_rot, float* dw, float* dx, int* rows_per_block,
                     void* stream);
int pf_op_pn_stem_bwd(const float* pin, const float* dS, const float* w, int B, int OH, int OW, float* dw, float* dpin, int* rows_per_block,
                      void* stream);
int pf_op_pn_fields_grad(const float* dpin, int B, int IH, int IW, int OH, int OW, float* dgrav, float* dlat, void* stream);
int pf_op_pn_tail_bwd(const float* feat, int n, int HW, const float* nw, const float* nb, const float* hw, const float* draw, float* dx,
                      float* grads, void* stream);
int pf_op_pn_pw2_grads(const float* G, const float* sdy, int C, int K, const float* gamma, const void* w_hi, const void* w_lo, const float* b,
                       float* dW, float* db, float* dgamma, void* stream);
int pf_op_pn_gelu_bwd(const float* dh, float* u, int64_t n, void* hi, void* lo, void* stream);
int pf_op_pn_scale_split(const float* src, const float* scale, int64_t n, int C, void* hi, void* lo, void* stream);
int pf_op_pn_col2im2(const float* dP, int B, int H, int W, int C, float* out, void* stream);
int pf_op_layernorm(const float* x, float* y, int64_t rows, int C, const float* w, const float* b, float eps, void* stream);
int pf_op_attention_tc(const float* q, const float* kv, float* out, int B, int N, int C, int heads, void* stream);   /* q / kv split into bf16 hi/lo planes first, then the mma.sync core as the forward graph runs it */
int pf_op_attention_tc_bf16(const float* q, const float* kv, float* out, int B, int N, int C, int heads, void* stream); /* the same in the bf16 precision mode: one mma.sync per product on bf16(q), bf16(k), bf16(P), bf16(v) */
/* pf_op_attention_tc / _bf16 (bf16 != 0) with NKV keys per image (kv: [B,NKV,2C]), 1..256: 100 runs the 320 x 320 kernel, other
 * counts up to 112 the single-block kernel with a run-time count, larger ones the key-block (online-softmax) kernel */
int pf_op_attention_tc_keys(const float* q, const float* kv, float* out, int B, int N, int NKV, int C, int heads, int bf16, void* stream);
int pf_op_dwconv3x3_gelu(const float* x, float* y, int B, int H, int W, int C, const float* w9c, const float* bias, void* stream);
int pf_op_dwconv7x7(const float* x, float* y, int B, int H, int W, int C, const float* w49c, const float* bias, void* stream);
int pf_op_upsample2x(const float* x, float* y, int B, int H, int W, int C, void* stream);
/* The forward graph's CUDA-core kernels one launch at a time, each through the host helper pf_forward launches it with (same
 * grid, block and arguments); pf_op_layernorm, pf_op_dwconv3x3_gelu, pf_op_dwconv7x7 and pf_op_upsample2x above go the same
 * way.  DEVICE pointers; the call ends with a stream synchronisation.  Every argument is checked before anything is launched
 * (PF_ERR_ARG), including shapes whose indices would leave the 32-bit range the kernel computes them in.  Pointers read or
 * written 16 bytes at a time (NHWC activations, split planes, weights of the depthwise convs) must be 16-byte aligned.  A split
 * output is a pair of bf16 planes hi / lo with hi + lo = the fp32 result (hi = its round-to-nearest-even bf16).
 *   layernorm_ex: LayerNorm over rows of C channels (a multiple of 4 up to 768) into any non-empty set of y (fp32), hi / lo (split,
 *     row order) and phi / plo (split, the im2col order of a k = s = sr convolution on RH x RW maps: token (b, y, x) goes to row
 *     (b, y / sr, x / sr), columns ((y % sr) sr + x % sr) C ..; RH, RW multiples of sr, rows a multiple of RH RW).
 *   dwconv3x3_gelu_ex: depthwise 3x3 (pad 1) + bias + GELU on NHWC [B, H, W, C] into y and / or hi / lo.
 *   upsample2x_ex: x2 bilinear upsample of channels icoff .. icoff + C - 1 of [B, H, W, ldi] into channels ocoff .. of
 *     [B, 2H, 2W, ldo], as y and / or hi / lo (pitch ldo); all four multiples of 4.
 *   stem_gather: the 7 x 7 / stride (2 or 4) / pad 3 patch matrix of channels 0-2 of x0 [B, IH, IW, 4] as split planes
 *     [B * OH * OW][160], columns (ky, kx, c), 147 .. 159 zero; OH = (IH - 1) / stride + 1, OW likewise.
 *   pn_stem: ParamNet stem conv 4 x 4 / 4 + bias of channels 0-2 of pin [B, SH, SW, 4] -> [B, SH / 4, SW / 4, 96]; w [(ky, kx, ci)][96].
 *   pack_fields: up fields [B, 2, IH, IW] and latitude [B, 1, IH, IW] nearest-resampled to [B, OH, OW, 4] (channel 3 zero).
 *   param_tail: ParamNet tail of feat [n, HW, 768]: mean pool, LayerNorm (eps 1e-6; nw, nb), Linear 768 -> 5 (hw [5][768], hb),
 *     parameter scaling of kind PF_PARAM_CENTERED / PF_PARAM_UNCENTERED into params [n][8] (pf_batch.params); raw [n][5] may be NULL.
 *   pred_tail: 1x1 conv 32 -> NC (w [NC][32], b [NC]) of channels coff .. coff + 31 of feat [B * HW, ld] -> NCHW out [B, NC, HW];
 *     mode 0 raw, 1 F.normalize over 2 channels (NC = 2), 2 clamp to [-1, 1]; NC <= 256. */
int pf_op_layernorm_ex(const float* x, float* y, void* hi, void* lo, void* phi, void* plo, int64_t rows, int C, const float* w, const float* b,
                       float eps, int RH, int RW, int sr, void* stream);
int pf_op_dwconv3x3_gelu_ex(const float* x, int B, int H, int W, int C, const float* w9c, const float* bias, float* y, void* hi, void* lo, void* stream);
int pf_op_upsample2x_ex(const float* x, int ldi, int icoff, float* y, int ldo, int ocoff, void* hi, void* lo, int B, int H, int W, int C, void* stream);
int pf_op_stem_gather(const float* x0, int B, int IH, int IW, int stride, void* hi, void* lo, void* stream);
int pf_op_pn_stem(const float* pin, int B, int SH, int SW, const float* w, const float* b, float* out, void* stream);
int pf_op_pack_fields(const float* grav, const float* lat, int B, int IH, int IW, int OH, int OW, float* out, void* stream);
int pf_op_param_tail(const float* feat, int n, int HW, const float* nw, const float* nb, const float* hw, const float* hb, int kind, float* params,
                     float* raw, void* stream);
int pf_op_pred_tail(const float* feat, int ld, int coff, const float* w, const float* b, float* out, int B, int HW, int NC, int mode, void* stream);
/* Pillow-exact resize + normalise of ONE uint8 HWC image -> [320,320,4] fp32 (b,g,r,0). */
int pf_op_preprocess(const uint8_t* img_dev, int H, int W, const float* mean3, const float* std3, float* y, void* stream);
/* the same to [net_h,net_w,4] (a working size pf_create_sized accepts) */
int pf_op_preprocess_sized(const uint8_t* img_dev, int H, int W, int net_h, int net_w, const float* mean3, const float* std3, float* y, void* stream);
/* ResizeTransform.apply_image (perspectivefields.py:34-67) on the device, HWC in -> HWC out, C channels:
 *   uint8 (PIL branch, :38-46): Pillow-exact antialiased bilinear (the same integer kernel as pf_forward's pre-process);
 *   float32 (:47-66): F.interpolate(mode="bilinear", align_corners=False), no antialias. */
int pf_op_resize_u8(const uint8_t* img_dev, int H, int W, int new_h, int new_w, uint8_t* out_dev, void* stream);   /* C = 3 */
int pf_op_resize_f32(const float* img_dev, int H, int W, int C, int new_h, int new_w, float* out_dev, void* stream);
/* write-only bandwidth probe: fills dst[numel] (numel % 4 == 0, 16-byte aligned) with 16-byte streaming stores (bench.py measures
 * the store roofline of the write-out kernels with it). */
int pf_op_fill_stream(float* dst, int64_t numel, float value, void* stream);
/* argmax over channels + bin decode of NCHW logits [B,NC,HW] (gravity_head.py:243-244 + utils/utils.py:114-130 when
 * is_gravity, field [B,2,HW]; latitude_head.py:205-208 + utils/utils.py:148-162 otherwise, field [B,1,HW] in degrees). */
int pf_op_argmax_decode(const float* logits, float* field, int B, int HW, int NC, int is_gravity, void* stream);
/* the same decode WITHOUT materialised logits (option "decode_only"): 1x1 conv 32 -> NC on feat [B*HW, ld] (channels coff..coff+31,
 * weights [NC][32], bias [NC]) + argmax + bin decode in one kernel; logits bit-identical to the separate 1x1 conv kernel. */
int pf_op_pred_argmax_decode(const float* feat, int ld, int coff, const float* w, const float* bias, float* field, int B, int HW, int NC,
                             int is_gravity, void* stream);
/* resample of decoded fields to the original sizes (gravity_head.py:246-256, latitude_head.py:209-219, utils/utils.py:483-507):
 * vec [n,2,320,320], lat [n,1,320,320] -> blobs as in pf_batch; lat_is_sin: lat holds sin(latitude) (regression head). */
int pf_op_postprocess(const float* vec, const float* lat, int n, const int32_t* height, const int32_t* width,
                      float* gravity_original, const int64_t* gravity_original_offset, float* latitude_original,
                      const int64_t* latitude_original_offset, int lat_is_sin, void* stream);
/* the same from fields at the working size net_h x net_w: vec [n,2,net_h,net_w], lat [n,1,net_h,net_w] (crop to and scale by
 * the net size as gravity_head.py:248-256 does with image_size) */
int pf_op_postprocess_sized(const float* vec, const float* lat, int n, int net_h, int net_w, const int32_t* height, const int32_t* width,
                            float* gravity_original, const int64_t* gravity_original_offset, float* latitude_original,
                            const int64_t* latitude_original_offset, int lat_is_sin, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* PF_B200_H_ */
