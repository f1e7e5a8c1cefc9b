/*
 * whenet_b200.h - C ABI of the H100-native WHENet per-crop forward.
 *
 * The reference has no FFI of its own: its whole hot path is the Python class
 * in reference whenet.py (WHENet.__init__ :7-20, WHENet.get_angle :22-34,
 * self.model.predict :27) sitting on Keras/TensorFlow.  This header is the
 * boundary a host in any language binds instead of Keras; each entry point
 * cites the reference line(s) it replaces.  Plain C types only, no C++
 * exceptions cross it.  Every function returns 0 on success or a negative
 * WHENET_E* code; whenet_last_error() returns the message of the last failure
 * on the calling thread.
 *
 * A context is bound to one device and one stream and is NOT thread-safe
 * (the reference is single-threaded and synchronous as well: demo_video.py:49-63).
 * Use one context per GPU / per host thread.
 */
#ifndef WHENET_B200_H
#define WHENET_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define WHENET_OK              0
#define WHENET_EINVAL         -1   /* bad argument (NULL, n<1, n>max_batch, wrong shape)      */
#define WHENET_ECUDA          -2   /* a CUDA runtime/driver call failed (message has details) */
#define WHENET_ENOWEIGHTS     -3   /* forward called before whenet_load_weights               */
#define WHENET_ESHAPE         -4   /* a weight tensor is missing or has the wrong shape       */
#define WHENET_ENOTFOUND      -5   /* unknown tap / kernel name                               */

#define WHENET_PRECISION_FP32  0   /* fp32 storage + fp32 FMA: the parity mode                */
#define WHENET_PRECISION_BF16  1   /* bf16 activations, fp32 accumulate: the throughput mode  */
#define WHENET_PRECISION_FP16  2   /* fp16 activations, fp32 accumulate                       */

/* Planar YUV 4:2:0 video frames (the *_yuv_u8 entries): cv2's contiguous (H * 3/2) x W uint8 layout, H and W even - the
 * H x W Y plane, then for NV12 one (H/2) x W plane of interleaved U, V pairs (U first), for I420 the (H/2) x (W/2) U plane
 * followed by the (H/2) x (W/2) V plane.  Each pixel is converted as it is read with cv2.cvtColor's COLOR_YUV2BGR_NV12 /
 * COLOR_YUV2BGR_I420 arithmetic (BT.601 limited range, 20-bit fixed point), so every result is the bits the BGR entry gives
 * on cvtColor's output. */
#define WHENET_YUV_NV12        1
#define WHENET_YUV_I420        2
/* Packed YUV 4:2:2 frames (the *_yuv422_u8 entries, and whenet_yuv_to_bgr_*): H x W x 2 uint8, W even, any H, as cameras,
 * V4L2, GStreamer and HDMI capture cards hand them out.  Row y holds W/2 pixel pairs; pair p is the bytes Y0 U Y1 V (YUYV,
 * also called YUY2) or U Y0 V Y1 (UYVY) at 4p, and both pixels share its U and V.  The arithmetic is that of the 4:2:0
 * layouts: cv2.cvtColor's COLOR_YUV2BGR_YUYV / COLOR_YUV2BGR_UYVY. */
#define WHENET_YUV_YUYV        3
#define WHENET_YUV_UYVY        4

#define WHENET_IMG        224
#define WHENET_N_YAW      120      /* reference whenet.py:11 */
#define WHENET_N_PITCH     66      /* reference whenet.py:12 */
#define WHENET_N_ROLL      66      /* reference whenet.py:13 */
#define WHENET_N_LOGITS   252

typedef struct whenet_ctx whenet_ctx;

/* One named float32 tensor of the Keras weights file ("conv2d_1/kernel:0", ...),
 * row-major in the file's own layout (conv HWIO, depthwise [kh,kw,C,1], BN [C],
 * Dense [in,out]).  Borrowed for the duration of whenet_load_weights only. */
typedef struct {
    const char*  name;
    const float* data;
    int32_t      ndim;
    int64_t      dims[4];
} whenet_tensor;

/* Per-kernel device timings of the last profiled forward (CUDA events on the
 * context's stream).  bytes/flops are the ALGORITHMIC figures of DESIGN.md. */
typedef struct {
    char   name[48];
    float  ms;          /* summed over `launches` launches                 */
    int    launches;
    double bytes;       /* algorithmic HBM bytes those launches must move   */
    double flops;       /* algorithmic flops (2*MAC) of those launches      */
} whenet_kernel_stat;

/* replaces: graph construction, reference whenet.py:8-14 (+ device choice via
 * CUDA_VISIBLE_DEVICES, demo_video.py:79-80).  `max_batch` bounds n of one
 * forward call (activation workspace is sized for min(max_batch, chunk)). */
int whenet_create(whenet_ctx** out, int device, int max_batch, int precision);

/* replaces: self.model.load_weights(snapshot), reference whenet.py:15-16.
 * Takes the file's raw tensors by name; folds BatchNorm (eps 1e-3) into the
 * preceding conv, re-lays weights out for the kernels and uploads them. */
int whenet_load_weights(whenet_ctx* ctx, const whenet_tensor* tensors, int n_tensors);

/* Persisted packed artefact (SURVEY.md 8f-2): the device image whenet_load_weights built - BatchNorm folded, 1x1 kernels
 * transposed to K-major and rounded to the context's storage type, K1 constants pre-halved - as two flat arenas plus an
 * index of offsets.  Export: call with NULL buffers to get sizes[3] = {fp32 elements, 16-bit elements, index entries}, then
 * with buffers of those sizes.  Import replaces whenet_load_weights (reference whenet.py:15-16) for a context of the SAME
 * precision: no HDF5 walk, no folding, no repacking - one validation pass over the index and two uploads. */
int whenet_export_packed(whenet_ctx* ctx, float* arena_f32, uint16_t* arena_16, int64_t* index, int64_t sizes[3]);
int whenet_import_packed(whenet_ctx* ctx, const float* arena_f32, int64_t n_f32, const uint16_t* arena_16, int64_t n_16,
                         const int64_t* index, int64_t n_index);

/* Run on an existing CUDA stream (cudaStream_t / CUstream) instead of the
 * context's own; NULL restores the internal stream.  Every call of the context
 * orders its device work after what was queued on its stream before the call,
 * and work queued on the stream after the call sees its results.  Switching to
 * another stream keeps that order: work queued after the switch runs after all
 * work queued before it, and whenet_synchronize covers both.  The previous
 * stream must still exist at the switch; setting the current stream again is a
 * no-op.  Host inputs of the forward entries are the exception: they are read
 * on the context's copy stream, which does not wait for the caller's stream (so
 * that the upload of one batch overlaps the compute of the previous one), so a
 * host input must hold its data when the call is made. */
int whenet_set_stream(whenet_ctx* ctx, void* cuda_stream);

/* replaces: WHENet.get_angle(img), reference whenet.py:22-34, for uint8 input.
 * `nhwc_rgb`: n x 224 x 224 x 3 RGB bytes (host memory, or device memory when
 * in_is_device != 0).  Normalisation (whenet.py:25-26) happens on the device
 * through a 3x256 table holding float32(((v/255)-mean)/std) evaluated in
 * float64 exactly as numpy does there.  `angles_out`: n x 3 floats
 * (yaw, pitch, roll in degrees) ; `logits_out`: NULL or n x 252 floats
 * (yaw 120 | pitch 66 | roll 66) = what self.model.predict returns
 * (whenet.py:27).  Outputs go to host memory, or to device memory when
 * out_is_device != 0 (then the call is asynchronous on the context's stream). */
int whenet_forward_u8(whenet_ctx* ctx, const uint8_t* nhwc_rgb, int n, int in_is_device,
                      float* angles_out, float* logits_out, int out_is_device);

/* Asynchronous form of whenet_forward_u8 for HOST buffers (both must be pinned, see whenet_host_alloc): queues the
 * H2D copy (copy stream), the forward and the D2H of the results, then returns.  Up to TWO calls may be in flight
 * (input staging and result buffers are double-buffered), so the upload of batch i+1 overlaps the compute of batch i.
 * Call whenet_synchronize before reading `angles_host` / `logits_host` or reusing `in_host`. */
int whenet_forward_u8_async(whenet_ctx* ctx, const uint8_t* in_host, int n, float* angles_host, float* logits_host);

/* replaces: self.model.predict(img, batch_size=8), reference whenet.py:27, for
 * an already normalised float32 n x 224 x 224 x 3 input. */
int whenet_forward_f32(whenet_ctx* ctx, const float* nhwc_normalised, int n, int in_is_device,
                       float* angles_out, float* logits_out, int out_is_device);

/* Crop front-end of the stream path; replaces, for ALL heads of a frame at once, the per-head
 * slice + cv2.cvtColor(BGR2RGB) + cv2.resize(.., (224,224)) of reference demo_video.py:21-23 (and demo.py:10-11).
 * `frame`: H x W x 3 uint8 (host, or device when frame_is_device); `rects`: m x 4 int32 host array of slice
 * bounds (y0, y1, x0, x1) with 0 <= y0 < y1 <= H, 0 <= x0 < x1 <= W (the margin arithmetic of
 * demo_video.py:13-19 is host-side, see whenet_b200/crops.py); `swap_rb` != 0 converts BGR -> RGB.
 * `crops_out`: m x 224 x 224 x 3 uint8 in DEVICE memory (feed it to whenet_forward_u8 with in_is_device=1),
 * bit-identical to OpenCV's 8-bit INTER_LINEAR resize.  Asynchronous on the context's stream. */
int whenet_crop_resize_u8(whenet_ctx* ctx, const uint8_t* frame, int H, int W, int frame_is_device,
                          const int32_t* rects, int m, int swap_rb, uint8_t* crops_out);

/* replaces, for the heads of n frames at once, reference demo_video.py:13-23: the margin arithmetic (:13-19), the slice,
 * cv2.cvtColor(BGR2RGB) and cv2.resize(.., (224,224)).  `frames`: n (1..64) x H x W x 3 uint8 (host, or device when
 * frames_are_device); `boxes`: m x 4 float32 host array in the detector's order (y_min, x_min, y_max, x_max), unclipped,
 * original pixels; `frame_of`: m int32 host frame indices in [0, n).  The margin arithmetic runs on the host in float32,
 * bit for bit what whenet_b200/crops.py enlarge_box computes with numpy; a box whose slice is empty or leaves the frame
 * (where cv2.resize would raise) gets valid_out 0 and an all-zero crop.  `crops_out`: m x 224 x 224 x 3 uint8 in DEVICE
 * memory; `rects_out` (m x 4 slice bounds (y0, y1, x0, x1), zeros for an invalid box) and `valid_out` (m int32) are host
 * arrays, each may be NULL, filled before the call returns.  The crops are asynchronous on the context's stream: feed them to
 * whenet_forward_u8 with in_is_device=1.  One launch serves every crop; host frames are uploaded once per call. */
int whenet_crop_boxes_u8(whenet_ctx* ctx, const uint8_t* frames, int n, int H, int W, int frames_are_device,
                         const float* boxes, const int32_t* frame_of, int m, int swap_rb,
                         uint8_t* crops_out, int32_t* rects_out, int32_t* valid_out);

/* whenet_crop_boxes_u8 for n (1..64) frames that each have their own size: `frames` is a host array of n frame pointers,
 * frame i is hw[2i] x hw[2i+1] x 3 uint8 (each side 1..16384), all in host memory or all in device memory on the context's
 * device (frames_are_device).  Each box's margin arithmetic uses its own frame's H and W; the outputs are laid out as
 * whenet_crop_boxes_u8's, and each crop is the bytes whenet_crop_boxes_u8 gives that box on its frame alone.  Host frames are
 * uploaded once per call into the context's staging buffer; device frames are read in place.  Every argument but the
 * context is checked before anything touches a device. */
int whenet_crop_boxes_ragged_u8(whenet_ctx* ctx, const uint8_t* const* frames, const int32_t* hw, int n, int frames_are_device,
                                const float* boxes, const int32_t* frame_of, int m, int swap_rb,
                                uint8_t* crops_out, int32_t* rects_out, int32_t* valid_out);

/* whenet_crop_boxes_u8 and whenet_crop_boxes_ragged_u8 on YUV 4:2:0 frames (WHENET_YUV_NV12 / WHENET_YUV_I420 in
 * `yuv_layout`, in place of swap_rb): H, W and hw are the image sizes (each side even, at most 16384), each frame is
 * H * W * 3/2 bytes.  The margin arithmetic and validity are those of the BGR entries; each crop is RGB, the bytes the BGR
 * entry with swap_rb gives on cv2.cvtColor(frame, COLOR_YUV2BGR_NV12 / _I420).  Every argument but the context is checked
 * before anything touches a device. */
int whenet_crop_boxes_yuv_u8(whenet_ctx* ctx, const uint8_t* frames, int n, int H, int W, int frames_are_device,
                             const float* boxes, const int32_t* frame_of, int m, int yuv_layout,
                             uint8_t* crops_out, int32_t* rects_out, int32_t* valid_out);
int whenet_crop_boxes_ragged_yuv_u8(whenet_ctx* ctx, const uint8_t* const* frames, const int32_t* hw, int n, int frames_are_device,
                                    const float* boxes, const int32_t* frame_of, int m, int yuv_layout,
                                    uint8_t* crops_out, int32_t* rects_out, int32_t* valid_out);

/* whenet_crop_boxes_u8 and whenet_crop_boxes_ragged_u8 on packed YUV 4:2:2 frames (WHENET_YUV_YUYV / WHENET_YUV_UYVY in
 * `yuv422_layout`, in place of swap_rb): H, W and hw are the image sizes (W even in [2, 16384], H in [1, 16384]), each frame
 * is H * W * 2 bytes.  Otherwise as the 4:2:0 entries above: each crop is RGB, the bytes the BGR entry with swap_rb gives on
 * cv2.cvtColor(frame, COLOR_YUV2BGR_YUYV / _UYVY), and every argument but the context is checked before anything touches a
 * device. */
int whenet_crop_boxes_yuv422_u8(whenet_ctx* ctx, const uint8_t* frames, int n, int H, int W, int frames_are_device,
                                const float* boxes, const int32_t* frame_of, int m, int yuv422_layout,
                                uint8_t* crops_out, int32_t* rects_out, int32_t* valid_out);
int whenet_crop_boxes_ragged_yuv422_u8(whenet_ctx* ctx, const uint8_t* const* frames, const int32_t* hw, int n, int frames_are_device,
                                       const float* boxes, const int32_t* frame_of, int m, int yuv422_layout,
                                       uint8_t* crops_out, int32_t* rects_out, int32_t* valid_out);

/* YUV frames -> BGR frames on the device, bit-identical to cv2.cvtColor(frame, COLOR_YUV2BGR_NV12 / _I420 / _YUYV / _UYVY)
 * for `layout` WHENET_YUV_NV12, _I420, _YUYV or _UYVY: the frames whenet_draw_heads_u8 and whenet_encode_jpeg_u8 take.
 * `frames`: n (1..64) frames of one size back to back, host memory or device memory on the context's device
 * (frames_are_device); H and W are the image size, sides in [1, 16384] (4:2:0: both even; 4:2:2: W even), so a frame is
 * H * W * 3/2 or H * W * 2 bytes.  `out_frames`: n x H x W x 3 bytes in caller-owned device memory.  Host frames are uploaded
 * into the context's staging buffer.  Every argument but the context is checked before any device call.  Asynchronous on the
 * context's stream: work queued on it later sees the frames; synchronise it (whenet_synchronize) before reading them on
 * another stream. */
int whenet_yuv_to_bgr_u8(whenet_ctx* ctx, const uint8_t* frames, int n, int H, int W, int frames_are_device, int layout,
                         uint8_t* out_frames);
/* the same on n frames of their own sizes: frames[i] is frame i (all host or all device), hw = n x (H_i, W_i) int32 on the
 * host, out_frames[i] the caller's H_i x W_i x 3 device frame */
int whenet_yuv_to_bgr_ragged_u8(whenet_ctx* ctx, const uint8_t* const* frames, const int32_t* hw, int n, int frames_are_device,
                                int layout, uint8_t* const* out_frames);

/* Block until everything queued by this context has finished. */
int whenet_synchronize(whenet_ctx* ctx);

/* Pinned host memory for asynchronous input staging (optional). */
void* whenet_host_alloc(size_t bytes);
void  whenet_host_free(void* p);

/* ---- test / measurement hooks (no reference counterpart) ---- */

/* Keep float32 copies of intermediate tensors of the NEXT forwards ("stem", "dw1".."dw16" or "dwg1".."dwg16",
 * "gate1".."gate16", "block1".."block16", "head", "pooled"), crop-major, one row per tapped crop.
 * enable = 0: off.
 * enable = 1: the first chunk of the call, if it has at most 8 crops.  The forward then runs on one stream and leaves every
 *   depthwise output ungated ("dw%d"), so its route can differ from the untapped one.
 * enable = 2: every chunk and both halves of a two-stream pass, at any batch, on the untapped route: the launches and every
 *   kernel parameter are those of the same call without taps.  The one difference: where the one-CTA head kernel alone has
 *   the pooled vector (batches below 64), it also writes it out for the "pooled" tap.  A block whose depthwise output was
 *   gated in place (the SE tails' scale_out) records the 16-bit d * g as "dwg%d" instead of "dw%d".  The tap buffers are
 *   allocated before the first kernel.  Without a selection (whenet_debug_tap_crops) every crop is tapped: 12.8 MB per crop.
 * Every forward invalidates the previous taps; a tapped forward under enable != 0 never replays a captured graph. */
int whenet_debug_enable_taps(whenet_ctx* ctx, int enable);
/* Mode 2: tap only crops idx[0..k) of each call, in that order (k <= 64; k = 0 taps every crop).  A forward with an index
 * >= its batch fails with WHENET_EINVAL before its first launch. */
int whenet_debug_tap_crops(whenet_ctx* ctx, const int* idx, int k);
/* Copy a tap to host; *n_elems receives its element count (call with out=NULL to query).  WHENET_ENOTFOUND for a tap the
 * last forward did not write. */
int whenet_debug_tap(whenet_ctx* ctx, const char* name, float* out, size_t cap_elems, size_t* n_elems);

/* Run ONE 1x1 convolution through the kernel family chosen by use_tc (0 CUDA-core, 1 tensor core):
 * out[m,n] = act(bias[n] + sum_k A[m,k]*gate[m/hw,k]*W[k,n]) (+ resid[m,n]).  All arrays are host
 * float32 (converted to the context's storage type on the way in and back on the way out);
 * gate / resid may be NULL.  Returns WHENET_EINVAL when the family cannot run the shape. */
int whenet_debug_conv1x1(whenet_ctx* ctx, int use_tc, const float* A, const float* W, const float* bias,
                         const float* gate, const float* resid, float* out,
                         int64_t M, int K, int N, int hw, int swish);

/* Tuning hook: force the K1 (fused expand+depthwise) tile plan of block `block` (2..16): output tile
 * th x tw, strips of r outputs, cc expanded channels per chunk, nt threads per CTA (256 or 512), nb crops
 * per CTA (2 only where one tile is the whole image).  WHENET_EINVAL if the plan cannot run. */
int whenet_debug_set_k1_plan(whenet_ctx* ctx, int block, int th, int tw, int r, int cc, int nt, int nb);

/* Decode only: n x 252 host logits -> n x 3 host angles through the SAME device function the head kernel uses
 * (softmax of reference utils.py:7-11, expectation of whenet.py:31-33).  Synchronous. */
int whenet_debug_decode(whenet_ctx* ctx, const float* logits_host, int n, float* angles_host);

/* A device kernel raises the context's mbarrier-timeout flag (what a tensor-core kernel does when a bounded wait expires):
 * the next synchronising call (host-output forward, whenet_synchronize) must return WHENET_ECUDA. */
int whenet_debug_raise_timeout(whenet_ctx* ctx);

/* The margin arithmetic of whenet_crop_boxes_u8 alone, on the host (no context, no GPU): m boxes of an H x W frame ->
 * rects_out / valid_out as that call fills them (each may be NULL). */
int whenet_debug_enlarge_boxes(const float* boxes, int m, int H, int W, int32_t* rects_out, int32_t* valid_out);
/* Head overlay (DESIGN.md section 8.7): draws, for each of m heads, what reference demo_video.py:26,29 draws with
   display="simple" - a black thickness-2 rectangle around the margin-enlarged box, then the red, green and blue pose axes
   (utils.py:40-42) - into device BGR frames IN PLACE on the context's stream, pixel-identical to OpenCV's cv2.rectangle /
   cv2.line.  Heads are drawn in order, a later one over an earlier one.  boxes: m x (y_min, x_min, y_max, x_max) float32,
   angles: m x (yaw, pitch, roll) float32 degrees, frame_of: m frame indices, all on the host.  A head is drawn exactly when
   the reference would draw it without raising: its enlarged slice is valid (as the crop entries' valid_out) and its three
   float32 radians are finite; drawn_out (optional, m int32) says which were.  m = 0 is a no-op.  n in [1, 64], sides in
   [1, 16384].  frames: n frames of H x W x 3 bytes back to back. */
int whenet_draw_heads_u8(whenet_ctx* ctx, uint8_t* frames, int n, int H, int W, const float* boxes, const float* angles,
                         const int32_t* frame_of, int m, int32_t* drawn_out);
/* the same on n device frames of their own sizes: frames[i] is H_i x W_i x 3, hw = n x (H_i, W_i) int32 on the host */
int whenet_draw_heads_ragged_u8(whenet_ctx* ctx, uint8_t* const* frames, const int32_t* hw, int n, const float* boxes,
                                const float* angles, const int32_t* frame_of, int m, int32_t* drawn_out);
/* The overlay's host geometry without a GPU: per head 7 segments (x0, y0, x1, y1) int32 in draw order - the rectangle's
   top, right, bottom and left edges, then the red, green and blue axes - zeros for a head not drawn (drawn_out[i] = 0). */
int whenet_debug_overlay_segments(const float* boxes, const float* angles, int m, int H, int W, int32_t* seg_out, int32_t* drawn_out);
/* Head overlay with a display mode (DESIGN.md section 8.8): display 0 draws exactly what whenet_draw_heads_u8 draws
   (display="simple"); display 1 ("full") adds, after each drawn head's rectangle and axes, the three labels of reference
   demo_video.py:31-34: cv2.putText(img, "yaw: {}".format(np.round(yaw)), (int(x_min), int(y_min)), FONT_HERSHEY_SIMPLEX,
   0.4, (100, 255, 0), 1), then "pitch: " 15 rows and "roll: " 30 rows higher, the numbers formatted from the float32 angles
   as the reference formats them ("-12.0", "-0.0").  Any other display is WHENET_EINVAL; with display 1, m is at most 65536;
   every other argument as whenet_draw_heads_u8. */
int whenet_draw_heads_ex_u8(whenet_ctx* ctx, uint8_t* frames, int n, int H, int W, const float* boxes, const float* angles,
                            const int32_t* frame_of, int m, int display, int32_t* drawn_out);
int whenet_draw_heads_ex_ragged_u8(whenet_ctx* ctx, uint8_t* const* frames, const int32_t* hw, int n, const float* boxes,
                                   const float* angles, const int32_t* frame_of, int m, int display, int32_t* drawn_out);
/* Text on device BGR frames in place, pixel-identical to cv2.putText(img, texts[i], (org[2i], org[2i+1]),
   FONT_HERSHEY_SIMPLEX, scale[i], (bgr[3i], bgr[3i+1], bgr[3i+2]), thickness[i]) with LINE_8 and bottomLeftOrigin=false, for
   m items drawn in order into frame frame_of[i].  texts: NUL-terminated printable ASCII (32..126), at most 4096
   characters each and 2^22 in all; m at most 2^20; thickness must be 1; scale in (0, 256]; origin coordinates within
   +-2^24.  Anything else, or more segments than an int indexes, is WHENET_EINVAL.
   m = 0 is a no-op; n and frame sizes as whenet_draw_heads_u8.  All arrays are on the host. */
int whenet_put_text_u8(whenet_ctx* ctx, uint8_t* frames, int n, int H, int W, const int32_t* frame_of, const char* const* texts,
                       const int32_t* org, const double* scale, const uint8_t* bgr, const int32_t* thickness, int m);
int whenet_put_text_ragged_u8(whenet_ctx* ctx, uint8_t* const* frames, const int32_t* hw, int n, const int32_t* frame_of,
                              const char* const* texts, const int32_t* org, const double* scale, const uint8_t* bgr,
                              const int32_t* thickness, int m);
/* The text geometry without a GPU: the 16.16 segments (x1, y1, x2, y2) int64 putText strokes for one item, in draw order.
   *count_out = their number; at most cap are written to seg_out (either may be NULL).  Arguments checked as above. */
int whenet_debug_text_segments(const char* text, int org_x, int org_y, double scale, int thickness, int64_t* seg_out, int cap,
                               int32_t* count_out);
/* The number of each display="full" label: str(np.round(np.float32(a))) for m float32 angles, NUL-terminated, one per
   `stride` (>= 32) bytes of out. */
int whenet_debug_label_text(const float* angles, int m, char* out, int stride);
/* Baseline JPEG files of n BGR frames (DESIGN.md section 8.9; options in section 8.11), byte-identical to
   cv2.imencode(".jpg", frame, [cv2.IMWRITE_JPEG_QUALITY, quality]): 4:2:0, the Annex K tables scaled by the IJG quality
   rule, no restart markers.  frames: n frames of H x W x 3 bytes back to back, in device memory (frames_are_device = 1) or
   host memory (0).  n in [1, 64], sides in [1, 16384], quality in [1, 100]; anything else is WHENET_EINVAL before any device
   call.  Runs on the context's stream and returns when the files are on the host: *data_out points into a pinned buffer
   the context owns, valid until its next encode call; offsets_out (n + 1 int64 on the host): file i is
   data[offsets[i] : offsets[i + 1]].  Scratch grows with the call and is freed with the context. */
int whenet_encode_jpeg_u8(whenet_ctx* ctx, const uint8_t* frames, int n, int H, int W, int frames_are_device, int quality,
                          const uint8_t** data_out, int64_t* offsets_out);
/* the same on n frames of their own sizes: frames[i] is H_i x W_i x 3, hw = n x (H_i, W_i) int32 on the host */
int whenet_encode_jpeg_ragged_u8(whenet_ctx* ctx, const uint8_t* const* frames, const int32_t* hw, int n, int frames_are_device,
                                 int quality, const uint8_t** data_out, int64_t* offsets_out);
/* The bytes of a file before its entropy-coded data (SOI .. SOS, 623 bytes) without a GPU; cap >= 623. */
int whenet_debug_jpeg_header(int H, int W, int quality, uint8_t* out, int cap, int* len);
/* JPEG options (DESIGN.md section 8.11).  A call with them equals cv2.imencode(".jpg", frame, params) where params are
   IMWRITE_JPEG_QUALITY quality (or, when chroma_quality != quality, IMWRITE_JPEG_LUMA_QUALITY quality and
   IMWRITE_JPEG_CHROMA_QUALITY chroma_quality), IMWRITE_JPEG_SAMPLING_FACTOR sampling, IMWRITE_JPEG_RST_INTERVAL
   restart_interval and IMWRITE_JPEG_OPTIMIZE optimize; a one-channel frame is the (H, W) image cv2 codes as gray. */
typedef struct whenet_jpeg_options {
    int quality;            /* 1..100: the luma table, and the chroma table unless chroma_quality differs */
    int chroma_quality;     /* 1..100; != quality needs sampling 444 (libjpeg codes it as 4:4:4 whatever the sampling) */
    int sampling;           /* 420, 422 or 444: luma sampling 2x2, 2x1 or 1x1; Cb and Cr 1x1 */
    int restart_interval;   /* 0..65535 MCUs per restart interval; 0 = no restart markers */
    int optimize;           /* 0: Annex K Huffman tables; 1: optimal tables per frame (libjpeg's jpeg_gen_optimal_table) */
    int progressive;        /* 0: baseline (SOF0); 1: progressive (SOF2, DESIGN.md section 8.12), equal to cv2 with
                               IMWRITE_JPEG_PROGRESSIVE 1: libjpeg's scan script with optimal tables per scan, so optimize is
                               ignored, as cv2 ignores it.  Left out of an initialiser it is 0, the baseline file. */
} whenet_jpeg_options;
/* whenet_encode_jpeg_ragged_u8 with options: frames[i] is H_i x W_i x channels (1 = gray, 3 = BGR); a gray call takes
   sampling 420 and chroma_quality == quality.  Every argument is checked as above, WHENET_EINVAL before any device call.
   whenet_encode_jpeg_u8 and _ragged_u8 are this call with channels 3 and {quality, quality, 420, 0, 0, 0}. */
int whenet_encode_jpeg_ex_u8(whenet_ctx* ctx, const uint8_t* const* frames, const int32_t* hw, int n, int channels,
                             int frames_are_device, const whenet_jpeg_options* opts, const uint8_t** data_out, int64_t* offsets_out);
/* The header (SOI .. SOS, at most 629 bytes) of a file with options (optimize 0 and progressive 0 only: those headers
   depend on the frame's symbols) without a GPU; *len = its bytes. */
int whenet_debug_jpeg_header_ex(int H, int W, int channels, const whenet_jpeg_options* opts, uint8_t* out, int cap, int* len);
/* libjpeg's jpeg_gen_optimal_table on 256 symbol counts (>= 0) on the host: bits_out[16] = codes per length 1..16,
   vals_out[*nvals_out] = the symbols by length, then value.  WHENET_EINVAL for a code past 32 bits, as libjpeg refuses it.
   The _gpu variant runs the encoder's device kernel on the context's stream and returns when done. */
int whenet_debug_jpeg_optimal_table(const int32_t* counts, uint8_t* bits_out, uint8_t* vals_out, int* nvals_out);
int whenet_debug_jpeg_optimal_table_gpu(whenet_ctx* ctx, const int32_t* counts, uint8_t* bits_out, uint8_t* vals_out, int* nvals_out);
/* JPEG decoding (DESIGN.md section 8.10), pixel-identical to cv2.imdecode(buf, cv2.IMREAD_COLOR): SOF0 / SOF1 8-bit Huffman,
   one interleaved scan, 1 component (replicated to B = G = R) or 3 (YCbCr) at 4:4:4, 4:2:2 or 4:2:0, restart intervals,
   Annex K tables where no DHT defines one, EXIF orientation 1..8 applied, sides 1..16384.
   whenet_jpeg_info parses a file's header on the host without a GPU: hw_out = (H, W) of the decoded frame (after the
   orientation), or WHENET_EINVAL with the reason in msg (cap bytes, may be NULL) and whenet_last_error(). */
int whenet_jpeg_info(const uint8_t* data, int64_t len, int32_t* hw_out, char* msg, int cap);
/* Decode n (1..64) host files (files[i], sizes[i] bytes) into caller-owned device frames out_frames[i], each H_i x W_i x 3
   BGR as whenet_jpeg_info gives.  A header error is WHENET_EINVAL naming the file before any device call.  Runs on the
   context's device and stream and returns when the frames are complete.  status_out (n int32 on the host, may be NULL):
   per file 0, or bits 1 truncated data, 2 restart markers out of sequence or miscounted, 4 a marker inside the entropy-coded
   data, 8 an invalid Huffman code, 16 an AC run past coefficient 63, 32 more or fewer blocks than the MCUs; any nonzero
   status makes the call return WHENET_EINVAL (that file's frame is then undefined) and leaves the context usable.  Scratch
   grows with the call and is freed with the context. */
int whenet_decode_jpeg_u8(whenet_ctx* ctx, const uint8_t* const* files, const int64_t* sizes, int n, uint8_t* const* out_frames,
                          int32_t* status_out);
/* Reduced and gray decoding (DESIGN.md section 8.13): scale_denom 1, 2, 4 or 8 and channels 3 (BGR) or 1 (the luma plane),
   pixel-identical to cv2.imdecode with IMREAD_REDUCED_COLOR_d / IMREAD_REDUCED_GRAYSCALE_d (IMREAD_COLOR / IMREAD_GRAYSCALE at
   d = 1).  whenet_jpeg_info_ex gives hw_out = (ceil(H / d), ceil(W / d)) after the orientation; whenet_decode_jpeg_ex_u8 writes
   H_i x W_i x channels frames of that size.  Otherwise as whenet_jpeg_info / whenet_decode_jpeg_u8, which are the (1, 3)
   case; a scale_denom or channels outside those sets is WHENET_EINVAL before any device call. */
int whenet_jpeg_info_ex(const uint8_t* data, int64_t len, int scale_denom, int channels, int32_t* hw_out, char* msg, int cap);
int whenet_decode_jpeg_ex_u8(whenet_ctx* ctx, const uint8_t* const* files, const int64_t* sizes, int n, int scale_denom,
                             int channels, uint8_t* const* out_frames, int32_t* status_out);
/* Bits per subsequence of the self-synchronising Huffman decode, 32..65536, or 0 for the default (2048). */
int whenet_debug_jpeg_piece_bits(whenet_ctx* ctx, int bits);


/* Time every kernel of the NEXT forwards with CUDA events. */
int whenet_profile_enable(whenet_ctx* ctx, int enable);
/* Read (and reset) the accumulated per-kernel statistics; returns the count written. */
int whenet_profile_read(whenet_ctx* ctx, whenet_kernel_stat* out, int cap);

/* Kernels launched by this context since creation (the bench's gpu_launches). */
int64_t whenet_launch_count(whenet_ctx* ctx);

/* Tuning / ablation switches (all have measured defaults; see DESIGN.md and profiles/README.md):
 *   "chunk"          crops per pass through the network (default max_batch: one pass)
 *   "streams"        1..4 batch parts running concurrently on internal streams (default 2)
 *   "graph"          1: replay device-resident forwards from a captured CUDA graph (default 0)
 *   "tensor_cores"   16-bit modes: 0 = CUDA-core kernels for every 1x1 conv, 1 = tensor core, wgmma (default 1).
 *                    fp32 mode: 0 = fp32 FMA kernels (default), 1 = the 1x1 convs on the tensor core through the bf16 hi/lo split
 *                    (three MMAs per product, fp32 accumulation: 6e-4 deg from the float64 oracle on the golden crops)
 *   "fused"          1: K1 (expand + depthwise fused, expanded tensor in shared memory) for blocks 2..fused_max_block
 *   "pw_variant"     2 = pw_tc2 (one tile per CTA, cp.async ring), 3 = K2 (persistent, TMA, warp-specialised), 4 = per layer (default):
 *                    K2 for the ungated / small-map convs that have at least 2 x 148 tiles, pw_tc2 otherwise
 *   "kd_from"        bf16: blocks >= this (default 7) run KD (expand conv on chip + depthwise + squeeze; at small batches expand
 *                    GEMM (fp16 E) + KD over TMA tiles) instead of K1; 0 = K1 on every block.  "kd_tail" 1: KD computes the SE gate
 *                    and gates its output itself (default 0: se_gate + gated project); "dw1_kd" 0: block 1's depthwise on K1's depthwise
 *                    half over a bf16 stem output (default 1: KD over an fp16 stem output); "pw3" 0: block-1 project on pw_tc2
 *   "se_batch", "head_batch"   batches >= 64: four crops per CTA in the SE gate / in the Dense + decode head (default 1; same bits)
 *   "stage_threads"  host threads that stage PAGEABLE inputs of 8 MB and more into the context's pinned buffer (default 8; 0 = plain
 *                    cudaMemcpyAsync from the caller's buffer)
 *   "fused_max_block", "dw1_fused", "k1_split_ctas",
 *   "se_fused", "se_tail" (K1 CTAs that hold whole crops compute the SE gate themselves, default 1), "se_scale_out", "se_wide",
 *   "pw_stage_cap", "pw_smem_kb", "pw_min_ctas" (split N until the grid has this many CTAs),
 *   "dw_variant", "stem_variant", "host_chunk".
 * Unknown keys return WHENET_ENOTFOUND. */
int whenet_set_option(whenet_ctx* ctx, const char* key, int value);

const char* whenet_last_error(void);
const char* whenet_version(void);
void whenet_destroy(whenet_ctx* ctx);

/* ==== YOLOv3 head detector (reference yolo_v3/yolo_postprocess.py:26-205, yolo_v3/model.py) ====
 * A detector handle is bound to one device, one stream and one model input size (multiples of 32 in [32, 608], or up to 4096
 * through whenet_det_create_large; the reference's model_image_size, default 416 x 416) and is NOT thread-safe.  Errors use the WHENET_E* codes and
 * whenet_last_error().  Storage is bf16, accumulation fp32; the head logits stay fp32 (whenet_det_create).  The fp32
 * parity mode (whenet_det_create_ex with WHENET_PRECISION_FP32) keeps every activation in fp32 and runs each conv as three
 * bf16 MMAs on the hi / lo split of activations and weights, with fp32 accumulation (DESIGN.md 8.3). */
typedef struct whenet_det whenet_det;

/* replaces: YOLO.__init__ graph construction (yolo_postprocess.py:44-50, 77-78 yolo_body).  `max_frames` bounds n of one
 * detect call (1..64). */
int whenet_det_create(whenet_det** out, int device, int input_h, int input_w, int max_frames);
/* whenet_det_create with a precision: WHENET_PRECISION_BF16 (what whenet_det_create makes) or WHENET_PRECISION_FP32 (the
 * parity mode); any other value is WHENET_EINVAL.  The activation buffers of one frame take, for one class, 77 MB at 416 x 416
 * and 164 MB at 608 x 608 in bf16 (tiny YOLOv3: 15 and 32 MB), and twice that in fp32: 153 and 328 MB (tiny: 30 and 63 MB);
 * they are allocated for `max_frames` frames. */
int whenet_det_create_ex(whenet_det** out, int device, int input_h, int input_w, int max_frames, int precision);

/* whenet_det_create_ex for model inputs up to 4096 x 4096: both sides multiples of 32 in [32, 4096], either precision, either
 * network; anything else is WHENET_EINVAL before a device is touched.  A 1080p frame letterboxes to 1088 x 1920 without a
 * downscale (1056 x 1920 is the reference's image-sized mode, model_image_size=(None, None), on 1080p).  Every other entry
 * works on such a detector unchanged.  Above 24,576 candidates per frame (3 * (H/32) * (W/32) * 21, tiny: * 5) decode and
 * NMS run as three kernels with the one-CTA kernel's results; conv launches with more than 65,535 M tiles run as groups of
 * whole frames.  Device memory per frame (activations, canvas, decode workspaces; one class), from the layer table:
 *                       YOLOv3 bf16   YOLOv3 fp32   tiny bf16   tiny fp32
 *   1088 x 1920            936 MB       1.86 GB      186 MB      364 MB
 *   2176 x 3840           3.75 GB       7.44 GB      743 MB     1.46 GB
 *   4096 x 4096           7.52 GB       14.9 GB     1.49 GB     2.92 GB
 * all of it allocated for `max_frames` frames (most of it by whenet_det_load_weights).  A request larger than the whole device
 * is refused before its first buffer with WHENET_ECUDA naming the bytes it needs: at create when even tiny YOLOv3 with one
 * class would not fit, at whenet_det_load_weights (the detector left as it was) for the network loaded.  An allocation that
 * fails otherwise returns WHENET_ECUDA naming its bytes; the detector is then left without weights (or, at create, not
 * made), and the device keeps working. */
int whenet_det_create_large(whenet_det** out, int device, int input_h, int input_w, int max_frames, int precision);

/* The detector's precision (WHENET_PRECISION_BF16 or WHENET_PRECISION_FP32). */
int whenet_det_precision(whenet_det* det);

/* replaces: load_model / yolo_model.load_weights(model_path) (yolo_postprocess.py:74-79) and _get_anchors (:59-64).
 * `anchors`: 9 (w, h) pairs in input pixels for YOLOv3 (yolo_body), 6 for tiny YOLOv3 (tiny_yolo_body, model.py:92-122);
 * any other count is WHENET_EINVAL.  `tensors`: the network's 75 (tiny: 13) convs in Keras weight order
 * (whenet_b200/yolo_arch.py), each its kernel [k,k,cin,cout] followed by BatchNorm gamma, beta, moving_mean,
 * moving_variance (bias-free convs) or by its bias (the output convs); BatchNorm (eps 1e-3) is folded in double and the
 * kernels rounded once to bf16 (fp32 detector: to fp32, then split into bf16 hi = bf16(w) and lo = bf16(w - hi)).  The class count follows from the output convs' width 3 * (5 + classes).  Loading the
 * other network or another class count into a live detector rebuilds its buffers and captured graphs. */
int whenet_det_load_weights(whenet_det* det, const whenet_tensor* tensors, int n_tensors, const float* anchors, int n_anchors);

/* Number of classes of the loaded weights (0 before whenet_det_load_weights). */
int whenet_det_num_classes(whenet_det* det);

/* Run on an existing CUDA stream; NULL restores the internal one. */
int whenet_det_set_stream(whenet_det* det, void* cuda_stream);

/* replaces: YOLO.detect (yolo_postprocess.py:180-205) for n frames of one size at once: letterbox_image (utils.py:23-34,
 * bit-exact with Pillow's BICUBIC), /255, the body, yolo_eval (model.py:190-232: decode, yolo_correct_boxes, per-class
 * score >= `score`, greedy NMS with IoU > `iou` suppressing, at most `max_boxes` (1..256) per class; equal scores keep
 * the lower candidate index first).  `frames`: n x H x W x 3 uint8, host or device memory; swap_rb != 0 reads BGR.
 * Outputs (host): per frame num_classes * max_boxes slots of boxes (y_min, x_min, y_max, x_max, original pixels,
 * unclipped), scores and classes, filled class by class; counts[i] = slots used by frame i.  The forward is a CUDA graph
 * captured on the first call for each (n, H, W) and replayed after.  Synchronous. */
int whenet_det_detect_u8(whenet_det* det, const uint8_t* frames, int n, int H, int W, int frames_are_device, int swap_rb,
                         float score, float iou, int max_boxes, float* boxes, float* scores, int32_t* classes, int32_t* counts);

/* whenet_det_detect_u8 for n (1..max_frames) frames that each have their own size, in one forward: `frames` is a host array
 * of n frame pointers, frame i is hw[2i] x hw[2i+1] x 3 uint8 (each side 1..16384), all in host memory or all in device
 * memory on the detector's device (frames_are_device).  Each frame is letterboxed with its own tables onto the model-size
 * canvas; the body, decode and NMS then run on all n canvases at once, and frame i's outputs (laid out as
 * whenet_det_detect_u8's) are the bits whenet_det_detect_u8 gives it alone.  The frames are copied into the detector's
 * frame buffer; the forward is a CUDA graph captured on the first call for each ordered list of sizes and swap_rb (at most
 * 16 such lists are kept, apart from the one-size graphs) and replayed after.  Every argument but the detector is checked
 * before anything touches a device.  Synchronous. */
int whenet_det_detect_ragged_u8(whenet_det* det, const uint8_t* const* frames, const int32_t* hw, int n, int frames_are_device,
                                int swap_rb, float score, float iou, int max_boxes,
                                float* boxes, float* scores, int32_t* classes, int32_t* counts);

/* whenet_det_detect_u8 and whenet_det_detect_ragged_u8 on YUV 4:2:0 frames (WHENET_YUV_NV12 / WHENET_YUV_I420 in
 * `yuv_layout`, in place of swap_rb): H, W and hw are the image sizes (each side even, 2..16384), each frame is H * W * 3/2
 * bytes.  The letterbox converts each source pixel as it reads it; everything after it is the BGR path's, and the outputs are
 * the bits the BGR entry with swap_rb gives on cv2.cvtColor(frame, COLOR_YUV2BGR_NV12 / _I420).  The graph caches key on the
 * layout too.  Every argument but the detector (and n against its max_frames) is checked before anything touches a device. */
int whenet_det_detect_yuv_u8(whenet_det* det, const uint8_t* frames, int n, int H, int W, int frames_are_device, int yuv_layout,
                             float score, float iou, int max_boxes, float* boxes, float* scores, int32_t* classes, int32_t* counts);
int whenet_det_detect_ragged_yuv_u8(whenet_det* det, const uint8_t* const* frames, const int32_t* hw, int n, int frames_are_device,
                                    int yuv_layout, float score, float iou, int max_boxes,
                                    float* boxes, float* scores, int32_t* classes, int32_t* counts);

/* whenet_det_detect_u8 and whenet_det_detect_ragged_u8 on packed YUV 4:2:2 frames (WHENET_YUV_YUYV / WHENET_YUV_UYVY in
 * `yuv422_layout`, in place of swap_rb): H, W and hw are the image sizes (W even in [2, 16384], H in [1, 16384]), each frame
 * is H * W * 2 bytes.  Otherwise as the 4:2:0 entries above: the outputs are the bits the BGR entry with swap_rb gives on
 * cv2.cvtColor(frame, COLOR_YUV2BGR_YUYV / _UYVY), and the graph caches key on the layout. */
int whenet_det_detect_yuv422_u8(whenet_det* det, const uint8_t* frames, int n, int H, int W, int frames_are_device, int yuv422_layout,
                                float score, float iou, int max_boxes, float* boxes, float* scores, int32_t* classes, int32_t* counts);
int whenet_det_detect_ragged_yuv422_u8(whenet_det* det, const uint8_t* const* frames, const int32_t* hw, int n, int frames_are_device,
                                       int yuv422_layout, float score, float iou, int max_boxes,
                                       float* boxes, float* scores, int32_t* classes, int32_t* counts);

/* Block until everything queued by this detector has finished. */
int whenet_det_synchronize(whenet_det* det);
void whenet_det_destroy(whenet_det* det);

/* ---- detector test hooks (no reference counterpart) ---- */
/* On an fp32 detector the hooks below take and return its fp32 values: taps are the fp32 activations, and debug_conv /
 * debug_maxpool use the host float32 inputs as given (no bf16 rounding) and run the fp32 kernels. */
/* float32 copy of the output of conv `layer` (0..74, tiny: 0..12, table order) of the last detect call (n x Ho x Wo x Cout),
 * with layer = -1 of its letterboxed uint8 canvas (n x input_h x input_w x 3), or with layer = 100 + i of the max-pooled
 * input of tiny conv i (i = 1..6; n x Hi x Wi x Cin). out=NULL queries the element count. */
int whenet_det_debug_tap(whenet_det* det, int layer, float* out, size_t cap_elems, size_t* n_elems);
/* One conv through the detector's implicit-GEMM kernel on host float32 arrays (rounded to bf16 on the way in):
 * x n x H x W x (cin - c_up); `up` NULL or the concat source n x H/2 x W/2 x c_up (put first, read upsampled x2);
 * w [k][k][cin][cout]; k = 1 or 3, stride 1 or 2 (3x3 only; padding 1 top/left; a concat conv has stride 1);
 * leaky != 0: bias + LeakyReLU(0.1) (+ resid n x Ho x Wo x cout) rounded to bf16, leaky = 0: bias only, fp32 output
 * (the output convs). */
int whenet_det_debug_conv(whenet_det* det, const float* x, const float* up, int n, int H, int W, int cin, int c_up,
                          const float* w, const float* bias, int k, int stride, int cout, int leaky, const float* resid, float* out);
/* The detector's 2x2 max-pool (tiny YOLOv3's MaxPooling2D, padding 'same': n x ceil(H/stride) x ceil(W/stride) x C, padded
 * cells never win) on host float32 arrays rounded to bf16 on the way in; x n x H x W x C, C a multiple of 8, stride 1 or 2. */
int whenet_det_debug_maxpool(whenet_det* det, const float* x, int n, int H, int W, int C, int stride, float* out);
/* Decode + NMS alone: host fp32 head logits (n x gh_l x gw_l x 3(5+C) for the detector's input size) of frames of
 * img_h x img_w pixels -> the outputs of whenet_det_detect_u8.  A tiny YOLOv3 detector has two heads: head2 is ignored and
 * may be NULL. */
int whenet_det_debug_decode(whenet_det* det, const float* head0, const float* head1, const float* head2, int n, int img_h, int img_w,
                            float score, float iou, int max_boxes, float* boxes, float* scores, int32_t* classes, int32_t* counts);

/* Test hook: on != 0 runs every later decode + NMS of this detector through the route for more than 24,576 candidates
 * (decode, per-class NMS and pack kernels) whatever its candidate count, so that both routes can be compared where both run;
 * 0 restores the choice by candidate count. */
int whenet_det_debug_force_large_decode(whenet_det* det, int on);

#ifdef __cplusplus
}
#endif
#endif /* WHENET_B200_H */
