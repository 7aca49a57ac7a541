/* mivos_b200 — C ABI of the H100-native mask-propagation hot path.
 *
 * The reference (hkchengrex/MiVOS) has no FFI: its hot path is PyTorch library calls made from
 * `PropagationNetwork` / `InferenceCore` (SURVEY.md §8b).  This header is the boundary a
 * maintainer would bind instead of those calls; every entry point names the reference code it
 * replaces (paths relative to the reference root).  Plain pointers and sizes only — no torch
 * types.  All pointers are DEVICE pointers unless a parameter says "host"; all work is enqueued
 * on `stream` and is stream-ordered; no entry point allocates device memory or synchronises.
 * Every function returns MIVOS_OK (0) or a negative MIVOS_ERR_* code; `mivos_last_error()` gives
 * the message for the calling thread's last failure.
 *
 * Data layouts
 *   NCHW   : the reference's layout, fp32 contiguous.
 *   HALO   : our resident activation layout, fp32 [N][H+2][W+2][C] (pixel-major, channels
 *            contiguous, C a multiple of 4) with a one-pixel zero border, so that a 3x3/pad-1
 *            convolution tap is a constant row offset in the flattened [N*(H+2)*(W+2), C] matrix.
 *            Borders are never written by any kernel (buffers are zeroed once by the owner).
 *   BANK   : memory bank, slot-major: keys fp32 [K][slots][128], values fp32 [K][slots][512],
 *            slot = t*HW + pixel (the transpose of the reference's [K,C,T,H,W]).
 */
#ifndef MIVOS_B200_H_
#define MIVOS_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define MIVOS_API __attribute__((visibility("default")))
#else
#define MIVOS_API
#endif

typedef struct CUstream_st* mivos_stream_t;

enum {
  MIVOS_OK = 0,
  MIVOS_ERR_INVALID = -1,  /* bad argument (shape, alignment, null pointer) */
  MIVOS_ERR_CUDA = -2,     /* a CUDA runtime/driver call failed */
  MIVOS_ERR_DEVICE = -3,   /* not an sm_90 device */
  MIVOS_ERR_KERNEL = -4    /* a kernel raised its error flag (bounded wait expired, overflow) */
};

/* Library / device ------------------------------------------------------------------------- */
#define MIVOS_ABI_VERSION 4 /* 2: element-type flags (fp16 / fp32 HALO maps) on the HALO operators;
                               3: + the S2M operators (stem_gather_frames ... halo_upsample_to_plane);
                               4: + attention_weights (get_W); batched forms for lock-step clips: query sets
                                  (memory_read q_div), groups (stem_gather, upsample4x_sigmoid_aggregate),
                                  skip_n (upsample2x_add) */
/* Largest object count of one clip: the u8 label map holds K objects + background.  The memory read takes up to
 * 256 object banks per call; the aggregation kernels of mivos_upsample4x_sigmoid_aggregate / mivos_aggregate_wbg
 * hold a pixel's objects in registers and take up to 16; their *_planes forms take any count up to this. */
#define MIVOS_MAX_OBJECTS 255
MIVOS_API int mivos_abi_version(void);
MIVOS_API const char* mivos_last_error(void);
/* MIVOS_OK iff the current device is compute capability 9.0 (there is no other code path). */
MIVOS_API int mivos_check_device(void);
/* Reads (and clears) the device-side error flag set by kernels; synchronises `stream`. */
MIVOS_API int mivos_poll_kernel_error(mivos_stream_t stream, int* code_out);
/* Number of kernels this library has launched since load (bench.py's gpu_launches). */
MIVOS_API int64_t mivos_launch_count(void);
/* Accounts for kernels executed by replaying a CUDA graph captured from this library's launches. */
MIVOS_API int64_t mivos_add_launch_count(int64_t n);

/* Writes up to four int32 scalars into device memory from launch arguments (stream-ordered): the
 * per-frame bank counters (`dyn_slots`, `dyn_t` below) that a replayed CUDA graph reads.          */
MIVOS_API int mivos_store_i32(int32_t* dst, int n, int v0, int v1, int v2, int v3, mivos_stream_t stream);
/* The same for a whole frame of a replayed graph in ONE launch: up to 64 int64 words (device pointers that change
 * from frame to frame: `vals64` is read at call time) and up to 4 int32 words.                                     */
MIVOS_API int mivos_store_words(int64_t* dst64, int n64, const int64_t* vals64, int32_t* dst32, int n32,
                      int v0, int v1, int v2, int v3, mivos_stream_t stream);
/* n segment copies (16-byte multiples, 16-byte aligned) with ONE side read from device memory at run time: segment
 * i copies bytes[i] bytes from dyn[i] to fixed[i] (dyn_is_src != 0) or from fixed[i] to dyn[i]; dyn[i] == 0 skips it.
 * Recorded into the per-frame graph, it stages the frame's cached query features / delivers the result planes of
 * frame ti (InferenceCore.prob[:, ti], inference_core.py:194) without eager copies between graph replays.            */
MIVOS_API int mivos_copy_segments(const int64_t* fixed, const int64_t* dyn, const int64_t* bytes, int n,
                        int dyn_is_src, int64_t max_bytes, mivos_stream_t stream);
/* Result delivery to host volumes (InferenceCore(result_dev="cpu")): one launch delivers the result planes of every
 * clip of a tick, reading each plane once from device memory.  `table` holds MIVOS_DELIVER_WORDS int64 words per
 * clip, read on the device when the (captured) launch runs:
 *   [0] address of the clip's probability volume at frame ti, prob[0, ti] of [(K+1), T, 1, nh, nw] fp32; 0 skips
 *   [1] the volume's plane stride in elements (T * nh * nw)
 *   [2] address of the padded label map at frame ti ([T, 1, nh, nw] u8)
 *   [3] address of the unpadded label map at frame ti ([T, h, w] u8)
 *   [4] low 32 bits: index of the clip's first plane in `planes`; high 32 bits: its plane count K+1 (1 to 256)
 *   [5] pad_l | pad_t << 32      [6] h | w << 32      [7] unused
 * Clip c copies planes[first + j] (j < K+1) to its volume's plane j at frame ti in 16-byte stores, and writes the
 * frame's argmax over the K+1 planes (the first maximum wins, as mivos_argmax_unpad) padded and unpadded.  The
 * destinations may be host-mapped addresses (mivos_host_register); volume, stride and padded labels must be 16-byte
 * aligned.  A record whose plane count is out of range is skipped.  nh * nw must be a multiple of 16.           */
#define MIVOS_DELIVER_WORDS 8
MIVOS_API int mivos_deliver_planes(const float* planes, const int64_t* table, int clips, int nh, int nw,
                         mivos_stream_t stream);
/* Page-locks `bytes` of pageable host memory at `host` (cudaHostRegister, mapped and portable) and returns in
 * *dev_out the address kernels use for it (cudaHostGetDevicePointer; not assumed equal to `host`).  Host code
 * allocates the memory; the library allocates nothing.  mivos_host_unregister undoes it.                        */
MIVOS_API int mivos_host_register(void* host, int64_t bytes, void** dev_out);
MIVOS_API int mivos_host_unregister(void* host);

/* Convolution as implicit GEMM on wgmma (TF32 in, FP32 accumulate) ----------------------------
 * Replaces nn.Conv2d (+ eval BatchNorm2d folded into weight/bias, + ReLU, + residual add) as
 * used by model/propagation/modules.py:15-35,38-89,92-114, mod_resnet.py:76-112,
 * prop_net.py:14-31 and model/fusion_net.py:8-50.
 * out[r, out_coff + co] = act( bias[co] + sum_{t,ci} in[r + off(t), in_coff + ci] * w[t][co][ci]
 *                              (+ residual[r, res_coff + co]) )     for interior rows r only,
 * rows r index the HALO matrix of an (n, h, w) map; taps = 9 means 3x3/stride 1/pad 1 with
 * off(t) = (t/3 - 1)*(w+2) + (t%3 - 1); taps = 1 means a 1x1 conv or a pre-gathered (im2col)
 * matrix whose rows are HALO rows of the OUTPUT map; taps = 4 means four VERTICAL taps off(t) = (t-2)*(w+2)
 * over such a matrix (the 7x7/stride-2 stems through mivos_stem_gather_s2d).  cin_pad (K per tap) is a multiple of 32
 * (64 for fp16 operands), cout_pad a multiple of 32.  Weight is packed [taps][cout_pad][cin_pad]
 * in the operand type, bias [cout_pad] is always fp32.  Activations may be fp32 (TF32 MMAs) or
 * fp16 (the precision the reference GUI itself runs in: torch.cuda.amp.autocast,
 * interactive_gui.py:990); accumulation is always fp32.                                          */
typedef struct {
  const void* in;  /* fp32 or fp16 (in_f16) */
  int64_t in_rows; /* rows of the input matrix that exist (TMA zero-fills beyond) */
  int in_cstride;  /* floats per input row */
  int in_coff;     /* first input channel used */
  int n, h, w;     /* logical output map; HALO rows = n*(h+2)*(w+2) */
  int cin_pad;
  int taps;
  const void* weight;
  const float* bias;
  int cout;
  int cout_pad;
  void* out;  /* fp32 or fp16 (out_f16) */
  int out_cstride;
  int out_coff;
  const void* residual; /* optional, HALO with res_cstride/res_coff */
  int res_cstride;
  int res_coff;
  void* out_relu; /* optional second output: max(out, 0) */
  int out_relu_cstride;
  int out_relu_coff;
  int relu; /* bit 0: ReLU on the primary output; bit 1: round outputs to TF32 (rna) so the next
               conv's operand truncation is exact */
  int in_f16;  /* 1: `in` and `weight` are IEEE fp16 (kind::f16 MMAs, K per tap a multiple of 64);
                  0: fp32 storage, TF32 MMAs */
  int out_f16; /* 1: `out`, `residual`, `out_relu` are fp16 HALO maps; 0: fp32 */
  void* splitk_ws; /* optional split-K scratch (device, 256-byte aligned): lets layers whose row tiles
                      cannot fill the SMs split the K range of a tile over several CTAs; the fp32
                      partial tiles are parked here and summed (in a fixed order) by a second,
                      PDL-chained launch that applies the epilogue.  Must not be shared by launches
                      that may run concurrently.  NULL: never split. */
  int64_t splitk_ws_bytes; /* 64 KB reserved + partial tiles (48 MB covers every layer of cfg-5) */
} mivos_conv_args;
MIVOS_API int mivos_conv_gemm(const mivos_conv_args* a, mivos_stream_t stream);
/* The tile width (32/64/128/256) and split-K factor mivos_conv_gemm would use for `a` on a device
 * with `sms` SMs (0: the current device).  Pure host arithmetic: no pointer in `a` is dereferenced
 * (only tested for NULL), no device is needed when sms > 0.                                        */
MIVOS_API int mivos_conv_plan(const mivos_conv_args* a, int sms, int* bn, int* splits);
/* Tuning hook: force the plan of the following mivos_conv_gemm calls (process-wide; mivos_conv_plan
 * reports it).  (0, 0): automatic choice.  bn = 32/64/128/256, splits = 0: that output-channel tile
 * width, no split-K.  splits >= 2 (only with bn > 0): also that split-K factor; a call it applies to
 * then fails unless it attaches a workspace of at least 64 KB + tiles * splits * 128 * bn * 4 bytes
 * and splits <= taps * cin_pad / k-block (every split owns a non-empty K range).
 * Results do not depend on the tile width, bit for bit (tests/test_gpu_conv_plans.py); another split-K
 * factor is another fp32 summation order.                                                             */
MIVOS_API int mivos_conv_tile_override(int bn, int splits);
/* CTAs per SM (1 or 2) mivos_conv_gemm would run `a`'s plan with on a device with `sms` SMs (0: the
 * current device).  Two CTAs per SM take tiles of up to 64 columns: each one's fill and epilogue run
 * under the other's main loop.  The residency never changes the tile width or split-K factor, nor any
 * result bit.  Pure host arithmetic, like mivos_conv_plan.                                             */
MIVOS_API int mivos_conv_plan_residency(const mivos_conv_args* a, int sms, int* ctas);
/* Tuning hook: force the residency of the following mivos_conv_gemm calls (process-wide;
 * mivos_conv_plan_residency reports it).  0: automatic, 1 or 2 CTAs per SM.  2 is rejected while a
 * tile override forces a tile wider than 64 columns (and such a tile override while 2 is forced); a
 * call whose automatic tile is wider than 64 columns fails under 2.                                     */
MIVOS_API int mivos_conv_residency_override(int ctas);

/* Gather kernels that feed mivos_conv_gemm ---------------------------------------------------
 * Every HALO-map operator below takes an element-type flag (`f16`, `out_f16`, `src_f16` ...):
 * 0 = fp32 maps (TF32 conv path), 1 = IEEE fp16 maps.  NCHW tensors at the API boundary, the
 * key/value bank, query keys, logits and probabilities are always fp32.
 * 7x7/stride-2/pad-3 stem gather (modules.py:52-58 conv1 of MaskRGBEncoder with cat(frame,
 * mask, others), modules.py:80-82 conv1 of RGBEncoder).  frame NCHW [1,3,H,W]; masks NCHW
 * [K,1,H,W] or NULL (cin = 3: `frame` is then a BATCH [k_objects,3,H,W] of frames); `others` =
 * sum of the other objects' masks is formed on the fly (prop_net.py:150-157).  Output: matrix
 * [K*(H/2+2)*(W/2+2), kpad], k = (ky*7+kx)*cin + c.  `groups` > 1 (mask form only): that many independent
 * (frame, K masks) sets in one launch — the clips of a lock-step step — group g reading
 * frame + g*frame_gstride and masks + g*mask_gstride (strides in elements), output images group-major. */
MIVOS_API int mivos_stem_gather(const float* frame, const float* masks, int k_objects, int h, int w,
                      void* out, int kpad, int out_f16, int groups, int64_t frame_gstride,
                      int64_t mask_gstride, mivos_stream_t stream);
/* The same stems WITHOUT the 49-tap im2col matrix (54 MB per 480p frame).  A 7x7/stride-2/pad-3 convolution is a
 * 4x4/stride-1 convolution over the space-to-depth input S[(py,px,c), Y, X] = in[c, 2Y+py, 2X+px] (taps dy, dx in
 * -2..1; ky = 2dy+py+3, kx = 2dx+px+3, weight 0 where an index is -1).  This gather writes, for every HALO row (Y, X)
 * of the half-resolution OUTPUT map, the 2 x 8 input pixels the four horizontal taps read:
 *   out[row(Y,X), py*8*cin + j*cin + c] = in[c, 2Y+py, 2X-4+j],  j = 0..7 (zero outside the image; border rows zero)
 * — [rows, kpad >= 16*cin], 13 MB per 480p frame at cin 3 — and mivos_conv_gemm runs the four vertical taps
 * (taps = 4) as row shifts of that matrix with weights packed [dy][cout][py*8*cin + (dx+2)*2*cin + px*cin + c].
 * Same (frame | frame + K masks | groups) forms as mivos_stem_gather; cin = 3 or 5.                              */
MIVOS_API int mivos_stem_gather_s2d(const float* frame, const float* masks, int k_objects, int h, int w,
                          void* out, int kpad, int out_f16, int groups, int64_t frame_gstride,
                          int64_t mask_gstride, mivos_stream_t stream);
/* The K-mask form of mivos_stem_gather_s2d for objects [obj0, obj0 + n_obj) of the K only: out holds n_obj images,
 * image i being object obj0 + i with its "others" channel summed over ALL K masks except its own, in object order
 * (prop_net.py:150-157).  Runs a memorize in object chunks with the bits of the whole-clip gather.                */
MIVOS_API int mivos_stem_gather_s2d_range(const float* frame, const float* masks, int k_objects, int obj0, int n_obj,
                                int h, int w, void* out, int kpad, int out_f16, mivos_stream_t stream);
/* Generic strided gather from a HALO map: out[r_out, (ky*ks+kx)*c + ci] for kernel ks (1 or 3),
 * stride 2, pad ks/2 (mod_resnet.py:83-84,140-144 with stride=2).                               */
MIVOS_API int mivos_gather_s2(const void* in, int n, int h, int w, int c, int in_cstride, int ks,
                    void* out, int out_cstride, int f16, mivos_stream_t stream);
/* 3x3/stride-2/pad-1 max pool on HALO maps (mod_resnet.py:122).                                 */
MIVOS_API int mivos_maxpool3x3s2(const void* in, int n, int h, int w, int c, void* out, int f16,
                       mivos_stream_t stream);
/* x[r] += bilinear_x2(up)[r] on HALO maps, optional relu copy (modules.py:100-103 followed by
 * the F.relu at modules.py:29).  up is (n, h/2, w/2, c); x is (n, h, w, c).  With `skip` (skip_n HALO
 * maps, map j broadcast over images [j*n/skip_n, (j+1)*n/skip_n) like the reference's
 * `x + interpolate(up_f)` does for the batch-1 skip path of a frame) the result is
 * x = skip + bilinear_x2(up) instead.                                                              */
MIVOS_API int mivos_upsample2x_add(void* x, const void* up, int n, int h, int w, int c, void* x_relu,
                         const void* skip, int skip_n, int f16, mivos_stream_t stream);

/* Channel-window copy between HALO maps (torch.cat at prop_net.py:178-179, F.relu at
 * modules.py:29): dst[i, :, :, dst_coff:+c] = (relu?) src[i / (n / src_n), :, :, src_coff:+c] — src_n maps,
 * each broadcast over n / src_n consecutive images (src_n == n: plain copy; 1: one map for all).     */
MIVOS_API int mivos_halo_copy(const void* src, int src_n, int src_cstride, int src_coff, void* dst,
                    int dst_cstride, int dst_coff, int n, int h, int w, int c, int relu, int src_f16,
                    int dst_f16, mivos_stream_t stream);

/* Layout conversion at the API boundary ------------------------------------------------------ */
MIVOS_API int mivos_halo_to_nchw(const void* halo, int n, int h, int w, int cstride, int coff, int c,
                       float* nchw, int f16, mivos_stream_t stream);
MIVOS_API int mivos_nchw_to_halo(const float* nchw, int n, int h, int w, int c, void* halo, int cstride,
                       int coff, int relu, int f16, mivos_stream_t stream);
/* HALO channel window -> pixel-major [n][h*w][c] (no border): query keys for the memory read.  */
MIVOS_API int mivos_halo_to_pixels(const float* halo, int n, int h, int w, int cstride, int coff, int c,
                         float* out, mivos_stream_t stream);
/* HALO [K, h, w, cstride] (key at coff_k, value at coff_v) -> BANK slot t of K objects.        */
MIVOS_API int mivos_bank_write(const float* halo, int k_objects, int h, int w, int cstride, int coff_k,
                     int coff_v, float* bank_k, float* bank_v, int64_t slots_cap, int t,
                     const int32_t* dyn_t, mivos_stream_t stream);
/* Per-set form of mivos_bank_write: the K objects are `sets` consecutive sets of K / sets objects (the clips of a
 * lock-step step), and set s writes bank frame dyn_t[s] (DEVICE array of `sets` int32, read at run time; required).
 * t_max is the largest frame that may occur (capacity check); a set whose frame lies outside [0, t_max] writes
 * nothing.  `sets` must divide k_objects.                                                                          */
MIVOS_API int mivos_bank_write_sets(const float* halo, int k_objects, int sets, int h, int w, int cstride, int coff_k,
                          int coff_v, float* bank_k, float* bank_v, int64_t slots_cap, int t_max,
                          const int32_t* dyn_t, mivos_stream_t stream);
/* Reference-layout bank [K,C,T,h,w] -> BANK (used when a caller hands us torch tensors).        */
MIVOS_API int mivos_bank_from_nchw(const float* keys, const float* values, int k_objects, int t, int hw,
                         float* bank_k, float* bank_v, int64_t slots_cap, mivos_stream_t stream);

/* Space-time memory read — EvalMemoryReader.forward + softmax_w_g_top (prop_net.py:47-73,
 * 81-108): for every query pixel q, affinity over all `slots` bank slots (keys . qk / sqrt(128)),
 * top-k over the memory axis, softmax over the k survivors, value-weighted read-out.
 * qk: HALO-free pixel-major [sets][hw][128]; object o reads query set o / q_div (q_div = 0: every object
 * reads set 0, the reference's one query frame per call; lock-step clips pass q_div = K objects per clip
 * and one set per clip, so the reads of C clips are ONE call).  out: HALO map channel block (n = K objects)
 * or pixel-major when out_halo_w == 0.  Never materialises the [slots, hw] affinity.
 * `workspace` sized by mivos_memory_read_workspace().  If topk_idx/topk_val are non-NULL they
 * receive the selected slot indices (int32, descending score order, [K][hw][k]) and scores.
 * dyn_slots / dyn_t (optional DEVICE scalars): when non-NULL the live slot count / bank frame is
 * read on the device at run time and the host argument only sizes the launch (`slots` = bank
 * capacity, `t` = largest frame index) — this is what lets one captured CUDA graph serve every
 * frame of a pass while the bank grows.                                                          */
MIVOS_API int64_t mivos_memory_read_workspace(int k_objects, int64_t slots, int hw, int top_k);
MIVOS_API int mivos_memory_read(const float* bank_k, const float* bank_v, int64_t slots_cap,
                      int k_objects, int64_t slots, const float* qk, int hw, int q_div, int top_k,
                      void* out, int out_cstride, int out_coff, int out_halo_h, int out_halo_w,
                      int32_t* topk_idx, float* topk_val, void* workspace, int64_t workspace_bytes,
                      int algo, const int32_t* dyn_slots, int out_f16, mivos_stream_t stream);
/* Dense space-time memory read — EvalMemoryReader.forward with top_k=None (prop_net.py:99-102): for
 * every query pixel q, softmax over ALL `slots` live bank slots of keys . qk / sqrt(128), then the
 * value-weighted read-out (the full 2*(128+512)*slots*hw flops per object, on the tensor cores:
 * 3xTF32 scores, online softmax, TF32 P.V, a second launch merging the chunks of the memory axis).
 * Operands, query sets (q_div), output window (out_cstride / out_coff / out_halo_h,w, out_f16) and
 * dyn_slots as for mivos_memory_read; 1 <= slots <= slots_cap.  Slots at or past the live count take
 * no part (they may hold stale data or NaN).  The partition of the memory axis depends on hw alone,
 * so eager (slots = n) and graph-sized (dyn_slots = n) reads, one q_div call and the per-set calls,
 * and repeated calls give the same bits.  `workspace` sized by mivos_memory_read_dense_workspace()
 * for the bank capacity (256-byte aligned); returns -1 on bad arguments.                         */
MIVOS_API int64_t mivos_memory_read_dense_workspace(int k_objects, int64_t slots_cap, int hw);
MIVOS_API int mivos_memory_read_dense(const float* bank_k, const float* bank_v, int64_t slots_cap,
                      int k_objects, int64_t slots, const float* qk, int hw, int q_div,
                      void* out, int out_cstride, int out_coff, int out_halo_h, int out_halo_w,
                      void* workspace, int64_t workspace_bytes, const int32_t* dyn_slots, int out_f16,
                      mivos_stream_t stream);
/* Wide top-k memory read — EvalMemoryReader.forward + softmax_w_g_top (prop_net.py:47-73, 81-108) for
 * 1 <= top_k <= 1024: the semantics of mivos_memory_read (exact fp32 scores, total order score desc /
 * slot asc, softmax over the k survivors, read-out in ascending slot order) and, for top_k <= 64, its
 * bits.  Operands, query sets, output window, dyn_slots and topk_idx / topk_val as for
 * mivos_memory_read; top_k <= slots <= slots_cap.  Scores are exact fp32 on CUDA cores: two histogram
 * sweeps find each query's threshold, a third emits the candidates, one CTA per query sorts them
 * (ties and near-ties beyond a query's candidate region: an exact radix select in that CTA).
 * `workspace` sized by mivos_memory_read_wide_workspace() (it depends on k_objects and hw alone;
 * 256-byte aligned); returns -1 on bad arguments.                                                  */
MIVOS_API int64_t mivos_memory_read_wide_workspace(int k_objects, int64_t slots_cap, int hw, int top_k);
MIVOS_API int mivos_memory_read_wide(const float* bank_k, const float* bank_v, int64_t slots_cap,
                      int k_objects, int64_t slots, const float* qk, int hw, int q_div, int top_k,
                      void* out, int out_cstride, int out_coff, int out_halo_h, int out_halo_w,
                      int32_t* topk_idx, float* topk_val, void* workspace, int64_t workspace_bytes,
                      const int32_t* dyn_slots, int out_f16, mivos_stream_t stream);
/* Per-set forms of the three reads: lock-step clips whose banks hold different numbers of live slots.  The
 * objects are `sets` consecutive sets of k_objects / sets (`sets` must divide k_objects); object o reads query
 * set o / (k_objects / sets) of qk [sets][hw][128] and the live slots 0 .. dyn_slots[s] - 1 of its own bank, where
 * dyn_slots is a DEVICE array of `sets` int32 counts read at run time (required).  `slots` (top_k <= slots <=
 * slots_cap; 1 <= slots for the dense read) sizes the launch and the workspace and bounds no count: each count is
 * clamped to slots_cap.  Slots at or past a set's count take no part in that set's read (they may hold stale data
 * or NaN).  Everything else — operands, output window, workspace sizes, topk_idx / topk_val, algo — is that of the
 * scalar form; with every count equal to n a per-set read gives the bits of the scalar read with dyn_slots = n and
 * q_div = k_objects / sets.  A count below top_k (`slots` bounds no count) selects every live slot: topk_idx is padded
 * with -1 and topk_val with 0 past them, the read-out is the softmax over the live slots, and a count of 0 writes
 * zeros; the top-k and wide reads give the same bits there as well (top_k <= 64).                                  */
MIVOS_API int mivos_memory_read_sets(const float* bank_k, const float* bank_v, int64_t slots_cap,
                      int k_objects, int64_t slots, const float* qk, int hw, int sets, int top_k,
                      void* out, int out_cstride, int out_coff, int out_halo_h, int out_halo_w,
                      int32_t* topk_idx, float* topk_val, void* workspace, int64_t workspace_bytes,
                      int algo, const int32_t* dyn_slots, int out_f16, mivos_stream_t stream);
MIVOS_API int mivos_memory_read_dense_sets(const float* bank_k, const float* bank_v, int64_t slots_cap,
                      int k_objects, int64_t slots, const float* qk, int hw, int sets,
                      void* out, int out_cstride, int out_coff, int out_halo_h, int out_halo_w,
                      void* workspace, int64_t workspace_bytes, const int32_t* dyn_slots, int out_f16,
                      mivos_stream_t stream);
MIVOS_API int mivos_memory_read_wide_sets(const float* bank_k, const float* bank_v, int64_t slots_cap,
                      int k_objects, int64_t slots, const float* qk, int hw, int sets, int top_k,
                      void* out, int out_cstride, int out_coff, int out_halo_h, int out_halo_w,
                      int32_t* topk_idx, float* topk_val, void* workspace, int64_t workspace_bytes,
                      const int32_t* dyn_slots, int out_f16, mivos_stream_t stream);

/* Object-group forms: lock-step clips with different object counts.  A batch of `maps` object maps (k_objects for
 * the reads) is split into `groups` runs of consecutive maps by `first`, a DEVICE array of groups + 1 int32 entries
 * read at run time (required): the exclusive prefix sums of the groups' object counts, so group g owns maps
 * [first[g], first[g+1]) and first[groups] = maps.  1 <= groups <= maps.  The host cannot check the table: a map
 * that no group inside [0, maps] holds (an empty group, a group past `maps`, a table that is not ascending) takes
 * part in nothing and never causes a fault; a table that is not ascending may also make groups overlap, and the
 * maps they share then get the (racing) result of either group — never a write outside the operands.  With the uniform table first = [0, K, 2K, ...] each form gives the bits
 * of the per-set / groups / skip_n / src_n form it generalises.
 * - the three reads: object o of group g reads query set g of qk [groups][hw][128] and the live slots
 *   0 .. dyn_slots[g] - 1 of its own bank (one count per group); everything else as the per-set forms.  An object in
 *   no group reads no slot.
 * - mivos_bank_write_groups: group g writes its maps to bank frame dyn_t[g] (outside [0, t_max]: nothing).
 * - mivos_stem_gather_s2d_groups (the memorize stem, kpad >= 80): image i, object j = i - first[g] of group g, reads
 *   frame g (frames frame_gstride floats apart) and the PACKED planes [maps + groups, H, W] of `planes`: group g's
 *   background plane first[g] + g, then its objects; the "others" channel sums group g's other objects only.
 * - mivos_upsample2x_add_groups (`skip` required) / mivos_halo_copy_groups: skip / source map g is broadcast over the
 *   images of group g (the HALO maps of n images; an image in no group is not written).
 * - mivos_upsample4x_sigmoid_aggregate_groups: the register kernel of mivos_upsample4x_sigmoid_aggregate within each
 *   group of at most 16 maps (maps <= 16 * groups; a larger group writes nothing): raw_out plane first[g] + j,
 *   prob_out PACKED planes [maps + groups, 1, H, W], group g's background at first[g] + g, then its objects.       */
MIVOS_API int mivos_memory_read_groups(const float* bank_k, const float* bank_v, int64_t slots_cap,
                      int k_objects, int64_t slots, const float* qk, int hw, int groups, const int32_t* first,
                      int top_k, void* out, int out_cstride, int out_coff, int out_halo_h, int out_halo_w,
                      int32_t* topk_idx, float* topk_val, void* workspace, int64_t workspace_bytes,
                      int algo, const int32_t* dyn_slots, int out_f16, mivos_stream_t stream);
MIVOS_API int mivos_memory_read_dense_groups(const float* bank_k, const float* bank_v, int64_t slots_cap,
                      int k_objects, int64_t slots, const float* qk, int hw, int groups, const int32_t* first,
                      void* out, int out_cstride, int out_coff, int out_halo_h, int out_halo_w,
                      void* workspace, int64_t workspace_bytes, const int32_t* dyn_slots, int out_f16,
                      mivos_stream_t stream);
MIVOS_API int mivos_memory_read_wide_groups(const float* bank_k, const float* bank_v, int64_t slots_cap,
                      int k_objects, int64_t slots, const float* qk, int hw, int groups, const int32_t* first,
                      int top_k, void* out, int out_cstride, int out_coff, int out_halo_h, int out_halo_w,
                      int32_t* topk_idx, float* topk_val, void* workspace, int64_t workspace_bytes,
                      const int32_t* dyn_slots, int out_f16, mivos_stream_t stream);
MIVOS_API int mivos_bank_write_groups(const float* halo, int maps, int groups, const int32_t* first, int h, int w,
                      int cstride, int coff_k, int coff_v, float* bank_k, float* bank_v, int64_t slots_cap,
                      int t_max, const int32_t* dyn_t, mivos_stream_t stream);
MIVOS_API int mivos_stem_gather_s2d_groups(const float* frame, const float* planes, int maps, int groups,
                      const int32_t* first, int h, int w, void* out, int kpad, int out_f16, int64_t frame_gstride,
                      mivos_stream_t stream);
MIVOS_API int mivos_upsample2x_add_groups(void* x, const void* up, int n, int h, int w, int c, void* x_relu,
                      const void* skip, int groups, const int32_t* first, int f16, mivos_stream_t stream);
MIVOS_API int mivos_halo_copy_groups(const void* src, int groups, const int32_t* first, int src_cstride,
                      int src_coff, void* dst, int dst_cstride, int dst_coff, int n, int h, int w, int c, int relu,
                      int src_f16, int dst_f16, mivos_stream_t stream);
MIVOS_API int mivos_upsample4x_sigmoid_aggregate_groups(const float* logits, int maps, int groups,
                      const int32_t* first, int h4, int w4, int cstride, int coff, float* raw_out, float* prob_out,
                      mivos_stream_t stream);
/* Diagnostic, synchronising: candidate statistics of the last tensor-core-path read in `workspace`:
 * out[0] total candidates, out[1] max per (object, query), out[2] queries served by the exact
 * fallback, out[3] splits of the memory axis.                                                    */
MIVOS_API int mivos_memory_read_stats(const void* workspace, int k_objects, int64_t slots, int hw, int top_k,
                            int64_t* out);
enum { MIVOS_MEMREAD_AUTO = 0, MIVOS_MEMREAD_EXACT_SIMT = 1, MIVOS_MEMREAD_TCGEN05 = 2 };  /* (name kept for ABI stability: the tensor-core candidate path, wgmma on sm_90) */

/* Decoder tail + soft aggregation — prop_net.py:30 (bilinear x4, align_corners=False),
 * prop_net.py:181 (sigmoid) and aggregate_wbg (aggregate.py:22-37, keep_bg=True).
 * logits: HALO (K, h4, w4, cstride) channel coff.  prob_out NCHW [(K+1),1,4*h4,4*w4].
 * raw_out (optional) NCHW [K,1,H,W] = sigmoid(upsampled) before aggregation.  `groups` G > 1: G independent
 * sets of K objects in one launch (the clips of a lock-step step): logits (G*K, ...), raw_out [G*K,...],
 * prob_out [G,(K+1),1,H,W]; the aggregation runs within a set.                                    */
MIVOS_API int mivos_upsample4x_sigmoid_aggregate(const float* logits, int k_objects, int h4, int w4,
                                       int cstride, int coff, float* raw_out, float* prob_out, int groups,
                                       mivos_stream_t stream);
/* aggregate_wbg on NCHW probabilities [K,1,H,W] -> [(K+1),1,H,W] (aggregate.py:22-37).
 * hard bit 0 multiplies the logits by 1000; hard bit 1 uses the constant 0.5 background of
 * aggregate_sbg (aggregate.py:4-20); keep_bg == 0 drops row 0 from the output.                  */
MIVOS_API int mivos_aggregate_wbg(const float* prob, int k_objects, int64_t hw, int keep_bg, int hard,
                        float* out, mivos_stream_t stream);
/* The same two operators for 1 <= K <= MIVOS_MAX_OBJECTS, with no per-thread object arrays: the sigmoid
 * planes are written first (the object planes of prob_out) and the aggregation makes per-pixel passes over
 * them — background product, logits and their maximum, exp-sum, normalisation — in the operation order of the
 * register kernels, whose bits they give for K <= 16.  prob_out may not alias raw_out.                       */
MIVOS_API int mivos_upsample4x_sigmoid_aggregate_planes(const float* logits, int k_objects, int h4, int w4,
                                              int cstride, int coff, float* raw_out, float* prob_out, int groups,
                                              mivos_stream_t stream);
MIVOS_API int mivos_aggregate_wbg_planes(const float* prob, int k_objects, int64_t hw, int keep_bg, int hard,
                               float* out, mivos_stream_t stream);
/* argmax over the K+1 rows of prob [(K+1), T, 1, nh, nw] for frame range, fused with unpad:
 * writes masks_padded [T,1,nh,nw] u8 and (optional) masks_out [T,h,w] u8
 * (inference_core.py:259-269).                                                                  */
MIVOS_API int mivos_argmax_unpad(const float* prob, int k_plus_1, int t, int nh, int nw, int pad_l,
                       int pad_t, int h, int w, uint8_t* masks_padded, uint8_t* masks_out,
                       mivos_stream_t stream);
/* Frame ingest — images_to_torch (interact/interactive_utils.py:18-23) / ToTensor + im_normalization
 * (dataset/davis_test_dataset.py:49-52, dataset/range_transform.py:5-8): u8 frames [t,h,w,3] ->
 * normalised fp32 [t,3,h,w]; bit-identical to `x.float()/255` then `(x - mean) / std` on the CPU.  */
MIVOS_API int mivos_frames_u8_normalize(const uint8_t* frames_hwc, int t, int h, int w, float* out,
                              mivos_stream_t stream);
/* pad_divide_by / unpad (util/tensor_util.py:62-87) on [planes, h, w] fp32.                     */
MIVOS_API int mivos_pad2d(const float* in, int planes, int h, int w, int pad_l, int pad_r, int pad_t,
                int pad_b, float* out, mivos_stream_t stream);

/* Fusion attention — PropagationNetwork.get_attention / AttentionMemory.forward
 * (prop_net.py:115-129,187-200): W = softmax over the memory axis of mk^T qk / sqrt(128)
 * (T = 1, no top-k); area-pool pos/neg [1,1,H,W] by 16; row-vector @ W; bilinear to (H,W).
 * mk, qk pixel-major [hw][128]; out NCHW [1,2,H,W].  scratch: 4*hw floats.                           */
MIVOS_API int mivos_attention_map(const float* mk, const float* qk, int h16, int w16, const float* pos,
                        const float* neg, float* out, float* scratch, mivos_stream_t stream);
/* PropagationNetwork.get_W (prop_net.py:183) = AttentionMemory.forward (prop_net.py:115-129): the
 * affinity itself, w_out[i][j] = softmax over memory pixels i of mk[i] . qk[j] / sqrt(128), [hw][hw]
 * fp32 row-major.  mk, qk pixel-major [hw][128]; scratch: 4*hw floats.                            */
MIVOS_API int mivos_attention_weights(const float* mk, const float* qk, int hw, float* w_out, float* scratch,
                            mivos_stream_t stream);
/* Whether mivos_attention_map / mivos_attention_weights take hw key pixels: *resident = 1 when one logit row per
 * query of the CTA fits their shared-memory tile (hw <= 6912), 0 otherwise.  Pure host arithmetic, no device.     */
MIVOS_API int mivos_attention_plan(int hw, int* resident);
/* The same two operators for ANY hw >= 1 (a 1080p frame pads to 68 x 120 = 8160 key pixels, 4K to 135 x 240):
 * prop_net.py:115-129,187-200 (get_attention) and prop_net.py:183 (get_W), same arguments, layouts and scratch
 * (4*hw floats) as mivos_attention_map / mivos_attention_weights.  The memory keys are streamed through shared
 * memory in tiles and the softmax over the memory axis is computed online (running maximum, partial sums
 * rescaled when it grows); the logits are the same fp32 fma chains as the resident kernel's.  The weights form
 * makes one such pass for the column maximum and denominator, then writes w_out row by row.                    */
MIVOS_API int mivos_attention_map_streamed(const float* mk, const float* qk, int h16, int w16, const float* pos,
                                 const float* neg, float* out, float* scratch, mivos_stream_t stream);
MIVOS_API int mivos_attention_weights_streamed(const float* mk, const float* qk, int hw, float* w_out,
                                     float* scratch, mivos_stream_t stream);
/* FusionNet input gather (fusion_net.py:35-40): cat(im, seg1, seg2, attn, time) -> HALO
 * (1, H, W, cpad) with channels 9..cpad-1 zero.                                                 */
MIVOS_API int mivos_fusion_gather(const float* im, const float* seg1, const float* seg2, const float* attn,
                        float nc, float nr, int h, int w, void* out_halo, int cpad, int f16,
                        mivos_stream_t stream);
/* sigmoid of a HALO logit channel into an NCHW plane (inference_core.py:214).                   */
MIVOS_API int mivos_halo_sigmoid_to_plane(const float* halo, int h, int w, int cstride, int coff,
                                float* plane, mivos_stream_t stream);

/* Scribble-to-Mask network (S2M, SURVEY.md 8f-3): the DeepLabV3+ head and dilated ResNet-50 stage of
 * model/s2m reuse mivos_conv_gemm; these are the HBM-bound operators around it. ------------------
 * 7x7/stride-2/pad-3 stem gather of a BATCH of cin-channel NCHW images [n,cin,H,W], cin = 3 or 6
 * (s2m_resnet.py:93-94: the 6-channel conv1 over cat(image, previous mask, +/- scribbles),
 * davis_processor.py:66 / interact/s2m_controller.py:34).  Output as mivos_stem_gather.          */
MIVOS_API int mivos_stem_gather_frames(const float* frames, int n, int cin, int h, int w, void* out, int kpad,
                             int out_f16, mivos_stream_t stream);
/* Whether mivos_stem_gather_frames takes cin-channel frames w pixels wide: *untiled = 1 when 7 whole input rows
 * fit its shared memory (cin 6: w <= 1376 in fp32, w <= 2760 in fp16), 0 otherwise.  Pure host arithmetic.       */
MIVOS_API int mivos_stem_frames_plan(int cin, int w, int out_f16, int* untiled);
/* mivos_stem_gather_frames for the 6-channel S2M stem (s2m_resnet.py:93-94) at ANY frame width: the output row
 * is gathered in windows of output columns, each staging only the input columns it reads (zero padding at the
 * image edges only).  Same output matrix as mivos_stem_gather_frames, bit for bit.                              */
MIVOS_API int mivos_stem_gather_frames_tiled(const float* frames, int n, int h, int w, void* out, int kpad,
                                   int out_f16, mivos_stream_t stream);
/* Dilated 3x3/stride-1/pad=dilation gather from a HALO map into an im2col matrix whose rows are
 * the HALO rows of the output map: out[r, (ky*3+kx)*c + ci] (s2m_resnet.py:19-20 conv3x3 with
 * dilation 2 in layer4; _deeplab.py:119-124 ASPPConv with rates 6/12/18).                        */
MIVOS_API int mivos_gather_dilated(const void* in, int n, int h, int w, int c, int in_cstride, int dilation,
                         void* out, int out_cstride, int f16, mivos_stream_t stream);
/* AdaptiveAvgPool2d(1) + bilinear resize of the 1x1 map back to (h, w) (_deeplab.py:126-138):
 * out[i, y, x, out_coff + ch] = mean over the interior pixels of in[i, :, :, in_coff + ch].      */
MIVOS_API int mivos_halo_avgpool_broadcast(const void* in, int n, int h, int w, int c, int in_cstride, int in_coff,
                                 void* out, int out_cstride, int out_coff, int f16, mivos_stream_t stream);
/* Bilinear resize (align_corners=False, F.interpolate(size=...)) of a HALO map (n,hs,ws) channel
 * window into a channel window of a HALO map (n,h,w) (_deeplab.py:50-52: resize + torch.cat).    */
MIVOS_API int mivos_upsample_bilinear(const void* src, int n, int hs, int ws, int src_cstride, int src_coff,
                            void* dst, int h, int w, int dst_cstride, int dst_coff, int c, int f16,
                            mivos_stream_t stream);
/* One fp32 HALO channel (n,hs,ws) -> NCHW planes [n,1,out_h,out_w], bilinear (align_corners=False),
 * optionally through a sigmoid (model/s2m/utils.py:20; davis_processor.py:68).                   */
MIVOS_API int mivos_halo_upsample_to_plane(const float* halo, int n, int hs, int ws, int cstride, int coff,
                                 int out_h, int out_w, int apply_sigmoid, float* out, mivos_stream_t stream);

/* Mask egress (SURVEY.md 8f-4): overlay_davis / overlay_davis_fade, the GUI's per-frame display
 * composite (interact/interactive_utils.py:119-143).  image u8 [t,h,w,3], mask u8 [t,h,w] labels,
 * colors u8 [ncolors,3] (the GUI table has 7 rows; the reference raises on a label beyond its table,
 * here such a label takes colour 0).  Labelled pixels: trunc(image*alpha + (1-alpha)*colour) in
 * float64; the 4-connected outer contour of the labelled region: 0; fade: other pixels * 0.6.      */
MIVOS_API int mivos_overlay_davis(const uint8_t* image_hwc, const uint8_t* mask, int t, int h, int w,
                        const uint8_t* colors, int ncolors, double alpha, int fade, uint8_t* out,
                        mivos_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* MIVOS_B200_H_ */
