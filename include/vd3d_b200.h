/*
 * vd3d_b200.h — C ABI of libvd3d_b200.so: hand-written sm_90a (H100) kernels for visualDet3D's inference hot path.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless the name ends in _host; `stream` is a cudaStream_t passed as void*.
 *   - activations are fp32, "NHWC" = [B][H][W][C] with an explicit channel pitch (`*_cs`, floats between two
 *     pixels) and channel offset (`*_co`) so a kernel can read / write a channel slice of a wider tensor
 *     (this is how every torch.cat on the path is fused away).
 *   - every entry returns 0 on success, a negative VD3D_E* code otherwise; it never exits the process
 *     (the reference's iou3d.cpp:13-21 CHECK_ERROR calls exit()).  vd3d_last_error() gives the message.
 *   - all launches are asynchronous on `stream`; no entry synchronises unless documented.
 *
 * Reference interfaces replaced (R/ = visualDet3D/networks in the reference tree) are cited per entry.
 */
#ifndef VD3D_B200_H
#define VD3D_B200_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VD3D_OK 0
#define VD3D_EINVAL -1   /* bad argument (shape / alignment / unsupported configuration) */
#define VD3D_ECUDA -2    /* CUDA runtime / launch error */
#define VD3D_ECAP -3     /* fixed-capacity buffer overflow (reported through a device flag, see decode) */

const char* vd3d_last_error(void);
int vd3d_version(void);
/* number of kernel launches issued through this library since the last reset (bench.py's gpu_launches) */
long long vd3d_launch_count(void);
void vd3d_launch_count_reset(void);

/* ---- layout helpers -------------------------------------------------------------------------------------- */
/* [B][C][H][W] -> [B][H][W][out_cs] (+out_co).  Input side of the detectors (testers.py:24-25,39 hand NCHW). */
int vd3d_nchw_to_nhwc(const float* in, float* out, int B, int C, int H, int W, int out_cs, int out_co, void* stream);
/* [B][H][W][in_cs](+in_co) -> [B][C][H][W].  Used by the NCHW-facing op mirrors and the tests. */
int vd3d_nhwc_to_nchw(const float* in, float* out, int B, int C, int H, int W, int in_cs, int in_co, void* stream);

/* ---- dense convolution (SIMT fp32 implicit GEMM) ----------------------------------------------------------
 * Replaces nn.Conv2d + folded eval-mode BatchNorm2d (+ReLU) (+residual add) as used by
 * R/backbones/resnet.py:23-91,184-198, R/lib/ghost_module.py:27-31, R/lib/blocks.py:24-43,
 * R/heads/detection_3d_head.py:47-82,500-533.
 *   in   : NHWC [B][H][W] pitch in_cs, channels [in_co, in_co+Cin)
 *   wgt  : [KH*KW*Cin][Cout]  (k = (kh*KW + kw)*Cin + ci), BN scale already folded in
 *   bias : [Cout] (folded BN shift + conv bias) or NULL
 *   res  : optional residual NHWC (same spatial size as out), added before the ReLU
 *   out  : NHWC [B][Ho][Wo] pitch out_cs, channels [out_co, out_co+Cout)
 *   Ho = (H + 2*pad - dil*(KH-1) - 1)/stride + 1 (same for Wo).  Requires Cout % 4 == 0, pitches/offsets % 4 == 0.
 */
int vd3d_conv2d_nhwc(const float* in, int B, int H, int W, int Cin, int in_cs, int in_co,
                     const float* wgt, const float* bias, int KH, int KW, int stride, int pad, int dil,
                     const float* res, int res_cs, int res_co,
                     float* out, int Cout, int out_cs, int out_co, int relu, void* stream);

/* ---- dense convolution (wgmma tensor cores, "3xTF32" split accumulation) ----------------------------------------
 * Same op as vd3d_conv2d_nhwc for stride-1 convs with Cin % 32 == 0 and Cout % 16 == 0, on the Hopper tensor cores:
 * operands staged by TMA (4-D box per filter tap, zero padding = TMA out-of-bounds fill), wgmma kind tf32 with the
 * fp32 accumulator in registers.  fp32-grade accuracy comes from splitting every operand v = hi + lo with
 * hi = v & 0xFFFFE000 (what the MMA reads when handed v) and accumulating A*Whi + Alo*Whi + A*Wlo (passes = 3).
 *   in / in_lo   : NHWC activation and its lo companion (in_lo may be NULL when passes == 1)
 *   w_hi / w_lo  : [Cout][KH*KW*Cin] (k = (kh*KW + kw)*Cin + ci), BN folded, split on the host
 *   out / out_lo : NHWC result and (optional) its lo companion, written by the epilogue
 *   bn           : output-channel tile (multiple of 16, <= 256; tiles wider than 128 run as two equal halves); 0 = vd3d_tc_pick_bn(Cout)
 * passes == 1 is plain single-pass TF32 (diagnostics only: ~1e-3 relative error, not parity-grade). */
int vd3d_tc_pick_bn(int Cout);
/* tile width of the persistent fp16-split engine (default of vd3d_conv2d_tc16 when bn == 0): Cout split evenly into
 * ceil(Cout / 128) tiles of 16-column granules (128 columns: the widest accumulator the consumer warpgroups hold in registers) */
int vd3d_tc_pick_bn_persistent(int Cout);
int vd3d_conv2d_tc(const float* in, const float* in_lo, int B, int H, int W, int Cin, int in_cs, int in_co,
                   const float* w_hi, const float* w_lo, const float* bias, int KH, int KW, int pad, int dil,
                   const float* res, int res_cs, int res_co,
                   float* out, float* out_lo, int Cout, int out_cs, int out_co, int relu, int passes, int bn, void* stream);
/* Same convolution with fp16-split operands ("3xFP16"): every operand v is kept as two fp16 planes hi = rn16(v), lo = rn16(v - hi)
 * (22 significant bits); three kind::f16 MMAs per k-step (Alo*Whi + Ahi*Wlo + Ahi*Whi), 64 channels per k-block: half the
 * shared-memory / L2 operand bytes and twice the MMA rate of the tf32 form at the same accuracy.  Weights are pre-scaled by a
 * power of two S on the host (so that their lo parts stay normal fp16 numbers); out_scale = 1/S is applied to the accumulator.
 * One launch runs the conv over L <= 5 tensors of different sizes ("levels": the shared-weight RetinaNet head over the pyramid, whole
 * batch; L = 1 for an ordinary conv).  Every tensor argument is an array of L pointers, one per level; the M tiles of all levels form one
 * persistent tile schedule, bit-identical to L separate launches (same K order per output pixel).
 *   in_hi / in_lo     : fp16 NHWC planes [B][H[l]][W[l]] with the same pitch / offset convention as the fp32 tensors (each level its own padding)
 *   w_hi / w_lo       : fp16 [Cout][KH*KW*cin_pad], cin_pad = Cin rounded up to 64 (zero filled)
 *   out               : fp32 NHWC result (NULL: not written); out_hi16 / out_lo16 (optional pair): its fp16 planes for the next conv.
 *                       Between two tensor-core convs an activation may exist as its planes only: half the output bytes of a layer.
 *   res               : optional fp32 residual; res_W[l] > 0 (res_H / res_W may be NULL): level l's residual is [B][res_H[l]][res_W[l]] at
 *                       exactly half the output size, added nearest-upsampled (the FPN top-down add, R/detectors/retinanet_2d.py:49-52)
 *   res_hi16 / res_lo16: or the residual as fp16 planes (value = hi + lo; L = 1, 3 passes); res_cs / res_co apply to either form
 *   passes            : 3, or 2 (error-budget experiments: the A_lo * W_hi product dropped); bn <= 0: the library's tile policy
 * With L > 1 every output form (and res) of level l must lie at a whole-pixel offset from level 0's, the same for all forms (levels
 * concatenated in one allocation per form).  stride 1..4 (strided convs load every stride-th pixel through the TMA traversal stride);
 * Cin % 8 == 0, Cout % 4 == 0. */
int vd3d_conv2d_tc16(int L, const void* const* in_hi, const void* const* in_lo, const int* H, const int* W, int B, int Cin, int in_cs,
                     int in_co, const void* w_hi, const void* w_lo, float out_scale, const float* bias, int KH, int KW, int pad,
                     int dil, int stride, const void* const* res, const void* const* res_hi16, const void* const* res_lo16,
                     const int* res_H, const int* res_W, int res_cs, int res_co,
                     const void* const* out, const void* const* out_hi16, const void* const* out_lo16,
                     int Cout, int out_cs, int out_co, int relu, int passes, int bn, void* stream);
/* Few-channel KHxKW convolution (the ResNet / DLA stem: conv1 7x7 stride 2, R/backbones/resnet.py:120,186) on the tensor cores.
 * The image is held as fp16 (hi, lo) planes [B][H][Wp][4] (pixel x at column x + pad, zeros elsewhere: the buffer must be
 * zero-initialised once); Wp = vd3d_stem_row_pitch(W, KW, stride, pad).  vd3d_image_to_h16_rows fills the planes from an
 * NCHW fp32 image (C <= 4; xoff = pad).  `win` = window elements per filter row (32: 8 pixels, 64-byte swizzle rows; 64: 16 pixels,
 * 128-byte rows), win >= 4 * KW.  Weights: fp16 (hi, lo) [Cout][KH][win] with column kw*4 + c (zero beyond KW*4 and for c >= C),
 * scaled by a power of two like vd3d_conv2d_tc16; even stride, Cout % 16 == 0, Cout <= 256. */
int vd3d_stem_row_pitch(int W, int KW, int stride, int pad);
int vd3d_image_to_h16_rows(const float* img_nchw, int B, int C, int H, int W, void* hi16, void* lo16, int Wp, int xoff, void* stream);
int vd3d_conv2d_tc16_stem(const void* in_hi, const void* in_lo, int B, int H, int W, int Wp, int KH, int KW, int stride, int pad, int win,
                          const void* w_hi, const void* w_lo, float out_scale, const float* bias,
                          float* out, void* out_hi16, void* out_lo16, int Cout, int out_cs, int out_co, int relu, void* stream);
/* Stem conv + BN + ReLU + MaxPool2d(kernel 3, stride 2, padding 1) in ONE kernel (R/backbones/resnet.py:186-189): same inputs as
 * vd3d_conv2d_tc16_stem; the conv output is never written: every 8 x 16 tile is pooled in shared memory by the epilogue and only the pooled
 * tensor pool_out NHWC [B][(Ho + 1) / 2][(Wo + 1) / 2][pool_cs] (channels [pool_co, pool_co + 64)) goes to HBM (pooled positions whose window
 * straddles two tiles are combined with atomicMax on the bit pattern: exact because of the ReLU).  Cout == 64. */
int vd3d_conv2d_tc16_stem_pool(const void* in_hi, const void* in_lo, int B, int H, int W, int Wp, int KH, int KW, int stride, int pad, int win,
                               const void* w_hi, const void* w_lo, float out_scale, const float* bias,
                               float* pool_out, int Cout, int pool_cs, int pool_co, void* stream);
/* The ResNet stem as one persistent row-strip kernel (stem_pool_kernel, csrc/row_conv.cu): conv 7x7 / stride 2 / pad 3 (<= 4 -> 64 channels) + folded BN + ReLU +
 * MaxPool2d(3, 2, 1) (R/networks/backbones/resnet.py:120-122,186-189).  Replaces vd3d_conv2d_tc16_stem_pool: no window re-reads (the wgmma
 * descriptor walks the overlapping 8-pixel windows inside one staged image row), no atomics, pooled tensor written as fp32 (`out`, may be
 * NULL) and / or fp16 (hi, lo) planes (may be NULL) NHWC [B][Hq][Wq][out_cs], channels [out_co, out_co + 64).
 * in_hi / in_lo: row planes [B][H][Wp][4] made by vd3d_image_to_h16_rows with xoff = vd3d_stem_pool_xoff() and Wp = vd3d_stem_pool_row_pitch(W)
 * (the buffer must be zero outside the image columns); w_hi / w_lo: the [64][7 * 32] matrices of the 32-element-window stem.
 * Results are bit-identical to vd3d_conv2d_tc16_stem + vd3d_maxpool3x3s2_nhwc. */
int vd3d_stem_pool_row_pitch(int W);
int vd3d_stem_pool_xoff(void);
int vd3d_stem_pool_fused(const void* in_hi, const void* in_lo, int B, int H, int W, int Wp, const void* w_hi, const void* w_lo, float out_scale,
                         const float* bias, float* out, void* out_hi16, void* out_lo16, int out_cs, int out_co, void* stream);
/* Few-channel convolutions on the tensor cores as row-strip kernels (csrc/row_conv.cu): the DLA-34 front end (base_layer 7x7 3 -> 16, level0 3x3
 * 16 -> 16, level1 3x3 / 2 16 -> 32; R/networks/backbones/dla.py:246-262), i.e. the layers with Cin < 32 that vd3d_conv2d_tc16 does not take.
 * Input: fp16 (hi, lo) ROW PLANES [B][H][Wp][pc] (pc = 4, 8 or 16 channels per pixel, image column x at pixel xoff + x, xoff >= pad, zero outside the
 * image columns; Wp >= vd3d_row_conv_pitch(...)); weights [N][KH * KS * 16] fp16 (hi, lo), k = ky * KS * 16 + kx * pc + c, KS = 2 if KW * pc <= 32 else 4,
 * scaled by a power of two undone by out_scale; N = 16 or 32.  Output: NHWC [B][Ho][out_W][out_cs] channels [out_co, out_co + N) as fp32 (may be NULL)
 * and / or fp16 (hi, lo) planes (may be NULL), image column x at out_xoff + x (so the output can be the next row conv's input planes).
 * vd3d_image_to_h16_rows_c: NCHW float image -> row planes with cpad = 4 or 8 channels per pixel. */
int vd3d_row_conv_pitch(int W, int pc, int KW, int S, int P, int xoff);
int vd3d_image_to_h16_rows_c(const float* img, int B, int C, int H, int W, void* hi16, void* lo16, int Wp, int xoff, int cpad, void* stream);
int vd3d_row_conv(const void* in_hi, const void* in_lo, int B, int H, int W, int Wp, int xoff, int pc, int KH, int KW, int S, int P,
                  const void* w_hi, const void* w_lo, float out_scale, const float* bias, int relu, int N,
                  float* out, void* out_hi16, void* out_lo16, int out_W, int out_xoff, int out_cs, int out_co, void* stream);
/* Diagnostics: when set, CTA 0 of every persistent tensor-core conv writes clock64 stamps into a [12][n] int64 device buffer: per k-block
 * 0 stage free / 1 loads issued / 2 MMA thread waits / 3 stage landed / 4 MMAs issued / 9 ring slot (a value, not a stamp), per tile
 * 5 last MMAs done / 6 staged and handed to the epilogue warps / 7 epilogue start / 8 stage released / 10 times the producer passed over
 * the held slot (a count) / 11 epilogue done; NULL disables (tools/trace_conv.py). */
void vd3d_tc_set_trace(void* dev_i64, int n);
/* fp32 channel slice -> fp16 (hi, lo) planes (producers that are not tensor-core convs). */
int vd3d_split_h16_nhwc(const float* in, void* hi16, void* lo16, long long npix, int C, int cs, int co, void* stream);
/* lo[pix][c] = in[pix][c] - (in[pix][c] & 0xFFFFE000) on a channel slice (producers that are not tensor-core convs). */
int vd3d_split_lo_nhwc(const float* in, float* lo, long long npix, int C, int cs, int co, void* stream);

/* depthwise 3x3 (stride 1, pad 1) + folded BN + ReLU: GhostModule.cheap_operation (R/lib/ghost_module.py:33-38).
 * wgt [9][C] (tap-major), bias [C]. */
int vd3d_dwconv3x3_nhwc(const float* in, int B, int H, int W, int C, int in_cs, int in_co,
                        const float* wgt, const float* bias, float* out, int out_cs, int out_co, int relu, void* stream);

/* nn.MaxPool2d(3, stride 2, pad 1) (R/backbones/resnet.py:123,190). */
int vd3d_maxpool3x3s2_nhwc(const float* in, int B, int H, int W, int C, int in_cs, int in_co,
                           float* out, int out_cs, int out_co, void* stream);
/* nn.AvgPool2d(2) (R/detectors/yolostereo3d_core.py:25,34). H, W even. */
int vd3d_avgpool2_nhwc(const float* in, int B, int H, int W, int C, int in_cs, int in_co,
                       float* out, int out_cs, int out_co, void* stream);
/* nn.MaxPool2d(2, stride=2) (DLA Tree.downsample, R/backbones/dla.py:203-204). */
int vd3d_maxpool2x2s2_nhwc(const float* in, int B, int H, int W, int C, int in_cs, int in_co,
                           float* out, int out_cs, int out_co, void* stream);
/* depthwise nn.ConvTranspose2d(C, C, 2f, stride=f, padding=f//2, groups=C, bias=False) (IDAUp.up_i, R/backbones/dla_utils.py:69-72)
 * with the `layers[i] + layers[i-1]` add of IDAUp.forward (:84) fused: out = up(in) + addend (addend may be NULL).
 * wgt [2f*2f][C] (tap-major); out is [B][H*f][W*f]. */
int vd3d_dw_convtranspose_nhwc(const float* in, int B, int H, int W, int C, int in_cs, int in_co, const float* wgt, int f,
                               const float* addend, int add_cs, int add_co, float* out, int out_cs, int out_co, void* stream);
/* channel-slice copy (the torch.cat legs that cannot be fused into a producer). */
int vd3d_copy_channels_nhwc(const float* in, int npix, int C, int in_cs, int in_co, float* out, int out_cs, int out_co, void* stream);

/* ---- stereo cost volumes ---------------------------------------------------------------------------------
 * PSMCosineModule.forward (R/lib/PSM_cost_volume.py:76-91):
 *   out[b,h,w,i] = (1/C) * sum_c L[b,h,w,c] * R[b,h,w-i,c]   if w >= i else 0,   i in [0, D)
 * L, R NHWC (pitch lr_cs, offset lr_co), out NHWC slice.  Algorithmic HBM bytes: 4*B*H*W*(2C + D). */
int vd3d_psm_cosine_nhwc(const float* L, const float* R, int B, int H, int W, int C, int lr_cs, int lr_co,
                         int D, float* out, int out_cs, int out_co, void* stream);
/* Same op on the reference's own layout: left/right [B][C][H][W] -> cost [B][D][H][W] (op-level mirror). */
int vd3d_psm_cosine_nchw(const float* L, const float* R, int B, int C, int H, int W, int D, float* out, void* stream);

/* PSMCosine on the tensor cores (R/lib/PSM_cost_volume.py:76-91), features given as the fp16 (hi, lo) planes the tensor-core
 * convs write (hi = rn16(v), lo = rn16(v - hi)); pixels are addressed flat (npix = B*H*W of ONE side), out[q][d] =
 * (q mod W >= d) ? mean_c L[q][c] * R[q-d][c] : 0.   C % 64 == 0, D % 4 == 0, D <= 32; cs / co: fp16 plane pitch / offset.    */
int vd3d_psm_cosine_h16(const void* l_hi, const void* l_lo, const void* r_hi, const void* r_lo, long long npix, int W, int C,
                        int cs, int co, int D, float* out, int out_cs, int out_co, void* stream);
/* CostVolume.forward after the 1x1 down_sample (R/lib/PSM_cost_volume.py:44-63): concat volume
 *   vol[b, c, i, h, w] = lf[b,h,w,c] (c < F) | rf[b,h,w-i,c-F] (c >= F)  if w >= i else 0
 * gathered on the fly (never materialised) into Conv3d(2F->F,3,pad 1)+BN3d+ReLU; then Conv3d(F->F)+BN3d+ReLU.
 *   lf, rf : NHWC [B][H][W][F] dense;  w1 [27][2F][F], b1 [F];  w2 [27][F][F], b2 [F]  (BN folded, tap = (kd*3+kh)*3+kw)
 *   mid    : scratch [B][D][H][W][F]
 *   out    : NHWC slice, channel = f*D + i  (the reshape at PSM_cost_volume.py:62)
 * F must be 8. */
int vd3d_concat_volume_conv3d(const float* lf, const float* rf, int B, int H, int W, int F, int D,
                              const float* w1, const float* b1, const float* w2, const float* b2,
                              float* mid, float* out, int out_cs, int out_co, void* stream);

/* ---- anchors / decode / NMS ------------------------------------------------------------------------------
 * Anchors.forward useful-mask (R/heads/anchors.py:93-111): mask[b,n] = any_t(-0.5 < y3d < 1.8 && |x3d| < 40).
 *   anchors [N][4] f32, means_z [T][N] f32 (prior z mean per type), P2 [B][3][4] f32 -> mask [B][N] u8 */
int vd3d_anchor_mask(const float* anchors, const float* means_z, const float* P2, int B, int N, int T,
                     float y_min, float y_max, float x_thr, uint8_t* mask, void* stream);

/* AnchorBasedDetection3DHead.get_bboxes (R/heads/detection_3d_head.py:341-400) + _decode (:218-263) +
 * ClipBoxes (R/utils/utils.py:181-196) + torchvision.ops.nms (class-agnostic, IoU > thr suppresses), batched.
 *   cls [B][N][ncls+1], reg [B][N][12], anchors [N][4], mean_std [N][T][6][2], mask [B][N] u8
 *   workspace: ws, at least vd3d_decode_nms_workspace(B, cap) bytes
 *   outputs (fixed capacity `cap` rows per image, rows >= count are undefined):
 *     out_scores [B][cap] f32 (descending), out_boxes [B][cap][11] f32, out_cls [B][cap] i64,
 *     out_anchor [B][cap] i32 (anchor index n of every kept row), out_count [B] i32 (kept rows),
 *     out_ncand [B] i32 (candidates before NMS; > cap means overflow: count is then -1 for that image)
 */
long long vd3d_decode_nms_workspace(int B, int cap);
int vd3d_decode_nms(const float* cls, const float* reg, const float* anchors, const float* mean_std,
                    const uint8_t* mask, int B, int N, int ncls, int T, float score_thr, double iou_thr,
                    float img_w, float img_h, int cap, void* ws,
                    float* out_scores, float* out_boxes, int64_t* out_cls, int32_t* out_anchor,
                    int32_t* out_count, int32_t* out_ncand, void* stream);

/* RetinanetHead.get_bboxes (R/heads/retinanet_head.py:257-307, test mode) batched: max-sigmoid score and label per anchor, top-k
 * (k = min(nms_pre, N); nms_pre <= 0: k = N) by radix select on the key (score desc, anchor index asc), _decode (:227-255, no clipping),
 * class-agnostic torchvision NMS (the vd3d_decode_nms sort / NMS stage) and the post-NMS `score > score_thr` as a prefix count.
 *   level l (of L <= 8) of the head outputs: cls_levels[l] NHWC [B][level_pix[l]][cls_cs] (anchor a, class c at channel a * ncls + c),
 *   reg_levels[l] [B][level_pix[l]][reg_cs] (a * 4 + j); anchor n = level offset + pixel * A + a; anchors [N][4] f32;
 *   means4 / stds4: host float[4] (target_means / target_stds).  The arrays cls_levels, reg_levels, level_pix are read on the host.
 *   workspace: ws, at least vd3d_retina_decode_workspace(B, N, cap) bytes; k must not exceed cap (<= 4096).
 *   outputs as vd3d_decode_nms (box columns 4..10 are zero; out_count = rows above score_thr) */
long long vd3d_retina_decode_workspace(int B, int N, int cap);
int vd3d_retina_decode(int L, const void* const* cls_levels, const void* const* reg_levels, const int* level_pix, int cls_cs, int reg_cs,
                       const float* anchors, int B, int N, int A, int ncls, int nms_pre, const float* means4, const float* stds4,
                       float score_thr, double iou_thr, int cap, void* ws,
                       float* out_scores, float* out_boxes, int64_t* out_cls, int32_t* out_anchor,
                       int32_t* out_count, int32_t* out_ncand, void* stream);

/* fp16-range guard of the fp16-split tensor-core engine.  Activations travel between tensor-core convs as two fp16 planes (hi, lo) of
 * the UNSCALED fp32 value (the reference's fp32 path has no such limit): |v| >= 65520 would become hi = inf.  Every kernel that writes
 * such planes (conv epilogues, vd3d_split_h16_nhwc, vd3d_image_to_h16_rows, vd3d_deform_im2col_h16) ORs a per-device word when it meets
 * such a value; vd3d_fp16_range_check reads it (synchronises `stream`), optionally clears it, and the record kernels report it as
 * count = -2 so that no result computed from an overflowed plane is ever returned silently. */
int vd3d_fp16_range_check(int* overflow_out, int reset, void* stream);

/* Record block for the multi-GPU all-gather (SURVEY.md 8(e)): rec [B][1 + kmax*13] f32 = count, then kmax rows of
 * (11 box floats, score, class); count = -1 flags a capacity overflow, -2 the fp16-range guard.  Built on the device from the vd3d_decode_nms outputs. */
int vd3d_pack_records(const float* scores, const float* boxes, const int64_t* cls, const int32_t* count, int B, int cap, int kmax,
                      float* rec, void* stream);

/* ---- CenterNet-style decode of the MonoFlex head (MonoFlexHead.get_bboxes, R/heads/monoflex_head.py:114-179) ----------
 * heads: NHWC [B][H][W][cs] holding all head outputs at the given channel offsets (hm: ncls, bbox2d 4, hps 20, rot 8, dim 3,
 * reg 2, depth 1, depth_uncertainty 1, corner_uncertainty 3); P2 [B][3][4].  sigmoid + 3x3 peak test + top-K + gather +
 * depth merge + alpha + x4 + clip + class-agnostic NMS, all on the device.  Outputs like vd3d_decode_nms
 * (out_index = flat (c*H + y)*W + x of every kept peak). */
long long vd3d_monoflex_decode_workspace(int B, int cap);
int vd3d_monoflex_decode(const float* heads, int B, int H, int W, int ncls, int cs, int hm_co, int bbox2d_co, int hps_co, int rot_co,
                         int dim_co, int reg_co, int depth_co, int dunc_co, int cunc_co, const float* P2,
                         float score_thr, double iou_thr, int K, float unc_lo, float unc_hi, float img_w, float img_h,
                         int cap, void* ws, int out_cap, float* out_scores, float* out_boxes, long long* out_cls,
                         int* out_index, int* out_count, int* out_ncand, void* stream);

/* KM3DHead.get_bboxes / _decode (R/heads/km3d_head.py:155-314) + gen_position (R/utils/rtm3d_utils.py:314-455): peaks + top-K,
 * keypoint refinement against the per-joint heat-map peaks, float64 3x3 least-squares position solve (the reference's 1e-8
 * random jitter of A^T A is omitted), projection, ClipBoxes, class-agnostic NMS.  heads channels: hm ncls, wh 2, hps 18, rot 8,
 * dim 3, prob 1, reg 2, hm_hp 9, hp_offset 2. */
long long vd3d_km3d_decode_workspace(int B, int cap, int hp_cap);
int vd3d_km3d_decode(const float* heads, int B, int H, int W, int ncls, int cs, int hm_co, int wh_co, int hps_co, int rot_co,
                     int dim_co, int prob_co, int reg_co, int hm_hp_co, int hp_offset_co, const float* P2,
                     float score_thr, double iou_thr, int K, float img_w, float img_h, int cap, int hp_cap, void* ws,
                     int out_cap, float* out_scores, float* out_boxes, long long* out_cls, int* out_index, int* out_count,
                     int* out_ncand, void* stream);

/* ---- image input pipelines (R/data/pipeline/stereo_augmentator.py: the test_augmentation and the shipped train_augmentation lists) ----
 * uint8 HWC frame (C == 3) -> geometry -> photometric program -> mirror -> (v / 255 - mean[c]) / std[c] -> [3][Ho][Wo] float32.
 * vd3d_train_augment_describe packs one frame's descriptor of vd3d_train_augment_desc_bytes() bytes (`pitch` bytes per frame row):
 *   geom 0: CropTop(crop_top) + Resize(preserve aspect, height Ho) cropped / zero padded on the right to Wo; the photometric program runs
 *           on the source pixels before the interpolation (source step <= 2 per axis);
 *   geom 1 / 2: cv2.warpAffine of the float32 forward matrix `affine` [2][3] on the uint8 frame (1) or on its float32 copy (2); the
 *           program runs on the warped values;
 *   mirror: flip the finished Wo-wide image;  ops[nops <= 8] / args[nops]: 1 brightness +=, 2 contrast *=, 3 RGB->HSV, 4 saturation *=,
 *           5 hue += with the 360 wrap, 6 HSV->RGB, 7 eigenvalue noise += noise[3] (float64).
 * Geometry 0 with no ops and no mirror is the test-time pipeline (ConvertToFloat, CropTop, Resize, Normalize: visualdet3d_b200/preprocess.py
 * and pipeline.StreamedInference.submit_frames).
 * vd3d_train_augment_host runs one descriptor on the HOST (src a host pointer; the parity checker); vd3d_train_augment is the CUDA form:
 * `descs_dev` = n descriptors with device `src` pointers (frames of different sizes, both cameras of a stereo batch), out = [n][3][Ho][Wo],
 * one launch.  Random draws, calibration and label updates are host work (visualdet3d_b200/train_augment.py, preprocess.adjust_calib). */
int vd3d_train_augment_desc_bytes(void);
int vd3d_train_augment_describe(void* desc, const unsigned char* src, int H, int W, int C, int pitch, int geom, int crop_top, int Ho, int Wo,
                                const float* affine, int mirror, int nops, const int* ops, const float* args, const double* noise);
int vd3d_train_augment_host(const void* desc, int C, int Ho, int Wo, const float* mean, const float* stdv, float* out);
int vd3d_train_augment(const void* descs_dev, int n, int C, int Ho, int Wo, const float* mean, const float* stdv, float* out, void* stream);

/* ---- KM3D / MonoFlex training targets (R/data/kitti/dataset/KM3D_dataset.py:57-221 KittiRTM3DDataset._build_target, :346-527
 * KittiMonoFlexDataset._build_target; R/networks/utils/rtm3d_utils.py:52-109 gaussian_radius / gaussian2D / gen_hm_radius) ----
 * vd3d_center_targets_pack fills one image's record of vd3d_center_targets_record_bytes() bytes: mode 0 KM3D (9 keypoints) / 1 MonoFlex
 * (10 keypoints), the augmented image's img_h x img_w, num_classes, the float64 P2 [3][4], n <= 32 objects as float64
 * objs[n][11] = x, y, z, w, h, l, ry, bbox_l, bbox_t, bbox_r, bbox_b and their class indices cls[n].
 * outs = 21 pointers, in this order: hm, hm_hp, hps, reg, hp_offset, dim, rots, rotbin, rotres, dep, ind, hp_ind, reg_mask, hps_mask,
 * hp_mask, wh, location, ori, kp_detph_mask, bboxes2d, bboxes2d_target (the reference's dtypes: float32, int64 for rotbin / ind / hp_ind,
 * uint8 for the three masks but kp_detph_mask, which is float32; the last three are MonoFlex's and may be null for KM3D).
 * vd3d_center_targets_host computes one image on the HOST (the parity checker; outs = that image's arrays).  vd3d_center_targets is the
 * CUDA form: recs_dev = B records of one mode / size / class count, outs = a HOST array of DEVICE pointers to [B, ...] arrays,
 * splats_dev = B * vd3d_center_targets_splat_bytes() bytes of scratch; two launches, no synchronisation.  edge_indices is a constant of
 * the image size and is built on the host (visualdet3d_b200/center_targets.py). */
int vd3d_center_targets_record_bytes(void);
int vd3d_center_targets_splat_bytes(void);
int vd3d_center_targets_pack(void* rec, int mode, int img_h, int img_w, int num_classes, const double* P2, int n, const double* objs,
                             const int* cls);
int vd3d_center_targets_host(const void* rec, int mode, int img_h, int img_w, int num_classes, void* const* outs);
int vd3d_center_targets(const void* recs_dev, int B, int mode, int img_h, int img_w, int num_classes, void* const* outs, void* splats_dev,
                        void* stream);

/* ---- post-optimisation of the yaw by hill climbing (R/lib/fast_utils/hill_climbing.py:24-122; caller detection_3d_head.py:294-308) ----
 * For each detection the yaw ry is moved in +-step_r steps (halved when neither direction improves, until step_r <= r_lim) to maximise
 * the IoU between the detected 2-D box and the hull of the projected 3-D box (clipped to img_w x img_h; the reference hard-codes 1280 x 288).
 * vd3d_post_opt_host runs on the HOST (float64, the reference's numba arithmetic): p2 / p2_inv row-major 4x4, box2d [n][4] f32,
 * (cx, cy) projected centre in pixels, z / w / h / l / theta0 as float32 values; theta_out [n] (wrapped like the reference), iou_out [n] or NULL.
 * vd3d_post_opt is the same routine as one CUDA thread per detection on the fixed-capacity NMS output (boxes [B][cap][11], cls [B][cap] i64,
 * count [B] i32, P2 [B][3][4] of KITTI shape), rewriting alpha in place for rows with cls == label and z > min_depth; no host round trip. */
int vd3d_post_opt_host(const double* p2, const double* p2_inv, int n, const float* box2d, const double* cx, const double* cy,
                       const float* z, const float* w, const float* h, const float* l, const float* theta0,
                       double img_w, double img_h, double step_r_init, double r_lim, double* theta_out, double* iou_out);
int vd3d_post_opt(float* boxes, const long long* cls, const int* count, const float* P2, int B, int cap,
                  float img_w, float img_h, float step_r_init, float r_lim, float min_depth, int label, void* stream);

/* ---- post-forward geometry (SURVEY.md 8(f) rank 1; `test_one`, R/networks/pipelines/evaluators.py:112-131) -------------------------------
 * On the fixed-capacity NMS output (boxes [B][cap][11] = x1, y1, x2, y2, cx, cy, z, w, h, l, alpha; count [B]; P2 [B][3][4]):
 *   box3d [B][cap][7]  = BackProjection (R/networks/utils/utils.py:256-278): (x, y, z, w, h, l, alpha) in the camera frame,
 *   theta [B][cap]     = alpha2theta_3d (visualDet3D/utils/utils.py:47-62) as BBox3dProjector returns it (R/networks/utils/utils.py:229),
 *   box2d [B][cap][4]  = the 2-D box shifted / scaled to the pixels of the original frame through original_P [B][3][4]
 *                        (evaluators.py:118-127); original_P == NULL copies the boxes,
 *   corners / homo [B][cap][8][3] (optional, NULL to skip) = BBox3dProjector's camera-frame and image-plane corners (:230-253).
 * float32 in the reference's operation order (x, y, box2d bit-identical to the reference's tensors); rows past count[b] are zero-filled.
 * vd3d_pack_records_geo builds the all-gather record block with these columns appended: rec [B][1 + kmax*20] =
 * count, then kmax rows of (11 box floats, score, class, x3d, y3d, theta, 4 rescaled box floats). */
int vd3d_post_forward(const float* boxes, const int32_t* count, const float* P2, const float* original_P, int B, int cap,
                      float* box3d, float* theta, float* box2d, float* corners, float* homo, void* stream);
int vd3d_pack_records_geo(const float* scores, const float* boxes, const int64_t* cls, const int32_t* count, const float* box3d,
                          const float* theta, const float* box2d, int B, int cap, int kmax, float* rec, void* stream);

/* ---- deformable convolution (R/lib/ops/dcn, make.sh) ----------------------------------------------------------
 * Deformable / modulated-deformable im2col on NHWC activations; the GEMM that the reference runs per image with cuBLAS
 * (deform_conv_cuda.cpp:540-556) is then ONE batched 1x1 convolution on vd3d_conv2d_tc over K = KH*KW*C.
 *   col[pix][k*C + c] = mask[pix][k] * bilinear(x[b,:,:,c], ho*s - pad + kh*dil + dh_k, wo*s - pad + kw*dil + dw_k)
 * sampling rule of modulated_deformable_im2col_gpu_kernel / dmcn_im2col_bilinear (deform_conv_cuda_kernel.cu:467-497,570-633;
 * DCNv1 :190-243 is the same with mask == 1, msk = NULL).
 *   off : NHWC, channel off_co + g*2*K + 2*k = dh, +1 = dw of tap k of deformable group g   (the (dh,dw)-interleaved layout)
 *   msk : NHWC, channel msk_co + g*K + k; mask_sigmoid != 0 applies the sigmoid of ModulatedDeformConvPack.forward (deform_conv.py:463)
 *   col / col_lo : [B*Ho*Wo][col_cs] columns and their lo companion (col_lo may be NULL)                                      */
int vd3d_deform_im2col_nhwc(const float* x, int B, int H, int W, int C, int x_cs, int x_co,
                            const float* off, int off_cs, int off_co,
                            const float* msk, int msk_cs, int msk_co, int mask_sigmoid,
                            int KH, int KW, int stride, int pad, int dil, int deform_groups,
                            float* col, float* col_lo, int col_cs, void* stream);
/* Same gather writing the fp16 (hi, lo) planes of the columns that vd3d_conv2d_tc16 reads (hi = rn16(v), lo = rn16(v - hi));
 * col (the fp32 columns) may be NULL: the planes alone feed the GEMM (no vd3d_split_h16_nhwc pass over 9*C floats per pixel). */
int vd3d_deform_im2col_h16(const float* x, int B, int H, int W, int C, int x_cs, int x_co,
                           const float* off, int off_cs, int off_co,
                           const float* msk, int msk_cs, int msk_co, int mask_sigmoid,
                           int KH, int KW, int stride, int pad, int dil, int deform_groups, int k_order,
                           float* col, void* col_hi16, void* col_lo16, int col_cs, void* stream);

/* ---- Ground-Aware Convolution sampling (LookGround.forward, R/lib/look_ground.py:24-71) ---------------------------
 * x NHWC [B][H][W] (stride-16 features), dconv = output of disp_create's 3x3 conv (channel d_co; tanh applied here),
 * P2 [B][3][4] (full-resolution calibration; rows 0..1 are divided by 16 here like :29-30).
 * out[pix] = [grid_sample(x) (C) | grid_sample(disparity plane) (1) | untouched padding], out_lo its lo companion (or NULL);
 * the 1x1 `extract` conv + alpha + residual + ReLU (:71) is a vd3d_conv2d_tc call on `out`. */
int vd3d_look_ground_sample(const float* x, int B, int H, int W, int C, int x_cs, int x_co,
                            const float* dconv, int d_cs, int d_co, const float* P2,
                            float baseline, float relative_elevation,
                            float* out, float* out_lo, int out_cs, void* stream);

/* Fused (modulated) deformable convolution: the bilinear gather writes the fp16 (hi, lo) A operand of the wgmma GEMM straight into
 * shared memory (SWIZZLE_128B K-major layout + fence.proxy.async), so the column tensor of the reference (deform_conv_cuda.cpp:539-556)
 * never exists in HBM.  x: NHWC fp32; om: NHWC at output resolution holding the offsets (channel off_co + 2k = dh, + 1 = dw) and, when
 * has_mask, the modulation (msk_co + k; mask_sigmoid applies the sigmoid of ModulatedDeformConvPack.forward); weights: the fp16 (hi, lo)
 * [Cout][KH*KW*C] matrix of vd3d_conv2d_tc16 (k = tap*C + c) with its power-of-two out_scale; epilogue (bias, residual, ReLU, fp32 output and
 * optional fp16 planes) as vd3d_conv2d_tc16.  One deformable group, KH*KW <= 9, C % 64 == 0.  Bit-identical to vd3d_deform_im2col_h16 followed
 * by vd3d_conv2d_tc16 (same K order, same gather arithmetic).
 * k_order: order of the K dimension of the weight matrix: 0 = tap * C + c; 1 = (chunk * KH*KW + tap) * 64 + c % 64 (64-channel chunk outermost).
 * With k_order = 1 and a 3x3 / stride 1 / pad 1 / dilation 1 layer the STAGED kernel runs: the input neighbourhood of every 8 x 16 tile (12 x 20
 * pixels x 64 channels, fp32) is brought into shared memory by TMA once per (tile, chunk), zero-filled outside the image, and the nine taps gather
 * from shared memory (corners farther than the staged halo fall back to global loads).  VD3D_DCN_STAGED=0 selects the global-gather kernel. */
int vd3d_deform_conv_fused(const float* x, int B, int H, int W, int C, int x_cs, int x_co,
                           const float* om, int om_cs, int off_co, int msk_co, int has_mask, int mask_sigmoid,
                           int KH, int KW, int stride, int pad, int dil, int k_order,
                           const void* w_hi, const void* w_lo, float out_scale, const float* bias,
                           const float* res, int res_cs, int res_co,
                           float* out, void* out_hi16, void* out_lo16, int Cout, int out_cs, int out_co, int relu, void* stream);

/* Backward of the deformable convolutions (training side, SURVEY.md 8(f) rank 4): the reference's col2im + col2im_coord kernels
 * (deform_conv_cuda_kernel.cu:635-767 modulated, :279-436 DCNv1) fused into one pass over the column gradients
 *   colgrad [B*Ho*Wo][cg_cs], channel k*C + c  =  sum_o W[o, c, k] * grad_out[pix][o]     (a plain GEMM, done by the caller)
 * writing grad_x (NHWC, ACCUMULATED into with 16-byte vector reductions: zero-fill it first), grad_off [pix][.. g*2K + 2k (+1)] and
 * grad_msk [pix][.. g*K + k] (both ASSIGNED; grad_msk / msk NULL for DCNv1).  Any of the three outputs may be NULL.  `msk` holds the
 * modulation values as used by the forward (after the sigmoid).  Same layout conventions as vd3d_deform_im2col_nhwc. */
int vd3d_deform_col2im_nhwc(const float* x, int B, int H, int W, int C, int x_cs, int x_co,
                            const float* off, int off_cs, int off_co, const float* msk, int msk_cs, int msk_co,
                            int KH, int KW, int stride, int pad, int dil, int deform_groups,
                            const float* colgrad, int cg_cs,
                            float* grad_x, int gx_cs, int gx_co, float* grad_off, int go_cs, int go_co,
                            float* grad_msk, int gm_cs, int gm_co, void* stream);

/* ---- iou3d (R/lib/ops/iou3d, make.sh) ---------------------------------------------------------------------------
 * boxes [n][5] = (x1, y1, x2, y2, ry) f32.  Replace iou3d_cuda.boxes_overlap_bev_gpu / boxes_iou_bev_gpu (iou3d.cpp:31-71,
 * kernels iou3d_kernel.cu:223-248) and nms_gpu / nms_normal_gpu (iou3d.cpp:73-170, kernels :250-348).  NMS runs entirely on
 * the device: keep [N] i64 and count [1] i32 are DEVICE buffers; boxes must be sorted by descending score by the caller
 * (as in the reference); rotated != 0 -> rotated IoU (nms_gpu), 0 -> axis-aligned IoU (nms_normal_gpu). */
int vd3d_boxes_overlap_bev(const float* a, int M, const float* b, int N, float* out, void* stream);
int vd3d_boxes_iou_bev(const float* a, int M, const float* b, int N, float* out, void* stream);
long long vd3d_nms_bev_workspace(int N);
int vd3d_nms_bev(const float* boxes, int N, float thresh, int rotated, void* ws, long long* keep, int* count, void* stream);

/* ---- KITTI object evaluator (visualDet3D/evaluator/kitti in the reference tree) ----------------------------------
 * vd3d_kitti_rotate_iou replaces rotate_iou.py rotate_iou_gpu_eval (the numba kernel rotate_iou_kernel_eval, :261-291):
 * boxes [N][5], qboxes [K][5] = (x, y, dx, dy, angle) f32; iou [N][K] f32 = devRotateIoUEval(qboxes[k], boxes[n], criterion),
 * criterion -1 IoU, 0 / 1 intersection over the query / box area, 2 intersection area.
 *
 * vd3d_kitti_eval replaces eval.py eval_class (:476-594) for the three metrics of do_eval_v3 (:650-673) with difficulties 0, 1, 2:
 * calculate_iou_partly, clean_data, compute_statistics_jit, get_thresholds and fused_compute_statistics, per image.
 *   gt [n_gt][15] f64 = bbox x1 y1 x2 y2, alpha, dims l h w, location x y z, rotation_y, truncated, occluded, class code;
 *   dt [n_dt][16] f64 = the same columns + score.  Class code: index into the reference's CLASS_NAMES of the lower-cased name
 *   ('car' 0, 'pedestrian' 1, 'cyclist' 2, 'van' 3, 'person_sitting' 4, 'tractor' 6, 'trailer' 7), -2 for "DontCare", else -1.
 *   offs [4][n_img+1] i64 = CSR offsets of gt rows, dt rows, [dt][gt] overlap blocks (n_pairs in all) and 32-bit detection-flag
 *   words (ceil(dt rows / 32) per image, n_words in all); classes [n_cls] i32; min_overlaps [2][3][n_cls] f64.
 * Outputs, configuration cfg = ((metric * n_cls + class) * 3 + difficulty) * 2 + min_overlap index:
 *   overlaps [3][n_pairs] (bbox, BEV, 3-D), precision / thresholds [18 n_cls][41], n_thresh [18 n_cls], orientation [6 n_cls][41]
 *   (metric 0 only; zeros unless compute_aos).  A configuration with n_thresh > 41 (the reference raises) has truncated thresholds.
 * workspace: vd3d_kitti_eval_workspace_bytes(...) bytes of device memory (a negative return is an error code). */
int vd3d_kitti_rotate_iou(const float* boxes, int N, const float* qboxes, int K, int criterion, float* iou, void* stream);
long long vd3d_kitti_eval_workspace_bytes(int n_img, long long n_gt, long long n_dt, long long n_words, int n_cls);
int vd3d_kitti_eval(const double* gt, const double* dt, const long long* offs, int n_img, long long n_gt, long long n_dt,
                    long long n_pairs, long long n_words, const int* classes, int n_cls, const double* min_overlaps, int compute_aos,
                    double* overlaps, double* precision, double* orientation, double* thresholds, int* n_thresh,
                    void* workspace, long long workspace_bytes, void* stream);

/* ---- training loss of the 3-D anchor head (AnchorBasedDetection3DHead.loss, R/networks/heads/detection_3d_head.py:402-498) -----------
 * cls [B][N][C+1] f32 (last column: alpha logit), reg [B][N][12] f32, anchors [N][4] f32 (16-byte aligned), mask [B][N] bool (u8),
 * mean_std [N][C][6][2] f32, ann [B][M][12] f32 (compound_annotation; class -1 rows are padding, anywhere).  C <= 8, M <= 512.
 * params (host) [7 + C + 13] f32 = fg_iou_threshold, bg_iou_threshold, min_iou_threshold, focal gamma, then float32 of 1/alpha,
 *   0.5*alpha and 0.5/alpha of ModifiedSmoothL1Loss, the balance weight of each class, the 13 regression weights.
 * vd3d_anchor_loss_forward: assign [B][N] i32 = the reference's assigned_gt_inds (1-based among the image's valid rows in their order,
 *   0 negative, -1 ignored; -1 for every anchor of an image without ground truth, -2 outside the mask); counts [B][3] i32 =
 *   positives assigned, positives kept by the prior's z_mean > 0, negatives; factors [B][2] f32 (read by the backward);
 *   cls_loss [1], reg_loss [1] f32.  Four launches, no host synchronisation, no float atomics (bit-reproducible).
 *   workspace: vd3d_anchor_loss_workspace_bytes(B, N, M) bytes of device memory (a negative return is an error code).
 * vd3d_anchor_loss_backward: grad_out [2] f32 (device) = d/d cls_loss, d/d reg_loss; writes grad_cls [B][N][C+1] and grad_reg [B][N][12]
 *   in full (zeros where no term depends on the element), from the forward's assign and factors.  One launch. */
long long vd3d_anchor_loss_workspace_bytes(int B, int N, int M);
int vd3d_anchor_loss_forward(const float* cls, const float* reg, const float* anchors, const unsigned char* mask, const float* mean_std,
                             const float* ann, int B, int N, int C, int M, const float* params, int match_low_quality, int gt_max_assign_all,
                             void* workspace, long long workspace_bytes, int* assign, int* counts, float* factors, float* cls_loss, float* reg_loss,
                             void* stream);
int vd3d_anchor_loss_backward(const float* cls, const float* reg, const float* anchors, const float* mean_std, const float* ann,
                              int B, int N, int C, int M, const float* params, const int* assign, const float* factors, const float* grad_out,
                              float* grad_cls, float* grad_reg, void* stream);

/* ---- training loss of the RetinaNet head (RetinanetHead.loss, R/networks/heads/retinanet_head.py:309-362) ----------------------------
 * Replaces _assign / _sample / _encode / _decode (retinanet_head.py:99-255), SigmoidFocalLoss and IoULoss (losses.py:11-46, 93-120) and
 * calc_iou (R/networks/utils/utils.py:83-100).
 * cls [B][N][C] f32 logits, reg [B][N][4] f32 deltas, anchors [N][4] f32 (16-byte aligned), ann [B][M][K] f32 (x1 y1 x2 y2 class in the
 *   first five columns; class -1 rows are padding, anywhere).  C <= 64, M <= 512, K >= 5.
 * params (host) [12 + C] f32 = fg_iou_threshold, bg_iou_threshold, min_iou_threshold, focal gamma, target_means[4], target_stds[4], the
 *   balance weight of each class.
 * vd3d_retina_loss_forward: assign [B][N] i32 = the reference's assigned_gt_inds (1-based among the image's valid rows in their order,
 *   0 negative, -1 ignored; 0 for every anchor of an image without a valid row); counts [B][3] i32 = positives, negatives, ignored;
 *   scale [1] f32 = 1 / (positives of the batch + 1e-4) (read by the backward); cls_loss, reg_loss 0-d f32.  A positive whose class.long() lies
 *   outside [0, C) makes both losses and the scale NaN.  Four launches, no host synchronisation, no float atomics (bit-reproducible).
 *   workspace: vd3d_retina_loss_workspace_bytes(B, N, M) bytes of device memory (a negative return is an error code).
 * vd3d_retina_loss_backward: grad_out [2] f32 (device) = d/d cls_loss, d/d reg_loss; writes grad_cls [B][N][C] and grad_reg [B][N][4]
 *   (16-byte aligned) in full (zeros where no term depends on the element), from the forward's assign and scale.  One launch. */
long long vd3d_retina_loss_workspace_bytes(int B, int N, int M);
int vd3d_retina_loss_forward(const float* cls, const float* reg, const float* anchors, const float* ann, int B, int N, int C, int M, int K,
                             const float* params, int match_low_quality, int gt_max_assign_all, void* workspace, long long workspace_bytes,
                             int* assign, int* counts, float* scale, float* cls_loss, float* reg_loss, void* stream);
int vd3d_retina_loss_backward(const float* cls, const float* reg, const float* anchors, const float* ann, int B, int N, int C, int M, int K,
                              const float* params, const int* assign, const float* scale, const float* grad_out, float* grad_cls,
                              float* grad_reg, void* stream);

/* ---- training loss of the MonoFlex head (MonoFlexHead.loss, R/networks/heads/monoflex_head.py:181-236) ------------------------------
 * Replaces _neg_loss, _RegWeightedL1Loss and _RotLoss (km3d_head.py:61-130, compute_rot_loss rtm3d_utils.py:9-49), _gather_output and
 * the six gathered terms (monoflex_head.py:26-104, 194-219, decode_depth_from_keypoints rtm3d_utils.py:141-182, IoULoss losses.py:93-120).
 * maps (host array of 9 device pointers, f32 NCHW): hm [B][C][H][W] logits, bbox2d 4, hps 20, rot 8, dim 3, reg 2, depth 1,
 *   depth_uncertainty 1, corner_uncertainty 3 channels.
 * targets (host array of 13 device pointers): hm [B][C][H][W] f32, ind [B][K] i64, reg_mask [B][K] u8, hps [B][K][20] f32,
 *   hps_mask [B][K][20] u8, dep [B][K] f32, rotbin [B][K][2] i64, rotres [B][K][2] f32, bboxes2d_target [B][K][4] f32, dim [B][K][3] f32,
 *   reg [B][K][2] f32, kp_detph_mask [B][K][3] f32, P2 [B][3][4] f32.  K <= 128.
 * unc_lo / unc_hi / unc_w: the head's uncertainty_range and uncertainty_weight.
 * vd3d_monoflex_loss_forward: terms [9] f32 = hm, hp, box2d, off, dim, depth, kpd, rot, soft_depth (unweighted, as in loss_stats) and
 *   total [1] f32 = their sum weighted 1, 1, 1, 0.5, 1, 1, 0.2, 1, 0.2.  Three launches, no host synchronisation, no float atomics.
 *   With no reg_mask row in the batch the six gathered terms are 0.  An ind outside [0, H*W) in any row makes every loss NaN (the map is
 *   not read there).  workspace: vd3d_monoflex_loss_workspace_bytes(B, C, H, W, K) bytes of device memory (negative: error code); the
 *   backward reads the factors the forward leaves in it.
 * vd3d_monoflex_loss_backward: grad_terms [9] and grad_total [1] f32 (device; either may be null = zero) = d/d terms, d/d total; writes
 *   grads (host array of 9 device pointers, shaped like maps) in full.  One launch. */
long long vd3d_monoflex_loss_workspace_bytes(int B, int C, int H, int W, int K);
int vd3d_monoflex_loss_forward(const void* const* maps, const void* const* targets, int B, int C, int H, int W, int K, float unc_lo,
                               float unc_hi, float unc_w, void* workspace, long long workspace_bytes, float* terms, float* total, void* stream);
int vd3d_monoflex_loss_backward(const void* const* maps, const void* const* targets, int B, int C, int H, int W, int K, float unc_lo,
                                float unc_hi, float unc_w, const void* workspace, const float* grad_terms, const float* grad_total,
                                float* const* grads, void* stream);

/* ---- training loss of the KM3D head (KM3DHead.loss, R/networks/heads/km3d_head.py:316-351) ----------------------------------------
 * Replaces _neg_loss (hm and hm_hp), _RegWeightedL1Loss, _RegL1Loss (wh, dim, reg, hp_offset), _RotLoss (km3d_head.py:61-130,
 * compute_rot_loss rtm3d_utils.py:9-49) and Position_loss with gen_position (rtm3d_utils.py:230-455).
 * maps (host array of 9 device pointers, f32 NCHW): hm [B][C][H][W] logits, wh 2, hps 18, rot 8, dim 3, prob 1, reg 2, hm_hp 9 (logits),
 *   hp_offset 2 channels.
 * targets (host array of 18 device pointers): hm [B][C][H][W] f32, hm_hp [B][9][H][W] f32, ind [B][K] i64, reg_mask [B][K] u8,
 *   hps [B][K][18] f32, hps_mask [B][K][18] u8, dep [B][K] f32, rotbin [B][K][2] i64, rotres [B][K][2] f32, wh [B][K][2] f32,
 *   dim [B][K][3] f32, reg [B][K][2] f32, hp_ind [B][K*9] i64, hp_mask [B][K*9] u8, hp_offset [B][K*9][2] f32, location [B][K][3] f32,
 *   ori [B][K] f32, P2 [B][3][4] f32.  K <= 128; 9 keypoints per object.  Inputs are never written (the reference rewrites dep in place).
 * output_w: the loss config's output_w (the keypoint centre is (ind mod output_w, trunc(ind / output_w))); rampup: exp_rampup(epoch),
 *   the weight of prob_loss and coor_loss (a captured graph holds one epoch's value).
 * vd3d_km3d_loss_forward: terms [11] f32 = hm, hp, hm_hp, hp_offset, wh, off, dim, rot, prob, coor, box_score (unweighted, as in
 *   loss_stats) and total [1] f32 = the first ten weighted 1, 1, 1, 1, 0.1, 1, 2, 0.2, rampup, rampup.  Three launches, no host
 *   synchronisation, no float atomics.  An ind or hp_ind outside [0, H*W) in any row makes every loss NaN (the map is not read there).
 *   workspace: vd3d_km3d_loss_workspace_bytes(B, C, H, W, K) bytes of device memory (negative: error code); the backward reads the factors
 *   the forward leaves in it.
 * vd3d_km3d_loss_backward: grad_terms [11] and grad_total [1] f32 (device; either may be null = zero) = d/d terms, d/d total (box_score
 *   has no gradient); writes grads (host array of 9 device pointers, shaped like maps) in full.  One launch. */
long long vd3d_km3d_loss_workspace_bytes(int B, int C, int H, int W, int K);
int vd3d_km3d_loss_forward(const void* const* maps, const void* const* targets, int B, int C, int H, int W, int K, float output_w,
                           float rampup, void* workspace, long long workspace_bytes, float* terms, float* total, void* stream);
int vd3d_km3d_loss_backward(const void* const* maps, const void* const* targets, int B, int C, int H, int W, int K, float output_w,
                            float rampup, const void* workspace, const float* grad_terms, const float* grad_total, float* const* grads,
                            void* stream);

/* ---- disparity loss of Stereo3D (DisparityLoss(max_disp), R/networks/heads/losses.py:122-135) -----------------------------------------
 * Replaces StereoFocalLoss.loss_per_level with LaplaceDisp2Prob (R/networks/lib/disparity_loss/*.py) at the shipped settings: start_disp 0,
 * dilation 1, one level, focal_coefficient 0, variance 0.5, the label at the cost volume's H, W, and max_disp = D.
 * cost [B][D][H][W] f32 (logits), disp [B][H][W] f32 (the disparity label; 0 = no label).  2 <= D <= 1024, H*W < 2^31 - 256, offsets are
 *   64-bit.  Masks: outer = 0 < disp < D (the loss), inner = 0 < disp < D - 1 (the target); target p_c = softmax_c(-|c - disp*inner| / 0.5)
 *   * inner + 1e-40.  Inputs are never written.
 * vd3d_disparity_loss_forward: loss [1] f32 = -(1/(B*H*W)) sum_pixels outer * sum_c p_c log_softmax(cost)_c, and lse [B][H][W] f32 = each
 *   pixel's log-sum-exp over D (0 outside outer), which the backward reads.  Two launches, no host synchronisation, no float atomics; one
 *   read of the volume (none at pixels outside outer).  With no outer pixel the loss is 0; a non-finite disp value makes it NaN.
 *   workspace: vd3d_disparity_loss_workspace_bytes(B, D, H, W) bytes of device memory (negative: error code), one float64 per block.
 * vd3d_disparity_loss_backward: grad_loss [1] f32 (device) = d/d loss; writes grad_cost [B][D][H][W] in full (exact zeros outside outer).
 *   One launch. */
long long vd3d_disparity_loss_workspace_bytes(int B, int D, int H, int W);
int vd3d_disparity_loss_forward(const float* cost, const float* disp, int B, int D, int H, int W, void* workspace, long long workspace_bytes,
                                float* lse, float* loss, void* stream);
int vd3d_disparity_loss_backward(const float* cost, const float* disp, const float* lse, int B, int D, int H, int W, const float* grad_loss,
                                 float* grad_cost, void* stream);

/* ---- Stereo3D's disparity ground truth (scripts/disparity_compute.py: compute_dispairity_for_split) --------------------------------
 * StereoBM: cv2.StereoBM_create(192, 25).compute with cv2's defaults (XSOBEL prefilter, cap 31, texture threshold 10, uniqueness 15 %, no
 *   speckle filter, no left-right check, minDisparity 0), bit for bit.  left / right [B][H][W]; disp [B][H][W] int16 = 16 x disparity,
 *   -16 where filtered and on the border StereoBM never computes (rows < 12 or >= H-12, columns < 203 or >= W-12).  26 <= H, 216 <= W
 *   (cv2 has no defined output below), H, W <= 16384, B <= 65535.  workspace: vd3d_stereo_bm_workspace_bytes(B, H, W) bytes of device
 *   memory (the prefiltered frames; negative: error code).  Three launches.
 * vd3d_stereo_bm: uint8 grey frames.
 * vd3d_stereo_bm_f32: float32 [B][H][W][3] normalised network input (the test augmentation's output); each pixel is de-normalised as the
 *   script's denorm does (x * std + mean in float64, clipped to [0, 1], * 255, truncated) and converted with COLOR_BGR2GRAY (channel 0
 *   weighted as blue).  mean_host / std_host: 3 float64 each.  grey [2][B][H][W] uint8 (left frames, then right; may be null) receives
 *   the grey frames.
 * vd3d_disparity_block_max: skimage.measure.block_reduce(max(in, 0) as uint16, (4, 4), np.max): in [B][H][W] int16 (is_signed) or uint16,
 *   out [B][ceil(H/4)][ceil(W/4)] uint16, the far edges zero-padded.  One launch.
 * vd3d_velo_disparity: generate_dispariy_from_velo (R/data/kitti/utils.py:85-120) for one frame.  points [N][stride] float32 (x, y, z
 *   first; stride >= 3), R0_host / Tr_host the calibration's 4x4 R0_rect / Tr_velo_to_cam, P2_host [3][4], all float64 host arrays.
 *   full [H][W] uint16 = uint16(P2[0, 0] * baseline / depth * 16) of the LAST in-view point (cloud order) of each pixel, 0 where none.
 *   winner: H * W int32 of device scratch.  A memset and two launches.
 * The _host forms compute one frame on the host with the kernels' per-element routines (the parity checker). */
long long vd3d_stereo_bm_workspace_bytes(int B, int H, int W);
int vd3d_stereo_bm(const uint8_t* left, const uint8_t* right, int B, int H, int W, uint8_t* workspace, int16_t* disp, void* stream);
int vd3d_stereo_bm_f32(const float* left, const float* right, int B, int H, int W, const double* mean_host, const double* std_host,
                       uint8_t* workspace, uint8_t* grey, int16_t* disp, void* stream);
int vd3d_disparity_block_max(const void* in, int is_signed, int B, int H, int W, uint16_t* out, void* stream);
int vd3d_velo_disparity(const float* points, int N, int stride, const double* R0_host, const double* Tr_host, const double* P2_host,
                        double baseline, int H, int W, int* winner, uint16_t* full, void* stream);
int vd3d_disparity_grey_host(const float* img, int H, int W, const double* mean, const double* std, uint8_t* grey);
int vd3d_stereo_bm_host(const uint8_t* left, const uint8_t* right, int H, int W, int16_t* disp);
int vd3d_disparity_block_max_host(const void* in, int is_signed, int H, int W, uint16_t* out);
int vd3d_velo_disparity_host(const float* points, int N, int stride, const double* R0, const double* Tr, const double* P2,
                             double baseline, int H, int W, uint16_t* full);

/* ---- the 3-D anchor priors (scripts/imdb_precompute_3d.py: read_one_split, lines 106-135) ------------------------------------------
 * One batch of B frames x T classes.  anchors [N][4] float32 (Anchors.forward's table for the post-augmentation shape).  The anchors of
 *   bin k (scale row * n_ratios + ratio column, the reference's anchors2indexes on the float32 table) are order[bin_start[k] ..
 *   bin_start[k+1]), ascending; bin_start_host: n_bins + 1 ints on the host.  offsets_host: B*T + 1 ints on the host, segment s = b * T + t
 *   (frame b, class t) holding boxes offsets[s] .. offsets[s+1] (at most 512 each).  boxes [K_total][4] (x1, y1, x2, y2): float32, or
 *   float64 with boxes_f64 (the IoU's dtype; the threshold is compared in the same dtype).  gt3 [K_total][3] float64 (z, sin 2a, cos 2a).
 * For every segment and anchor: calc_iou against the segment's boxes, the first-maximum box, positive where the maximum is >
 *   fg_iou_threshold.  Each positive adds 1 to examine[t][bin], its gt3 row to sums[t][bin][3] and the row's squares to squared[t][bin][3],
 *   in frame, class, anchor order: the reference's sequential float64 sums, bit for bit.  usable[t] += the class's boxes whose maximum IoU
 *   over all anchors is > fg_iou_threshold.  The state (int64 / float64 device arrays) carries over from batch to batch.
 * vd3d_anchor_prior_accumulate: device pointers except the two _host arrays; workspace: vd3d_anchor_prior_workspace_bytes(N, n_bins, B, T,
 *   K_total) bytes of device memory (negative: error code).  A copy of the offsets, a memset and two launches; no synchronisation.
 * vd3d_anchor_prior_host: the same accumulation on host arrays in the reference's loop order (the parity checker); it also checks that
 *   order lists every anchor once, ascending within each bin. */
long long vd3d_anchor_prior_workspace_bytes(int N, int n_bins, int B, int T, int K_total);
int vd3d_anchor_prior_accumulate(const float* anchors, const int* order, const int* bin_start_host, int N, int n_bins,
                                 const int* offsets_host, int B, int T, const void* boxes, int boxes_f64, const double* gt3, int K_total,
                                 double fg_iou_threshold, long long* examine, double* sums, double* squared, long long* usable,
                                 void* workspace, long long workspace_bytes, void* stream);
int vd3d_anchor_prior_host(const float* anchors, const int* order, const int* bin_start, int N, int n_bins, const int* offsets, int B,
                           int T, const void* boxes, int boxes_f64, const double* gt3, int K_total, double fg_iou_threshold,
                           long long* examine, double* sums, double* squared, long long* usable);

#ifdef __cplusplus
}
#endif
#endif
