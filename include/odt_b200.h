/*
 * odt_b200.h -- C ABI of the H100-native (sm_90a) detection hot path.
 *
 * This is the drop-in boundary underneath the reference's Python surface
 * (SSD300.SSD300 / RetinaNet.RetinaNet / YOLOv3.YOLOv3 / FCOS.FCOS /
 * SSD512.SSD512 .test_one_image()).  The reference has no FFI of its own: all
 * of its arithmetic is executed by TensorFlow 1.13 ops called from Python.
 * Each entry point below replaces one class of TF op *call sites* on the
 * inference path; the call site it stands in for is cited as
 * "ref: <file>:<line>" (paths relative to the reference checkout).
 *
 * Conventions
 *   - extern "C", plain pointers and sizes, no torch / C++ types.
 *   - every pointer is a DEVICE pointer unless its name ends in _host.
 *   - every function is asynchronous on `stream` (a cudaStream_t passed as
 *     void*), never allocates, never synchronises, and returns ODT_OK (0) or a
 *     negative error code; odt_last_error() returns a thread-local message.
 *   - tensors are NHWC.  Boxes are (y1, x1, y2, x2) in input pixels
 *     (ref: SSD300.py:169-171).
 *   - dtype codes: ODT_F16 = 0 (IEEE half), ODT_F32 = 1.
 *   - thread-compatible: no mutable globals (the only global state is the
 *     lazily resolved driver entry points for cuTensorMapEncode*).
 */
#ifndef ODT_B200_H_
#define ODT_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ODT_OK 0
#define ODT_ERR_INVALID (-1)   /* bad argument                                 */
#define ODT_ERR_CUDA (-2)      /* a CUDA runtime / driver call failed          */
#define ODT_ERR_UNSUPPORTED (-3)
#define ODT_ERR_OVERFLOW (-4)  /* candidate list capacity exceeded (reported in
                                  the status word of odt_nms_per_class)        */

#define ODT_F16 0
#define ODT_F32 1

#define ODT_ACT_NONE 0
#define ODT_ACT_RELU 1
#define ODT_ACT_LEAKY 2 /* max(x, 0.1 x)  ref: YOLOv3.py:506 */

#define ODT_MAX_LEVELS 8
#define ODT_MAX_PRIORS 9

/* ---------------------------------------------------------------- misc --- */
int odt_abi_version(void);
/* host utility: CRC-32C of a host buffer continuing from `crc` (0 = fresh).  Used by the
 * tf.train.Saver V2 (TensorBundle) reader / writer that replaces NewCheckpointReader /
 * Saver.save / Saver.restore (SSD300.py:31,490-504; RetinaNet.py:505-557; YOLOv3.py:376-385). */
unsigned int odt_crc32c(unsigned int crc, const void* data, unsigned long long n);
const char* odt_last_error(void);
/* TF "SAME" geometry: out = ceil(in/stride); pad_before = pad_total/2.
 * ref: every tf.layers.conv2d/max_pooling2d(padding='same'), e.g. SSD300.py:524,540 */
int odt_same_pad(int in, int k, int stride, int dil, int* out, int* pad_before, int* pad_after);

/* --------------------------------------------------------------- input --- */
/* images - mean (RGB 123.68,116.779,103.979), fp32 [B,H,W,3] -> dtype [B,H,W,ld]
 * (channels >= 3 are zero).  ref: SSD300.py:52-66, RetinaNet.py:101-115,
 * YOLOv3.py:62-76, FCOS.py:51-65 */
int odt_normalize_input(const float* images, void* out, int out_dtype, int B, int H, int W,
                        int out_ld, const float* mean3_host, void* stream);

/* images - mean as fp16 RGBX: out [B][H+2*pad][W+2*pad][4] (4th channel 0), interior only -- the zero border of
 * `pad` pixels is the caller's (zero-fill the buffer once).  Input format of odt_conv2d_stem_rgbx.
 * ref: the same `images - mean` lines as odt_normalize_input */
int odt_pack_input_rgbx(const float* images, void* out_f16, int B, int H, int W, int pad,
                        const float* mean3_host, void* stream);

/* ---------------------------------------------------------------- conv --- */
typedef struct {
  /* input  [B,H,W,in_ld] (Cin real channels, in_ld >= Cin channel stride)    */
  int B, H, W, Cin, in_ld;
  /* output geometry (TF SAME) and filter                                      */
  int OH, OW, Cout;
  int R, S, stride, dil, pad_t, pad_l;
  /* weights: KRSC [Cout_pad][R][S][w_ld] in the activation dtype; rows
   * >= Cout and channels >= Cin must be zero.  (TF stores HWIO; the host
   * transposes at load -- ref: SSD300.py:519,524.)                            */
  int w_ld;      /* channel stride inside one filter tap (>= Cin)             */
  int Cout_pad;  /* number of filter rows present in memory                   */
  /* epilogue 1:  v = act(acc*scale[c] + shift[c]) (+ residual)  -> out0      */
  const float* scale; /* [Cout] or NULL (=1)  folded BN gamma*rsqrt(var+eps)  */
  const float* shift; /* [Cout] or NULL (=0)  bias / folded BN beta           */
  int act;
  const void* residual; /* activation dtype, same addressing as out0, or NULL */
  void* out0;           /* may be NULL when only out1 / out2 are wanted       */
  int out0_dtype;       /* ODT_F16 / ODT_F32                                  */
  long long out0_img_stride; /* elements between images                       */
  int out0_pix_stride;       /* elements between pixels                       */
  int out0_group;            /* channel regrouping: channel n is stored at    */
  int out0_group_stride;     /* (n/group)*group_stride + n%group; 0 = off     */
  /* epilogue 2 (pre-activation of the consumer):
   *   out1 = act2(v*scale2[c] + shift2[c]),  activation dtype                */
  const float* scale2;
  const float* shift2;
  int act2;
  void* out1; /* or NULL */
  long long out1_img_stride;
  int out1_pix_stride;
  /* epilogue 3: a second consumer pre-activation of the same value (RetinaNet's
   * identity and conv branches normalise the block input with different BNs,
   * RetinaNet.py:634-643):  out2 = act3(v*scale3[c] + shift3[c])              */
  const float* scale3;
  const float* shift3;
  int act3;
  void* out2; /* or NULL */
  long long out2_img_stride;
  int out2_pix_stride;
  /* halo layouts (tensor-core path only): 1 = the tensor is stored as
   * [B][H+2][W+2][ld] with a zero 1-pixel border that the kernels never dirty.
   * A halo input lets 3x3/stride-1 convolutions with Cout_pad <= 128 run in
   * "flat" mode: one [136 x 64] slab per (filter row, channel chunk) feeds the
   * three horizontal taps, cutting the activation traffic ~3x.  out0_img_stride
   * must then be (OH+2)*(OW+2)*out0_pix_stride; `residual` shares out0's layout. */
  int in_halo;
  int out0_halo;
  /* fused 2x2 / stride-2 max pooling (a4: SSD300.py:539-547 straight after the
   * VGG conv): out0_pool = 2 makes out0 the pooled tensor [B][OH/2][OW/2]
   * (strides and out0_halo describe THAT tensor; OH/OW stay the convolution's).
   * Tensor-core path only, for the halo-flat shapes (in_halo, 3x3, stride 1,
   * Cout_pad <= 128) with even OH and OW, fp16 out0, no residual / out1 /
   * regrouping.  0 = off.                                                      */
  int out0_pool;
  /* halo layout of the extra outputs (tensor-core path): 1 = out1 / out2 is stored as [B][OH+2][OW+2][pix_stride]
   * with a zero border (outK_img_stride = (OH+2)*(OW+2)*outK_pix_stride), so that the 3x3 convolution that consumes a
   * pre-activated tensor can run in the halo-flat / taps-as-N modes like any other 3x3 layer.                      */
  int out1_halo;
  int out2_halo;
} odt_conv_params;

/* wgmma / TMA implicit-GEMM forward convolution, fp16 in, fp32 accumulate.
 * Requires in_ld % 64 == 0, w_ld == in_ld, Cout_pad % 32 == 0.
 * ref: tf.nn.conv2d SSD300.py:519; tf.layers.conv2d SSD300.py:524,
 * RetinaNet.py:579,599,609, YOLOv3.py:495, FCOS.py:449,469,479; the fused
 * epilogue is bias_add/BN/ReLU SSD300.py:520-521,534-537 */
int odt_conv2d_f16_tc(const void* in, const void* weights, const odt_conv_params* p, void* stream);
/* the N tile (32 .. 128, or 256) odt_conv2d_f16_tc picks for an im2col-mode layer of M = B*OH*OW output
 * pixels, Cout_pad channels and kblocks = R*S*in_ld/64 K blocks (host only; honours ODT_TC_WIDE) */
int odt_conv_tc_pick_bn(int cout_pad, long long M, int kblocks);
/* whether odt_conv2d_f16_tc runs the layer on the transposed 64-cout x 256-pixel tiles (narrow 3x3 halo layers, fp16
 * out0 alone; host only; honours ODT_TC_SWAP): 1 and *rp = rows per row-block tile (0: halo-flat), *tiles = 256-pixel
 * tiles, *waste_permille = computed positions that are no output pixel, per thousand; else 0.  Outputs may be null. */
int odt_conv_tc_swap_plan(const odt_conv_params* p, int* rp, long long* tiles, int* waste_permille);
/* generic direct convolution on CUDA cores: any Cin/Cout/filter; `dtype` is
 * the activation dtype (ODT_F32: reference-precision path, ODT_F16: stems and
 * shapes the tensor-core kernel does not take).  Same call sites as above. */
int odt_conv2d_direct(const void* in, const void* weights, int dtype, const odt_conv_params* p,
                      void* stream);
/* stem variant: fp32 image minus mean is read directly (a1 fused), output dtype `dtype` */
int odt_conv2d_stem(const float* images, const float* mean3_host, const void* weights, int dtype,
                    const odt_conv_params* p, void* stream);

/* Tensor-core (wgmma) 7x7/stride-2 stem on the packed image of odt_pack_input_rgbx (p->in_ld = 4, p->in_halo = its
 * pad = 4), with even W / left pad and Cout <= 16 real outputs: it always computes and stores 16 channels, so
 * Cout_pad = 16 and weights / scale / shift hold 16 rows, zero past Cout, and out0_pix_stride >= 16;
 * every filter row of an output pixel is one aligned span of the image, so the im2col rows are built with
 * wide loads and no arithmetic.  ODT_ERR_UNSUPPORTED for other shapes (use odt_conv2d_stem).
 * ref: RetinaNet.py:260-265; FCOS.py:73-78 */
int odt_conv2d_stem_rgbx(const void* rgbx, const void* weights, const odt_conv_params* p, void* stream);

/* --------------------------------------------------------------- glue ---- */
/* max pooling, TF SAME (pads ignored).  in_halo / out_halo: the tensor is stored with a
 * zero 1-pixel border ([B][H+2][W+2][ld], see odt_conv_params).
 * ref: SSD300.py:539-547, RetinaNet.py:645-653 */
int odt_maxpool(const void* in, void* out, int dtype, int B, int H, int W, int C, int ld, int k,
                int stride, int in_halo, int out_halo, void* stream);
/* max pooling plus up to two per-channel affine + activation outputs of the pooled value:
 *   out (optional, may be NULL) = pool(in);  outK = actK(pool(in)*scaleK[c] + shiftK[c]), [B][OH][OW][ld] or, with outK_halo = 1,
 * [B][OH+2][OW+2][ld] with a zero border the kernel never writes.
 * One pass for the pooled stem of the pre-activation ResNets feeding the two BN+ReLU of block1_unit1.
 * ref: RetinaNet.py:645-653 (pool) + :594-597 (BN, ReLU of _bn_activation_conv); FCOS.py likewise */
int odt_maxpool_affine(const void* in, void* out, int dtype, int B, int H, int W, int C, int ld, int k, int stride,
                       int in_halo, int out_halo, const float* scale1, const float* shift1, int act1, void* out1,
                       int out1_halo, const float* scale2, const float* shift2, int act2, void* out2, int out2_halo,
                       void* stream);
/* x * rsqrt(max(sum_c x^2, 1e-12)) * gamma.  ref: SSD300.py:74-83 */
int odt_l2norm_scale(const void* in, void* out, int dtype, long long pixels, int C, int ld,
                     float gamma, void* stream);
/* y = act(x*scale[c] + shift[c])  (stand-alone BN/affine + activation).
 * ref: RetinaNet.py:594-597, SSD300.py:506-512 */
int odt_affine_act(const void* in, void* out, int dtype, long long pixels, int C, int ld,
                   const float* scale, const float* shift, int act, void* stream);
/* out = a + legacy_bilinear_resize(top) (TF1 align_corners=False, no half pixel).
 * ref: RetinaNet.py:309-310, FCOS.py:372-373.  Optional second output
 * out1 = act(out*scale2+shift2). */
int odt_upsample_bilinear_add(const void* top, const void* a, void* out, int dtype, int B, int TH,
                              int TW, int H, int W, int C, int ld, const float* scale2,
                              const float* shift2, int act2, void* out1, void* stream);
/* out[..., :Ca] = a ; out[..., Ca:Ca+Cb] = nearest_resize(b).  ref: YOLOv3.py:406-407 */
int odt_upsample_nearest_concat(const void* a, const void* b, void* out, int dtype, int B, int H,
                                int W, int Ca, int lda, int BH, int BW, int Cb, int ldb, int ldo,
                                void* stream);
/* GroupNorm(groups) statistics: stats[b][g] = (mean, rstd), eps inside; stats holds B*groups*2 floats.
 * One CTA per (group, image), two passes (mean, then the sum of squared deviations) in a fixed order: the result
 * does not depend on B or on scheduling.  ref: FCOS.py:438-446 */
int odt_groupnorm_stats(const void* in, float* stats, int dtype, int B, long long hw, int C,
                        int ld, int groups, float eps, void* stream);
/* y = act((x-mean)*rstd*gamma[c] + beta[c]) */
int odt_groupnorm_apply(const void* in, void* out, const float* stats, int dtype, int B,
                        long long hw, int C, int ld, int groups, const float* gamma,
                        const float* beta, int act, void* stream);
/* Bytes of the workspace odt_groupnorm_act needs for this shape; 0 when the shape is outside its two-launch path
 * (C and groups powers of two, C a multiple of the vector width (8 fp16 / 4 fp32) and at most 256 vectors,
 * groups <= 64, B*groups <= 6144). */
long long odt_groupnorm_act_workspace_bytes(int dtype, int B, long long hw, int C, int groups);
/* GroupNorm + activation in two launches.  Statistics: each image is cut into pixel slices chosen from (hw, C) alone;
 * every slice is reduced two-pass in a fixed order and the last CTA of the image merges the slices in a fixed order in
 * fp64, so the output is reproducible and does not depend on B.  `workspace`: odt_groupnorm_act_workspace_bytes()
 * bytes, 8-byte aligned, zeroed by the caller before its first use (the launch leaves it zeroed where that matters:
 * its per-image arrival counters).  Returns ODT_ERR_UNSUPPORTED (nothing launched) for other shapes or for tensors
 * that are not 16-byte aligned -- use stats + apply then. */
int odt_groupnorm_act(const void* in, void* out, void* workspace, int dtype, int B, long long hw, int C,
                      int ld, int groups, float eps, const float* gamma, const float* beta, int act,
                      void* stream);

/* ------------------------------------------------- decode + NMS tail ----- */
#define ODT_DECODE_SSD 0    /* SSD300/SSD512/RetinaNet: softmax+argmax+bg filter */
#define ODT_DECODE_YOLO3 1  /* sigmoid cls * sigmoid obj, additive exp           */
#define ODT_DECODE_FCOS 2   /* sigmoid cls * sigmoid ctr, exp(l,r,t,b)           */

typedef struct {
  int H, W, A;  /* feature grid and priors per cell                            */
  int offset;   /* first candidate row of this level                          */
  /* centre: cy = ((i+0.5)*cmul_y)/cdiv_y   (SSD: cmul=input, cdiv=H;
   *         RetinaNet: cmul = W_in/H_feat, cdiv = 1).  YOLO: cy = i+0.5.
   *         FCOS: cy = i.                                                     */
  float cmul_y, cdiv_y, cmul_x, cdiv_x;
  float out_mul; /* YOLO: 32,32,16 ; FCOS: stride                              */
  float prior_h[ODT_MAX_PRIORS], prior_w[ODT_MAX_PRIORS];
} odt_level;

typedef struct {
  int kind;       /* ODT_DECODE_*                                              */
  int num_levels;
  int N;          /* candidates (rows) per image                               */
  int num_fg;     /* classes thresholded (SSD/RetinaNet: 20 of 21; YOLOv3 /
                     FCOS: 1..128); a candidate row is num_fg + 5 floats       */
  int nms_classes;/* classes the NMS loop visits, 0..num_fg (FCOS: num_fg - 1,
                     ref FCOS.py:252)                                          */
  float score_thr, iou_thr;
  int max_boxes;
  int cap;        /* candidate capacity per (image, class)                     */
  odt_level level[ODT_MAX_LEVELS];
} odt_tail_params;

/* fused: score activation + anchor/prior generation + threshold + candidate
 * compaction.  head: fp32 [B,N,num_fg+5] rows (layout per kind, see DESIGN.md).
 * cand_keys: u64 [B,num_fg,cap]; cand_count: i32 [B,num_fg] (zeroed here).
 * ref: SSD300.py:157-172,323-343; RetinaNet.py:224-239,328-355;
 *      YOLOv3.py:320-351,419-433; FCOS.py:130-150,197-248 */
int odt_decode_candidates(const float* head, const odt_tail_params* p, int B,
                          unsigned long long* cand_keys, int* cand_count, void* stream);
/* per-(image,class) exact TF NonMaxSuppressionV3 + class-major compaction.
 * dets: f32 [B, nms_classes*max_boxes, 6] rows (score,y1,x1,y2,x2,class);
 * det_anchor: i32 same rows (candidate row index = the keep index);
 * det_count: i32 [B]; status: i32 [1] (zeroed by this call, then 0 ok / ODT_ERR_OVERFLOW if any
 * list overflowed `cap`).  dets_img_stride: floats between the images of `dets` (0 = dense,
 * D*6 with D = nms_classes*max_boxes); with a stride >= D*6+2 the two floats behind an image's D
 * rows receive (float) det_count and its overflow flag (0 / 1): `dets` is then the packed
 * fixed-size record [B, D*6+2] that one all-gather / one device->host copy ships.  work: i32 [round_up(B,2) + 2] zero-initialised, 8-byte aligned scratch
 * (per-image completion counters reset by the kernel, then the 64-bit bump pointer
 * of the box pool).  nms_classes = 0: no list is visited, only the counts / flags are written.
 * box_pool: optional f32 [box_pool_entries][4]
 * scratch where lists longer than the 1024-entry shared-memory window cache their
 * decoded boxes when they take the full-list path (the prefilter subset ran dry, or more
 * than 1024 scores tie at the top); NULL / exhausted -> boxes are re-decoded every round.
 * ref: SSD300.py:173-190; RetinaNet.py:240-256; YOLOv3.py:352-368; FCOS.py:249-264 */
int odt_nms_per_class(const float* head, const odt_tail_params* p, int B,
                      unsigned long long* cand_keys, const int* cand_count, float* dets,
                      int* det_anchor, int* det_count, int* sel_scratch, int* work, int* status,
                      float* box_pool, long long box_pool_entries, long long dets_img_stride,
                      void* stream);
/* bytes of sel_scratch needed by odt_nms_per_class */
long long odt_nms_scratch_bytes(const odt_tail_params* p, int B);

/* Training-loss forwards, one per family.  All four share one calling convention:
 *   head: the [B,N,num_fg+5] candidate rows the inference tail reads (SSD / RetinaNet: num_fg = 20;
 *   YOLOv3 / FCOS: 1..128); gt: f32 [B,G,5] rows (y,x,h,w,id)
 *   padded with -1 (G <= 128); loss_out: f32 [B] per-image loss (the reference averages them over the
 *   batch and adds weight decay on the host side of the graph);
 *   scratch: odt_<family>_loss_scratch_bytes(p, B) bytes, 8-byte aligned, owned by the call until it
 *   completes on `stream`.  The size queries return -1 for a null p, B <= 0 or p->N <= 0. */

/* RetinaNet softmax focal loss + smooth-L1 (anchor/GT matching included).
 * ref: RetinaNet.py:357-474 */
long long odt_retina_loss_scratch_bytes(const odt_tail_params* p, int B);
int odt_retina_loss_fwd(const float* head, const odt_tail_params* p, int B, const float* gt, int G,
                        float alpha, float gamma, void* scratch, float* loss_out, void* stream);
/* SSD300 / SSD512 training-loss forward (matching, cross-entropy, smooth-L1, hard-negative mining by
 * NonMaxSuppressionV3 over the negative anchors): replaces `_compute_one_image_loss`
 * SSD300.py:345-453 (SSD512.py same body).  info_out: i32 [B,3] (#positives, #negatives, #mined
 * negatives) per image, or NULL. */
long long odt_ssd_loss_scratch_bytes(const odt_tail_params* p, int B);
int odt_ssd_loss_fwd(const float* head, const odt_tail_params* p, int B, const float* gt, int G,
                     void* scratch, float* loss_out, int* info_out, void* stream);
/* FCOS training-loss forward (level assignment by GT size, inside-box targets, IoU loss, centre-ness
 * BCE, sigmoid focal loss): replaces FCOS.py:153-187 + `_compute_one_image_loss` FCOS.py:266-348 on
 * the candidate rows [20 cls, ctr, l, r, t, b (pre-exp)]. */
long long odt_fcos_loss_scratch_bytes(const odt_tail_params* p, int B);
int odt_fcos_loss_fwd(const float* head, const odt_tail_params* p, int B, const float* gt, int G,
                      void* scratch, float* loss_out, void* stream);
/* YOLOv3 training-loss forward (per-GT level / prior assignment by anchor IoU at the GT's cell,
 * sigmoid-CE centre / class / objectness terms, squared log-size term, no-object term over the cells
 * without a GT centre): replaces the loss section of `_build_graph` YOLOv3.py:115-318 on the candidate
 * rows [20 cls, y, x, h, w, obj].  The four scales are config['coord_scale' | 'noobj_scale' |
 * 'obj_scale' | 'class_scale'].  loss_out [B] is pos_loss + neg_loss per image (the graph then takes
 * 0.5 x the batch mean).  Every level holds the same number of priors A (1..ODT_MAX_PRIORS), its rows
 * cell after cell with the A priors of a cell consecutive: level.offset = rows of the levels before it,
 * N = sum of H*W*A; anything else is rejected before any launch.  The scratch holds one byte per cell. */
long long odt_yolo_loss_scratch_bytes(const odt_tail_params* p, int B);
int odt_yolo_loss_fwd(const float* head, const odt_tail_params* p, int B, const float* gt, int G,
                      float coord_scale, float noobj_scale, float obj_scale, float class_scale,
                      void* scratch, float* loss_out, void* stream);

/* Training-loss gradients, one per family: the family's loss forward (same kernels, same arguments, same
 * checks, loss_out / info_out bit-identical to the _fwd call) followed by its gradient kernel.
 *   grad_out: f32 [B,N,num_fg+5], every element written: d loss_out[b] / d head[b], zero where a row has no
 *   gradient.  It restates the gradient of the training step's autograd loss (odt_b200/train.py):
 *   RetinaNet: focal (through clamp(p, 1e-8, 1), zero outside) and smooth-L1, / #positives, ignored anchors 0;
 *   SSD: (softmax - one-hot) / #positives on positives, smooth-L1 / #positives on their boxes,
 *   (softmax - one-hot(background)) / #mined on the mined negatives only;
 *   FCOS: per level with GT, IoU loss through exp(), centre-ness BCE, sigmoid focal, / its positive class cells;
 *   YOLOv3: sigmoid-BCE and squared log-size terms of the assigned (cell, prior) rows, the no-object term on
 *   the objectness column under its mask, / #GT.
 * GTs sharing a row add up in GT order; no floating-point atomics: the gradient is bit-identical from run to
 * run and an image's gradient does not depend on its batch.  scratch: odt_<family>_loss_scratch_bytes. */
int odt_retina_loss_grad(const float* head, const odt_tail_params* p, int B, const float* gt, int G,
                         float alpha, float gamma, void* scratch, float* loss_out, float* grad_out, void* stream);
int odt_ssd_loss_grad(const float* head, const odt_tail_params* p, int B, const float* gt, int G,
                      void* scratch, float* loss_out, int* info_out, float* grad_out, void* stream);
int odt_fcos_loss_grad(const float* head, const odt_tail_params* p, int B, const float* gt, int G,
                       void* scratch, float* loss_out, float* grad_out, void* stream);
int odt_yolo_loss_grad(const float* head, const odt_tail_params* p, int B, const float* gt, int G,
                       float coord_scale, float noobj_scale, float obj_scale, float class_scale,
                       void* scratch, float* loss_out, float* grad_out, void* stream);

/* ------------------------------------------------- classification tail --- */
/* Global mean pool + arg-max (+ sparse softmax cross-entropy) of RetinaNet's ImageNet-pretraining mode.
 *   feat: activation `dtype` [B][H+2*halo][W+2*halo][ld], real channels [0, C) (C <= 4096, ld >= C); the halo
 *         border and channels >= C are never summed.
 *   logits: f32 [B,C] = (float)(sum over H x W, in fp64) / (H*W), rounded division;
 *   pred: i64 [B] = the first maximum of each row (tf.argmax);
 *   labels: i64 [B] and loss: f32 [B], both or neither: loss = log(sum_c exp(x_c - max)) - (x_label - max),
 *         NaN for a label outside [0, C) (the host rejects those before the call).
 * One CTA per image, fixed-order reductions: repeated calls give bit-identical results.
 * ref: RetinaNet.py:123-127 (reduce_mean over [1, 2], sparse_softmax_cross_entropy, argmax) */
int odt_pool_classify(const void* feat, int dtype, int B, int H, int W, int C, int ld, int halo, float* logits,
                      long long* pred, const long long* labels, float* loss, void* stream);

/* ------------------------------------------------------- multi-GPU ------- */
/* One process per GPU; images shard batch-parallel, weights are replicated, and the only data-path collective is
 * ONE all-gather of the packed detection records (the `dets` buffer of odt_nms_per_class with the record stride).
 * The context holds the NCCL communicator -- the library's only piece of cross-call state.  NCCL is loaded at run
 * time (libnccl.so.2, or ODT_NCCL_LIB); without it these calls return ODT_ERR_UNSUPPORTED.  The reference is
 * single-device (SSD300.py:458-462): no counterpart there.
 *   odt_ctx_unique_id : rank 0 fills a 128-byte id; the host ships it to the other ranks out of band
 *   odt_ctx_create    : collective over all ranks, binds the communicator to the CURRENT CUDA device
 *   odt_allgather_dets: rec_all[r*floats_per_rank ...] = rank r's rec_local, on `stream`
 *   odt_bcast_weights : in-place broadcast of `bytes` bytes from `root` (weight replication at start-up)          */
typedef struct odt_ctx odt_ctx;
int odt_ctx_unique_id(void* id128_host);
int odt_ctx_create(odt_ctx** ctx, int rank, int world, const void* id128_host);
int odt_ctx_destroy(odt_ctx* ctx);
int odt_allgather_dets(odt_ctx* ctx, const float* rec_local, float* rec_all, long long floats_per_rank,
                       void* stream);
int odt_bcast_weights(odt_ctx* ctx, void* buf, long long bytes, int root, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* ODT_B200_H_ */
