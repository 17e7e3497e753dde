/* propainter_b200 -- C ABI of the sm_90a hot-path kernels (libpropainter_b200.so).
 *
 * The reference (sczhou/ProPainter) has no native code and no FFI: every op below replaces a
 * *library call site* in the reference's Python (torch / torchvision), cited per entry point.
 * A reference-side binding is a ctypes stub (INTEGRATION.md).  Conventions (SURVEY.md §8b):
 *   - plain pointers + sizes, device pointers unless noted; no torch types
 *   - returns 0 or a negative PP_ERR_* code; never throws, never allocates, never synchronises
 *   - caller owns every buffer incl. workspace (size from pp_<op>_workspace_bytes)
 *   - stream-ordered on `stream`, re-entrant across streams, no global mutable state
 * Layouts: "planar" = [n][c][H][W] (reference API boundary); "pixel-major" = [n][H][W][ld], ld >= C
 * given explicitly so ops can read / write channel slices of wider concat buffers.  fp32 throughout.
 */
#ifndef PROPAINTER_B200_H
#define PROPAINTER_B200_H
#include <stddef.h>
#include <stdint.h>
#include <cuda_runtime_api.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PP_ABI_VERSION 2
int pp_abi_version(void);
const char* pp_error_string(int code);

/* ---- RAFT correlation (RAFT/corr.py) -------------------------------------------------------- */
/* CorrBlock.corr :52-60.  fmap pixel-major [frames][h*w][D]; pair p correlates frame idx1[p] with
 * idx2[p] (device int32 arrays).  Writes level 0: [n_pairs][h*w][h][ld0], ld0 = roundup4(w). */
int pp_corr_build(const float* fmap, int D, const int* idx1, const int* idx2, int n_pairs, float* lvl0, int h, int w,
                  cudaStream_t stream);
/* CorrBlock.__init__ :25-27 (3x avg_pool2d).  levels[l]: [planes][h>>l][roundup4(w>>l)] (host array of
 * 4 device pointers); level 0 must be filled. */
int pp_corr_pool_pyramid(float* const* levels, long planes, int h, int w, cudaStream_t stream);
/* CorrBlock.__call__ :29-50 + bilinear_sampler RAFT/utils/utils.py:57-71.
 * coords [n_pairs*h*w][2] (x,y) -> out pixel-major [n_pairs*h*w][324]. */
int pp_corr_lookup(const float* const* levels, const float* coords, float* out, long n_pairs, int h, int w,
                   cudaStream_t stream);
/* same contract, plain global loads instead of TMA staging (baseline for the ncu comparison) */
int pp_corr_lookup_ldg(const float* const* levels, const float* coords, float* out, long n_pairs, int h, int w,
                       cudaStream_t stream);
/* AlternateCorrBlock RAFT/corr.py:83-111 (the memory-free lookup behind args.alternate_corr, raft.py:44-45,106-109):
 * levels 1-3 of the per-frame feature pyramid, 2x2 average pooling with avg_pool2d's floor sizes.  fmap pixel-major
 * [frames][h*w][D] (D % 4 == 0); pooled: host array of 3 device pointers, pooled[l-1] = [frames][(h>>l)*(w>>l)][D]. */
int pp_corr_fmap_pyramid(const float* fmap, int D, int frames, int h, int w, float* const* pooled, cudaStream_t stream);
/* The lookup of AlternateCorrBlock: pair p correlates frame idx1[p] with idx2[p] of fmap (level 0) and pooled (levels
 * 1-3, from pp_corr_fmap_pyramid) at lookup time; D = 256.  Writes the tensor of pp_corr_lookup -- coords
 * [n_pairs*h*w][2] (x,y) -> out [n_pairs*h*w][324] -- with CorrBlock's channel order, /sqrt(D) scaling and sampling
 * rule (corr.py:29-50, bilinear_sampler RAFT/utils/utils.py:57-71), so no volume of n_pairs*(h*w)^2 floats is stored. */
int pp_corr_lookup_otf(const float* fmap, const float* const* pooled, int D, const int* idx1, const int* idx2, int n_pairs,
                       const float* coords, float* out, int h, int w, cudaStream_t stream);
/* RAFT.upsample_flow RAFT/raft.py:73-84.  mask pixel-major [n*h*w][ld_mask>=576] (unscaled conv output,
 * mask_scale = 0.25 from update.py:135); flow_lr [n][h][w][2]; out planar [n][2][8h][8w]. */
int pp_convex_upsample(const float* mask, int ld_mask, float mask_scale, const float* flow_lr, float* out, int n,
                       int h, int w, cudaStream_t stream);

/* ---- propagation ---------------------------------------------------------------------------- */
/* InpaintGenerator.img_propagation model/propainter.py:315-317 (BidirectionalPropagation :104-190,
 * learnable=False; flow_warp model/modules/flow_loss_utils.py:6-45; fbConsistencyCheck :22-31).
 * All planar, batch 1: frames [t][3][H][W], flows [t-1][2][H][W], masks [t][1][H][W]. nearest: 1|0. */
size_t pp_img_prop_scan_workspace_bytes(int t, int H, int W);
int pp_img_prop_scan(const float* frames, const float* flows_f, const float* flows_b, const float* masks,
                     float* out_frames, float* out_masks, void* workspace, size_t ws_bytes, int t, int H, int W,
                     int nearest, cudaStream_t stream);
/* One step's prologue of BidirectionalPropagation(learnable=True) model/propainter.py:144-166:
 * fb-check + bilinear flow_warp + the two torch.cat's.  Pixel-major features (C channels), flows /
 * masks pixel-interleaved [h][w][2].  cond = [cur | warped | fx fy | valid | m0 m1 | 0..],
 * bb = [cur | <slot for the aligned feature> | m0 m1 | 0..]; first!=0: no cond, slot := cur. */
int pp_prop_cond(const float* cur, int ld_cur, const float* prop, int ld_prop, const float* fprop,
                 const float* fcheck, const float* mcur, float* cond, int ld_cond, float* bb, int ld_bb, int h, int w,
                 int C, int first, cudaStream_t stream);
/* DeformableAlignment.forward model/propainter.py:57-69 and SecondOrderDeformableAlignment.forward
 * model/recurrent_flow_completion.py:31-44 after the conv_offset stack (torchvision.ops.deform_conv2d,
 * 3x3/s1/p1, 16 deform groups).  x pixel-major [H*W][ld_x] (Cin), o = raw conv_offset output
 * [H*W][ld_o>=432], flow [H*W][2] or NULL, w_packed [9*Cin][128] (row = tap*Cin + c), out [H*W][ld_out]. */
size_t pp_deform_align_workspace_bytes(int H, int W);   /* decoded tap records + split-K partial sums */
int pp_deform_align(const float* x, int ld_x, const float* o, int ld_o, const float* o_bias, const float* flow, float max_res,
                    const float* w_packed, const float* bias, float* out, int ld_out, int H, int W, int Cin, int Cout,
                    void* workspace, size_t ws_bytes, cudaStream_t stream);
/* ---- wgmma convolution (conv_umma.cu) ---------------------------------------------------------- */
/* Stride-1 "same" KHxKW convolution + the epilogue that follows it in the reference, as one kernel:
 *   out = post_relu?( act( conv(cat(seg...), W) + bias + pre ) + res )        [optionally rounded to TF32 on store]
 * Replaces F.conv2d / nn.Conv2d (cuDNN) + bias + nn.LeakyReLU/ReLU + residual add + torch.cat of the recurrent
 * propagation steps: model/propainter.py:42-50 (conv_offset), :86-96 (backbone / fuse), :146-176 (step);
 * model/recurrent_flow_completion.py:17-29, :60-66, :96-110; RAFT/update.py:33-60,79-97 (same op, 1x5 / 5x1 / 3x3).
 * With KH = KW = 1 over the columns written by pp_deform_gather it is the GEMM of torchvision.ops.deform_conv2d
 * (model/propainter.py:67-69, model/recurrent_flow_completion.py:42-44).
 * seg[i]: pixel-major input maps [n][H][W][ld] (C channels used, any C >= 1; ld % 4 == 0) concatenated along channels.
 * w_packed: [Cout][K], K = KH*KW*sum_i roundup32(C_i); inside segment i, 32-channel block b (global block index blk):
 *   k = ((blk*KH + dy)*KW + dx)*32 + c   (c = channel - 32*b; padded channels hold zeros).  TF32 products, fp32 accumulate.
 * bias [Cout] | NULL; pre (pre-activation addend) / res (post-activation residual): pixel-major [n*H*W][ld] | NULL.
 * act: 0 none, 1 relu, 2 leaky(slope), 3 sigmoid, 4 tanh.  Cout % 4 == 0.  bn / tile_w / tile_m: 0 = choose (see _plan). */
#define PP_CONV_MAX_SEG 4
typedef struct PPConvSeg { const float* x; int ld; int C; } PPConvSeg;
typedef struct PPConvParams {
  PPConvSeg seg[PP_CONV_MAX_SEG];
  int nseg;
  int n, H, W, KH, KW;
  const float* w_packed;
  int Cout;
  const float* bias;
  const float* pre; int ld_pre;
  const float* res; int ld_res;
  float* out; int ld_out;
  int act; float slope; int post_relu; int round_tf32;
  int bn, tile_w, tile_m;   /* tiling hints, 0 = choose: output channels per CTA (32|64|128), tile width (8|16), pixels per CTA (64|128) */
} PPConvParams;
int pp_conv2d_umma(const PPConvParams* prm, cudaStream_t stream);
/* the tiling pp_conv2d_umma will use for `prm` (no launch): pixel tile, output-channel tile, CTA count, dynamic smem */
int pp_conv2d_umma_plan(const PPConvParams* prm, int* tile_h, int* tile_w, int* bn, int* ctas, int* smem_bytes);
/* Sampling half of torchvision.ops.deform_conv2d for DeformableAlignment / SecondOrderDeformableAlignment (same call
 * sites as pp_deform_align): x [n][H][W][ld_x] (Cin = 128 | 256), o = raw conv_offset output [n*H*W][ld_o >= 432],
 * o_bias [432] | NULL, flow [n*H*W][2] | NULL -> cols [n*H*W][9*Cin] (k*Cin + c), modulated samples rounded to TF32.
 * x2 != NULL: channels [Cin/2, Cin) come from a second map x2 [n][H][W][ld_x2] (x then holds channels [0, Cin/2)). */
int pp_deform_gather(const float* x, int ld_x, const float* x2, int ld_x2, const float* o, int ld_o, const float* o_bias,
                     const float* flow, float max_res, float* cols, int n, int H, int W, int Cin, cudaStream_t stream);
/* flow_warp (model/modules/flow_loss_utils.py:6-45; bilinear, zeros padding, align_corners=True) of pixel-major feature
 * maps and fbConsistencyCheck (model/propainter.py:22-31), batched: feat [n][h][w][ld_f] (C channels), fprop / fcheck
 * [n][h][w][2] (x,y) -> warped [n][h][w][ld_w] (NULL to skip; feat may then be NULL), aux [n][h][w][ld_a >= 3] receives
 * (fprop.x, fprop.y, valid) (NULL to skip; fcheck may then be NULL).  The per-step prologue of
 * BidirectionalPropagation.forward model/propainter.py:146-148 when the concat buffers of pp_prop_cond are not wanted. */
int pp_flow_warp_fbcheck(const float* feat, int ld_f, const float* fprop, const float* fcheck, float* warped, int ld_w,
                         float* aux, int ld_a, int n, int h, int w, int C, int round_tf32, cudaStream_t stream);

/* ---- generator glue ------------------------------------------------------------------------- */
/* F.interpolate block of InpaintGenerator.forward model/propainter.py:338-342: flows planar
 * [lt-1][2][H][W] -> [lt-1][H/4][W/4][2] (/4); masks planar [>=lt][1][H][W] -> pmask [lt][H/4][W/4][2]. */
int pp_gen_prep(const float* flows_f, const float* flows_b, const float* masks_in, const float* masks_upd, float* dsf,
                float* dsb, float* pmask, int lt, int H, int W, cudaStream_t stream);
/* max_pool (model/propainter.py:349-350) + window max-pool/sum (sparse_transformer.py:224-229):
 * flags[nwh*nww] = 1 if any local frame has mask inside the window. */
int pp_window_mask(const float* pmask, int lt, int h, int w, int fh, int fw, int nwh, int nww, int* flags,
                   cudaStream_t stream);

typedef struct PPAttnParams {
  const float* qkv;     /* [t][NT][ld_qkv]: Q at +0, K at +C, V at +2C (padded token grid, NT tokens/frame) */
  const float* pool;    /* [t][NP][ld_pool]: pooled K at +0, V at +C */
  const int* key_tok;   /* [n_windows][NKO] token index of own (first WN) + rolled keys */
  const int* flags;     /* [n_windows] window masked? */
  float* out;           /* [t][NT][ld_out] head-concatenated attention output */
  int ld_qkv, ld_pool, ld_out;
  int t, NT, WN, NKO, NP, C;
  int kf_start, kf_step, nkf;   /* key frames T_ind = kf_start + i*kf_step, i < nkf */
  float scale_log2;             /* log2(e)/sqrt(head_dim) */
} PPAttnParams;
/* SparseWindowAttention.forward model/modules/sparse_transformer.py:177-275 (between q/k/v and proj). */
int pp_sparse_window_attn(const PPAttnParams* prm, int n_windows, cudaStream_t stream);
/* same contract; masked windows on the warp-level mma.sync kernel (baseline of the wgmma kernel) */
int pp_sparse_window_attn_mma(const PPAttnParams* prm, int n_windows, cudaStream_t stream);

/* FusionFeedForward.forward model/modules/sparse_transformer.py:81-100: fold -> /normalizer -> unfold -> GELU.
 * Y,Z [frames*fh*fw][ld], hidden columns tap-major (tap*CH + c). */
size_t pp_ffn_overlap_add_workspace_bytes(int frames, int h, int w, int CH);
int pp_ffn_overlap_add(const float* Y, int ldy, float* Z, int ldz, int frames, int h, int w, int CH, void* workspace,
                       size_t ws_bytes, cudaStream_t stream);

/* ---- transformer glue ------------------------------------------------------------------------ */
/* SparseWindowAttention.pool_layer (model/modules/sparse_transformer.py:131-133, used :203-206): depthwise Conv2d with
 * kernel = stride = (kh,kw), no padding.  x [n][H][W][C] pixel-major (pixel stride ld_x), w_taps [kh*kw][C],
 * out [n][H/kh][W/kw][C] dense. */
int pp_pool_depthwise(const float* x, int ld_x, const float* w_taps, const float* bias, float* out, int n, int H, int W, int C,
                      int kh, int kw, cudaStream_t stream);
/* TemporalSparseTransformer.forward model/modules/sparse_transformer.py:322-334: x_out = x + delta (residual),
 * y = LayerNorm(x_out) * gamma + beta, rows of C in {128,256,512,1024} floats.  delta NULL: plain LayerNorm. */
int pp_add_layernorm(const float* x, const float* delta, const float* gamma, const float* beta, float* x_out, float* y, long rows,
                     int C, float eps, cudaStream_t stream);

/* ---- RAFT SepConvGRU elementwise fusion (RAFT/update.py:45-60,95-97) ------------------------- */
/* zr: raw output of the fused z|r gate conv [npix][2C]; net: state slice of HX (ld_net); writes z [npix][C]
 * and r*net into the state slice of RX (ld_r).  bias [2C] and pre [npix][2C] are nullable addends: `pre` carries the
 * part of the gate convs that does not change over the refinement iterations (the context-feature input channels,
 * RAFT/update.py:129), convolved once per clip. */
int pp_gru_gate(const float* zr, const float* bias, const float* pre, const float* net, int ld_net, float* z, float* rnet,
                int ld_r, long npix, int C, cudaStream_t stream);
/* net = (1-z)*net + z*tanh(q + bias + pre), in place on the state slice of HX; net_copy (nullable, dense [npix][C]) also
 * receives the new state (input of the flow / mask heads, RAFT/update.py:133-136). */
int pp_gru_update(const float* q, const float* bias, const float* pre, const float* z, float* net, int ld_net, float* net_copy,
                  long npix, int C, cudaStream_t stream);
/* motion features: channels [0,126) of `mot` + the 2 flow channels -> the same 128-channel slot of d0 and d1.
 * bias != NULL: `mot` is the raw conv output and relu(mot + bias) (RAFT/update.py:96) is applied on the way. */
int pp_raft_pack_motion(const float* mot, int ld_mot, const float* bias, const float* flow, float* d0, float* d1, int ld,
                        long npix, cudaStream_t stream);

/* ---- conv epilogues ------------------------------------------------------------------------- */
/* out = post(act(x + bias[c]) + res) on pixel-major tensors [n_pix][C] with pixel strides ld_*: replaces the bias add of
 * F.conv2d, the ReLU / LeakyReLU / sigmoid / tanh that follows it at every conv of the three nets, the residual add
 * (+ ReLU) of RAFT/extractor.py:49-57, model/propainter.py:173-176, model/recurrent_flow_completion.py:108-110, and --
 * through a strided `out` -- the torch.cat of RAFT/update.py:95.  bias / res nullable; out may alias x.
 * act: 0 none, 1 relu, 2 leaky(slope), 3 sigmoid, 4 tanh; post_relu: final ReLU after the residual add. */
int pp_bias_act(const float* x, int ld_x, const float* bias, const float* res, int ld_res, float* out, int ld_out, long n_pix,
                int C, int act, float slope, int post_relu, cudaStream_t stream);
/* the same with a per-pixel pre-activation addend pre [n_pix][C] (stride ld_pre, nullable): out = post(act(x + bias + pre) + res).
 * conv(cat[a, b]) = conv_a(a) + conv_b(b): the share of a recurrent step's conv over step-independent inputs (current frame,
 * flow, masks; model/propainter.py:151,171, model/recurrent_flow_completion.py:96-106) is convolved once per scan and added here. */
int pp_bias_act_pre(const float* x, int ld_x, const float* bias, const float* pre, int ld_pre, const float* res, int ld_res,
                    float* out, int ld_out, long n_pix, int C, int act, float slope, int post_relu, cudaStream_t stream);

/* nn.InstanceNorm2d(affine=False, eps) of the RAFT feature encoder (RAFT/extractor.py:18-21,125,168-192) on channels-last
 * maps x [n][HW][C]: out = post(relu?((x - mean) * rstd) + res), statistics per (sample, channel), biased variance.
 * res nullable (dense, same shape); out may alias x. */
size_t pp_instance_norm_workspace_bytes(int n, long HW, int C);
int pp_instance_norm(const float* x, const float* res, float* out, int n, long HW, int C, float eps, int relu, int post_relu,
                     void* workspace, size_t ws_bytes, cudaStream_t stream);
/* `deconv` up-sampling, F.interpolate(scale_factor=2, bilinear, align_corners=True)
 * (model/propainter.py:248-253, model/recurrent_flow_completion.py:141-146); pixel-major [n][h][w][C] -> [n][2h][2w][C]. */
int pp_upsample2x_bilinear(const float* src, float* dst, int n, int h, int w, int C, cudaStream_t stream);

/* ---- driver-side pixel ops (inference_propainter.py) ----------------------------------------- */
/* read_mask's scipy.ndimage.binary_dilation(mask, iterations=k) (cross structure) + to_tensors (inference_propainter.py:93-107,
 * :265-266): uint8 masks [T][H][W] (non-zero = hole) -> float {0,1} [T][1][H][W]; iterations = 0 only binarises. */
int pp_mask_dilate(const uint8_t* src, float* dst, int T, int H, int W, int iterations, cudaStream_t stream);
/* to_tensors()(frames)*2-1  core/utils.py:130-170 + inference_propainter.py:264: uint8 [T][H][W][3] -> planar float */
int pp_u8_to_frames(const uint8_t* src, float* dst, int T, int H, int W, cudaStream_t stream);
/* ---- resizing around the path (inference_propainter.py:34-45 resize_frames, :95-96 mask resize, :469-470 output resize) --- */
/* HOST helpers (no GPU work): the per-axis tables of the three library resamplers the reference calls.
 * bicubic: Pillow's Image.resize(size) on 8-bit images (BICUBIC, 22-bit fixed point): bounds [out*2] = (first source index,
 * taps), kk [out*ksize]; returns ksize (kk == NULL: query only) or < 0.  nearest: Pillow's Image.resize(size, NEAREST): source
 * index per destination index.  linear_cv: OpenCV's 8-bit INTER_LINEAR: ofs [out], coef [out*2] (11-bit taps). */
int pp_resample_coeffs_bicubic(int in_size, int out_size, int* bounds, int* kk, long kk_capacity);
int pp_resample_index_nearest(int in_size, int out_size, int* idx);
int pp_resample_coeffs_linear_cv(int in_size, int out_size, int horizontal, int* ofs, short* coef);
/* Device passes; tables are device copies of the above.  uint8 [T][H][W][3] -> [T][Ho][Wo][3] (nearest: C channels). */
size_t pp_resize_u8_bicubic_workspace_bytes(int T, int H, int Wo);
int pp_resize_u8_bicubic(const uint8_t* src, uint8_t* dst, int T, int H, int W, int Ho, int Wo, const int* bounds_x, const int* kk_x,
                         int ksize_x, const int* bounds_y, const int* kk_y, int ksize_y, void* workspace, size_t ws_bytes,
                         cudaStream_t stream);
int pp_resize_u8_nearest(const uint8_t* src, uint8_t* dst, int T, int H, int W, int Ho, int Wo, int C, const int* idx_x, const int* idx_y,
                         cudaStream_t stream);
int pp_resize_u8_bilinear_cv(const uint8_t* src, uint8_t* dst, int T, int H, int W, int Ho, int Wo, const int* xofs, const short* alpha,
                             const int* yofs, const short* beta, cudaStream_t stream);
#define PP_MAX_WINDOW 32
typedef struct PPWindowIds { int n; int frame[PP_MAX_WINDOW]; int first[PP_MAX_WINDOW]; } PPWindowIds;
/* inference_propainter.py:437-450: pred planar [n][3][H][W] in (-1,1), masks planar [T][1][H][W],
 * ori/comp uint8 [T][H][W][3]; ids (host struct): target frame + first-visit flag per local frame. */
int pp_composite_blend_u8(const float* pred, const float* masks, const uint8_t* ori, uint8_t* comp,
                          const PPWindowIds* ids, int H, int W, cudaStream_t stream);
/* ---- video outpainting (inference_propainter.py --mode video_outpainting) --------------------------- */
/* extrapolation inference_propainter.py:117-156 + to_tensors of its masks (:265-266): uint8 frames [T][h][w][3] are
 * placed at (top, left) of a zero canvas [T][H][W][3]; flow_masks / masks_dilated float {0,1} [T][1][H][W] are 1 outside
 * [top+rim_h, top+h-rim_h) x [left+rim_w, left+w-rim_w) and outside the source rectangle respectively (an empty range
 * clears nothing, as numpy slicing does).  The reference's geometry: rim = 4 if offset > 10 else 0.
 * PP_ERR_SHAPE unless the source rectangle lies inside the canvas and the rims are >= 0. */
int pp_extrapolate_u8(const uint8_t* src, uint8_t* canvas, float* flow_masks, float* masks_dilated, int T, int h, int w, int H,
                      int W, int top, int left, int rim_h, int rim_w, cudaStream_t stream);
/* the masked-frame preview inference_propainter.py:250-261: per channel, in float64, fuse = 0.4*img + 0.6*(0,255,0),
 * mask*fuse + (1-mask)*img, truncated to uint8.  frames uint8 [T][H][W][3], masks [T][1][H][W] -> out uint8 [T][H][W][3]. */
int pp_mask_overlay_u8(const uint8_t* frames, const float* masks, uint8_t* out, int T, int H, int W, cudaStream_t stream);
/* ---- optical-flow colour coding (RAFT/utils/flow_viz.py, RAFT/utils/flow_viz_pt.py) ------------------- */
#define PP_FLOWVIZ_FRAME 0 /* flow_viz.py::flow_to_image per frame: rad_max + 1e-5, numpy >= 2 dtypes, rad > 1 -> x0.75 */
#define PP_FLOWVIZ_CLIP 1  /* flow_viz_pt.py::flow_to_image: max_norm + FLT_EPSILON over the whole batch, float32 */
/* Group maxima of sqrt(u^2 + v^2) over planar float32 flow [N][2][H][W], after np.clip(flow, 0, clip_flow) when
 * has_clip: maxima[N] (per_frame = 1) or maxima[1] (per_frame = 0), caller-owned; cleared on the stream first.
 * PP_ERR_SHAPE unless 1 <= N <= 65535 and H, W >= 1. */
int pp_flow_maxrad(const float* flow, float* maxima, int N, int H, int W, int per_frame, int has_clip, float clip_flow,
                   cudaStream_t stream);
/* The colour wheel of `variant` (PP_FLOWVIZ_*) over the same flow (clipped when has_clip), normalised by the maxima of
 * pp_flow_maxrad with the matching per_frame -> uint8 out [N][H][W][3], RGB (BGR when bgr). */
int pp_flow_to_image_u8(const float* flow, const float* maxima, uint8_t* out, int N, int H, int W, int variant, int has_clip,
                        float clip_flow, int bgr, cudaStream_t stream);

#ifdef __cplusplus
}
#endif
#endif
