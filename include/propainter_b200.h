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
 * 4 device pointers); level 0 must be filled.  Columns w>>l .. roundup4(w>>l)-1 of each row are padding: no entry point
 * of this section reads or writes them, so the levels may come from any allocation, zeroed or not. */
int pp_corr_pool_pyramid(float* const* levels, long planes, int h, int w, cudaStream_t stream);
/* CorrBlock.__call__ :29-50 + bilinear_sampler RAFT/utils/utils.py:57-71.
 * coords [n_pairs*h*w][2] (x,y) -> out pixel-major [n_pairs*h*w][324].  n_pairs = 0 returns PP_OK without a launch. */
int pp_corr_lookup(const float* const* levels, const float* coords, float* out, long n_pairs, int h, int w,
                   cudaStream_t stream);
/* same contract, plain global loads instead of TMA staging (baseline for the ncu comparison) */
int pp_corr_lookup_ldg(const float* const* levels, const float* coords, float* out, long n_pairs, int h, int w,
                       cudaStream_t stream);
/* pp_corr_lookup / pp_corr_lookup_ldg writing fp16 (each tap blended in fp32, rounded to nearest once) into rows of
 * ld_out >= 324 halves; channels [324, ld_out) are not written.  The operand of RAFT's half-precision convc1. */
int pp_corr_lookup_f16(const float* const* levels, const float* coords, void* out, int ld_out, long n_pairs, int h, int w,
                       cudaStream_t stream);
int pp_corr_lookup_ldg_f16(const float* const* levels, const float* coords, void* out, int ld_out, long n_pairs, int h, int w,
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
/* Radius-selectable lookups: radius 4 (the basic model, 324 channels) or 3 (RAFT-small, raft.py:29-33: 4 x 7 x 7 = 196
 * channels, l*49 + a*7 + b).  Same contracts as pp_corr_lookup / pp_corr_lookup_ldg / pp_corr_lookup_otf with
 * out [n_pairs*h*w][4*(2*radius+1)^2]; the on-the-fly lookup takes (D, radius) = (256, 4) or (128, 3) and divides by
 * sqrt(D) rounded to float, as CorrBlock.corr does (corr.py:60).  Any other radius or D: PP_ERR_SHAPE. */
int pp_corr_lookup_r(const float* const* levels, int radius, const float* coords, float* out, long n_pairs, int h, int w,
                     cudaStream_t stream);
int pp_corr_lookup_ldg_r(const float* const* levels, int radius, const float* coords, float* out, long n_pairs, int h, int w,
                         cudaStream_t stream);
int pp_corr_lookup_otf_r(const float* fmap, const float* const* pooled, int D, int radius, const int* idx1, const int* idx2,
                         int n_pairs, const float* coords, float* out, int h, int w, cudaStream_t stream);
/* upflow8 RAFT/utils/utils.py:80-82 (RAFT-small's upsampling, raft.py:136-137): 8 * bilinear (align_corners=True)
 * resize to 8h x 8w, bit-exact with ATen's CPU kernel.  flow_lr pixel-major [n][h][w][2] -> out planar [n][2][8h][8w]. */
int pp_upflow8(const float* flow_lr, float* out, int n, int h, int w, cudaStream_t stream);
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
/* The same scan on half-precision clip storage (InferenceConfig.half_storage), with the compositing of
 * inference_propainter.py:372, 389-390, 402 in its epilogue.  frames_u8 uint8 [t][H][W][3] (the clip's frames, masked
 * in-kernel: u8 -> [-1,1], times 1 - masks), masks float {0,1} [t][1][H][W], flows fp16 [t-1][2][H][W].  Writes frames
 * [lo, hi) only: out_frames fp16 [hi-lo][3][H][W] = rn16(frames * (1 - masks) + prop * masks), out_masks fp16
 * [hi-lo][1][H][W] (exact: {0,1}).  All arithmetic fp32, one fp16 rounding per output.  fp16 pointers 2-byte aligned,
 * masks / workspace 4-byte (PP_ERR_ALIGN); lo == hi: PP_OK without a launch. */
size_t pp_img_prop_scan_u8h_workspace_bytes(int t, int H, int W);
int pp_img_prop_scan_u8h(const uint8_t* frames_u8, const float* masks, const void* flows_f, const void* flows_b,
                         void* out_frames, void* out_masks, void* workspace, size_t ws_bytes, int t, int H, int W, int lo,
                         int hi, int nearest, cudaStream_t stream);
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
/* The same convolution on fp16 operands (f16 x f16 products, fp32 accumulate): seg[i].x and w_packed point to fp16 data,
 * segments ld % 8 == 0 and 16-byte aligned (else PP_ERR_ALIGN); w_packed [Cout][K] fp16 in 64-channel blocks,
 * K = KH*KW*sum_i roundup64(C_i), k = ((blk*KH + dy)*KW + dx)*64 + c.  bias / pre / res stay fp32 and the epilogue computes
 * in fp32.  It writes out (fp32, round_tf32 ignored) and / or out16 (fp16 [n*H*W][ld_out16], ld_out16 % 8 == 0, 16-byte
 * aligned, rounded to nearest once); at least one of them (else PP_ERR_SHAPE). */
int pp_conv2d_umma_f16(const PPConvParams* prm, void* out16, int ld_out16, cudaStream_t stream);
/* the tiling pp_conv2d_umma_f16 will use for `prm` (no launch) */
int pp_conv2d_umma_plan_f16(const PPConvParams* prm, int* tile_h, int* tile_w, int* bn, int* ctas, int* smem_bytes);
/* Sampling half of torchvision.ops.deform_conv2d for DeformableAlignment / SecondOrderDeformableAlignment (same call
 * sites as pp_deform_align): x [n][H][W][ld_x] (Cin = 128 | 256), o = raw conv_offset output [n*H*W][ld_o >= 432],
 * o_bias [432] | NULL, flow [n*H*W][2] | NULL -> cols [n*H*W][9*Cin] (k*Cin + c), modulated samples rounded to TF32.
 * x2 != NULL: channels [Cin/2, Cin) come from a second map x2 [n][H][W][ld_x2] (x then holds channels [0, Cin/2)). */
int pp_deform_gather(const float* x, int ld_x, const float* x2, int ld_x2, const float* o, int ld_o, const float* o_bias,
                     const float* flow, float max_res, float* cols, int n, int H, int W, int Cin, cudaStream_t stream);
/* pp_deform_gather with fp16 cols (16-byte aligned), each column rounded to nearest once: the A operand of the fp16
 * deformable GEMM (pp_conv2d_umma_f16).  Inputs and sampling arithmetic stay fp32. */
int pp_deform_gather_f16(const float* x, int ld_x, const float* x2, int ld_x2, const float* o, int ld_o, const float* o_bias,
                         const float* flow, float max_res, void* cols, int n, int H, int W, int Cin, cudaStream_t stream);
/* flow_warp (model/modules/flow_loss_utils.py:6-45; bilinear, zeros padding, align_corners=True) of pixel-major feature
 * maps and fbConsistencyCheck (model/propainter.py:22-31), batched: feat [n][h][w][ld_f] (C channels), fprop / fcheck
 * [n][h][w][2] (x,y) -> warped [n][h][w][ld_w] (NULL to skip; feat may then be NULL), aux [n][h][w][ld_a >= 3] receives
 * (fprop.x, fprop.y, valid) (NULL to skip; fcheck may then be NULL).  The per-step prologue of
 * BidirectionalPropagation.forward model/propainter.py:146-148 when the concat buffers of pp_prop_cond are not wanted. */
int pp_flow_warp_fbcheck(const float* feat, int ld_f, const float* fprop, const float* fcheck, float* warped, int ld_w,
                         float* aux, int ld_a, int n, int h, int w, int C, int round_tf32, cudaStream_t stream);
/* pp_flow_warp_fbcheck with fp16 warped (ld_w % 8 == 0, 16-byte aligned, else PP_ERR_ALIGN), rounded to nearest once: the
 * operand of the fp16 offset-net conv.  feat, the flows and aux stay fp32. */
int pp_flow_warp_fbcheck_f16(const float* feat, int ld_f, const float* fprop, const float* fcheck, void* warped, int ld_w,
                             float* aux, int ld_a, int n, int h, int w, int C, cudaStream_t stream);

/* ---- generator glue ------------------------------------------------------------------------- */
/* F.interpolate block of InpaintGenerator.forward model/propainter.py:338-342: flows planar
 * [lt-1][2][H][W] -> [lt-1][H/4][W/4][2] (/4); masks planar [>=lt][1][H][W] -> pmask [lt][H/4][W/4][2]. */
int pp_gen_prep(const float* flows_f, const float* flows_b, const float* masks_in, const float* masks_upd, float* dsf,
                float* dsb, float* pmask, int lt, int H, int W, cudaStream_t stream);
/* pp_gen_prep on fp16 clip-storage flows (2-byte aligned, widened on load); H = 0 or W = 0: PP_OK without a launch. */
int pp_gen_prep_f16(const void* flows_f, const void* flows_b, const float* masks_in, const float* masks_upd, float* dsf,
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
/* same window / key-table semantics (incl. nkf = 0 and flags) on fp16 operands: qkv [t][NT][3C] and pool [t][NP][2C] fp16,
 * out [t][NT][C] fp16 rounded to nearest; scores, softmax statistics and O accumulate in fp32 (Q is scaled in fp32 and rounded
 * once).  Masked windows: wgmma m64nNk16 f32.f16.f16; unmasked windows: mma.sync m16n8k16.  Rows 16-byte aligned and
 * ld_* % 8 == 0 (else PP_ERR_ALIGN); WN <= 48; t = 0 or n_windows = 0 returns PP_OK without a launch. */
int pp_sparse_window_attn_f16(const PPAttnParams* prm, int n_windows, cudaStream_t stream);

/* FusionFeedForward.forward model/modules/sparse_transformer.py:81-100: fold -> /normalizer -> unfold -> GELU.
 * Y,Z [frames*fh*fw][ld], hidden columns tap-major (tap*CH + c). */
size_t pp_ffn_overlap_add_workspace_bytes(int frames, int h, int w, int CH);
int pp_ffn_overlap_add(const float* Y, int ldy, float* Z, int ldz, int frames, int h, int w, int CH, void* workspace,
                       size_t ws_bytes, cudaStream_t stream);
/* the same on fp16 Y and Z (the half-operand fc1 output and fc2 operand): rows 16-byte aligned, ldy % 8 == ldz % 8 == 0
 * (else PP_ERR_ALIGN); the fold sums in fp32 in the same order into the fp32 workspace, Z is rounded to nearest once.
 * frames = 0 returns PP_OK without a launch. */
int pp_ffn_overlap_add_f16(const void* Y, int ldy, void* Z, int ldz, int frames, int h, int w, int CH, void* workspace,
                           size_t ws_bytes, cudaStream_t stream);
/* SoftComp's fold (model/modules/sparse_transformer.py:49-61) after its Linear layer ran as a GEMM into tap-major columns:
 * cols fp16 [frames*fh*fw][ldc] (column tap*C + c, fh = (h-1)/3+1, fw = (w-1)/3+1, ldc >= 49*C), bmap fp32 [h][w][C] (the
 * fold of the Linear bias) -> out fp16 [frames][h][w][C].  7x7 / stride 3 / pad 3 overlap-add, fp32 sums in a fixed order,
 * rounded to nearest once.  8-byte aligned fp16 rows, C % 4 == ldc % 4 == 0 (else PP_ERR_ALIGN); frames = 0 returns PP_OK
 * without a launch. */
int pp_sc_fold_f16(const void* cols, long ldc, const float* bmap, void* out, int frames, int h, int w, int C, cudaStream_t stream);

/* ---- transformer glue ------------------------------------------------------------------------ */
/* SparseWindowAttention.pool_layer (model/modules/sparse_transformer.py:131-133, used :203-206): depthwise Conv2d with
 * kernel = stride = (kh,kw), no padding.  x [n][H][W][C] pixel-major (pixel stride ld_x), w_taps [kh*kw][C],
 * out [n][H/kh][W/kw][C] dense. */
int pp_pool_depthwise(const float* x, int ld_x, const float* w_taps, const float* bias, float* out, int n, int H, int W, int C,
                      int kh, int kw, cudaStream_t stream);
/* the same on fp16 x and out (the half-operand LayerNorm output and the pooled K/V Linear's operand): weights, bias and the
 * sums fp32, out rounded to nearest; rows 16-byte aligned, C % 8 == ld_x % 8 == 0 (else PP_ERR_ALIGN); n = 0 returns PP_OK. */
int pp_pool_depthwise_f16(const void* x, int ld_x, const float* w_taps, const float* bias, void* out, int n, int H, int W, int C,
                          int kh, int kw, cudaStream_t stream);
/* TemporalSparseTransformer.forward model/modules/sparse_transformer.py:322-334: x_out = x + delta (residual),
 * y = LayerNorm(x_out) * gamma + beta, rows of C in {128,256,512,1024} floats.  delta NULL: plain LayerNorm. */
int pp_add_layernorm(const float* x, const float* delta, const float* gamma, const float* beta, float* x_out, float* y, long rows,
                     int C, float eps, cudaStream_t stream);
/* the same with an fp16 delta (delta_f16 != 0: the half-operand fc2 output) and / or an fp16 y (y_f16 != 0: the operand of the
 * half-operand fc1), rounded to nearest; x / x_out and the statistics stay fp32.  Rows 16-byte aligned (else PP_ERR_ALIGN);
 * rows = 0 returns PP_OK without a launch. */
int pp_add_layernorm_f16(const float* x, const void* delta, int delta_f16, const float* gamma, const float* beta, float* x_out,
                         void* y, int y_f16, long rows, int C, float eps, cudaStream_t stream);

/* ---- RAFT SepConvGRU elementwise fusion (RAFT/update.py:45-60,95-97) ------------------------- */
/* All of them read and write 4 channels at a time: every fp32 pointer must be 16-byte aligned and every stride a multiple
 * of 4 (else PP_ERR_ALIGN, checked before anything is launched); npix = 0 returns PP_OK without a launch. */
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
/* Half-operand variants (fp16 rows 8-byte aligned): the gate / candidate / motion conv outputs (zr, q, mot), rnet, h_img,
 * net_copy, d0 and d1 are fp16; the recurrent state net, z, bias, pre and flow stay fp32, all arithmetic is fp32 and every
 * fp16 store rounds to nearest.  pp_gru_update_f16 updates the fp32 state in place and writes its fp16 image to h_img
 * (the state slice of HX, stride ld_img, nullable) and net_copy (dense, nullable). */
int pp_gru_gate_f16(const void* zr, const float* bias, const float* pre, const float* net, int ld_net, float* z, void* rnet,
                    int ld_r, long npix, int C, cudaStream_t stream);
int pp_gru_update_f16(const void* q, const float* bias, const float* pre, const float* z, float* net, int ld_net, void* h_img,
                      int ld_img, void* net_copy, long npix, int C, cudaStream_t stream);
int pp_raft_pack_motion_f16(const void* mot, int ld_mot, const float* bias, const float* flow, void* d0, void* d1, int ld,
                            long npix, cudaStream_t stream);
/* the same for `cmot` motion channels (RAFT-small: 80, update.py:62-77): channels [0,cmot) of `mot` (+ bias, ReLU), then
 * the 2 flow channels, then zeros up to the slot width roundup4(cmot+2) (<= ld); d0 / d1 16-byte aligned, ld % 4 == 0. */
int pp_raft_pack_motion_n(const float* mot, int ld_mot, const float* bias, const float* flow, float* d0, float* d1, int ld,
                          long npix, int cmot, cudaStream_t stream);

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
/* pp_bias_act_pre with fp16 x (x_f16 != 0, 8-byte aligned rows) and / or fp16 out (out_f16 != 0, rounded to nearest);
 * bias, pre, res and the arithmetic stay fp32.  The epilogue of RAFT's half-precision refinement-loop convs. */
int pp_bias_act_f16(const void* x, int ld_x, int x_f16, const float* bias, const float* pre, int ld_pre, const float* res, int ld_res,
                    void* out, int ld_out, int out_f16, long n_pix, int C, int act, float slope, int post_relu, cudaStream_t stream);
/* pp_bias_act with fp16 x, residual res (may be NULL) and out, 8-byte aligned rows; bias and arithmetic fp32, out rounded
   to nearest once.  Returns PP_ERR_ALIGN / PP_ERR_SHAPE like pp_bias_act_f16. */
int pp_bias_act_f16_res(const void* x, int ld_x, const float* bias, const void* res, int ld_res, void* out, int ld_out, long n_pix,
                        int C, int act, float slope, int post_relu, cudaStream_t stream);

/* nn.InstanceNorm2d(affine=False, eps) of the RAFT feature encoder (RAFT/extractor.py:18-21,125,168-192) on channels-last
 * maps x [n][HW][C]: out = post(relu?((x - mean) * rstd) + res), statistics per (sample, channel), biased variance,
 * computed from double sums of x minus the channel's value at pixel 0 (no cancellation when |mean| >> std).
 * res nullable (dense, same shape); out may alias x. */
size_t pp_instance_norm_workspace_bytes(int n, long HW, int C);
int pp_instance_norm(const float* x, const float* res, float* out, int n, long HW, int C, float eps, int relu, int post_relu,
                     void* workspace, size_t ws_bytes, cudaStream_t stream);
/* `deconv` up-sampling, F.interpolate(scale_factor=2, bilinear, align_corners=True)
 * (model/propainter.py:248-253, model/recurrent_flow_completion.py:141-146); pixel-major [n][h][w][C] -> [n][2h][2w][C]. */
int pp_upsample2x_bilinear(const float* src, float* dst, int n, int h, int w, int C, cudaStream_t stream);
/* the same on fp16 rows (the half-operand decoder; 16-byte aligned rows, C % 8 == 0, else PP_ERR_ALIGN): blend in fp32, rounded to nearest once.
 * n = 0 returns PP_OK without a launch. */
int pp_upsample2x_bilinear_f16(const void* src, void* dst, int n, int h, int w, int C, cudaStream_t stream);

/* ---- driver-side pixel ops (inference_propainter.py) ----------------------------------------- */
/* read_mask's scipy.ndimage.binary_dilation(mask, iterations=k) (cross structure) + to_tensors (inference_propainter.py:93-107,
 * :265-266): uint8 masks [T][H][W] (non-zero = hole) -> float {0,1} [T][1][H][W]; iterations = 0 only binarises. */
int pp_mask_dilate(const uint8_t* src, float* dst, int T, int H, int W, int iterations, cudaStream_t stream);
/* to_tensors()(frames)*2-1  core/utils.py:130-170 + inference_propainter.py:264: uint8 [T][H][W][3] -> planar float */
int pp_u8_to_frames(const uint8_t* src, float* dst, int T, int H, int W, cudaStream_t stream);
/* scripts/compute_flow.py:67-92 (its frame preparation before RAFT): ToTensor (v / 255), F.interpolate(size=(h, w),
 * mode='bilinear', align_corners=False) and img*2 - 1, fused: uint8 RGB [T][H0][W0][3] -> planar float [T][3][h][w] in [-1,1],
 * equal to ATen's CPU resize bit for bit (pp_resize_coord in csrc/pp_elem.cuh); at h == H0, w == W0 equal to
 * pp_u8_to_frames.  Any size < 1: PP_ERR_SHAPE. */
int pp_u8_to_frames_resized(const uint8_t* src, float* dst, int T, int H0, int W0, int h, int w, cudaStream_t stream);
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
/* resize_flow (utils/flow_util.py:6-11) of the evaluation dataset (core/dataset.py:213-214): cv2.resize(INTER_LINEAR) of
 * float32 flows, then component 0 *= float32(Wo/W), component 1 *= float32(Ho/H).  Planar [N][2][H][W] -> [N][2][Ho][Wo].
 * HOST helper pp_resample_coeffs_linear_f32: OpenCV's float tables for one axis, ofs [out], coef [out*2] = (1-f, f).
 * Tables are device copies (unused, may be NULL, for the same size and for exact 2x down-scaling, which is OpenCV's
 * INTER_AREA fast path). */
int pp_resample_coeffs_linear_f32(int in_size, int out_size, int horizontal, int* ofs, float* coef);
int pp_resize_flow_linear_cv(const float* src, float* dst, int N, int H, int W, int Ho, int Wo, const int* xofs, const float* alpha,
                             const int* yofs, const float* beta, cudaStream_t stream);
#define PP_MAX_WINDOW 32
typedef struct PPWindowIds { int n; int frame[PP_MAX_WINDOW]; int first[PP_MAX_WINDOW]; } PPWindowIds;
/* inference_propainter.py:437-450: pred planar [n][3][H][W] in (-1,1), masks planar [T][1][H][W],
 * ori/comp uint8 [T][H][W][3]; ids (host struct): target frame + first-visit flag per local frame. */
int pp_composite_blend_u8(const float* pred, const float* masks, const uint8_t* ori, uint8_t* comp,
                          const PPWindowIds* ids, int H, int W, cudaStream_t stream);
/* scripts/evaluate_propainter.py:166-179: the same inputs, but comp is a float32 clip [T][H][W][3]: a first visit stores
 * the uint8 composite, a later one prev*0.5 + img*0.5 without truncation. */
int pp_composite_blend_f32(const float* pred, const float* masks, const uint8_t* ori, float* comp,
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
/* ---- temporal warping error E_warp ------------------------------------------------------------------------------- */
/* No reference line: the reference defers this metric to the evaluation of Lai et al., "Learning Blind Video Temporal
 * Consistency" (ECCV 2018), whose occlusion test is that of Ruder et al., "Artistic style transfer for videos" (GCPR
 * 2016).  Warps are FlowNet2 Resample2d's border-clamped bilinear sample (pp_clamp_taps in pp_elem.cuh).
 * Flows planar float32 [N][2][H][W], pair t: fw frame t -> t+1, bw frame t+1 -> t.
 * Occlusion map O_t -> occ uint8 [N][H][W], 1 = occluded: |F + w|^2 > 0.01 (|F|^2 + |w|^2) + 0.5 with w = bw sampled at
 * x + F(x), or the motion-boundary test |du|^2 + |dv|^2 > 0.01 |F|^2 + 0.002 (forward differences, 0 in the last
 * column / row).  PP_ERR_SHAPE unless N, H, W >= 1. */
int pp_flow_occlusion(const float* fw, const float* bw, uint8_t* occ, int N, int H, int W, cudaStream_t stream);
/* Per pair t of frames uint8 [T][H][W][3] (values / 255): out float64 [T-1][2] = (sum over pixels with O_t = 0 of
 * sum_c (S(frame t+1, fw_t) - frame t)^2, N_t = their count); E_t = sum / (3 N_t).  O_t is read from occ (uint8
 * [T-1][H][W], non-zero = occluded; bw unused, may be NULL) or, when occ is NULL, computed from fw / bw in the same pass.
 * fp32 per pixel, float64 sums in a fixed order without atomics: the same bits on every run.  Caller-owned workspace of
 * pp_warp_error_workspace_bytes(T, H, W) bytes (0 for an invalid shape).  PP_ERR_SHAPE unless 2 <= T <= 65536, H, W >= 1
 * and occ or bw is given. */
size_t pp_warp_error_workspace_bytes(int T, int H, int W);
int pp_warp_error(const uint8_t* frames, const float* fw, const float* bw, const uint8_t* occ, double* out, int T, int H, int W,
                  void* workspace, size_t workspace_bytes, cudaStream_t stream);
/* ---- I3D feature network of VFID (core/metrics.py:62-82,195-569) ---------------------------------------------- */
/* 'same' padding (Unit3D / MaxPool3dSamePadding.compute_pad, core/metrics.py:196-200,258-262): for a k-tap window of stride
 * s over n samples, pad = max(k - (n % s ? n % s : s), 0), front pad / 2, back the rest (pp_same_pad in pp_elem.cuh);
 * the output extent is (n + pad - k) / s + 1. */
/* to_tensors (core/utils.py:151-170) + transpose(1, 2) (core/metrics.py:183) + the F.pad of Conv3d_1a_7x7
 * (core/metrics.py:264-279, k = 7, s = 2 per axis): src uint8 frames [B][T][H][W][3] (src_u8 != 0, value u8 / 255) or
 * planar float [B][3][T][H][W] (src_u8 == 0, copied) -> dst float [B][T+pt][H+ph][W+pw][4] (16-byte aligned), zero
 * border and a zero 4th channel; conv1a then runs with padding 0. */
int pp_i3d_input(const void* src, int src_u8, float* dst, int B, int T, int H, int W, cudaStream_t stream);
/* MaxPool3dSamePadding (core/metrics.py:195-218): F.pad with zeros + nn.MaxPool3d((kt,kh,kw), (st,sh,sw)), NaN
 * propagating as ATen's max pooling does.  x [B][T][H][W][ld_x] -> out [B][To][Ho][Wo][ld_out] (channels [0, C) of its
 * rows, so out may be a channel slice); C, ld_x, ld_out multiples of 4, 16-byte aligned pointers. */
int pp_maxpool3d_same(const float* x, int ld_x, float* out, int ld_out, int B, int T, int H, int W, int C, int kt, int kh, int kw,
                      int st, int sh, int sw, cudaStream_t stream);
/* x.mean(4).mean(3).mean(2) of extract_features(target_endpoint='Logits') (core/metrics.py:566-567): x [B][N][ld]
 * (N = T*H*W pixels) -> out float [B][C], summed in float64 in a fixed order and rounded once. */
int pp_mean_thw(const float* x, int ld, float* out, int B, long N, int C, cudaStream_t stream);

/* ---- Cutie mask tracker (web-demos/hugging_face/tracker) ------------------------------------------------------------ */
/* The working-memory read of MemoryManager.read / _readout (tracker/inference/memory_manager.py:160-187,68-79) at top_k:
 * get_similarity (anisotropic L2, tracker/model/utils/memory_utils.py:6-42) of every memory token against each query
 * column, do_softmax's top-k + softmax (:45-73) and the bmm with each object's values, in one pass: neither the N x HW
 * similarity nor the dense affinity exists.  Memory lives in ring buffers of 1 + fifo_cap frame slots of HW tokens:
 * mem_key [slots*HW][64], mem_shrink [slots*HW], mem_value [num_objects][slots*HW][256] (object o at
 * o * value_obj_stride floats); slot 0 is the permanent frame, logical frame f >= 1 is slot 1 + (fifo_head + f - 1) %
 * fifo_cap, and n_frames frames are read (N = n_frames * HW tokens, in the reference's order).  qk, qe planar [64][HW];
 * out pixel-major [num_objects][HW][256]; mem_key, mem_value, out 16-byte aligned.  top_k <= 32; when N < top_k all N
 * tokens are kept.  Ties keep the lower token index (csrc/pp_topk.cuh).  sel_idx / sel_w (both or neither,
 * [HW][top_k]): the selected logical tokens in descending order and their softmax weights, -1 / 0 past min(top_k, N).  fp32 CUDA-core arithmetic throughout. */
int pp_cutie_topk_readout(const float* mem_key, const float* mem_shrink, const float* mem_value, long value_obj_stride,
                          int n_frames, int fifo_head, int fifo_cap, const float* qk, const float* qe, int HW, int num_objects,
                          int top_k, float* out, int* sel_idx, float* sel_w, cudaStream_t stream);
/* image_to_torch + pad_divide_by(16) + encode_image's normalisation (base_tracker.py:46-51, tracker/utils/tensor_utils.py:6-21,
 * tracker/model/cutie.py:59-62): uint8 frame [H][W][3] -> float planar [3][Hp][Wp], Hp / Wp the next multiples of 16,
 * the zero padding (floor half before) normalised as the reference's is. */
int pp_cutie_frame_in(const uint8_t* frame, float* out, int H, int W, cudaStream_t stream);
/* torch.argmax over K probability channels [K][Hp][Wp] (padded as pp_cutie_frame_in), unpad and the MaskMapper remapping
 * lut[K] (base_tracker.py:79-87) -> uint8 labels [H][W]. */
int pp_cutie_labels(const float* prob, int K, const uint8_t* lut, uint8_t* out, int H, int W, cudaStream_t stream);
/* The tracking preview: BaseTracker.track's painter loop (base_tracker.py:90-95) over a clip.  Every non-zero id k of
 * labels uint8 [T][H][W] present in a frame, in ascending order, goes through mask_painter (tools/painter.py:137-157,
 * contour width 3): fill with palette row k + 1 in float64 (frames * alpha[1] + row * alpha[0], truncated; alpha[1] is
 * 1 - alpha as the caller computes it), then palette row 1 on its contour.  frames uint8 [T][H][W][3] -> out (may be
 * frames); palette uint8 [n_colors][3], ids with k + 1 >= n_colors are left unpainted.  Byte-exact with the reference
 * (the rules are pp_paint_* in pp_elem.cuh).  Caller-owned workspace of pp_mask_paint_workspace_bytes(T, H, W) bytes (0
 * for an invalid shape), 4-byte aligned.  PP_ERR_SHAPE unless 1 <= T <= 65535, H, W >= 1 and n_colors >= 2. */
size_t pp_mask_paint_workspace_bytes(int T, int H, int W);
int pp_mask_paint_u8(const uint8_t* frames, const uint8_t* labels, const uint8_t* palette, int n_colors, const double* alpha,
                     uint8_t* out, int T, int H, int W, void* workspace, size_t workspace_bytes, cudaStream_t stream);

#ifdef __cplusplus
}
#endif
#endif
