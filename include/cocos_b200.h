/* cocos_b200 — C-ABI of the H100-native CoCosNet hot path (libcocos_b200.so).
 *
 * The reference (microsoft/CoCosNet) has no native boundary: its hot path is
 * Python calling ATen.  This header is the boundary we put underneath the
 * reference's module API (SURVEY.md 8b); each entry point cites the reference
 * expression it replaces.  Conventions:
 *   - every pointer is a DEVICE pointer owned by the caller (torch); the
 *     library never allocates or frees device memory and never synchronises;
 *   - work is enqueued on `stream` (a cudaStream_t passed as void*);
 *   - return 0 on success, negative on error; cocos_last_error() gives the
 *     message (thread local).  Nothing throws across the boundary;
 *   - fp16 operand buffers are produced by the cocos_pack_* entry points.
 */
#ifndef COCOS_B200_H
#define COCOS_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define COCOS_ABI_VERSION 8

/* Multi-block reductions (cocos_conv_wgrad, cocos_tapwgrad, cocos_sn_power_iter, cocos_in_stats_nhwc,
 * cocos_inst_act_nhwc_bwd, cocos_pair_loss_nhwc_fwd, cocos_colsum_nhwc, cocos_se_nhwc_fwd / _bwd) write one partial sum per block into a
 * caller-provided fp32 workspace and add the partials in a fixed order: the same inputs give the same bits on every
 * run.  Workspace arguments (ws, ws_floats): ws == NULL is a size query -- *ws_floats receives the floats needed and
 * nothing is launched; otherwise *ws_floats is the capacity of ws.  The workspace must stay untouched until the work
 * enqueued on `stream` has finished. */

int cocos_abi_version(void);
const char* cocos_last_error(void);

/* fp32 [B, C, N] (channel-major, the layout of theta/phi after
 * correspondence.py:274/276 view/unfold and :277-280 normalisation) ->
 * fp16 [B, N, Kt], Kt = Kp * (split_mode ? 3 : 1), Kp >= C zero padded, Kp%2==0.
 * This is the `theta.permute(0, 2, 1)` of correspondence.py:281 plus the
 * operand rounding.  split_mode: 0 = plain fp16; 1 = query side [hi, lo, hi];
 * 2 = key side [hi, hi, lo] (one GEMM then sums hi*hi + lo*hi + hi*lo); 4 = plain bf16 instead of fp16.
 * rowscale_out (may be NULL): if given, every position n is first multiplied by
 * r[b,n] = min(1 / max_c |src[b,c,n]|, 2^126) and r is written to rowscale_out [B,N] (used for
 * the upstream gradient dO in the backward so it always fits fp16). */
int cocos_pack_rows_f16(const float* src, void* dst, int B, int C, int N, int Kp, int split_mode, float* rowscale_out,
                        void* stream);

/* fp32 [B, Cv, Nk] (channel-major exemplar values: avg-pooled ref image
 * correspondence.py:313-315, unfolded patches :311, ref_seg :330-332) ->
 * fp16 (bf16 if `bf16` != 0) [B, Cvp, Nkp], zero padded; for K1: Cvp % 16 == 0, Nkp % 8 == 0. */
int cocos_pack_v_f16(const float* src, void* dst, int B, int Cv, int Nk, int Cvp, int Nkp, int bf16, void* stream);

/* K1, fused correlation + softmax + warp.  Replaces
 *   f = matmul(theta_permute, phi)          correspondence.py:291
 *   f_WTA = f / temperature                 correspondence.py:304
 *   f_div_C = softmax(f_WTA, -1)            correspondence.py:307
 *   y = matmul(f_div_C, ref)                correspondence.py:318 (and :334, :343-344,
 *                                           :362, :368, :370 with operands swapped)
 * q  : fp16 [B, Nq, Kd]   k : fp16 [B, Nk, Kd]   (Kd % 64 == 0)
 * vt : fp16 [B, Cvp, Nkp] (values, channel-major; cocos_pack_v_f16).  May be NULL when v32 is given and Cv <= 4.
 *      Any Cvp (% 16 == 0): beyond 256 the values run in chunks of 256 rows (the last one may be narrower), each of
 *      which recomputes the logits and the softmax, so the logit work grows by ceil(Cvp / 256).  Every chunk's
 *      output is bit for bit what a call on that chunk's channels alone gives; lse and corr come from the first.
 * v32: fp32 [B, Cv, Nk] the same values unpacked (may be NULL).  With Cv <= 4 (the avg-pooled RGB exemplar of
 *      correspondence.py:313-318) the product with the values runs on the CUDA cores inside the exp loop, in fp32.
 * out: fp32 [B, Cv, Nq]   = y.permute(0, 2, 1)  (correspondence.py:323)
 * lse: fp32 [B, Nq] natural-log row log-sum-exp of scale*f (may be NULL)
 * corr: fp32 [B, Nq, Nk] scaled logits f/temperature (may be NULL; the
 *       `return_corr=True` output of correspondence.py:305-306)
 * scale = 1 / temperature. */
int cocos_corr_warp_fwd(const void* q, const void* k, const void* vt, const float* v32, float* out, float* lse,
                        float* corr, int B, int Nq, int Nk, int Kd, int Cv, int Cvp, int Nkp, float scale,
                        void* stream);

/* Batched wgmma GEMM: C[b] (MxN fp32 row-major, ldc) = alpha * A[b] (MxK fp16,
 * K contiguous, lda) * B[b]^T (NxK fp16, ldb) (+ C[b] if accumulate); `bf16` != 0
 * treats both operands as bf16.  Strides in
 * elements.  The torch.matmul / 1x1-conv call sites of correspondence.py:291
 * (return_corr), architecture.py:116-125 and the K1 backward. */
int cocos_gemm_f16(const void* a, const void* b, float* c, int batch, int M, int N, int K, int lda, int ldb, int ldc,
                   long long stride_a, long long stride_b, long long stride_c, float alpha, int accumulate,
                   int bf16, void* stream);

/* K1 backward, stage A (what autograd does through correspondence.py:291-318):
 * recomputes S = q k^T and dP' = dO' V^T tile by tile and writes, as bf16,
 *   ds  [B, Nq, Nkp] = P * (dP' - D') * scale / r,   D'[i] = sum_c dO'[i,c] O[c,i]
 *   dst [B, Nk, Nqp] = ds^T,   pt [B, Nk, Nqp] = P^T (optional, may be NULL)
 * q,k as in cocos_corr_warp_fwd; do16 fp16 [B,Nq,Cvk] = row-scaled upstream gradient
 * dO' = r * dO with rscale = r [B,Nq] (cocos_pack_rows_f16 with rowscale_out), v16 fp16
 * [B,Nk,Cvk] = V position-major (Cvk % 64 == 0, any width: up to 192 dO and V stay resident in shared memory,
 * beyond that their 64-channel atoms are streamed; dS is still written once); out fp32 [B,Cv,Nq] and lse from the
 * forward.  The input gradients follow from three bf16 cocos_gemm_f16 calls:
 *   dq^T[Kd,Nq] = k_cm[Kd,Nk] x ds,  dk^T[Kd,Nk] = q_cm[Kd,Nq] x dst,  dv^T[Cv,Nk] = do_cm[Cv,Nq] x pt. */
int cocos_corr_warp_bwd_ds(const void* q, const void* k, const void* do16, const void* v16, const float* rscale,
                           const float* out, const float* lse, void* ds, void* dst, void* pt, int B, int Nq, int Nk,
                           int Kd, int Cv, int Cvk, int Nkp, int Nqp, float scale, void* stream);

/* Fused PONO + SPADE modulation + LeakyReLU + reflection pad, NCHW fp32:
 *   y[B,C,H+2p,W+2p] = reflect_pad_p( lrelu_slope( (x - mean_c)/sqrt(var_c + eps) * (1 + gamma) + beta ) )
 * with per-pixel statistics over channels, unbiased variance (normalization.py:63-68), the
 * modulation of normalization.py:149, architecture.py:94-95 (slope 0.2; pass 1.0 for the
 * shortcut's plain SPADE) and the ReflectionPad2d of architecture.py:73-74.  gb = [gamma ; beta]
 * as [B,2C,H,W].  mean/rstd [B,H,W] are saved for the backward, which returns dx [B,C,H,W] and
 * dgb [B,2C,H,W] from dy [B,C,H+2p,W+2p].  nhwc != 0: every tensor is channels-last ([B,H,W,C] in memory,
 * C % 4 == 0), one warp per pixel. */
int cocos_spade_mod_fwd(const float* x, const float* gb, float* y, float* mean, float* rstd, int B, int C, int H,
                        int W, int pad, float slope, float eps, int nhwc, void* stream);
int cocos_spade_mod_bwd(const float* dy, const float* x, const float* gb, const float* mean, const float* rstd,
                        float* dx, float* dgb, int B, int C, int H, int W, int pad, float slope, int nhwc,
                        void* stream);

/* K2: TMA-fed wgmma implicit-GEMM convolution, forward, KS in {1, 3}, stride 1 (the 3x3 convs of the SPADE blocks,
 * domain adaptor and residual blocks: architecture.py:31-33,73-74; normalization.py:112-120; correspondence.py:17-22).
 *   y[b,n,h,w] = bias[n] + sum_{r,s,c} x[b, h + r - off, w + s - off, c] * wt[n, (r*KS + s)*Cp + c]
 * x  : fp16 (bf16 if `bf16`) NHWC [B, Hin, Win, Cp], Cp % 64 == 0 (cocos_pack_rows_f16 of the NCHW tensor viewed as
 *      [B,C,Hin*Win]); reads outside [0,Hin)x[0,Win) are zero (TMA out-of-bounds fill).
 *      forward, producer already padded (reflection): Hin = H + KS - 1, off = 0; forward with zero padding: Hin = H,
 *      off = KS/2; backward-data (the same kernel): x = dy, wt = spatially flipped W^T, off = KS - 1 (- padding).
 * wt : fp16/bf16 [Cout, KS*KS*Cp].   bias: fp32 [Cout] or NULL.   y: fp32 NCHW [B, Cout, H, W]. */
int cocos_conv_fwd(const void* x, const void* wt, const float* bias, float* y, int B, int H, int W, int Hin, int Win,
                   int Cp, int Cout, int KS, int off, int bf16, void* stream);

/* fp32 [rows, Win] -> 16-bit (fp16, or bf16 if `bf16`) [nshift, rows, Wp], row pitch Wp >= Wout, Wp % 8 == 0 (TMA
 * needs 16-byte strides): dst[s][row][w] = src[row][w + s - off] for w < Wout, zero where that column does not exist.
 * Makes the NCHW 16-bit operand copies of cocos_conv_wgrad (dy: nshift 1, off 0; x: nshift KS column-shifted copies,
 * because a TMA box cannot start at an odd column). */
int cocos_cast_pitch(const float* src, void* dst, long long rows, int Win, int Wout, int Wp, int nshift, int off,
                     int bf16, void* stream);

/* K2w: convolution backward-weights (stride 1, KS in {1,3}) as a wgmma GEMM over the B*H*W pixels, split-K over the
 * grid.  Replaces the wgrad half of autograd's convolution_backward for the same nn.Conv2d call sites as
 * cocos_conv_fwd.
 *   ws[(r*KS + s), c, n] = sum_{b,h,w} dy[b, n, h, w] * x[b, c, h + r - off, w + s - off]
 * dy : 16-bit NCHW [B, Cout, H, Wp]  (Wp = W rounded up to 8);
 * x  : 16-bit [KS, B, Cin, Hin, Wp], the KS column-shifted copies cocos_cast_pitch(.., Win, W, Wp, KS, off, ..) makes;
 *      rows outside [0,Hin) are zero.  off = 0 when x carries its halo, KS/2 for zero padding.
 * W >= 64 only (narrower layers: error return; the host mirror sends them to the library wgrad); both operands bf16
 * (dy_bf16 = x_bf16 = 1): a bf16 x fp16 instruction descriptor is rejected by the hardware.
 * ws : fp32 [KS*KS, Cin, Cout], fully overwritten (split-K partials are added in split order: the same bits on every run). */
int cocos_conv_wgrad(const void* dy, const void* x, float* ws, int B, int H, int W, int Hin, int Win, int Cout, int Cin,
                     int KS, int off, int dy_bf16, int x_bf16, float* part, long long* part_floats, void* stream);

/* Fused operand prologue for `--PONO_C` (correspondence.py:273-281 / 283-289): x fp32 [B,C,h,w] (output of the theta
 * or phi 1x1 conv) -> unfold(match_kernel, zero pad) -> minus the mean over K = C*mk*mk -> / (L2 norm over K + eps)
 * -> fp16 [B, h*w, K], K laid out tap-major (k = tap*C + c; use the same call for both operands).  xt_workspace:
 * fp32 scratch of B*C*h*w elements.  match_kernel in {1, 3}; C % 4 == 0; K % 64 == 0.  mean_out / inv_out (both or
 * neither; [B, h*w] fp32): the per-position mean and 1 / (norm + eps), kept for the backward. */
int cocos_normalize_pack(const float* x, float* xt_workspace, void* out, float* mean_out, float* inv_out, int B, int C,
                         int h, int w, int match_kernel, float eps, void* stream);
/* Backward of cocos_normalize_pack (autograd through correspondence.py:273-289: normalise, centre, unfold):
 * g = dL/d(operand) fp32 [B, K, h*w] (k = tap*C + c, the layout cocos_gemm_f16 emits for K_cm . dS) -> dx fp32
 * [B,C,h,w]; a_ws / s_ws: fp32 scratch [B, h*w] each.  The unfolded [B, K, N] tensors never exist: the fold is a
 * 9-term gather per pixel. */
int cocos_normalize_pack_bwd(const float* g, const float* x, const float* mean, const float* inv, float* a_ws,
                             float* s_ws, float* dx, int B, int C, int h, int w, int match_kernel, void* stream);
/* fp16 [B, N, K] (a packed operand) -> bf16 [B, K, N]: the channel-major A operands of the dQ / dK GEMMs of the
 * correspondence backward without keeping the fp32 [B, K, N] tensors of the forward. */
int cocos_transpose_f16_bf16(const void* src, void* dst, int B, int N, int K, void* stream);

/* Fused InstanceNorm2d(affine=False, eps) + LeakyReLU(slope) over `planes` = B*C contiguous planes of HW fp32
 * elements (NCHW): the norm/activation pairs of the domain adaptor (generator.py:104-113,141-145) and of the
 * PatchGAN (discriminator.py:92-115; normalization.py:52-53).  mean/rstd [planes] are saved for the backward,
 * which returns dx from dy.  slope = 1 is the plain instance norm. */
int cocos_inst_act_fwd(const float* x, float* y, float* mean, float* rstd, int planes, int HW, float slope, float eps,
                       void* stream);
int cocos_inst_act_bwd(const float* dy, const float* x, const float* mean, const float* rstd, float* dx, int planes,
                       int HW, float slope, void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * 16-bit NHWC pipeline (round 2): every convolution of the generator / adaptor / residual blocks / PatchGAN / VGG19 is
 * ONE wgmma kernel over NHWC activations, described by a list of "tap groups"; the kernels between two
 * convolutions (normalisation, modulation, activation, halo) read and write the same 16-bit NHWC tensors, so an
 * activation crosses HBM once per producer / consumer instead of as fp32 NCHW + transposes + re-packs.
 * Tensor kinds: 1 = fp16, 2 = bf16, 3 = fp32 (all NHWC [B, H, W, Cs], channel stride Cs >= C); 0 = fp32 NCHW.
 * ------------------------------------------------------------------------------------------------------------------ */
#define COCOS_TAPCONV_MAX_GROUPS 48

/* Reflection halos: every NHWC entry point below that writes a halo of width pad (y_pad) fills it like
 * F.pad(mode="reflect"), and every one that reads a haloed gradient folds the halo back by the exact adjoint (each
 * halo pixel added onto its source).  Any width with pad < H and pad < W is accepted; the networks use 1 and the
 * dilations 2 and 4 of the dilated SPADE blocks (architecture.py:22-24 with --dilation_conv).
 * A dilated 3x3 convolution is the same nine tap groups at offsets dh = r*dilation - padding: no separate kernel. */

/* cocos_tapconv: y[b, h, w, n] = epilogue( sum_g sum_{c < 64*kchunks}
 *                    x[b, a_stride*h + dh[g], a_stride*w + dw[g], coff[g] + c] * w[n, (g*kchunks)*64 + c] )
 * Replaces nn.Conv2d forward (architecture.py:31-33,73-74; normalization.py:112-120; correspondence.py:17-22,79-146;
 * discriminator.py:92-115; generator.py:47,104-113) and the backward-data half of autograd's convolution_backward for
 * the same layers (x = dy, transposed / flipped weights; for stride-2 layers one launch per input parity class,
 * scattered through y_sh/y_sw/y_oh/y_ow).  Reads outside the image or beyond channel Ca are zero.
 *   x   : 16-bit (fp16, or bf16 if `bf16`) NHWC [B, Hin, Win, Ca], Ca % 8 == 0; a_stride 2 needs even Hin, Win.
 *   w   : same 16-bit type, [w_rows >= Cout, ngroups*kchunks*64] (cocos_pack_w), rows >= Cout zero.
 *   epilogue: * scale[0] (device fp32 scalar, may be NULL: the 1/sigma of a spectrally normalised layer,
 *             normalization.py:30-31 -- the weights stay un-normalised in w), + bias[n] (fp32, may be NULL),
 *             + res[b,h,w,n] (kind 1 or 3, channel stride res_Cs, may be NULL),
 *             act 0 none / 1 ReLU / 2 LeakyReLU(slope) / 3 tanh.
 *   y   : kind y_kind.  NHWC kinds: [B, y_H + 2*y_pad, y_W + 2*y_pad, y_Cs], channel offset y_coff; output pixel
 *         (h, w) lands at (h*y_sh + y_oh, w*y_sw + y_ow) (+ y_pad); y_reflect fills the y_pad-pixel halo by
 *         reflection (nn.ReflectionPad2d(y_pad) of the consumer: 1, or the dilation 2 / 4 of a dilated SPADE block;
 *         y_pad < y_H, y_W); y_lo_off != 0 (fp16 only) also stores lo = v - fp16(v) at channel
 *         offset + y_lo_off (2-term split operand).  y_kind 0: fp32 NCHW [B, y_Cs, y_H, y_W]. */
typedef struct cocos_tapconv_desc {
  const void* x;
  const void* w;
  const float* bias;
  const void* res;
  void* y;
  const float* scale;
  int B, Hin, Win, Ca, a_stride, bf16;
  int H, W, Cout, w_rows;
  int ngroups, kchunks;
  signed char dh[COCOS_TAPCONV_MAX_GROUPS];
  signed char dw[COCOS_TAPCONV_MAX_GROUPS];
  short coff[COCOS_TAPCONV_MAX_GROUPS];
  int res_kind, res_Cs, act;
  float slope;
  int y_kind, y_H, y_W, y_Cs, y_coff, y_lo_off, y_pad, y_reflect, y_sh, y_sw, y_oh, y_ow;
  /* SPADE modulation epilogue (mod_W = 64 | 128; 0 = off): the convolution is mlp_gamma and mlp_beta at once
   * (normalization.py:118-120,135-136) with Cout = 2C output rows ordered per N tile as [gamma of mod_W channels |
   * beta of the same channels], and the epilogue emits the operand of the NEXT convolution directly:
   *   y[b,h,w,c] = reflect_pad(lrelu(PONO(x)[b,h,w,c] * (1 + gamma) + beta, slope))   (normalization.py:63-68,149;
   *   architecture.py:73-74,94-95) -- y fp16 [B, H+2*y_pad, W+2*y_pad, y_Cs] with C channels (+ lo terms),
   *   mod_x the raw activation (kind 1|3, [B,H,W,mod_x_Cs]), mod_mean / mod_rstd its per-pixel PONO statistics
   *   (cocos_pono_stats_nhwc); gb (optional, kind 1|3, [B,H,W,gb_Cs >= 2C], same interleaved channel order as the
   *   rows) keeps the raw gamma / beta for cocos_spade_mod_nhwc_bwd.  act must be 2 (LeakyReLU; slope 1 = none). */
  int mod_W;
  const void* mod_x;
  int mod_x_kind, mod_x_Cs;
  const float* mod_mean;
  const float* mod_rstd;
  void* gb;
  int gb_kind, gb_Cs;
} cocos_tapconv_desc;
int cocos_tapconv(const cocos_tapconv_desc* desc, void* stream);

/* cocos_tapwgrad: ws[g, n, c] = sum_{b,h,w} dy[b,h,w,n] * x[b, a_stride*h + dh[g], a_stride*w + dw[g], coff[g] + c]
 * (the backward-weights half of convolution_backward for the layers cocos_tapconv serves).
 *   dy : bf16 NHWC [B, H, W, dy_Cs];  x: NHWC [B, Hin, Win, Ca] as the forward read it, fp16 (x_f16 = 1: converted
 *        to bf16 inside the kernel) or bf16;  ws: fp32 [ngroups, Cout, Cin_s], Cin_s >= Cin, Cin_s % 4 == 0, fully
 *        overwritten (columns >= Cin undefined).
 *   part / part_floats: split-K workspace and its capacity in floats (cocos_tapwgrad_workspace gives the need; 0:
 *        part may be NULL). */
typedef struct cocos_tapwgrad_desc {
  const void* dy;
  const void* x;
  float* ws;
  int B, H, W, dy_Cs, Cout;
  int Hin, Win, Ca, a_stride, x_f16;
  int Cin, Cin_s;
  int ngroups;
  signed char dh[COCOS_TAPCONV_MAX_GROUPS];
  signed char dw[COCOS_TAPCONV_MAX_GROUPS];
  short coff[COCOS_TAPCONV_MAX_GROUPS];
  float* part;
  long long part_floats;
} cocos_tapwgrad_desc;
int cocos_tapwgrad(const cocos_tapwgrad_desc* desc, void* stream);
int cocos_tapwgrad_workspace(const cocos_tapwgrad_desc* desc, long long* floats);

/* Weight matrix of a tap-group list from an nn.Conv2d weight fp32 [Cout, Cin, KS, KS]:
 * dst[row, g*Kc + c] (16-bit, fp16 or bf16) for row < rows_alloc, g < ngroups, c < Kc (Kc % 64 == 0); zero for
 * row >= rows and beyond the channel count.  transposed 0: row = output channel, c = input channel (forward);
 * 1: row = input channel, c = output channel (backward-data).  Group g takes filter tap (r[g], s[g]); term[g] = 1
 * stores the fp16 residual lo = fp16(v - fp16(v)) instead of fp16(v) (2-term split). */
int cocos_pack_w(const float* w, int Cout, int Cin, int KS, void* dst, int rows, int rows_alloc, int Kc, int ngroups,
                 const signed char* r, const signed char* s, const signed char* term, int transposed, int bf16,
                 void* stream);

/* PONO + SPADE modulation + LeakyReLU + ReflectionPad2d over NHWC tensors (normalization.py:63-68,149;
 * architecture.py:73-74,94-95):  y = reflect_pad_p( lrelu_slope( PONO(x) * (1 + gamma) + beta ) ).
 * x (kind 1|3, stride x_Cs), gb (kind 1|3, stride gb_Cs; gamma = channels [0,C), beta = [C,2C)) -> y fp16
 * [B,H+2p,W+2p,y_Cs] (+ lo term at channel offset y_lo_off if != 0); mean / rstd fp32 [B,H,W] saved for the backward:
 * dy bf16 [B,H+2p,W+2p,dy_Cs] -> dx bf16 [B,H,W,dx_Cs] (added to the existing content if dx_acc), dgb bf16
 * [B,H,W,dgb_Cs].  C % 4 == 0. */
int cocos_spade_mod_nhwc_fwd(const void* x, int x_kind, int x_Cs, const void* gb, int gb_kind, int gb_Cs, void* y,
                             int y_Cs, int y_lo_off, float* mean, float* rstd, int B, int C, int H, int W, int pad,
                             float slope, float eps, void* stream);
int cocos_spade_mod_nhwc_bwd(const void* dy, int dy_Cs, const void* x, int x_kind, int x_Cs, const void* gb,
                             int gb_kind, int gb_Cs, int gb_W, const float* mean, const float* rstd, void* dx,
                             int dx_Cs, int dx_acc, void* dgb, int dgb_Cs, int B, int C, int H, int W, int pad,
                             float slope, void* stream);
/* Contextual loss (models/networks/ContextualLoss.py:93-137, called from pix2pix_model.py:196-203) on the correlation
 * matrix S = Xhat^T Yhat, fp32 [B, N, N] with N <= 1024 (cocos_gemm_f16 on the normalised VGG features):
 *   cx[b, i] = max_j A_ij,  A = row-normalised exp((1 - d / (min_j d + eps)) / h),  d = 1 - S
 * (the loss of image b is -log(mean_i cx[b, i])), and its backward: dS (bf16, row pitch ldd >= N) from g = dL/dcx.
 * One warp per row; d, d_norm, w, A of the reference never reach memory. */
int cocos_ctx_rows_fwd(const float* S, float* cx, int B, int N, float h, float eps, void* stream);
int cocos_ctx_rows_bwd(const float* S, const float* g, void* dS, int B, int N, int ldd, float h, float eps,
                       void* stream);

/* Spectral normalisation (torch.nn.utils.spectral_norm as normalization.py:30-31 applies it) of n layers at once:
 * `table` = n device-resident records of 8 x int64 {W fp32 [rows, cols] (weight_orig), u [rows], v [cols], rows, cols,
 * first block of the layer in phase A (128 columns per block), first block in phase B (8 rows per block), offset
 * of the layer's [u | v] copy in `snapshot` (may be NULL; the vectors the backward of this forward needs)}.
 * training != 0: one power iteration, u and v updated in place (v <- normalize(W^T u), u <- normalize(W v)); then
 * inv_sigma[i] = 1 / (u^T W v).  The normalised weight is never formed: cocos_tapconv takes inv_sigma as `scale`.
 * scratch: 2n + blocks_a + blocks_b floats (per-layer |W^T u|^2 and |W v|^2, or u^T W v in evaluation, then the
 * per-block partials).  blocks_a / blocks_b: total blocks of the two phases. */
int cocos_sn_power_iter(const void* table, int n, int blocks_a, int blocks_b, float* scratch, float* inv_sigma,
                        float* snapshot, float eps, int training, void* stream);
/* Per-pixel PONO statistics of x (kind 1|3) [npix, Cs] over its C channels: mean and 1/sqrt(unbiased var + eps)
 * (normalization.py:63-68), for the SPADE epilogue of cocos_tapconv. */
int cocos_pono_stats_nhwc(const void* x, int kind, int Cs, int C, long long npix, float eps, float* mean, float* rstd,
                          void* stream);

/* InstanceNorm2d(affine=False) statistics over NHWC: stats[b, c] = {sum, sum of squares} over the HW pixels
 * (generator.py:104-113, discriminator.py:92-115, correspondence.py:19,23 with normalization.py:52-53). */
int cocos_in_stats_nhwc(const void* x, int kind, int Cs, int B, int C, int HW, float* stats, float* ws,
                        long long* ws_floats, void* stream);

/* y = act( instance_norm(x) [+ res] ), act = LeakyReLU(slope) or PReLU (slope_ptr: device scalar, correspondence.py:20)
 * [, reflection halo y_pad, lo term, second fp32 copy y2 without halo].  Backward: dy bf16 (halo folded) [+ dy2] ->
 * dx bf16, dres bf16 (optional), dslope += PReLU gradient (optional); bstats fp32 [B,C,2] scratch. */
int cocos_inst_act_nhwc_fwd(const void* x, int x_kind, int x_Cs, const float* stats, const void* res, int res_kind,
                            int res_Cs, const float* slope_ptr, float slope, void* y, int y_kind, int y_Cs,
                            int y_lo_off, int y_pad, void* y2, int y2_Cs, int B, int C, int H, int W, float eps,
                            const void* gb, int gb_kind, int gb_Cs, int batch_stats, void* stream);
int cocos_inst_act_nhwc_bwd(const void* dy, int dy_Cs, int dy_pad, const void* dy2, int dy2_Cs, const void* x,
                            int x_kind, int x_Cs, const float* stats, const void* res, int res_kind, int res_Cs,
                            const float* slope_ptr, float slope, float* bstats, float* dslope, void* dx, int dx_Cs,
                            int dx_acc, void* dres, int dres_Cs, int dres_acc, int B, int C, int H, int W, float eps,
                            const void* gb, int gb_kind, int gb_Cs, void* dgb, int dgb_Cs, int batch_stats,
                            int const_stats, int phase, float* ws, long long* ws_floats, void* stream);
/* The same two entry points serve SPADE with instance / batch statistics (normalization.py:96-104,132-149, the
 * celebahq / deepfashion configurations): gb (kind 1|3, [B,H,W,gb_Cs], gamma at channels [0,C), beta at [C,2C))
 * modulates the normalised value, z = norm(x) * (1 + gamma) + beta, and the backward also emits dgb (bf16);
 * batch_stats = 1: stats / bstats are [1][C][2] over B*H*W values (BatchNorm2d, training); const_stats = 1: the
 * statistics are constants (running estimates, eval mode); phase 1 / 2 = only the reduction / only the apply pass
 * (a synchronised BatchNorm all-reduces bstats in between), 0 = both. */

/* Backward of an activation fused into a cocos_tapconv epilogue (act 1 ReLU: normalization.py:114-117, correspondence.py
 * 107-146; act 2 LeakyReLU: discriminator.py:93): dz[b,h,w,c] = fold_halo(dy)[b,h,w,c] * act'(y[b,h+pad,w+pad,c]);
 * dy bf16 and y (kind 1|3) share the halo `pad`; dz bf16 [B,H,W,dz_Cs]. */
int cocos_act_bwd_nhwc(const void* dy, int dy_Cs, const void* y, int y_kind, int y_Cs, int pad, void* dz, int dz_Cs,
                       int B, int C, int H, int W, int act, float slope, void* stream);

/* fp32 NCHW [B, C, Hs, Ws] -> NHWC kind `kind` [B, H+2*pad, W+2*pad, Cs]: nearest down-sampling by the integer
 * factor f (F.interpolate(mode='nearest') of normalization.py:130), reflection halo, zero channels [C, Cs) and, for
 * lo_off != 0 (fp16, Cs == 2*lo_off), the lo terms at channel offset lo_off.  (c_lo, c_span): the source lands in
 * the channel window [c_lo, c_lo + c_span) of dst (zeros beyond C; c_span 0 = up to Cs) -- the torch.cat((semantics,
 * image), 1) of pix2pix_model.py:301-302 without the concatenated tensor. */
int cocos_nhwc_pack(const float* src, void* dst, int kind, int B, int C, int Cs, int lo_off, int c_lo, int c_span,
                    int Hs, int Ws, int H, int W, int f, int pad, void* stream);
/* Feature losses on fp16 NHWC tensors x, y [B, HW, Cs] (C % 8 == 0): out[0] += scale * sum_b w[b] * sum |x - y| (mode 0:
 * criterionFeat / weighted_l1_loss, pix2pix_model.py:240,253, util/util.py:36-40; w may be NULL) or (x - y)^2 (mode 1,
 * pix2pix_model.py:256), and the gradient w.r.t. x: dx (bf16, added to its content if acc) = g[0] * scale * w[b] *
 * d/dx.  The discriminator / VGG19 features are compared where they live instead of as fp32 NCHW copies. */
int cocos_pair_loss_nhwc_fwd(const void* x, int x_Cs, const void* y, int y_Cs, const float* w, int B, long long HW, int C,
                             float scale, int mode, float* out, float* ws, long long* ws_floats, void* stream);
int cocos_pair_loss_nhwc_bwd(const void* x, int x_Cs, const void* y, int y_Cs, const float* w, int B, long long HW, int C,
                             float scale, int mode, const float* g, void* dx, int dx_Cs, int acc, void* stream);
/* fp16 operand [npix, src_Cs] (hi at channels [0, dst_Cs), optional lo term at lo_off) -> bf16 [npix, dst_Cs] =
 * bf16(hi + lo): the X operand of cocos_tapwgrad (the weight-gradient half of autograd's convolution_backward),
 * converted once per tensor instead of inside the GEMM.  Channel counts are multiples of 8. */
int cocos_cast_op_bf16(const void* src, int src_Cs, int lo_off, void* dst, int dst_Cs, long long npix, void* stream);
/* nn.MaxPool2d(2, 2) of the VGG19 feature net (correspondence.py:84-100) over fp16 NHWC [B, 2*Ho, 2*Wo, Cs] ->
 * [B, Ho, Wo, Cs] and its backward (dy / dx bf16, the gradient goes to the first maximum in scan order). */
int cocos_maxpool2_nhwc_fwd(const void* x, void* y, int B, int Cs, int Ho, int Wo, void* stream);
int cocos_maxpool2_nhwc_bwd(const void* dy, const void* x, void* dx, int B, int Cs, int Ho, int Wo, void* stream);
/* NHWC kind `kind` [B, H+2*pad, W+2*pad, Cs], channels [c_lo, c_lo+C), halo folded back -> fp32 NCHW
 * dst[b, cd_lo + c, h*f, w*f] (dst is [B, Cd, Hd, Wd]); acc != 0 adds instead of overwriting. */
int cocos_nhwc_unpack(const void* src, int kind, int Cs, int c_lo, int C, int B, int H, int W, int pad, float* dst,
                      int Cd, int cd_lo, int Hd, int Wd, int f, int acc, void* stream);
/* out[c] = sum over the rows of x [rows, Cs] (kind 1|2|3), c < C: the bias gradient of a convolution. */
int cocos_colsum_nhwc(const void* x, int kind, int Cs, int C, long long rows, float* out, float* ws,
                      long long* ws_floats, void* stream);
/* Squeeze-excitation (SELayer, architecture.py:182-197) of a SPADE block's raw conv_1 output dx, fused with the
 * block's residual sum:  y = res + s[b,c] * dx,  s = sigmoid(W2 relu(W1 m)),  m[b,c] = mean over the HW pixels of dx.
 *   dx (kind 1|3, [B,HW,dx_Cs]), res (kind 1|3), y (kind 1|3, no halo); w1 fp32 [Cr, C], w2 fp32 [C, Cr] (bias-free
 *   nn.Linear weights, Cr = C / 16); m, s fp32 [B, C] and hid = relu(W1 m) fp32 [B, Cr] are written for the backward.
 *   The squeeze is cocos_in_stats_nhwc's fixed-order reduction.  C % 4 == 0, C <= 4096.
 * Backward from dy (bf16, gradient of y; the residual's gradient is dy itself):
 *   ds[b,c] = sum_hw dy * dx (fixed order), ddx = s * dy + dm[b,c] / HW (bf16, overwritten) with dm the gradient of
 *   m, dw1 fp32 [Cr, C] and dw2 fp32 [C, Cr] overwritten (images added in ascending order).
 * Both take the workspace protocol of the multi-block reductions (ws NULL: size query). */
int cocos_se_nhwc_fwd(const void* dx, int dx_kind, int dx_Cs, const void* res, int res_kind, int res_Cs, const float* w1,
                      const float* w2, void* y, int y_kind, int y_Cs, float* m, float* hid, float* s, int B, int C, int Cr,
                      int HW, float* ws, long long* ws_floats, void* stream);
int cocos_se_nhwc_bwd(const void* dy, int dy_Cs, const void* dx, int dx_kind, int dx_Cs, const float* w1, const float* w2,
                      const float* m, const float* hid, const float* s, void* ddx, int ddx_Cs, float* dw1, float* dw2,
                      int B, int C, int Cr, int HW, float* ws, long long* ws_floats, void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * SAGAN non-local block (Attention, architecture.py:97-127; the adaptor's --adaptor_nonlocal, generator.py:124-125,
 * 148-149) on the NHWC tape:  y = x + gamma * o(bmm(g, softmax(theta^T phi)^T)),  phi and g max-pooled 2x2.  The 1x1
 * convolutions theta | phi | g run as ONE cocos_tapconv with the three filters concatenated (raw output z, channels
 * [0, Kd) theta, [Kd, 2Kd) phi, [2Kd, 2Kd + Cv) g); the attend step is K1 at scale 1 and its backward stage A plus three
 * bf16 GEMMs; o runs as a cocos_tapconv with scale = gamma and res = x.  The entry points below are the layout and
 * gradient steps in between.  None of them reduces across threads: no atomics, no workspace, the same bits every run.
 * ------------------------------------------------------------------------------------------------------------------ */
/* Raw NHWC activation x (kind 1|3, [npix, Cs], Cs % 8 == 0, no halo) -> fp16 conv operand y [npix, y_Cs]: hi =
 * fp16(x) at channels [0, Cs) and, for lo_off != 0, lo = fp16(x - hi) at [lo_off, lo_off + Cs) (2-term split).  The
 * block's input x is both the theta | phi | g operand and the fp32 residual (architecture.py:116-118,127). */
int cocos_nhwc_to_op(const void* x, int x_kind, int Cs, void* y, int y_Cs, int lo_off, long long npix, void* stream);
/* Forward pack of the raw theta | phi | g output z (kind 1|3, [B, H, W, z_Cs], H and W even; Nq = H*W, Nk = Nq/4).
 * Replaces the view / max_pool2d / transpose steps of architecture.py:116-122 in front of K1.  Kp = Kd rounded up
 * to 64, Kt = Kp * (split ? 3 : 1):
 *   q    fp16 [B, Nq, Kt]  theta rows: [hi] or the query layout [hi, lo, hi] (cocos_pack_rows_f16 split mode 1)
 *   k    fp16 [B, Nk, Kt]  maxpool2(phi) rows: [hi] or the key layout [hi, hi, lo]
 *   vt   fp16 [B, Cvp, Nkp] maxpool2(g) channel-major, K1's V (Cvp % 16 == 0, Nkp % 8 == 0, zero padded)
 * and for the backward (all optional; q_cm and k_cm both or neither):
 *   v16  fp16 [B, Nk, Cvk] maxpool2(g) position-major (Cvk >= Cvp, Cvk % 64 == 0, zero beyond Cv): stage A's V, one
 *        cocos_corr_warp_bwd_ds call at any Cvk
 *   q_cm bf16 [B, Kd, Nqp], k_cm bf16 [B, Kd, Nkp]: theta and maxpool2(phi) channel-major, the A operands of the
 *        dQ / dK GEMMs (pitches multiples of 8; the padding columns are not written). */
int cocos_attn_pack_nhwc(const void* z, int z_kind, int z_Cs, int B, int H, int W, int Kd, int Cv, int split, void* q,
                         void* k, void* vt, int Cvp, int Nkp, void* v16, int Cvk, void* q_cm, int Nqp, void* k_cm,
                         void* stream);
/* dO rows of the attend backward from dy, the bf16 NHWC gradient of the attention output ([B, N, dy_Cs], Cv channels;
 * the gradient of bmm(g, beta^T) in architecture.py:126): do16 fp16 [B, N, Cvk] = r * dy (Cvk >= Cv, Cvk % 64 == 0,
 * zero beyond Cv) with r = min(1 / max_c |dy|, 2^126) (1 for an all-zero row) written to rscale [B, N] -- what
 * cocos_pack_rows_f16 with rowscale_out makes from fp32 channel-major -- and do_cm bf16 [B, Cv, Nqp] = dy
 * channel-major, the A operand of the dV GEMM. */
int cocos_attn_do_rows(const void* dy, int dy_Cs, int B, int N, int Cv, void* do16, int Cvk, float* rscale, void* do_cm,
                       int Nqp, void* stream);
/* Gradient of the theta | phi | g output from the three GEMM results dq fp32 [B, Kd, Nq], dk fp32 [B, Kd, Nk], dv fp32
 * [B, Cv, Nk] (channel-major, dense): dz bf16 [B, H, W, dz_Cs] (fully overwritten, zero beyond 2Kd + Cv) with theta's
 * channels = dq transposed and phi's / g's = dk / dv at the first maximum in scan order of each 2x2 window of z, zero
 * elsewhere -- the backward of F.max_pool2d (architecture.py:117-118), the argmax recomputed from the saved z. */
int cocos_attn_grad_unpack(const float* dq, const float* dk, const float* dv, const void* z, int z_kind, int z_Cs, int B,
                           int H, int W, int Kd, int Cv, void* dz, int dz_Cs, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* COCOS_B200_H */
