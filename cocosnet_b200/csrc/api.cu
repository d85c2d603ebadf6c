// extern "C" boundary of libcocos_b200.so — see include/cocos_b200.h.
#include "../../include/cocos_b200.h"

#include "corr_kernels.h"
#include "tmap.h"

using namespace cocos;

extern "C" {

int cocos_abi_version(void) { return COCOS_ABI_VERSION; }
const char* cocos_last_error(void) { return get_error(); }

int cocos_pack_rows_f16(const float* src, void* dst, int B, int C, int N, int Kp, int split_mode, float* rowscale_out,
                        void* stream) {
  return pack_rows_f16_launch(src, dst, B, C, N, Kp, split_mode, rowscale_out, static_cast<cudaStream_t>(stream));
}

int cocos_pack_v_f16(const float* src, void* dst, int B, int Cv, int Nk, int Cvp, int Nkp, int bf16, void* stream) {
  return pack_v_f16_launch(src, dst, B, Cv, Nk, Cvp, Nkp, bf16, static_cast<cudaStream_t>(stream));
}

// any Cvp % 16 == 0: beyond 256 value rows K1 runs in chunks of 256 (corr_fwd.cu)
int cocos_corr_warp_fwd(const void* q, const void* k, const void* vt, const float* v32, float* out, float* lse,
                        float* corr, int B, int Nq, int Nk, int Kd, int Cv, int Cvp, int Nkp, float scale,
                        void* stream) {
  if (!q || !k || (!vt && !v32) || !out) {
    set_error("cocos_corr_warp_fwd: null pointer argument");
    return -1;
  }
  return corr_warp_fwd_launch(q, k, vt, v32, out, lse, corr, B, Nq, Nk, Kd, Cv, Cvp, Nkp, scale,
                              static_cast<cudaStream_t>(stream));
}

int cocos_gemm_f16(const void* a, const void* b, float* c, int batch, int M, int N, int K, int lda, int ldb, int ldc,
                   long long stride_a, long long stride_b, long long stride_c, float alpha, int accumulate,
                   int bf16, void* stream) {
  if (!a || !b || !c) {
    set_error("cocos_gemm_f16: null pointer argument");
    return -1;
  }
  return gemm_f16_launch(a, b, c, batch, M, N, K, lda, ldb, ldc, stride_a, stride_b, stride_c, alpha, accumulate,
                         bf16, static_cast<cudaStream_t>(stream));
}

// any Cvk % 64 == 0: dO / V resident up to 192 channels, streamed through the operand ring beyond (corr_bwd.cu)
int cocos_corr_warp_bwd_ds(const void* q, const void* k, const void* do16, const void* v16, const float* rscale,
                           const float* out, const float* lse, void* ds, void* dst, void* pt, int B, int Nq, int Nk,
                           int Kd, int Cv, int Cvk, int Nkp, int Nqp, float scale, void* stream) {
  if (!q || !k || !do16 || !v16 || !rscale || !out || !lse || !ds || !dst) {
    set_error("cocos_corr_warp_bwd_ds: null pointer argument");
    return -1;
  }
  return corr_bwd_ds_launch(q, k, do16, v16, rscale, out, lse, ds, dst, pt, B, Nq, Nk, Kd, Cv, Cvk, Nkp, Nqp, scale,
                            static_cast<cudaStream_t>(stream));
}

int cocos_spade_mod_fwd(const float* x, const float* gb, float* y, float* mean, float* rstd, int B, int C, int H,
                        int W, int pad, float slope, float eps, int nhwc, void* stream) {
  if (!x || !gb || !y || !mean || !rstd) {
    set_error("cocos_spade_mod_fwd: null pointer argument");
    return -1;
  }
  return spade_mod_fwd_launch(x, gb, y, mean, rstd, B, C, H, W, pad, slope, eps, nhwc,
                              static_cast<cudaStream_t>(stream));
}

int cocos_spade_mod_bwd(const float* dy, const float* x, const float* gb, const float* mean, const float* rstd,
                        float* dx, float* dgb, int B, int C, int H, int W, int pad, float slope, int nhwc,
                        void* stream) {
  if (!dy || !x || !gb || !mean || !rstd || !dx || !dgb) {
    set_error("cocos_spade_mod_bwd: null pointer argument");
    return -1;
  }
  return spade_mod_bwd_launch(dy, x, gb, mean, rstd, dx, dgb, B, C, H, W, pad, slope, nhwc,
                              static_cast<cudaStream_t>(stream));
}

int cocos_inst_act_fwd(const float* x, float* y, float* mean, float* rstd, int planes, int HW, float slope, float eps,
                       void* stream) {
  if (!x || !y || !mean || !rstd) {
    set_error("cocos_inst_act_fwd: null pointer argument");
    return -1;
  }
  return inst_act_fwd_launch(x, y, mean, rstd, planes, HW, slope, eps, static_cast<cudaStream_t>(stream));
}

int cocos_inst_act_bwd(const float* dy, const float* x, const float* mean, const float* rstd, float* dx, int planes,
                       int HW, float slope, void* stream) {
  if (!dy || !x || !mean || !rstd || !dx) {
    set_error("cocos_inst_act_bwd: null pointer argument");
    return -1;
  }
  return inst_act_bwd_launch(dy, x, mean, rstd, dx, planes, HW, slope, static_cast<cudaStream_t>(stream));
}

int cocos_normalize_pack(const float* x, float* xt_workspace, void* out, float* mean_out, float* inv_out, int B, int C,
                         int h, int w, int match_kernel, float eps, void* stream) {
  if (!x || !xt_workspace || !out) {
    set_error("cocos_normalize_pack: null pointer argument");
    return -1;
  }
  return norm_pack_launch(x, xt_workspace, out, mean_out, inv_out, B, C, h, w, match_kernel, eps,
                          static_cast<cudaStream_t>(stream));
}

int cocos_normalize_pack_bwd(const float* g, const float* x, const float* mean, const float* inv, float* a_ws,
                             float* s_ws, float* dx, int B, int C, int h, int w, int match_kernel, void* stream) {
  if (!g || !x || !mean || !inv || !a_ws || !s_ws || !dx) {
    set_error("cocos_normalize_pack_bwd: null pointer argument");
    return -1;
  }
  return norm_pack_bwd_launch(g, x, mean, inv, a_ws, s_ws, dx, B, C, h, w, match_kernel,
                              static_cast<cudaStream_t>(stream));
}

int cocos_transpose_f16_bf16(const void* src, void* dst, int B, int N, int K, void* stream) {
  if (!src || !dst) {
    set_error("cocos_transpose_f16_bf16: null pointer argument");
    return -1;
  }
  return transpose_f16_bf16_launch(src, dst, B, N, K, static_cast<cudaStream_t>(stream));
}

int cocos_cast_pitch(const float* src, void* dst, long long rows, int Win, int Wout, int Wp, int nshift, int off,
                     int bf16, void* stream) {
  if (!src || !dst) {
    set_error("cast_pitch: null pointer");
    return -1;
  }
  return cast_pitch_launch(src, dst, rows, Win, Wout, Wp, nshift, off, bf16, static_cast<cudaStream_t>(stream));
}

int cocos_conv_wgrad(const void* dy, const void* x, float* ws, int B, int H, int W, int Hin, int Win, int Cout, int Cin,
                     int KS, int off, int dy_bf16, int x_bf16, float* part, long long* part_floats, void* stream) {
  if (part && (!dy || !x || !ws)) {
    set_error("conv_wgrad: null pointer");
    return -1;
  }
  return conv_wgrad_launch(dy, x, ws, B, H, W, Hin, Win, Cout, Cin, KS, off, dy_bf16, x_bf16, part, part_floats,
                           static_cast<cudaStream_t>(stream));
}

int cocos_conv_fwd(const void* x, const void* wt, const float* bias, float* y, int B, int H, int W, int Hin, int Win,
                   int Cp, int Cout, int KS, int off, int bf16, void* stream) {
  if (!x || !wt || !y) {
    set_error("cocos_conv_fwd: null pointer argument");
    return -1;
  }
  return conv_fwd_launch(x, wt, bias, y, B, H, W, Hin, Win, Cp, Cout, KS, off, bf16,
                         static_cast<cudaStream_t>(stream));
}

int cocos_tapconv(const cocos_tapconv_desc* desc, void* stream) {
  return tapconv_launch(desc, static_cast<cudaStream_t>(stream));
}

int cocos_tapwgrad(const cocos_tapwgrad_desc* desc, void* stream) {
  return tapwgrad_launch(desc, nullptr, static_cast<cudaStream_t>(stream));
}

int cocos_tapwgrad_workspace(const cocos_tapwgrad_desc* desc, long long* floats) {
  if (!floats) {
    set_error("cocos_tapwgrad_workspace: null pointer argument");
    return -1;
  }
  return tapwgrad_launch(desc, floats, nullptr);
}

int cocos_pack_w(const float* w, int Cout, int Cin, int KS, void* dst, int rows, int rows_alloc, int Kc, int ngroups,
                 const signed char* r, const signed char* s, const signed char* term, int transposed, int bf16,
                 void* stream) {
  return pack_w_launch(w, Cout, Cin, KS, dst, rows, rows_alloc, Kc, ngroups, r, s, term, transposed, bf16,
                       static_cast<cudaStream_t>(stream));
}

int cocos_spade_mod_nhwc_fwd(const void* x, int x_kind, int x_Cs, const void* gb, int gb_kind, int gb_Cs, void* y,
                             int y_Cs, int y_lo_off, float* mean, float* rstd, int B, int C, int H, int W, int pad,
                             float slope, float eps, void* stream) {
  if (!x || !gb || !y || !mean || !rstd) {
    set_error("cocos_spade_mod_nhwc_fwd: null pointer argument");
    return -1;
  }
  return spade_mod_nhwc_fwd_launch(x, x_kind, x_Cs, gb, gb_kind, gb_Cs, y, y_Cs, y_lo_off, mean, rstd, B, C, H, W, pad,
                                   slope, eps, static_cast<cudaStream_t>(stream));
}

int cocos_ctx_rows_fwd(const float* S, float* cx, int B, int N, float h, float eps, void* stream) {
  if (!S || !cx) {
    set_error("cocos_ctx_rows_fwd: null pointer argument");
    return -1;
  }
  return ctx_rows_fwd_launch(S, cx, B, N, h, eps, static_cast<cudaStream_t>(stream));
}

int cocos_ctx_rows_bwd(const float* S, const float* g, void* dS, int B, int N, int ldd, float h, float eps,
                       void* stream) {
  if (!S || !g || !dS) {
    set_error("cocos_ctx_rows_bwd: null pointer argument");
    return -1;
  }
  return ctx_rows_bwd_launch(S, g, dS, B, N, ldd, h, eps, static_cast<cudaStream_t>(stream));
}

int cocos_sn_power_iter(const void* table, int n, int blocks_a, int blocks_b, float* scratch, float* inv_sigma,
                        float* snapshot, float eps, int training, void* stream) {
  return sn_power_iter_launch(table, n, blocks_a, blocks_b, scratch, inv_sigma, snapshot, eps, training,
                              static_cast<cudaStream_t>(stream));
}

int cocos_pono_stats_nhwc(const void* x, int kind, int Cs, int C, long long npix, float eps, float* mean, float* rstd,
                          void* stream) {
  if (!x || !mean || !rstd) {
    set_error("cocos_pono_stats_nhwc: null pointer argument");
    return -1;
  }
  return pono_stats_nhwc_launch(x, kind, Cs, C, npix, eps, mean, rstd, static_cast<cudaStream_t>(stream));
}

int cocos_spade_mod_nhwc_bwd(const void* dy, int dy_Cs, const void* x, int x_kind, int x_Cs, const void* gb,
                             int gb_kind, int gb_Cs, int gb_W, const float* mean, const float* rstd, void* dx,
                             int dx_Cs, int dx_acc, void* dgb, int dgb_Cs, int B, int C, int H, int W, int pad,
                             float slope, void* stream) {
  if (!dy || !x || !gb || !mean || !rstd || !dx || !dgb) {
    set_error("cocos_spade_mod_nhwc_bwd: null pointer argument");
    return -1;
  }
  return spade_mod_nhwc_bwd_launch(dy, dy_Cs, x, x_kind, x_Cs, gb, gb_kind, gb_Cs, gb_W, mean, rstd, dx, dx_Cs, dx_acc, dgb,
                                   dgb_Cs, B, C, H, W, pad, slope, static_cast<cudaStream_t>(stream));
}

int cocos_in_stats_nhwc(const void* x, int kind, int Cs, int B, int C, int HW, float* stats, float* ws,
                        long long* ws_floats, void* stream) {
  if (ws && (!x || !stats)) {
    set_error("cocos_in_stats_nhwc: null pointer argument");
    return -1;
  }
  return in_stats_nhwc_launch(x, kind, Cs, B, C, HW, stats, ws, ws_floats, static_cast<cudaStream_t>(stream));
}

int cocos_inst_act_nhwc_fwd(const void* x, int x_kind, int x_Cs, const float* stats, const void* res, int res_kind,
                            int res_Cs, const float* slope_ptr, float slope, void* y, int y_kind, int y_Cs,
                            int y_lo_off, int y_pad, void* y2, int y2_Cs, int B, int C, int H, int W, float eps,
                            const void* gb, int gb_kind, int gb_Cs, int batch_stats, void* stream) {
  if (!x || !stats || !y) {
    set_error("cocos_inst_act_nhwc_fwd: null pointer argument");
    return -1;
  }
  return inst_act_nhwc_fwd_launch(x, x_kind, x_Cs, stats, res, res_kind, res_Cs, slope_ptr, slope, y, y_kind, y_Cs,
                                  y_lo_off, y_pad, y2, y2_Cs, B, C, H, W, eps, gb, gb_kind, gb_Cs, batch_stats,
                                  static_cast<cudaStream_t>(stream));
}

int cocos_inst_act_nhwc_bwd(const void* dy, int dy_Cs, int dy_pad, const void* dy2, int dy2_Cs, const void* x,
                            int x_kind, int x_Cs, const float* stats, const void* res, int res_kind, int res_Cs,
                            const float* slope_ptr, float slope, float* bstats, float* dslope, void* dx, int dx_Cs,
                            int dx_acc, void* dres, int dres_Cs, int dres_acc, int B, int C, int H, int W, float eps,
                            const void* gb, int gb_kind, int gb_Cs, void* dgb, int dgb_Cs, int batch_stats,
                            int const_stats, int phase, float* ws, long long* ws_floats, void* stream) {
  if (ws && (!dy || !x || !stats || !dx)) {
    set_error("cocos_inst_act_nhwc_bwd: null pointer argument");
    return -1;
  }
  return inst_act_nhwc_bwd_launch(dy, dy_Cs, dy_pad, dy2, dy2_Cs, x, x_kind, x_Cs, stats, res, res_kind, res_Cs,
                                  slope_ptr, slope, bstats, dslope, dx, dx_Cs, dx_acc, dres, dres_Cs, dres_acc, B, C,
                                  H, W, eps, gb, gb_kind, gb_Cs, dgb, dgb_Cs, batch_stats, const_stats, phase, ws,
                                  ws_floats, static_cast<cudaStream_t>(stream));
}

int cocos_act_bwd_nhwc(const void* dy, int dy_Cs, const void* y, int y_kind, int y_Cs, int pad, void* dz, int dz_Cs,
                       int B, int C, int H, int W, int act, float slope, void* stream) {
  if (!dy || !y || !dz) {
    set_error("cocos_act_bwd_nhwc: null pointer argument");
    return -1;
  }
  return act_bwd_nhwc_launch(dy, dy_Cs, y, y_kind, y_Cs, pad, dz, dz_Cs, B, C, H, W, act, slope,
                             static_cast<cudaStream_t>(stream));
}

int cocos_nhwc_pack(const float* src, void* dst, int kind, int B, int C, int Cs, int lo_off, int c_lo, int c_span,
                    int Hs, int Ws, int H, int W, int f, int pad, void* stream) {
  if (!src || !dst) {
    set_error("cocos_nhwc_pack: null pointer argument");
    return -1;
  }
  return nhwc_pack_launch(src, dst, kind, B, C, Cs, lo_off, c_lo, c_span, Hs, Ws, H, W, f, pad,
                          static_cast<cudaStream_t>(stream));
}

int cocos_pair_loss_nhwc_fwd(const void* x, int x_Cs, const void* y, int y_Cs, const float* w, int B, long long HW, int C,
                             float scale, int mode, float* out, float* ws, long long* ws_floats, void* stream) {
  if (ws && (!x || !y || !out)) {
    set_error("cocos_pair_loss_nhwc_fwd: null pointer argument");
    return -1;
  }
  return pair_loss_nhwc_fwd_launch(x, x_Cs, y, y_Cs, w, B, HW, C, scale, mode, out, ws, ws_floats,
                                   static_cast<cudaStream_t>(stream));
}

int cocos_pair_loss_nhwc_bwd(const void* x, int x_Cs, const void* y, int y_Cs, const float* w, int B, long long HW, int C,
                             float scale, int mode, const float* g, void* dx, int dx_Cs, int acc, void* stream) {
  if (!x || !y || !g || !dx) {
    set_error("cocos_pair_loss_nhwc_bwd: null pointer argument");
    return -1;
  }
  return pair_loss_nhwc_bwd_launch(x, x_Cs, y, y_Cs, w, B, HW, C, scale, mode, g, dx, dx_Cs, acc,
                                   static_cast<cudaStream_t>(stream));
}

int cocos_cast_op_bf16(const void* src, int src_Cs, int lo_off, void* dst, int dst_Cs, long long npix, void* stream) {
  if (!src || !dst) {
    set_error("cocos_cast_op_bf16: null pointer argument");
    return -1;
  }
  return cast_op_bf16_launch(src, src_Cs, lo_off, dst, dst_Cs, npix, static_cast<cudaStream_t>(stream));
}

int cocos_maxpool2_nhwc_fwd(const void* x, void* y, int B, int Cs, int Ho, int Wo, void* stream) {
  if (!x || !y) {
    set_error("cocos_maxpool2_nhwc_fwd: null pointer argument");
    return -1;
  }
  return maxpool2_nhwc_fwd_launch(x, y, B, Cs, Ho, Wo, static_cast<cudaStream_t>(stream));
}

int cocos_maxpool2_nhwc_bwd(const void* dy, const void* x, void* dx, int B, int Cs, int Ho, int Wo, void* stream) {
  if (!dy || !x || !dx) {
    set_error("cocos_maxpool2_nhwc_bwd: null pointer argument");
    return -1;
  }
  return maxpool2_nhwc_bwd_launch(dy, x, dx, B, Cs, Ho, Wo, static_cast<cudaStream_t>(stream));
}

int cocos_nhwc_unpack(const void* src, int kind, int Cs, int c_lo, int C, int B, int H, int W, int pad, float* dst,
                      int Cd, int cd_lo, int Hd, int Wd, int f, int acc, void* stream) {
  if (!src || !dst) {
    set_error("cocos_nhwc_unpack: null pointer argument");
    return -1;
  }
  return nhwc_unpack_launch(src, kind, Cs, c_lo, C, B, H, W, pad, dst, Cd, cd_lo, Hd, Wd, f, acc,
                            static_cast<cudaStream_t>(stream));
}

int cocos_colsum_nhwc(const void* x, int kind, int Cs, int C, long long rows, float* out, float* ws,
                      long long* ws_floats, void* stream) {
  if (ws && (!x || !out)) {
    set_error("cocos_colsum_nhwc: null pointer argument");
    return -1;
  }
  return colsum_nhwc_launch(x, kind, Cs, C, rows, out, ws, ws_floats, static_cast<cudaStream_t>(stream));
}

int cocos_se_nhwc_fwd(const void* dx, int dx_kind, int dx_Cs, const void* res, int res_kind, int res_Cs, const float* w1,
                      const float* w2, void* y, int y_kind, int y_Cs, float* m, float* hid, float* s, int B, int C, int Cr,
                      int HW, float* ws, long long* ws_floats, void* stream) {
  if (ws && (!dx || !res || !w1 || !w2 || !y || !m || !hid || !s)) {
    set_error("cocos_se_nhwc_fwd: null pointer argument");
    return -1;
  }
  return se_nhwc_fwd_launch(dx, dx_kind, dx_Cs, res, res_kind, res_Cs, w1, w2, y, y_kind, y_Cs, m, hid, s, B, C, Cr, HW,
                            ws, ws_floats, static_cast<cudaStream_t>(stream));
}

int cocos_se_nhwc_bwd(const void* dy, int dy_Cs, const void* dx, int dx_kind, int dx_Cs, const float* w1, const float* w2,
                      const float* m, const float* hid, const float* s, void* ddx, int ddx_Cs, float* dw1, float* dw2,
                      int B, int C, int Cr, int HW, float* ws, long long* ws_floats, void* stream) {
  if (ws && (!dy || !dx || !w1 || !w2 || !m || !hid || !s || !ddx || !dw1 || !dw2)) {
    set_error("cocos_se_nhwc_bwd: null pointer argument");
    return -1;
  }
  return se_nhwc_bwd_launch(dy, dy_Cs, dx, dx_kind, dx_Cs, w1, w2, m, hid, s, ddx, ddx_Cs, dw1, dw2, B, C, Cr, HW, ws,
                            ws_floats, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
