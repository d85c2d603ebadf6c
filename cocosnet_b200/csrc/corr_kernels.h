// Internal launch prototypes shared between the kernel translation units and
// the C-ABI (api.cu).  All pointers are device pointers; every launcher
// returns 0 or a negative error code after cocos::set_error().
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace cocos {

// v32 (optional): the values as fp32 [B, Cv, Nk]; with Cv <= 4 the P V product runs on the CUDA cores in fp32
int corr_warp_fwd_launch(const void* q, const void* k, const void* vt, const float* v32, float* out, float* lse,
                         float* corr, int B, int Nq, int Nk, int Kd, int Cv, int Cvp, int Nkp, float scale,
                         cudaStream_t stream);

// C[b] (MxN fp32, row-major, ldc) = alpha * A[b] (MxK fp16, K contiguous) * B[b]^T (NxK fp16) (+ C if accumulate)
int gemm_f16_launch(const void* a, const void* b, float* c, int batch, int M, int N, int K, int lda, int ldb,
                    int ldc, long long stride_a, long long stride_b, long long stride_c, float alpha,
                    int accumulate, int bf16, cudaStream_t stream);

int corr_bwd_ds_launch(const void* q, const void* k, const void* do16, const void* v16, const float* rscale,
                       const float* out, const float* lse, void* ds, void* dst, void* pt, int B, int Nq, int Nk,
                       int Kd, int Cv, int Cvk, int Nkp, int Nqp, float scale, cudaStream_t stream);

int pack_rows_f16_launch(const float* src, void* dst, int B, int C, int N, int Kp, int split_mode,
                         float* rowscale_out, cudaStream_t stream);
int pack_v_f16_launch(const float* src, void* dst, int B, int Cv, int Nk, int Cvp, int Nkp, int bf16,
                      cudaStream_t stream);

int cast_pitch_launch(const float* src, void* dst, long long rows, int Win, int Wout, int Wp, int nshift, int off,
                      int bf16, cudaStream_t stream);
int conv_wgrad_launch(const void* dy, const void* x, float* ws, int B, int H, int W, int Hin, int Win, int Cout, int Cin,
                      int KS, int off, int a_bf16, int b_bf16, float* ws_part, long long* ws_floats,
                      cudaStream_t stream);
int conv_fwd_launch(const void* x, const void* wt, const float* bias, float* y, int B, int H, int W, int Hin, int Win,
                    int Cp, int Cout, int KS, int off, int bf16, cudaStream_t stream);

int norm_pack_launch(const float* x, float* xt_workspace, void* out, float* mean_out, float* inv_out, int B, int C, int h,
                     int w, int mk, float eps, cudaStream_t stream);
int norm_pack_bwd_launch(const float* g, const float* x, const float* mean, const float* inv, float* a_ws, float* s_ws,
                         float* dx, int B, int C, int h, int w, int mk, cudaStream_t stream);
int transpose_f16_bf16_launch(const void* src, void* dst, int B, int N, int K, cudaStream_t stream);

int inst_act_fwd_launch(const float* x, float* y, float* mean, float* rstd, int planes, int HW, float slope, float eps,
                        cudaStream_t stream);
int inst_act_bwd_launch(const float* dy, const float* x, const float* mean, const float* rstd, float* dx, int planes,
                        int HW, float slope, cudaStream_t stream);

int spade_mod_fwd_launch(const float* x, const float* gb, float* y, float* mean, float* rstd, int B, int C, int H,
                         int W, int pad, float slope, float eps, int nhwc, cudaStream_t stream);
int spade_mod_bwd_launch(const float* dy, const float* x, const float* gb, const float* mean, const float* rstd,
                         float* dx, float* dgb, int B, int C, int H, int W, int pad, float slope, int nhwc,
                         cudaStream_t stream);

}  // namespace cocos

struct cocos_tapconv_desc;
struct cocos_tapwgrad_desc;
namespace cocos {
// 16-bit NHWC pipeline (tapconv.cu, tapwgrad.cu, ew_nhwc.cu)
int tapconv_launch(const cocos_tapconv_desc* d, cudaStream_t stream);
void tapconv_tile_shape(int B, int H, int W, int* TB, int* TH, int* TW);
int tapwgrad_launch(const cocos_tapwgrad_desc* d, long long* need_out, cudaStream_t stream);
int spade_mod_nhwc_fwd_launch(const void* x, int x_kind, int x_Cs, const void* gb, int gb_kind, int gb_Cs, void* y,
                              int y_Cs, int y_lo_off, float* mean, float* rstd, int B, int C, int H, int W, int pad,
                              float slope, float eps, cudaStream_t stream);
int ctx_rows_fwd_launch(const float* S, float* cx, int B, int N, float h, float eps, cudaStream_t stream);
int ctx_rows_bwd_launch(const float* S, const float* g, void* dS, int B, int N, int ldd, float h, float eps,
                        cudaStream_t stream);
int sn_power_iter_launch(const void* table, int n, int blocks_a, int blocks_b, float* scratch, float* inv_sigma,
                         float* snapshot, float eps, int training, cudaStream_t stream);
int pono_stats_nhwc_launch(const void* x, int kind, int Cs, int C, long long npix, float eps, float* mean, float* rstd,
                           cudaStream_t stream);
int spade_mod_nhwc_bwd_launch(const void* dy, int dy_Cs, const void* x, int x_kind, int x_Cs, const void* gb,
                              int gb_kind, int gb_Cs, int gb_W, const float* mean, const float* rstd, void* dx, int dx_Cs,
                              int dx_acc, void* dgb, int dgb_Cs, int B, int C, int H, int W, int pad, float slope,
                              cudaStream_t stream);
int in_stats_nhwc_launch(const void* x, int kind, int Cs, int B, int C, int HW, float* stats, float* ws,
                         long long* ws_floats, cudaStream_t stream);
int inst_act_nhwc_fwd_launch(const void* x, int x_kind, int x_Cs, const float* stats, const void* res, int res_kind,
                             int res_Cs, const float* slope_ptr, float slope, void* y, int y_kind, int y_Cs,
                             int y_lo_off, int y_pad, void* y2, int y2_Cs, int B, int C, int H, int W, float eps,
                             const void* gb, int gb_kind, int gb_Cs, int batch_stats, cudaStream_t stream);
int inst_act_nhwc_bwd_launch(const void* dy, int dy_Cs, int dy_pad, const void* dy2, int dy2_Cs, const void* x,
                             int x_kind, int x_Cs, const float* stats, const void* res, int res_kind, int res_Cs,
                             const float* slope_ptr, float slope, float* bstats, float* dslope, void* dx, int dx_Cs,
                             int dx_acc, void* dres, int dres_Cs, int dres_acc, int B, int C, int H, int W, float eps,
                             const void* gb, int gb_kind, int gb_Cs, void* dgb, int dgb_Cs, int batch_stats,
                             int const_stats, int phase, float* ws, long long* ws_floats, cudaStream_t stream);
int act_bwd_nhwc_launch(const void* dy, int dy_Cs, const void* y, int y_kind, int y_Cs, int pad, void* dz, int dz_Cs,
                        int B, int C, int H, int W, int act, float slope, cudaStream_t stream);
int nhwc_pack_launch(const float* src, void* dst, int kind, int B, int C, int Cs, int lo_off, int c_lo, int c_span,
                     int Hs, int Ws, int H, int W, int f, int pad, cudaStream_t stream);
int pair_loss_nhwc_fwd_launch(const void* x, int x_Cs, const void* y, int y_Cs, const float* w, int B, long long HW, int C,
                              float scale, int mode, float* out, float* ws, long long* ws_floats, cudaStream_t stream);
int pair_loss_nhwc_bwd_launch(const void* x, int x_Cs, const void* y, int y_Cs, const float* w, int B, long long HW, int C,
                              float scale, int mode, const float* g, void* dx, int dx_Cs, int acc, cudaStream_t stream);
int cast_op_bf16_launch(const void* src, int src_Cs, int lo_off, void* dst, int dst_Cs, long long npix,
                        cudaStream_t stream);
int maxpool2_nhwc_fwd_launch(const void* x, void* y, int B, int Cs, int Ho, int Wo, cudaStream_t stream);
int maxpool2_nhwc_bwd_launch(const void* dy, const void* x, void* dx, int B, int Cs, int Ho, int Wo,
                             cudaStream_t stream);
int nhwc_unpack_launch(const void* src, int kind, int Cs, int c_lo, int C, int B, int H, int W, int pad, float* dst,
                       int Cd, int cd_lo, int Hd, int Wd, int f, int acc, cudaStream_t stream);
int colsum_nhwc_launch(const void* x, int kind, int Cs, int C, long long rows, float* out, float* ws,
                       long long* ws_floats, cudaStream_t stream);
int pack_w_launch(const float* w, int Cout, int Cin, int KS, void* dst, int rows, int rows_alloc, int Kc, int ngroups,
                  const signed char* r, const signed char* s, const signed char* term, int transposed, int bf16,
                  cudaStream_t stream);
int se_nhwc_fwd_launch(const void* dx, int dx_kind, int dx_Cs, const void* res, int res_kind, int res_Cs,
                       const float* w1, const float* w2, void* y, int y_kind, int y_Cs, float* m, float* hid, float* s,
                       int B, int C, int Cr, int HW, float* ws, long long* ws_floats, cudaStream_t stream);
int se_nhwc_bwd_launch(const void* dy, int dy_Cs, const void* dx, int dx_kind, int dx_Cs, const float* w1,
                       const float* w2, const float* m, const float* hid, const float* s, void* ddx, int ddx_Cs,
                       float* dw1, float* dw2, int B, int C, int Cr, int HW, float* ws, long long* ws_floats,
                       cudaStream_t stream);
}  // namespace cocos
