/* saicv_b200.h — C ABI of libsaicv_b200.so: the sm_90a kernels behind the SimpleAICV
 * data-parallel training hot path (conv / ViT backbones forward + backward).
 *
 * The reference (zgcr/SimpleAICV_pytorch_training_examples) ships no native code; every entry
 * point below replaces a torch library call made from the reference file:line that is cited.
 * Conventions: raw device pointers + sizes, `stream` is a cudaStream_t passed as void*, the
 * library never allocates or frees device memory, never synchronises, never touches the
 * default stream unless stream == NULL is passed by the caller.  Every function returns 0 on
 * success and a non-zero code otherwise; saicv_last_error() returns a thread-local message.
 * Activations are NHWC bf16, parameters are fp32 in the reference's own layouts; bf16 operand
 * copies of weights are made by saicv_prep_conv_weight / saicv_cast_bf16.
 */
#ifndef SAICV_B200_H_
#define SAICV_B200_H_
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* epilogue flags for the GEMM family */
#define SAICV_EPI_BIAS 1
#define SAICV_EPI_RELU 2
#define SAICV_EPI_GELU 4
#define SAICV_EPI_DIRECT 8 /* debugging: registers -> global without the TMA store path */
#define SAICV_EPI_RESID 16 /* += fp32 residual[M, N] */
#define SAICV_EPI_ADD_BF16 32   /* saicv_linear_dgrad: the aux bf16 operand is ADDED to dx */
#define SAICV_EPI_MUL_DRELU 512 /* saicv_linear_dgrad: the aux bf16 operand is a ReLU output; dx *= (aux > 0) */

int saicv_version(void);
const char* saicv_last_error(void);
/* Number of SMs the persistent kernels size their grids for (132 on H100 SXM). */
int saicv_sm_count(void);
/* Kernels launched by this library in this process so far (bench.py reports the delta). */
long long saicv_launch_count(void);

/* ---- dense layers: nn.Linear (vit.py:57-58,87-89; resnet.py:204) ------------------------ */
/* y[M,N] = resid + row_scale[row / rows_per_scale] * act(x[M,K] w[N,K]^T + bias); x,w bf16; y bf16
 * or fp32 (out_f32); bias [N] fp32, resid [M,N] fp32 and row_scale (drop-path, vit.py:118-135) may
 * be NULL. */
int saicv_linear_fwd(const void* x, const void* w, const float* bias, const float* resid,
                     const float* row_scale, int rows_per_scale, float* stats_partial, void* y,
                     int M, int N, int K, int flags, int out_f32, void* stream);
/* Forward GEMMs (saicv_linear_fwd / saicv_conv_fprop) can accumulate the BatchNorm statistics of
 * their own (bf16) output in the epilogue: pass stats_partial (saicv_gemm_stats_rows(M, N) * 2 * N
 * floats, <= SAICV_BN_PARTIAL_ROWS rows) and hand it to saicv_bn_finalize with that row count. */
int saicv_gemm_stats_rows(long long out_rows, int out_cols);
/* dx[M,K] = (dy[M,N] w[N,K]) (* gelu'(gelu_pre[M,K])) (+ resid[M,K]); dy,w,gelu_pre bf16; dx bf16
 * or fp32; gelu_pre (the pre-activation saved by the forward, vit.py:87-89) and resid may be NULL.
 * With SAICV_EPI_MUL_DRELU / SAICV_EPI_ADD_BF16 in flags the bf16 operand passed as gelu_pre is instead a
 * ReLU output used as a mask (van.py:46-51: fc2 <- relu) / a second bf16 gradient added to dx. */
int saicv_linear_dgrad(const void* dy, const void* w, const float* resid, const void* gelu_pre,
                       void* dx, int M, int N, int K, int flags, int out_f32, void* stream);
/* dw_partial[splits][N][K] (fp32) = dy[M,N]^T x[M,K], reduction over M split `splits` ways.
 * Pass splits = saicv_wgrad_splits(...) and reduce with saicv_reduce_partials. */
int saicv_linear_wgrad(const void* dy, const void* x, float* dw_partial, int M, int N, int K,
                       int splits, void* stream);
int saicv_wgrad_splits(int out_rows, int out_cols, long long reduce_len);
/* 1 when the weight gradient dW [out_rows, out_cols] is computed as dW^T (fewer padded 128-row tiles: few filters).
 * saicv_conv_wgrad then writes dw_partial [splits][r*s*c][k]; linear_wgrad callers swap dy and x themselves. */
int saicv_wgrad_transposed(int out_rows, int out_cols);

/* ---- convolutions: nn.Conv2d inside ConvBnActBlock (resnet.py:33-39, darknet.py:49-56) ---- */
typedef struct {
  int n, h, w, c; /* input  NHWC */
  int k, r, s;    /* filters, taps; weights bf16 [k][r][s][c] */
  int stride, pad;
} saicv_conv_shape;
/* y[n,p,q,k] bf16; requires c % 64 == 0 (the 3-channel stem goes through saicv_stem_im2col +
 * saicv_linear_fwd). */
int saicv_conv_fprop(const void* x, const void* w, float* stats_partial, void* y,
                     const saicv_conv_shape* cs, int flags, void* stream);
/* dx[n,h,w,c] = sum dy[n, h+pad-r, w+pad-s, k] w[k,r,s,c] (+ add[n,h,w,c]) (* mask): stride-1 data
 * gradient; `add` (bf16, may be NULL) is the gradient arriving over the shortcut, fused into the
 * epilogue.  `mask_bits` (may be NULL): the [n*h*w][c/32] ReLU mask written by saicv_bn_apply; the
 * result (after the add) is multiplied by its bit, i.e. dx is the gradient behind that ReLU.
 * `dy` has spatial extent (h, w).  requires k % 64 == 0, c % 64 == 0.
 * stride = 2 (3x3, pad 1, even h and w, w <= 256, no `add` / `mask_bits`): `dy` is the compact [n, h/2, w/2, k]
 * gradient of the strided conv; each output phase (h mod 2, w mod 2) reduces only the taps that reach it, in the order
 * the stride-1 path reduces them, so dx equals that path's bit for bit up to the sign of exact zeros.  Other
 * stride-2 convs: pass the zero-upsampled dy (saicv_zero_upsample2) and stride = 1. */
int saicv_conv_dgrad(const void* dy, const void* w, const void* add, const uint32_t* mask_bits, void* dx,
                     const saicv_conv_shape* cs, void* stream);
/* dw_partial[splits][k][r*s*c] fp32 = sum over output pixels dy[pix,k] * x[patch(pix), (r,s,c)]; laid out
 * [splits][r*s*c][k] (dW^T) when saicv_wgrad_transposed(k, r*s*c).  splits = saicv_wgrad_splits(k, r*s*c, pixels) in
 * both layouts, so every element is the same sum. */
int saicv_conv_wgrad(const void* dy, const void* x, float* dw_partial, const saicv_conv_shape* cs,
                     int splits, void* stream);

/* ---- layout / weight preparation ---------------------------------------------------------- */
/* fp32 [k][c][r][s] (torch Conv2d.weight) -> bf16 [k][kpad], zero padded to kpad (kpad >=
 * r*s*c, multiple of 8).  order 0: column (r*S+s)*C + c, the implicit-GEMM layout of
 * saicv_conv_*; order 1: column (c*R+r)*S + s, the layout of saicv_stem_im2col.  kp / cp (0 = k / c):
 * rows and per-tap channels padded with zeros (networks whose channel counts are not multiples of
 * 64 run on channel-padded activations, e.g. DarkNet's 32-channel stem). */
int saicv_prep_conv_weight(const float* w, void* w_bf16, int k, int c, int r, int s, int kpad,
                           int order, int kp, int cp, void* stream);
/* sum of fp32 partials [splits][k][kpad] (columns in `order`; transposed != 0: [splits][kpad][k]) -> fp32 grad in
 * torch layout [k][c][r][s]; accumulate != 0 adds to the destination (gradient accumulation). */
int saicv_finish_conv_wgrad(const float* partial, float* grad, int splits, int k, int c, int r,
                            int s, int kpad, int accumulate, int order, int kp, int cp, int transposed, void* stream);
/* out[i] (+)= sum_s partial[s][i]; plain reduction for linear wgrad. */
int saicv_reduce_partials(const float* partial, float* out, int splits, long long n,
                          int accumulate, void* stream);
int saicv_cast_bf16(const float* src, void* dst, long long n, void* stream);
/* NCHW fp32 image batch -> NHWC bf16 */
int saicv_nchw_to_nhwc_bf16(const float* x, void* y, int n, int c, int h, int w, void* stream);
/* NCHW fp32 image batch -> im2col matrix [n*p*q][kpad] bf16 for the 3-channel stem conv
 * (resnet.py:173-180 7x7/2, resnetforcifar.py:38-45 3x3/1; vit.py:31-37 16x16/16 patches);
 * column (ch*R+r)*S8 + s with S8 = S rounded up to a multiple of 8 (every filter row is a whole number of 16-byte
 * vectors; padding columns are zero).  kpad = saicv_stem_kpad(c, r, s) = c*r*S8 rounded up to 64; the weight operand
 * uses the same column order (saicv_prep_conv_weight / saicv_finish_conv_wgrad with order 1). */
int saicv_stem_kpad(int c, int r, int s);
int saicv_stem_im2col(const float* x, void* cols, int n, int c, int h, int w, int r, int s,
                      int stride, int pad, int kpad, void* stream);
/* u[n, 2p, 2q, c] = dy[n,p,q,c], zero elsewhere; u is [n,h,w,c]. */
int saicv_zero_upsample2(const void* dy, void* u, int n, int p, int q, int h, int w, int c,
                         void* stream);
/* dx[n,2p,2q,c] += dd[n,p,q,c]  (data gradient of a 1x1 stride-2 conv added in place). */
int saicv_add_strided2(void* dx, const void* dd, int n, int p, int q, int h, int w, int c,
                       void* stream);

/* ---- BatchNorm2d (training) + ReLU + residual (resnet.py:40-42,152-153) ------------------- */
/* Column reductions are deterministic (no atomics): every block writes one row of partial sums
 * into a caller-provided workspace `partials` of SAICV_BN_PARTIAL_ROWS * 2 * c floats, folded in a
 * fixed order by the next call. */
#define SAICV_BN_PARTIAL_ROWS 264
/* per-channel partial sum / sum of squares of y[rows][c] (bf16) -> partials. */
int saicv_bn_stats(const void* y, float* partials, long long rows, int c, void* stream);
/* folds `partial_rows` rows of `partials` (0: the row count saicv_bn_stats used for this rows, c;
 * otherwise the count returned by saicv_gemm_stats_rows for an epilogue-fused reduction) ->
 * mean/var -> scale_shift[2][c], saved[2][c] = (mean, rstd); running stats updated with `momentum`
 * and the unbiased variance exactly like nn.BatchNorm2d (running_* may be NULL). */
int saicv_bn_finalize(const float* partials, int partial_rows, const float* gamma, const float* beta,
                      float* running_mean, float* running_var, float* scale_shift, float* saved,
                      long long rows, int c, float eps, float momentum, void* stream);
/* out = act(y*scale+shift + res) ; res optional, itself optionally batch-normalised with
 * res_scale_shift (downsample branch).  act: 0 none, 1 ReLU, 2 LeakyReLU(0.1); act | 8: the
 * residual is added after the activation, out = act(y*scale+shift) + res (darknet.py:141-144).
 * mask_bits (may be NULL; act == 1 and c % 32 == 0): receives the ReLU mask of `out` packed as
 * uint32 [rows][c/32], bit j of word w set where out[row][32w + j] > 0. */
int saicv_bn_apply(const void* y, const float* scale_shift, const void* res,
                   const float* res_scale_shift, void* out, uint32_t* mask_bits, long long rows, int c,
                   int act, void* stream);
/* backward reductions: g = dout * act'(out); sums[0][c] = sum g, sums[1][c] = sum g * xhat
 * (xhat from y, saved mean/rstd).  The activation mask comes from `out` (activated output) when
 * it is non-NULL; else from `bits` (the ReLU mask of saicv_bn_apply, act == 1) when it is
 * non-NULL; otherwise, for a unit without residual input, it is recomputed from
 * sign(y*scale+shift) using `scale_shift` (saves reading `out`).  All may be NULL when act == 0.
 * `partials`: workspace as above; `sums[2][c]` receives the folded result. */
int saicv_bn_bwd_reduce(const void* dout, const void* out, const uint32_t* bits, const void* y,
                        const float* saved, const float* scale_shift, float* partials, float* sums,
                        long long rows, int c, int act, void* stream);
/* dy = gamma*rstd*(g - sum_g/rows - xhat*sum_gx/rows) bf16; writes dgamma/dbeta (fp32, (+)=)
 * and optionally dres = g (gradient flowing into the residual input). */
int saicv_bn_bwd_apply(const void* dout, const void* out, const uint32_t* bits, const void* y,
                       const float* saved, const float* gamma, const float* scale_shift, float* sums,
                       void* dy, void* dres, float* dgamma, float* dbeta, long long rows, int c, int act,
                       int accumulate, void* stream);
/* The same two passes for two BatchNorms A and B with one gradient g and the same rows, c (the last
 * BatchNorm and the downsample BatchNorm of a residual block): g = g_in * bits (bits may be NULL:
 * g_in is already masked).  `partials`: SAICV_BN_PARTIAL_ROWS * 4 * c floats; sums[4][c] = A's
 * sums[2][c] then B's.  Sums, dy and dgamma / dbeta equal two saicv_bn_bwd_reduce /
 * saicv_bn_bwd_apply calls bit for bit. */
int saicv_bn_bwd_reduce2(const void* g, const uint32_t* bits, const void* y_a, const void* y_b,
                         const float* saved_a, const float* saved_b, float* partials, float* sums,
                         long long rows, int c, void* stream);
int saicv_bn_bwd_apply2(const void* g, const uint32_t* bits, const void* y_a, const void* y_b,
                        const float* saved_a, const float* saved_b, const float* gamma_a,
                        const float* gamma_b, const float* sums, void* dy_a, void* dy_b,
                        float* dgamma_a, float* dbeta_a, float* dgamma_b, float* dbeta_b,
                        long long rows, int c, int accumulate_a, int accumulate_b, void* stream);
/* a = a + b (bf16), used where two gradient paths meet. */
int saicv_add_bf16(void* a, const void* b, long long n, void* stream);

/* ---- pooling (resnet.py:184,203) ----------------------------------------------------------- */
int saicv_maxpool3x3s2_fwd(const void* x, void* y, uint8_t* argmax, int n, int h, int w, int c,
                           void* stream);
int saicv_maxpool3x3s2_bwd(const void* dy, const uint8_t* argmax, void* dx, int n, int h, int w,
                           int c, void* stream);
/* General nn.MaxPool2d(k, stride) on NHWC bf16 (darknet.py:105,161-213: 2x2/2 pools; :212-213
 * ZeroPad2d((0,1,0,1)) + MaxPool2d(2,1) = pad 0, pad_hi 1, oob_zero 1: padded taps count as 0 and
 * get no gradient).  Output extent (h + pad + pad_hi - k) / stride + 1; argmax byte = r*k + s. */
int saicv_maxpool_fwd(const void* x, void* y, uint8_t* argmax, int n, int h, int w, int c, int k,
                      int stride, int pad, int pad_hi, int oob_zero, void* stream);
int saicv_maxpool_bwd(const void* dy, const uint8_t* argmax, void* dx, int n, int h, int w, int c,
                      int k, int stride, int pad, int pad_hi, void* stream);
int saicv_avgpool_fwd(const void* x, void* y, int n, int hw, int c, void* stream);
int saicv_avgpool_bwd(const void* dy, void* dx, int n, int hw, int c, void* stream);
/* column sums of a bf16 (or fp32 when is_f32) [rows][c] matrix into fp32 out[c] ((+)= when
 * accumulate): bias gradients.  `partials`: SAICV_BN_PARTIAL_ROWS * c floats (unused for fp32). */
int saicv_colsum(const void* x, float* partials, float* out, long long rows, int c, int accumulate,
                 int is_f32, void* stream);

/* ---- ViT blocks (SimpleAICV/classification/backbones/vit.py) --------------------------------- */
/* nn.LayerNorm(eps=1e-6) (vit.py:147,151,225): x fp32 [rows][c] -> y bf16; stats[2][rows] =
 * (mean, rstd) kept for the backward.  c in {128, 256, 768, 1024, 1280}. */
int saicv_layernorm_fwd(const float* x, const float* gamma, const float* beta, void* y,
                        float* stats, long long rows, int c, float eps, void* stream);
/* dx (fp32) = dres + LN'(dy) with dres the residual-stream gradient (may be NULL); optional bf16
 * copy of dx for the next GEMM, optionally pre-multiplied per row by
 * bf16_row_scale[row / rows_per_scale] (the drop-path scale of the branch that consumes it);
 * dgamma/dbeta (+)= column reductions (zeroed first unless accumulate). */
int saicv_layernorm_bwd(const void* dy, const float* x, const float* gamma, const float* stats,
                        const float* dres, float* dx, void* dx_bf16, const float* bf16_row_scale,
                        int rows_per_scale, float* partials /* [SAICV_BN_PARTIAL_ROWS][2*c] workspace */,
                        float* dgamma, float* dbeta, long long rows, int c, int accumulate, void* stream);
/* nn.GELU() exact erf (vit.py:87-89): h = gelu(u); du = dh * gelu'(u); bf16, n % 8 == 0. */
int saicv_gelu_fwd(const void* u, void* h, long long n, void* stream);
int saicv_gelu_bwd(const void* dh, const void* u, void* du, long long n, void* stream);
/* x[b,0] = cls + pos[0]; x[b,1+i] = patch[b*np+i] + pos[1+i] (vit.py:242-243); all fp32. */
int saicv_vit_assemble_tokens(const float* patch, const float* cls, const float* pos, float* x,
                              int b, int np, int c, void* stream);
/* dpos (+)= sum_b dx[b]; dcls (+)= sum_b dx[b,0]; dpatch[b*np+i] = bf16(dx[b,1+i]). */
int saicv_vit_assemble_tokens_bwd(const float* dx, float* dpos, float* dcls, void* dpatch, int b,
                                  int np, int c, int accumulate, void* stream);
/* pooled[b] = mean of tokens 1..l-1 (mean_pool, vit.py:252-255) or token 0 (vit.py:257-258). */
int saicv_token_pool_fwd(const float* x, float* pooled, int b, int l, int c, int mean_pool,
                         void* stream);
int saicv_token_pool_bwd(const float* dpooled, float* dx, void* dx_bf16, const float* bf16_row_scale,
                         int b, int l, int c, int mean_pool, void* stream);
/* ---- VAN (SimpleAICV/classification/backbones/van.py) ------------------------------------------------
 * Depthwise convolution k x k (3, 5, 7), dilation dil, 'same' padding dil*(k-1)/2, stride 1, NHWC bf16
 * (van.py:20-35 DWConv 3x3; :63-77 LKA 5x5 and 7x7 dilation 3).  w: fp32 [C][1][k][k] (torch layout),
 * bias fp32 [C] or NULL; relu: fused ReLU (van.py:49-50); flip: mirrored taps = the data gradient. */
int saicv_dwconv_fwd(const void* x, const float* w, const float* bias, void* y, int n, int h, int wd,
                     int c, int k, int dil, int relu, int flip, void* stream);
/* ConvFormer SepConv (SimpleAICV/classification/backbones/convformer.py:64-79: dwconv(relu(pwconv1(x)))):
 * dx = dwconv^T(dy) * (mask > 0), the data gradient of the 7x7 depthwise conv (dilation 1, no bias) masked by
 * the ReLU in front of it; mask bf16 [n][h][wd][c] = that ReLU's output.  Replaces the autograd pair
 * conv-backward + threshold_backward of :68-70.  k must be 7. */
int saicv_dwconv_dgrad_masked(const void* dy, const float* w, const void* mask, void* dx, int n, int h,
                              int wd, int c, int k, void* stream);
/* Global average pool of an NHWC stream x [n][hw][c], bf16 or fp32 (x_f32), summed in fp32 and written once
 * as the head GEMM's bf16 operand y [n][c] (convformer.py:251-254: AdaptiveAvgPool2d of the fp32 or bf16
 * stream, then autocast's cast for the Linear).  Backward: dx [n][hw][c] (fp32 when dx_f32, else bf16) =
 * dy [n][c] (bf16) / hw. */
int saicv_avgpool_stream_fwd(const void* x, int x_f32, void* y, int n, int hw, int c, void* stream);
int saicv_avgpool_stream_bwd(const void* dy, void* dx, int dx_f32, int n, int hw, int c, void* stream);
/* dw[C][1][k][k] (+)= sum over pixels dy * shifted x; partial: fp32 workspace
 * [saicv_dwconv_wgrad_blocks(n*h*w)][k*k][C]; fixed-order two-stage reduction. */
int saicv_dwconv_wgrad_blocks(long long npix);
int saicv_dwconv_wgrad(const void* dy, const void* x, float* partial, float* dw, int n, int h, int wd,
                       int c, int k, int dil, int accumulate, void* stream);
/* out = a * b (LKA gate u * attn, van.py:91, and its gradient w.r.t. attn); bf16, n % 8 == 0. */
int saicv_mul_bf16(const void* a, const void* b, void* out, long long n, void* stream);
/* out = (dg * c1 + dlk) * (p1 > 0): gradient at the input of the ReLU that produced p1 (van.py:106-108),
 * from the gate (dg * c1) and from the LKA convolutions (dlk). */
int saicv_gate_bwd(const void* dg, const void* c1, const void* dlk, const void* p1, void* out,
                   long long n, void* stream);
/* Residual update with layer scale (van.py:183-184): out(fp32) = x + row_scale[row/rows_per_scale] *
 * ls[c] * (branch [+ shortcut]); x bf16 or fp32 (x_f32), branch / shortcut bf16 [rows][c], shortcut and
 * row_scale (drop path, van.py:118-151) may be NULL. */
int saicv_ls_residual_fwd(const void* x, int x_f32, const void* branch, const void* shortcut,
                          const float* ls, const float* row_scale, int rows_per_scale, float* out,
                          long long rows, int c, void* stream);
/* dy(bf16) = row_scale * ls[c] * dxn; dls[c] (+)= sum_rows row_scale * dxn * (branch [+ shortcut]);
 * partial: fp32 workspace [SAICV_BN_PARTIAL_ROWS][c]. */
int saicv_ls_residual_bwd(const float* dxn, const void* branch, const void* shortcut, const float* ls,
                          const float* row_scale, int rows_per_scale, void* dy, float* partial,
                          float* dls, long long rows, int c, int accumulate, void* stream);
/* Train-mode BatchNorm2d over [rows][c] with bf16 OR fp32 input / output (van.py:160-165,205-207: BN of the
 * fp32 residual stream feeding bf16 GEMMs; :200-207 BN of the bf16 patch-embedding conv into the stream).
 * stats: partial sums [saicv_bn_generic_partial_rows(rows, c)][2][c] for saicv_bn_finalize; apply:
 * out = x*scale + shift; bwd: dx = BN'(g) [+ dres fp32], dgamma/dbeta (+)=; partial [..][2][c], sums [2][c]. */
int saicv_bn_generic_partial_rows(long long rows, int c);
int saicv_bn_stats_generic(const void* x, int x_f32, float* partial, long long rows, int c, void* stream);
int saicv_bn_apply_generic(const void* x, int x_f32, const float* scale_shift, void* out, int out_f32,
                           long long rows, int c, void* stream);
int saicv_bn_bwd_generic(const void* x, int x_f32, const void* g, int g_f32, const float* saved,
                         const float* gamma, const float* dres, float* partial, float* sums, void* dx,
                         int dx_f32, float* dgamma, float* dbeta, long long rows, int c, int accumulate,
                         void* stream);
/* NHWC bf16 im2col / col2im for the strided patch-embedding convolutions whose channel counts are not
 * multiples of 64 (van.py:189-208: 3x3 stride 2): cols[(n,p,q)][(r*k+s)*c + ch]. */
int saicv_im2col_nhwc(const void* x, void* cols, int n, int h, int w, int c, int k, int stride, int pad,
                      void* stream);
int saicv_col2im_nhwc(const void* dcols, void* dx, int n, int h, int w, int c, int k, int stride, int pad,
                      void* stream);

/* ---- SAM image encoder (segment_anything/image_encoder.py) ---------------------------------------------
 * Window partition with zero padding (:32-55) / unpartition (:58-79) of NHWC bf16 tokens:
 * windows [b*nwy*nwx][ws*ws][c], nwy = ceil(h/ws), nwx = ceil(w/ws). */
int saicv_window_partition(const void* x, void* windows, int b, int h, int w, int c, int ws, void* stream);
int saicv_window_unpartition(const void* windows, void* x, int b, int h, int w, int c, int ws, void* stream);
/* x[b][...] += pos[...] (fp32, in place): tokens + pos_embed (:315); per_batch = elements of pos. */
int saicv_add_pos_embed(float* x, const float* pos, int b, long long per_batch, void* stream);
/* Decomposed relative-position bias as extra score columns (image_encoder.py:82-144): the bias terms are dot products
 * of q rows with rel-pos table rows, so they run as GEMMs of the tensor-core engine; these entries move / re-index data
 * around them.  qkv: bf16 [bw][l = sh*sw][3][heads][hd]; per-head operand rows r are ordered (window, head, token);
 * nip: a multiple of 8 >= (2sh-1) + (2sw-1); dqk: a multiple of 8 >= hd + sh + sw.
 *   pack_q:   qc bf16 [rows][hd] = the q rows (unscaled)
 *   table:    rtab bf16 [nip][hd] = [rel_pos_h ; rel_pos_w ; 0]
 *   (T bf16 [rows][nip] = saicv_linear_fwd(qc, rtab))
 *   gather:   qe = [q*scale | T[r][qh-kh+sh-1] | T[r][(2sh-1)+qw-kw+sw-1] | 0], ke = [k | onehot(kh) | onehot(kw) | 0]
 *   shift:    ef bf16 [rows][nip] = the bias-column gradients of dqe re-indexed so that column idx is its table row
 *   (dqx fp32 [rows][hd] = saicv_linear_dgrad(ef, rtab); [d rel_pos_h ; d rel_pos_w] = saicv_linear_wgrad(ef, qc))
 *   dq_combine: q slot of dqkv = bf16(scale * dqe[r][0:hd] + dqx[r]) */
int saicv_relpos_pack_q(const void* qkv, void* qc, int bw, int heads, int hd, int l, void* stream);
int saicv_relpos_table(const float* rel_pos_h, const float* rel_pos_w, void* rtab, int sh, int sw, int nip, int hd,
                       void* stream);
int saicv_relpos_gather(const void* qkv, const void* t, void* qe, void* ke, int bw, int heads, int hd, int sh, int sw,
                        int dqk, int nip, float scale, void* stream);
int saicv_relpos_shift(const void* dqe, void* ef, int bw, int heads, int hd, int sh, int sw, int dqk, int nip,
                       void* stream);
int saicv_relpos_dq_combine(const void* dqe, const float* dqx, void* dqkv, int bw, int heads, int hd, int l, int dqk,
                            float scale, void* stream);

/* ---- fused multi-head attention on wgmma (csrc/attn_sm90.cuh) ------------------------------
 * Replaces the materialised attention of the reference: vit.py:62-80 (q k^T * scale, softmax, @ v),
 * segment_anything/image_encoder.py:167-184 (+ decomposed rel-pos bias, folded into extra score columns by
 * the caller: dqk = head_dim + bias columns), detection/models/detr.py:54-56,103-109 (nn.MultiheadAttention
 * with key_padding_mask, self- and cross-attention).
 *   S = Q K^T * scale  [lq x lk]; masked keys -> -inf; P = softmax(S); out = P V; the l x l matrices never
 *   touch HBM.  q, k: bf16 rows of dqk elements; v, out: bf16 rows of dv elements; every tensor is addressed
 *   as [b][h][row] through element strides {batch, head, row} (rows contiguous, 16-byte aligned), so packed
 *   qkv [b][l][3][h][d], [b*h][l][d] and [b][l][h*d] layouts are all views.  lse [b][h][lq] fp32 holds
 *   log2(sum exp2(s*scale*log2e)) for the backward.  key_mask_bits: [b][mask_words] uint32, bit k%32 of
 *   word k/32 set = key k is padding (NULL: none); mask_words*32 >= lk rounded up to 128.
 *   Supported (dqk, dv): (32,32) (64,64) (80,80) (96,64) (112,64) (112,80) (128,80) (192,64) (208,80). */
typedef struct {
  const void* q; const void* k; const void* v;
  void* out;
  float* lse;
  long long q_strides[3], k_strides[3], v_strides[3], o_strides[3];
  const unsigned int* key_mask_bits;
  int mask_words;
  int b, h, lq, lk, dqk, dv;
  float scale;
  /* attention-probability dropout (nn.MultiheadAttention(dropout=p), detr.py:55-57): probability dropout_p of
   * zeroing softmax(S)[q, k], survivors scaled by 1 / (1 - p); the mask is the counter hash of csrc/dropout_hash.cuh
   * over (row (b*h + head)*lq + q, column k) under dropout_seed, recomputed by the backward.  0 = off. */
  float dropout_p;
  unsigned long long dropout_seed;
  const unsigned long long* dropout_seed_base;  /* device word added to dropout_seed (nullable), see saicv_dropout */
} saicv_attn_args;
int saicv_attn_fwd(const saicv_attn_args* a, void* stream);
/* Backward: fwd holds the forward's arguments (out = the forward output, lse as written by it); dout has the
 * layout of out.  delta: fp32 workspace [b][h][lq] (rowsum(dout * out), written here).  dq rows have dqk
 * columns; dk rows get their leading dk_cols columns (0 = all dqk; the bias columns of k carry no gradient);
 * dv rows dv columns.  Two deterministic phases (no atomics): dQ per query tile, dK/dV per key tile. */
typedef struct {
  saicv_attn_args fwd;
  const void* dout;
  float* delta;
  void* dq; void* dk; void* dv;
  long long dq_strides[3], dk_strides[3], dv_strides[3];
  int dk_cols;
} saicv_attn_bwd_args;
int saicv_attn_bwd(const saicv_attn_bwd_args* a, void* stream);
/* ViT convenience entries (vit.py:66-76): qkv bf16 [b][l][3][h][d] -> out bf16 [b][l][h*d]; lse [b][h][l];
 * backward writes dqkv in the layout of qkv; delta: fp32 workspace [b][h][l]. */
int saicv_attention_fwd(const void* qkv, void* out, float* lse, int b, int l, int h, int d,
                        float scale, void* stream);
int saicv_attention_bwd(const void* qkv, const void* out, const void* dout, const float* lse,
                        float* delta, void* dqkv, int b, int l, int h, int d, float scale, void* stream);

/* ---- DETR transformer glue (SimpleAICV/detection/models/detr.py:44-180; csrc/capi_detr.cu) -------------------
 * Post-LayerNorm on the fp32 token stream: y = LN(z) (nullable), yb = bf16(y) (nullable),
 * ypb = bf16(y + pos[row % pos_rows]) (nullable; pos fp32 [pos_rows][c]); stats fp32 [2][rows] (mean | rstd).
 * c in {128, 256, 384, 512}. */
int saicv_postln_fwd(const float* z, const float* gamma, const float* beta, float eps, float* y, void* yb,
                     const float* pos, long long pos_rows, void* ypb, float* stats, long long rows, int c,
                     void* stream);
/* dz = LN'(dy) (+ dres), dy fp32: dz fp32 (nullable), dzb = bf16(dz) (nullable); dgamma / dbeta (+)= through the
 * fp32 workspace partials [SAICV_BN_PARTIAL_ROWS][2*c] in a fixed order (bit-reproducible). */
int saicv_postln_bwd(const float* dy, const float* z, const float* gamma, const float* stats, const float* dres,
                     float* dz, void* dzb, float* partials, float* dgamma, float* dbeta, long long rows, int c,
                     int accumulate, void* stream);
/* xb = bf16(x) (nullable), xpb = bf16(x + pos[row % pos_rows]) (nullable); x fp32 [rows][c]. */
int saicv_add_pos_cast(const float* x, const float* pos, long long pos_rows, void* xb, void* xpb, long long rows,
                       int c, void* stream);
/* Dropout with the counter hash of csrc/dropout_hash.cuh over the element index:
 * out = (keep ? in / (1 - p) : 0) * (row_scale ? row_scale[index / elems_per_scale] : 1) (+ resid, fp32, only with an
 * fp32 out).  row_scale is the per-sample drop-path scale of the branch (vit.py:102-135).  in / out are bf16 or fp32
 * (flags); the same call on a gradient with the same seed is the backward pass.  n %% 4 == 0.  The effective seed is
 * seed + *seed_base when seed_base (a device pointer) is given: a training step captured in a CUDA graph refreshes the
 * device word every replay, so the masks change from step to step although `seed` is a constant of the graph. */
int saicv_dropout(const void* in, int in_f32, const float* resid, const float* row_scale, long long elems_per_scale,
                  void* out, int out_f32, long long n, float p, unsigned long long seed,
                  const unsigned long long* seed_base, void* stream);
/* Per-head packing of projected rows into a score operand: dst bf16 [b][h][l][dp],
 * dst[.., 0:hd] = src[(b*l + l') * ld + col0 + head*hd + :] * scale, dst[.., hd] = extra ? extra[b*l + l'] :
 * extra_const (the column that carries nn.MultiheadAttention's additive float key_padding_mask against a constant-1
 * column of the query operand), remaining columns 0.  unpack is the inverse on the leading hd columns. */
int saicv_heads_pack(const void* src, int ld, int col0, const float* extra, float extra_const, void* dst, int b,
                     int l, int h, int hd, int dp, float scale, void* stream);
int saicv_heads_unpack(const void* src, void* dst, int ld, int col0, int b, int l, int h, int hd, int dp, float scale,
                       void* stream);

/* ---- SAMLoss on full-resolution mask logits (interactive_segmentation/losses.py:11-198; csrc/capi_loss.cu) ------------
 * logits: fp32 or bf16 [b][m][n] (n = H*W pixels, n %% 4 == 0); targets: fp32 [b][n] (one plane per image, shared by its
 * m masks).  sums: fp32 [b*m][6] = { sum focal_weight*bce, sum sigmoid(x)*t, sum sigmoid(x), sum t,
 * #(x > thr & t > thr), #(x > thr | t > thr) } — everything focal_loss (:126-146), dice_loss (:148-170) and
 * iou_predict_loss (:172-198) reduce over the pixels, in ONE pass.  partials: fp32 workspace of
 * saicv_sam_loss_partial_floats(b, m, n) floats (per-block partial sums, folded in a fixed order).
 * Backward: dlogits[b][m][i] = coef[p][0] * d(focal_weight*bce)/dx + sigmoid'(x) * (coef[p][1] * t + coef[p][2]),
 * p = b*m_count + m; coef fp32 [b*m][3] (upstream gradients folded with 1/(n b) and the dice quotient rule). */
int saicv_sam_loss_partial_floats(int b, int m, long long n);
int saicv_sam_loss_sums(const void* logits, int logits_bf16, const float* targets, float* partials, float* sums, int b,
                        int m, long long n, float alpha, float gamma, float mask_threshold, void* stream);
int saicv_sam_loss_bwd(const void* logits, int logits_bf16, const float* targets, const float* coef, void* dlogits,
                       int dl_bf16, int b, int m, long long n, float alpha, float gamma, void* stream);

/* ---- multi-tensor optimizer step (SURVEY.md 8 f2; csrc/capi_optim.cu) --------------------------------------------------
 * Replaces torch.optim.SGD / torch.optim.AdamW as the reference builds them (tools/utils.py:292-600, stepped at
 * tools/scripts.py:209-248) with ONE launch over all parameters, the refresh of the bf16 GEMM-operand copies and the
 * global-norm gradient clip (torch.nn.utils.clip_grad_norm_, tools/scripts.py:226-236) fused in.
 * tensors: device array of saicv_opt_tensor; chunk_tensor / chunk_index: device int arrays, block b updates elements
 * [chunk_index[b] * SAICV_OPT_CHUNK, +SAICV_OPT_CHUNK) of tensor chunk_tensor[b].
 * hyper: device fp32 [SAICV_OPT_RING][n_groups][8]; the update reads table (*step %% SAICV_OPT_RING) and a one-thread
 * kernel then advances *step (device int).  Rows:
 *   SGD   {lr, weight_decay, momentum, nesterov, 0...}       (dampening 0; buf = momentum buf + (g + wd p); p -= lr buf)
 *   AdamW {lr, weight_decay, beta1, beta2, eps, 1 - beta1^t, sqrt(1 - beta2^t), 0}   (torch.optim.AdamW's update)
 * clip: device fp32 [2] = {gradient scale, global norm} written by saicv_multi_tensor_clip_coef, or NULL.  All launch
 * arguments are step-invariant: a captured step replays with new learning rates once the host has rewritten slot
 * t %% SAICV_OPT_RING of the (pinned) table the captured copy brings in. */
#define SAICV_OPT_CHUNK 8192
#define SAICV_OPT_RING 8
typedef struct {
  float* p;            /* fp32 master parameter */
  const float* g;      /* fp32 gradient */
  float* s1;           /* SGD momentum buffer / AdamW exp_avg */
  float* s2;           /* AdamW exp_avg_sq (NULL for SGD) */
  void* shadow;        /* bf16 operand copy refreshed in the same pass, or NULL */
  long long numel;
  int group;           /* row of `hyper` */
  int rs;              /* shadow layout: 0 = same linear index ([N][K] Linear weights); > 0 = conv weight [K][C][rs taps]
                          -> [K][kpad] with column tap * cp + c (saicv_prep_conv_weight order 0) */
  int c, cp, kpad;
  int pad_;
} saicv_opt_tensor;
int saicv_opt_chunk(void);
int saicv_multi_tensor_sgd(const void* tensors, const int* chunk_tensor, const int* chunk_index, int n_chunks,
                           const float* hyper, int n_groups, int* step, const float* clip, void* stream);
int saicv_multi_tensor_adamw(const void* tensors, const int* chunk_tensor, const int* chunk_index, int n_chunks,
                             const float* hyper, int n_groups, int* step, const float* clip, void* stream);
/* partial: fp32 [n_chunks] workspace; clip = {min(1, max_norm / (norm + 1e-6)), norm}; fixed summation order. */
int saicv_multi_tensor_clip_coef(const void* tensors, const int* chunk_tensor, const int* chunk_index, int n_chunks,
                                 float max_norm, float* partial, float* clip, void* stream);

/* ---- input-pipeline edge (SURVEY.md 8 f3; csrc/capi_input.cu) ---------------------------------------------------------
 * out fp32 [n][3][h][w] = (float(in uint8 [n][h][w][3]) / 255 - mean[c]) / std[c]: ToTensor + Normalize of
 * classification/common.py:228-248 followed by the collater's NHWC -> NCHW permute (:645-665), on the device, bit-identical
 * to the host arithmetic (IEEE divisions in the same order).  mean3 / std3 are HOST pointers to 3 floats. */
int saicv_u8_nhwc_to_nchw_norm(const void* in, float* out, int n, int h, int w, const float* mean3, const float* std3,
                               void* stream);

/* ---- token gather / scatter for masked-token models (SURVEY.md 8 f4; csrc/capi_tokens.cu) -----------------------------
 * out fp32 [b][r][c] = (idx[b][r] >= 0 ? src[b][idx[b][r]][:] : fill[:]) + (pos ? pos[pos_idx ? pos_idx[b][r] : r][:] : 0);
 * src fp32 [b][src_rows][c].  One call is the torch.gather + cat(cls / mask token) + position-encoding add of
 * masked_image_modeling/models/vit_mae.py:171-186 (encoder: keep the visible patches) and :339-354 (decoder: un-shuffle).
 * Backward: dsrc[b][idx][:] = dout[b][r][:] for idx >= 0 (fp32 or bf16; rows never referenced must be pre-zeroed by the
 * caller) and fill_partial[slab][c] = sum of the dout rows with idx < 0 (saicv_token_fill_slabs(b * r) slabs, to be folded
 * with saicv_reduce_partials: the gradient of the cls / mask token).  Either output may be NULL.  c %% 4 == 0. */
int saicv_token_gather_fwd(const float* src, long long src_rows, const int* idx, const float* fill, const float* pos,
                           const int* pos_idx, float* out, int b, int r, int c, void* stream);
int saicv_token_fill_slabs(long long rows);
int saicv_token_gather_bwd(const float* dout, const int* idx, void* dsrc, int dsrc_bf16, long long src_rows,
                           float* fill_partial, int b, int r, int c, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SAICV_B200_H_ */
