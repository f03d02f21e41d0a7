/* pdae_b200 -- C-ABI of the Hopper-native (H100) PDAE hot path (libpdae_b200.so).
 *
 * The reference (ckczzj/PDAE) has no FFI: its hot path is PyTorch ATen dispatches issued from
 * model/module.py, model/unet.py, model/shift_unet.py, diffusion/ddim.py and
 * diffusion/gaussian_diffusion.py.  Each entry point below replaces the ATen call group named in
 * its comment (reference file:line) with one hand-written sm_90a kernel launch.
 *
 * Conventions
 *   - plain pointers and sizes only; every pointer is DEVICE memory owned by the caller;
 *   - activations are NHWC ("channels last", [B][H][W][C]) unless a flag says NCHW;
 *   - every call is asynchronous on `stream` (a cudaStream_t), allocates nothing, and is legal
 *     inside CUDA-graph capture;
 *   - return 0 on success, a negative PDAE_E* code otherwise; pdae_last_error() gives the message
 *     (thread-local).  Nothing throws or aborts.
 *   - there is NO CPU fallback: without an sm_90 device every compute entry point fails.
 */
#ifndef PDAE_B200_H
#define PDAE_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* pdae_stream_t; /* cudaStream_t */

#define PDAE_OK 0
#define PDAE_EINVAL (-1)  /* bad argument / unsupported shape */
#define PDAE_ECUDA (-2)   /* CUDA runtime / launch error      */
#define PDAE_ENODEV (-3)  /* no sm_90 device                  */

#define PDAE_F32 0
#define PDAE_BF16 1

#define PDAE_RESAMPLE_NONE 0
#define PDAE_RESAMPLE_UP2 1   /* nearest x2   (model/module.py:162-172) */
#define PDAE_RESAMPLE_DOWN2 2 /* avgpool 2x2  (model/module.py:200-202) */

const char* pdae_last_error(void);
int pdae_abi_version(void);
/* 0 if the current device is sm_90 (H100), PDAE_ENODEV otherwise. */
int pdae_device_check(void);

/* ---- implicit-GEMM convolution / linear, fp32 CUDA-core math ("parity mode") -------------------
 * out[b,oy,ox,n] = bias[n] + residual[b,oy,ox,n] + sum_{ky,kx,c} w[ky*k+kx][c][n] * f(in[b, oy*s-p+ky, ox*s-p+kx, c])
 * f = SiLU if a_silu else identity.  Replaces nn.Conv2d / nn.Conv1d(k=1) / nn.Linear (H=W=1,k=1)
 * at model/module.py:241-243,255-266,268-276,410,420; unet.py:51-55; shift_unet.py:52-63;
 * encoder/ffhq.py:12-35; mlp_skip_net.py:96,99.
 * w_packed: fp32 [k*k][Cin][Cout].  in_nchw / out_nchw select NCHW addressing for that tensor
 * (fp32 only).  residual (optional) is fp32 NHWC shaped like out.                                   */
int pdae_conv2d_simt(const void* in, int in_dtype, int in_nchw, const float* w_packed, const float* bias,
                     const float* residual, float* out, int out_nchw, int B, int H, int W, int Cin, int Cout,
                     int ksize, int stride, int pad, int a_silu, pdae_stream_t stream);

/* 3x3 pad-1 stride-1 conv with Cout <= 4 (the UNet `out` / `shift_out` heads, unet.py:171-175,
 * shift_unet.py:239-249): bandwidth kernel, NHWC in (fp32|bf16), NCHW fp32 out.
 * w_packed4: fp32 [9][Cin][4] (zero-padded over Cout).                                              */
int pdae_conv3x3_smalln(const void* in, int in_dtype, const float* w_packed4, const float* bias, float* out_nchw,
                        int B, int H, int W, int Cin, int Cout, pdae_stream_t stream);

/* ---- GroupNorm(32, C) split into stats -> per-(b,c) affine coefficients -> apply ------------------
 * Replaces F.group_norm + SiLU + AdaGN modulation + F.interpolate / AvgPool2d + torch.cat
 * (model/module.py:56-63,278-297,361-384,162-172,200-202; unet.py:199-200; shift_unet.py:276-281). */

/* sums[b][g] = (sum x, sum x^2) in fp64 over the virtual channel-concat [src1 (C1) | src2 (C2)].
 * src2 may be NULL (C2 = 0).  C1, C2 multiples of 4; (C1+C2) % 32 == 0.                              */
int pdae_gn_stats(const float* src1, int C1, const float* src2, int C2, int B, int HW, double* sums,
                  pdae_stream_t stream);

/* ab[b][0][c] = a, ab[b][1][c] = b with  y = a*x + b  ==  (1+zs)*((x-mu)*rstd*gamma+beta)*(1+s)+sh)+zsh.
 * emb / embz (optional) are rows of 2C floats (scale | shift) with leading dimension *_ld.            */
int pdae_gn_coef(const double* sums, const float* gamma, const float* beta, int B, int C, int HW, float eps,
                 const float* emb, int emb_ld, const float* embz, int embz_ld, float* ab, pdae_stream_t stream);

/* out_act = resample( f(a*x+b) ) over the virtual concat; f = SiLU if silu.  ab == NULL -> a=1,b=0.
 * out_raw (optional) = resample(x) (the un-normalised input, for the skip path).  H, W are the SOURCE
 * dims; outputs are [B][H'][W'][C1+C2] with H' = 2H (UP2), H/2 (DOWN2) or H.                          */
int pdae_gn_apply(const void* src1, int src1_dtype, int C1, const void* src2, int src2_dtype, int C2, const float* ab,
                  int silu, int resample, int B, int H, int W, void* out_act, int act_dtype, void* out_raw, int raw_dtype,
                  pdae_stream_t stream);

/* "bf16x3" precision (fp32-grade results from bf16 tensor-core MMAs): like pdae_gn_apply with fp32 sources, but the
 * activation is written as three bf16 channel blocks [hi | lo | hi] per pixel (out_act3: [B][Ho][Wo][3*(C1+C2)],
 * hi = bf16(a), lo = bf16(a - hi)); a conv whose weights are packed [W_hi | W_hi | W_lo] along Cin then yields
 * a_hi*W_hi + a_lo*W_hi + a_hi*W_lo.  out_raw (optional): fp32 plain [..][C] or bf16 split [..][3C] per raw_dtype.        */
int pdae_gn_apply_split3(const float* src1, int C1, const float* src2, int C2, const float* ab, int silu, int resample, int B,
                         int H, int W, void* out_act3_bf16, void* out_raw, int raw_dtype, pdae_stream_t stream);
/* Per-channel variant of the statistics (what the tensor-core conv epilogue accumulates): chs[b][c] = (sum, sum^2)
 * in fp32.  pdae_ch_stats fills it for a tensor that no conv epilogue produced; pdae_gn_coef_ch forms the 32 group
 * statistics over the virtual concat [chs1 | chs2] (groups may straddle the seam) and folds the affine / AdaGN terms. */
int pdae_zero(void* ptr, int64_t bytes, pdae_stream_t stream);
int pdae_ch_stats(const float* src, int B, int HW, int C, float* chs, pdae_stream_t stream);
int pdae_gn_coef_ch(const float* chs1, int C1, const float* chs2, int C2, const float* gamma, const float* beta, int B,
                    int HW, float eps, const float* emb, int emb_ld, const float* embz, int embz_ld, float* ab,
                    pdae_stream_t stream);
/* Deterministic forms (torch.use_deterministic_algorithms): bitwise-identical results for identical inputs, no float atomics.
 * Each CTA writes its per-channel partials to its own slot of the caller-owned workspace (no initialisation needed) and the
 * slots are summed in a fixed order; an image's CTAs follow HW only, so its results do not depend on B or on its place in the
 * batch.  workspace: pdae_stats_det_workspace_bytes(B, HW, C) = B x that of one image, with C = C1 + C2 for pdae_gn_stats_det
 * (a negative size: bad arguments).  Same outputs and shapes as pdae_ch_stats /
 * pdae_gn_stats (C <= 6144).                                                                                                */
int64_t pdae_stats_det_workspace_bytes(int B, int HW, int C);
int pdae_ch_stats_det(const float* src, int B, int HW, int C, float* chs, float* workspace, int64_t workspace_bytes,
                      pdae_stream_t stream);
int pdae_gn_stats_det(const float* src1, int C1, const float* src2, int C2, int B, int HW, double* sums, float* workspace,
                      int64_t workspace_bytes, pdae_stream_t stream);

/* ---- attention (model/module.py:422-488) ---------------------------------------------------------
 * qkv: fp32 [B][T][3C] token-major.  legacy != 0: per-head channel blocks [q|k|v] (QKVAttentionLegacy);
 * else [all q | all k | all v] (QKVAttention).  out: fp32 [B][T][C], head h at channels h*ch.
 * scratch: fp32 [B*heads][T][T].                                                                     */
int pdae_attention_simt(const float* qkv, float* out, float* scratch, int B, int T, int C, int heads, int legacy,
                        pdae_stream_t stream);

/* ---- embeddings -------------------------------------------------------------------------------- */
/* model/module.py:66-84: out[b] = [cos(t*f) | sin(t*f) | 0 if dim odd]; freqs = device fp32 [dim/2],
 * f_i = exp(-ln(1e4) i/half) evaluated by the caller with the reference's fp32 op order.             */
int pdae_timestep_embedding(const int64_t* t, int B, int dim, const float* freqs, float* out, pdae_stream_t stream);
/* unet.py:190-192: emb[b] += table[idx[b]].                                                          */
int pdae_embedding_add(float* emb, const float* table, const int64_t* idx, int B, int E, pdae_stream_t stream);

/* ---- per-step diffusion arithmetic -------------------------------------------------------------- */
/* ddim.py:43-55,66-79,91-107,123-138.  Tables are the fp32 DDIM tables indexed by t[b]:
 * e = eps - s1m[t]*grad (if grad); x0 = clamp(A[t]*x - Bm[t]*e, -1, 1); e' = (A[t]*x - x0)/Bm[t];
 * out = x0*sqrt(ab[t]) + sqrt(1-ab[t])*e'  with ab = alphas_cumprod_prev (sample) or _next (encode).  */
int pdae_ddim_step(const float* x, const float* eps, const float* grad, const int64_t* t, const float* tab_A,
                   const float* tab_Bm, const float* tab_s1m, const float* tab_ab, float* out, int B,
                   int64_t per_sample, pdae_stream_t stream);
/* Loop bookkeeping of the DDIM loops (ddim.py:57-64,81-88,110-120,140-147: `for i in ...: t = full(i)` + t_transform,
 * ddim.py:39-41) on the device, so a whole step (select -> network -> update) is one CUDA-graph replay:
 * i = *counter; t_loc[b] = i; t_net[b] = timestep_map[i]; *counter = i + delta.                         */
int pdae_ddim_select_t(int64_t* counter, int delta, const int64_t* timestep_map, int map_len, int64_t* t_loc,
                       int64_t* t_net, int B, pdae_stream_t stream);
/* gaussian_diffusion.py:98-103: out = c1[t]*x0 + c2[t]*noise.                                         */
int pdae_q_sample(const float* x0, const float* noise, const int64_t* t, const float* tab_c1, const float* tab_c2,
                  float* out, int B, int64_t per_sample, pdae_stream_t stream);
/* gaussian_diffusion.py:112-126,148-154: DDPM ancestral step with caller-provided N(0,1) noise.
 * learned_range optional (then tab_logbeta is log(betas)).                                           */
int pdae_noise_p_sample(const float* x, const float* eps, const float* noise, const float* learned_range,
                        const int64_t* t, const float* tab_cx, const float* tab_ce, const float* tab_logvar,
                        const float* tab_logbeta, float* out, int B, int64_t per_sample, pdae_stream_t stream);
/* pdae_noise_p_sample on a network's raw outputs (gaussian_diffusion.py:216-229, :257-270): eps and learned_range are read
 * at per-sample stride eps_ld (>= per_sample; 2*per_sample with learned_range = eps + per_sample: the two halves of a
 * learned-sigma output); with grad (optional, then tab_shift = shift_coef) the epsilon is eps + shift[t]*grad, one rounding
 * after the product and one after the sum.  out may alias x.                                          */
int pdae_noise_p_sample_shift(const float* x, const float* eps, const float* grad, const float* tab_shift, const float* noise,
                              const float* learned_range, int64_t eps_ld, const int64_t* t, const float* tab_cx,
                              const float* tab_ce, const float* tab_logvar, const float* tab_logbeta, float* out, int B,
                              int64_t per_sample, pdae_stream_t stream);
/* ddim.py:168 trajectory-interpolation gradient: out = ab[0]*g1 + ab[1]*g2 (fp32, one rounding per product and sum), with
 * ab = { fp32(1 - alpha), fp32(alpha) } in DEVICE memory.  out may alias g1 or g2.                      */
int pdae_grad_blend(const float* g1, const float* g2, const float* ab, float* out, int64_t n, pdae_stream_t stream);
/* gaussian_diffusion.py:292-318 gap measure, one timestep: per element (fp32, one rounding per product and sum, tables indexed
 * by t[b]) true = c0*x0 + c1*x_t; m1 = c0*(A*x_t - Bm*eps) + c1*x_t; m2 = the same with eps + shift*grad; then
 * out[2*t[0]] = mean((true - m1)^2), out[2*t[0] + 1] = mean((true - m2)^2) over all B*per_sample elements (the loop's t is
 * shared by the batch, so t[0] picks the row on the device).  Tables: x_0_posterior_mean_x_0_coef, _x_t_coef,
 * sqrt_recip_alphas_cumprod, _m1, shift_coef.  Deterministic: fp64 block partials over a grid fixed by the element count, summed
 * in a fixed order, no atomics.  workspace: caller-owned device memory of pdae_gap_terms_workspace_bytes(B*per_sample) bytes
 * (a negative result: total <= 0).                                                                                    */
int64_t pdae_gap_terms_workspace_bytes(int64_t total);
int pdae_gap_terms(const float* x0, const float* x_t, const float* eps, const float* grad, const int64_t* t, const float* tab_c0,
                   const float* tab_c1, const float* tab_A, const float* tab_Bm, const float* tab_shift, double* workspace,
                   int64_t workspace_bytes, float* out, int B, int64_t per_sample, pdae_stream_t stream);

/* ---- latent MLP row op (mlp_skip_net.py:123-141) -------------------------------------------------
 * y = act( LN( h * (1 + cond) ) ) per row; cond/ln_w optional; act = SiLU if silu.  out has row stride
 * out_ld (so it can land inside the [h | x] concat buffer of the next layer).                         */
int pdae_mlp_mod_ln_act(const float* h, const float* cond, const float* ln_w, const float* ln_b, float eps,
                        int silu, float* out, int out_ld, int B, int N, pdae_stream_t stream);
/* dst[b][col0 + j] = src[b][j], j < N (row strides dst_ld / N).                                       */
int pdae_copy_cols(const float* src, float* dst, int dst_ld, int col0, int B, int N, pdae_stream_t stream);
/* bf16 operands of the autocast latent training step.  pdae_mlp_mod_ln_act_bf16: cond row b at cond + b * cond_ld; with a
 * mask the value is then multiplied by mask[b][j] * mask_scale; out (bf16) = bf16_rn of exactly what pdae_mlp_mod_ln_act
 * followed by pdae_mul_mask_cols writes in fp32.  pdae_copy_cols_bf16: pdae_copy_cols into a bf16 dst.                  */
int pdae_mlp_mod_ln_act_bf16(const float* h, const float* cond, int cond_ld, const float* ln_w, const float* ln_b, float eps,
                             int silu, const float* mask, float mask_scale, void* out_bf16, int out_ld, int B, int N,
                             pdae_stream_t stream);
int pdae_copy_cols_bf16(const float* src, void* dst_bf16, int dst_ld, int col0, int B, int N, pdae_stream_t stream);
/* split operands of the latent MLP's sampling forward in the tensor-core modes.  out / dst: bf16 [B][3 * ld], the column
 * blocks [hi | lo | hi] of a split-operand concat buffer (hi = bf16_rn(v), lo = bf16_rn(v - hi), as pdae_gn_apply_split3
 * rounds them); columns col0 .. col0 + N - 1 of each block are written (col0 + N <= ld).
 * pdae_mlp_mod_ln_act_split3: v = exactly what pdae_mlp_mod_ln_act computes in fp32, cond row b at cond + b * cond_ld;
 * cond_ld = 0 reads one cond row for every row (a batch that shares its timestep).
 * pdae_copy_cols_split3: v = src[b][j] (src row stride N).                                                            */
int pdae_mlp_mod_ln_act_split3(const float* h, const float* cond, int cond_ld, const float* ln_w, const float* ln_b, float eps,
                               int silu, void* out_split3, int ld, int col0, int B, int N, pdae_stream_t stream);
int pdae_copy_cols_split3(const float* src, void* dst_split3, int ld, int col0, int B, int N, pdae_stream_t stream);


/* ---- backward (training config: autograd through module.py:278-297,361-384,422-428 and the encoders), fp32 ---------
 * dgrad: dx[B,H,W,Cin] (+)= conv^T(dy[B,Ho,Wo,Cout]); w_tco fp32 [k*k][Cout][Cin].
 * wgrad: dw_tcico[k*k][Cin][Cout] += sum_pixels f(x) * dy  (caller zeroes; f = SiLU if a_silu).  colsum: out[n] += sum_m dy. */
int pdae_conv2d_dgrad_simt(const float* dy, const float* w_tco, float* dx, int B, int H, int W, int Cin, int Cout, int ksize,
                           int stride, int pad, int accumulate, pdae_stream_t stream);
int pdae_conv2d_wgrad_simt(const float* x, int in_nchw, int a_silu, const float* dy, float* dw_tcico, int B, int H, int W,
                           int Cin, int Cout, int ksize, int stride, int pad, pdae_stream_t stream);
int pdae_colsum(const float* dy, int64_t M, int N, float* out, pdae_stream_t stream);
/* GroupNorm(+AdaGN)+SiLU(+resample) backward in three passes (forward: y = R(f(a*x+b)), see pdae_gn_apply):
 *  sums : S[b][c] = (sum du, sum du*x), du = f'(u) * R^T(dy)           (dy has the RESAMPLED spatial size, C channels)
 *  coef : kk[b][3][C] with dx = k0*du + k1*x + k2; accumulates dgamma/dbeta; writes the (scale|shift) grads of emb/embz
 *  apply: dx1[B,H,W,C1] (and, if dx2 != NULL, dx2[B,H,W,C2] for the skip source) = k0*du + k1*x + k2 (+ R^T(add)).         */
int pdae_gn_bwd_sums(const float* src1, int C1, const float* src2, int C2, const float* ab, const float* dy, int silu,
                     int resample, int B, int H, int W, float* S, pdae_stream_t stream);
int pdae_gn_bwd_coef(const float* S, const double* sums, const float* gamma, const float* beta, const float* emb, int emb_ld,
                     const float* embz, int embz_ld, int B, int C, int HW, float eps, float* kk, float* dgamma, float* dbeta,
                     float* demb, int demb_ld, float* dembz, int dembz_ld, pdae_stream_t stream);
int pdae_gn_bwd_apply(const float* src1, int C1, const float* src2, int C2, const float* ab, const float* kk, const float* dy,
                      int silu, int resample, int B, int H, int W, const float* add, int add_ld, float* dx1, float* dx2,
                      pdae_stream_t stream);
int pdae_embedding_bwd(const float* d_emb, const int64_t* idx, float* dw, int B, int E, pdae_stream_t stream);
int pdae_softmax_bwd(const float* P, float* dP, int64_t rows, int cols, float alpha, pdae_stream_t stream);
int pdae_dsilu_mul(const float* g, const float* x, float* out, int64_t n, pdae_stream_t stream);
int pdae_add_inplace(float* a, const float* b, int64_t n, pdae_stream_t stream);
/* inverted dropout (nn.Dropout in out_layers, module.py:259): a *= mask * scale with a caller-drawn 0/1 mask.            */
int pdae_mul_mask(float* a, const float* mask, float scale, int64_t n, pdae_stream_t stream);
/* Deterministic forms of the backward (torch.use_deterministic_algorithms in training): no float atomics; every partial result
 * is stored in its own slot of the caller-owned workspace (no initialisation needed; *_workspace_bytes bytes, 0 = none needed,
 * negative = bad arguments) and the slots are summed in a fixed order.  Split and chunk counts follow the shapes only.  The
 * outputs are WRITTEN, not added to: dw, out, S, dgamma / dbeta and the embedding gradient need no zeroing.
 *  wgrad_simt_det: pixel chunk z -> slot z of [chunks][k*k*Cin][Cout], summed in chunk order (one chunk: straight into dw).
 *  dgrad_simt_det: as pdae_conv2d_dgrad_simt; the wide-Linear split-K form (H = W = 1, Cout >= 1024) slots [Cout/64][B][Cin].
 *  colsum_det:     row chunk -> slot of [chunks][N].
 *  gn_bwd_sums_det: per-CTA (sum du, sum du*x) slots [B][P][C][2] reduced in P order into S [B][C][2] (same layout).
 *  gn_bwd_coef_det: group sums added in channel order; dgamma / dbeta through per-image slots [2][B][C] summed over b in order
 *                   (workspace only when dgamma or dbeta is given; C % 32 == 0, C <= 2048).
 *  embedding_bwd_det: dw[rows][E] = for every row r, the sum over b (in order) of d_emb[b] with idx[b] == r.                  */
int64_t pdae_conv2d_wgrad_simt_det_workspace_bytes(int B, int H, int W, int Cin, int Cout, int ksize, int stride, int pad);
int pdae_conv2d_wgrad_simt_det(const float* x, int in_nchw, int a_silu, const float* dy, float* dw_tcico, int B, int H, int W,
                               int Cin, int Cout, int ksize, int stride, int pad, float* workspace, int64_t workspace_bytes,
                               pdae_stream_t stream);
int64_t pdae_conv2d_dgrad_simt_det_workspace_bytes(int B, int H, int W, int Cin, int Cout, int ksize, int stride, int pad,
                                                   int accumulate);
int pdae_conv2d_dgrad_simt_det(const float* dy, const float* w_tco, float* dx, int B, int H, int W, int Cin, int Cout, int ksize,
                               int stride, int pad, int accumulate, float* workspace, int64_t workspace_bytes, pdae_stream_t stream);
int64_t pdae_colsum_det_workspace_bytes(int64_t M, int N);
int pdae_colsum_det(const float* dy, int64_t M, int N, float* out, float* workspace, int64_t workspace_bytes, pdae_stream_t stream);
int64_t pdae_gn_bwd_sums_det_workspace_bytes(int B, int H, int W, int C);
int pdae_gn_bwd_sums_det(const float* src1, int C1, const float* src2, int C2, const float* ab, const float* dy, int silu,
                         int resample, int B, int H, int W, float* S, float* workspace, int64_t workspace_bytes,
                         pdae_stream_t stream);
int64_t pdae_gn_bwd_coef_det_workspace_bytes(int B, int C);
int pdae_gn_bwd_coef_det(const float* S, const double* sums, const float* gamma, const float* beta, const float* emb, int emb_ld,
                         const float* embz, int embz_ld, int B, int C, int HW, float eps, float* kk, float* dgamma, float* dbeta,
                         float* demb, int demb_ld, float* dembz, int dembz_ld, float* workspace, int64_t workspace_bytes,
                         pdae_stream_t stream);
int pdae_embedding_bwd_det(const float* d_emb, const int64_t* idx, float* dw, int B, int E, int rows, pdae_stream_t stream);
/* MLPLNAct backward (model/mlp_skip_net.py:123-141; latent DPM training, gaussian_diffusion.py:373-398): given
 * dy = grad of y = SiLU(LN(h*(1+cond))) (read with leading dimension dy_ld) -> dh, dcond [B][N] and the LayerNorm
 * parameter gradients accumulated into d_ln_w / d_ln_b (zero them first).  ln_w == NULL: no LayerNorm.                  */
int pdae_mlp_mod_ln_act_bwd(const float* h, const float* cond, const float* ln_w, const float* ln_b, float eps, int silu,
                            const float* dy, int dy_ld, float* dh, float* dcond, float* d_ln_w, float* d_ln_b, int B, int N,
                            pdae_stream_t stream);
/* The same for the autocast step: cond and dcond rows at leading dimension cond_ld (a layer's column block of the bank),
 * dy multiplied by mask[b][j] * mask_scale as it is read (mask may be NULL), and dh / dcond written in fp32 and, in the
 * same pass, as their bf16 roundings (dh_bf16 [B][N], dcond_bf16 with leading dimension cond_ld).  The fp32 outputs equal
 * pdae_mul_mask_cols + pdae_mlp_mod_ln_act_bwd's bit for bit.                                                        */
int pdae_mlp_mod_ln_act_bwd_bf16(const float* h, const float* cond, int cond_ld, const float* ln_w, const float* ln_b, float eps,
                                 int silu, const float* dy, int dy_ld, const float* mask, float mask_scale, float* dh,
                                 void* dh_bf16, float* dcond, void* dcond_bf16, float* d_ln_w, float* d_ln_b, int B, int N,
                                 pdae_stream_t stream);
/* a[b][0..N) *= mask[b][0..N) * scale on a row-major [B][ld] matrix (dropout, mlp_skip_net.py:140, on the concat buffer). */
int pdae_mul_mask_cols(float* a, int ld, const float* mask, float scale, int B, int N, pdae_stream_t stream);
int pdae_nchw_to_nhwc(const float* src, float* dst, int B, int C, int HW, pdae_stream_t stream);
int pdae_gemm_batched_simt(const float* A, int64_t lda, int64_t a_bs, int64_t a_hs, int transA, const float* Bm, int64_t ldb,
                           int64_t b_bs, int64_t b_hs, int transB, float* C, int64_t ldc, int64_t c_bs, int64_t c_hs, int M,
                           int N, int K, int batch, int heads, float alpha, pdae_stream_t stream);

/* v3: the fused ResBlock convolution (model/module.py:278-297, 361-384).  out = conv3x3(SiLU(a*cat(src1, src2) + b)) + bias
 * [+ residual] [+ cat(skp1, skp2) * w_skip^T]: the GroupNorm / AdaGN / z-modulation coefficients (a, b) ([B][2][C1+C2] fp32
 * from pdae_gn_coef_ch) and the SiLU are applied while the tensor-core operand is built (one swizzled 18 x 10-pixel halo tile
 * per 64-channel block, all nine taps address it through row-shifted UMMA descriptors), so the activated tensor is never
 * written to HBM; the concatenated skip input (unet.py:199) is never materialised either.  src_dtype PDAE_BF16: bf16 NHWC
 * sources, weights bf16 [9][Cout][Cin] (w_skip [Cout][S1+S2]).  src_dtype PDAE_F32 = split-operand mode: fp32 NHWC sources
 * are split hi/lo in the prologue, weights are (hi, lo) pairs [9][2][Cout][Cin] (w_skip [2][Cout][S1+S2]) and every
 * product is a_hi*W_hi + a_lo*W_hi + a_hi*W_lo (fp32-grade).  H % 16 == 0, W % 8 == 0, every channel count % 64 == 0
 * (pdae_conv_tc3_supported).  Residual / ch_stats / out_dtype as for pdae_conv_tc2_create; the fused skip conv's bias must
 * be folded into `bias`. */
typedef struct pdae_conv_tc3_plan pdae_conv_tc3_plan;
int pdae_conv_tc3_supported(int H, int W, int Cin, int Cout);
int pdae_conv_tc3_create(pdae_conv_tc3_plan** plan, const void* src1, int C1, const void* src2, int C2, int src_dtype,
                         const float* ab, int silu, const void* w, const float* bias, const void* skp1, int S1,
                         const void* skp2, int S2, const void* w_skip, const void* residual, void* out, int out_dtype,
                         float* ch_stats, int B, int H, int W, int Cout, int bn_override);
int pdae_conv_tc3_run(const pdae_conv_tc3_plan* plan, pdae_stream_t stream);
/* Deterministic statistics: the DET kernel stores each 16 x 8 tile's per-channel sums in the tile's own slot and the run sums
 * an image's slots in order into ch_stats.  Call once, after create and before the first run; workspace: caller-owned,
 * pdae_conv_tc3_det_workspace_bytes(plan) bytes (0: one tile per image or no statistics; the slots are then ch_stats itself).  */
int64_t pdae_conv_tc3_det_workspace_bytes(const pdae_conv_tc3_plan* plan);
int pdae_conv_tc3_set_deterministic(pdae_conv_tc3_plan* plan, float* workspace, int64_t workspace_bytes);
void pdae_conv_tc3_destroy(pdae_conv_tc3_plan* plan);

/* Weight gradient of a stride-1 3x3 / 1x1 "same" convolution on the tensor cores (what autograd computes for conv weights
 * under trainer/train_representation_learning.py:112 loss.backward(); convs of model/module.py:241-259, 278-297):
 * dw[tap][cin][cout] += sum_{b,y,x} act[b, y+dy, x+dx, cin] * dy[b, y, x, cout].  act3 / dy3: bf16 NHWC with 3*C channels,
 * split-operand blocks [hi | lo | hi] (pdae_gn_apply_split3); every product is a_hi*d_hi + a_lo*d_hi + a_hi*d_lo with fp32
 * accumulation in registers (fp32-grade).  dw must be zeroed by the caller (split-K partial sums are added with fp32 reductions).
 * Shapes: Cin % 64 == 0, Cout % 64 == 0, images tileable by 64-pixel TMA boxes (pdae_wgrad_tc_supported). */
typedef struct pdae_wgrad_tc_plan pdae_wgrad_tc_plan;
int pdae_wgrad_tc_supported(int H, int W, int Cin, int Cout, int ksize);
int pdae_wgrad_tc_create(pdae_wgrad_tc_plan** plan, const void* act3_bf16, const void* dy3_bf16, float* dw, int B, int H, int W,
                         int Cin, int Cout, int ksize);
/* Single-pass variant (bf16 autocast training): act / dy are plain bf16 NHWC tensors with Cin / Cout channels and every product
 * is one bf16 MMA with fp32 accumulation.  Same shapes, zeroing contract and run / destroy functions as above. */
int pdae_wgrad_tc_create_bf16(pdae_wgrad_tc_plan** plan, const void* act_bf16, const void* dy_bf16, float* dw, int B, int H, int W,
                              int Cin, int Cout, int ksize);
/* Weight gradient of a 3x3, stride-2, pad-1 conv on plain bf16 operands (the semantic encoder under autocast):
 * dw[3 ky + kx][cin][cout] += sum_{b,oy,ox} act[b, 2 oy + ky - 1, 2 ox + kx - 1, cin] * dy[b, oy, ox, cout].  act: [B][H][W][Cin],
 * dy: [B][H/2][W/2][Cout], H and W even, channels as pdae_conv_s2_tc_supported.  Same zeroing contract and run / destroy. */
int pdae_wgrad_tc_create_bf16_s2(pdae_wgrad_tc_plan** plan, const void* act_bf16, const void* dy_bf16, float* dw, int B, int H,
                                 int W, int Cin, int Cout);
/* Deterministic plans: switch any wgrad_tc plan to its DET kernel (no float atomics).  Work unit = (output tile group, pixel
 * split); each split stores its partial dw into its own slot [splits][k*k][Cin][Cout] of the caller-owned workspace and the run
 * adds the slots in split order into dw, which then needs no zeroing.  The split count follows the shape only (about one wave
 * of units on a 132-SM H100); with one split (workspace 0) the kernel stores straight into dw.  Call once, after create and
 * before the first run; workspace: pdae_wgrad_tc_det_workspace_bytes(plan) bytes.                                          */
int64_t pdae_wgrad_tc_det_workspace_bytes(const pdae_wgrad_tc_plan* plan);
int pdae_wgrad_tc_set_deterministic(pdae_wgrad_tc_plan* plan, float* workspace, int64_t workspace_bytes);
int pdae_wgrad_tc_run(const pdae_wgrad_tc_plan* plan, pdae_stream_t stream);
void pdae_wgrad_tc_destroy(pdae_wgrad_tc_plan* plan);

/* ---- tensor-core convolution: TMA -> wgmma (bf16 x bf16 -> fp32 in registers) ---------------------
 * Same contract as pdae_conv2d_simt for ksize in {1,3}, stride 1, pad ksize/2, Cin % 64 == 0,
 * Cout % 64 == 0, bf16 NHWC input (already normalised/activated by pdae_gn_apply), weights bf16
 * [k*k][Cout][Cin].  A plan owns the TMA descriptors for fixed buffers; run it any number of times.
 * Persistent CTAs, two consumer warpgroups with register accumulators (the producer runs ahead into the next tile), TMA-store
 * epilogue.  out_dtype PDAE_F32|PDAE_BF16; ch_stats (optional) fp32 [B][Cout][2] accumulates per-channel (sum, sum^2)
 * of the stored values (zero it first); a residual is read in the OUTPUT's dtype.  cout_valid > 0 selects the image-head variant:
 * Cout must be 16 (weights zero-padded), `out` is NCHW fp32 [B][cout_valid][H][W].  bn_override: 0 = auto.              */
typedef struct pdae_conv_tc2_plan pdae_conv_tc2_plan;
int pdae_conv_tc2_create(pdae_conv_tc2_plan** plan, const void* in_bf16, const void* w_bf16, const float* bias,
                         const void* residual, void* out, int out_dtype, float* ch_stats, int B, int H, int W, int Cin,
                         int Cout, int ksize, int cout_valid, int bn_override);
/* Same, with the ResBlock's 1x1 skip conv (model/module.py:268-276,297) folded in as extra K blocks:
 * out = conv(in, w) + in2[B,H,W,Cin2] * w2[Cout][Cin2]^T + bias   (bias = conv bias + skip bias, combined by the caller). */
int pdae_conv_tc2_create_skip(pdae_conv_tc2_plan** plan, const void* in_bf16, const void* w_bf16, const float* bias,
                              const void* in2_bf16, const void* w2_bf16, int Cin2, void* out, int out_dtype, float* ch_stats,
                              int B, int H, int W, int Cin, int Cout, int ksize, int bn_override);
/* Same, the skip conv's input being cat([in2a (Cin2a ch), in2b (Cin2b ch)], channel) of two NHWC bf16 tensors, never
 * materialised (unet.py:199 `torch.cat([h, hs.pop()], dim=1)` feeding module.py:297); Cin2a, Cin2b multiples of 64.     */
int pdae_conv_tc2_create_skip2(pdae_conv_tc2_plan** plan, const void* in_bf16, const void* w_bf16, const float* bias,
                               const void* in2a_bf16, int Cin2a, const void* in2b_bf16, int Cin2b, const void* w2_bf16,
                               void* out, int out_dtype, float* ch_stats, int B, int H, int W, int Cin, int Cout, int ksize,
                               int bn_override);
/* Batched GEMM on the same kernel (tensor-core attention, model/module.py:452-456,483-487): for each batch item
 * out[M x N] = A[M x K] * Bm[N x K]^T, both operands bf16 K-major; *_ld = elements between rows, *_bs = between items.
 * M % 128 == 0, N % 64 == 0, K % 64 == 0.                                                                             */
int pdae_gemm_tc2_create(pdae_conv_tc2_plan** plan, const void* a_bf16, long long a_ld, long long a_bs, const void* b_bf16,
                         long long b_ld, long long b_bs, void* out, int out_dtype, long long out_ld, long long out_bs,
                         int batch, int M, int N, int K);
/* P_i = softmax_rows(alpha * A_i * Bm_i^T) stored as bf16 (ld / batch strides as above): attention probabilities with the
 * softmax (module.py:455, :486) folded into the GEMM epilogue -- the fp32 scores never leave the registers.  N in {64,128,256}.     */
int pdae_gemm_tc2_softmax_create(pdae_conv_tc2_plan** plan, const void* a_bf16, long long a_ld, long long a_bs,
                                 const void* b_bf16, long long b_ld, long long b_bs, void* out_bf16, long long out_ld,
                                 long long out_bs, int batch, int M, int N, int K, float alpha);
/* Attention backward under autocast (bf16 operands, fp32 accumulation).  Batched GEMM with per-operand majors: out_i[M x N]
 * (fp32) = A_i * B_i^T, where a_mn / b_mn = 0 means A_i is stored [M][K] / B_i [N][K] (K-major, as above) and 1 means A_i is
 * stored [K][M] / B_i [K][N] (MN-major); *_ld = elements between consecutive stored rows, *_bs = between batch items
 * (multiples of 8).  M % 128 == 0, N % 64 == 0, K % 64 == 0.  All arguments are checked before any CUDA call.              */
int pdae_gemm_tc2_create_major(pdae_conv_tc2_plan** plan, const void* a_bf16, int a_mn, long long a_ld, long long a_bs,
                               const void* b_bf16, int b_mn, long long b_ld, long long b_bs, float* out, long long out_ld,
                               long long out_bs, int batch, int M, int N, int K);
/* Softmax gradient: dS_i = alpha * P_i * (dP_i - rowsum(P_i * dP_i)) stored as bf16, with dP_i = dO_i * V_i^T (both K-major)
 * accumulated in fp32 and consumed in the GEMM epilogue; P_i (bf16) has the output's [M][N] shape with strides p_ld / p_bs.
 * N in {64, 128, 256}, alpha > 0, other bounds as above.  Run / destroy: pdae_conv_tc2_run / pdae_conv_tc2_destroy.           */
int pdae_gemm_tc2_softmax_grad_create(pdae_conv_tc2_plan** plan, const void* do_bf16, long long a_ld, long long a_bs,
                                      const void* v_bf16, long long b_ld, long long b_bs, const void* p_bf16, long long p_ld,
                                      long long p_bs, void* ds_bf16, long long out_ld, long long out_bs, int batch, int M, int N,
                                      int K, float alpha);
/* 3x3, stride-2, pad-1 convs on plain bf16 operands with fp32 accumulation (the semantic encoder's training step under
 * autocast, model/representation_learning/encoder).  H, W: the conv's input size, both even; Cin % 64 == 0, Cout % 64 == 0
 * (pdae_conv_s2_tc_supported).  Forward: out[B][H/2][W/2][Cout] fp32 = conv(in[B][H][W][Cin] bf16, w[9][Cout][Cin] bf16)
 * + bias (optional).  Data gradient: dx[B][H][W][Cin] fp32 (every element written) from dy[B][H/2][W/2][Cout] bf16 and
 * wt[9][Cin][Cout] bf16, wt[3 ky + kx][ci][co] = w[co][ci][ky][kx] (transposed, not flipped).  Run / destroy as above.  */
int pdae_conv_s2_tc_supported(int H, int W, int Cin, int Cout);
int pdae_conv_tc2_create_s2(pdae_conv_tc2_plan** plan, const void* in_bf16, const void* w_bf16, const float* bias, float* out,
                            int B, int H, int W, int Cin, int Cout);
int pdae_conv_tc2_create_s2_dgrad(pdae_conv_tc2_plan** plan, const void* dy_bf16, const void* wt_bf16, float* dx, int B, int H,
                                  int W, int Cin, int Cout);
/* The same stride-2 forward with the stride-1 epilogue's options (the encoder's forward in the "bf16" and "bf16x3" modes):
 * out[B][H/2][W/2][Cout] in out_dtype (PDAE_F32 or PDAE_BF16) and, if ch_stats != NULL ([B][Cout][2] fp32, 8-byte aligned,
 * zero it first), the per-channel (sum, sum^2) of the stored values.  Cin is the operand's channel count: a split-operand
 * input [B][H][W][hi | lo | hi] passes 3 C with weights [9][Cout][W_hi | W_hi | W_lo] for fp32-grade products.
 * pdae_conv_tc2_create_s2 is this entry point with PDAE_F32 and no statistics.  Run / destroy as above.                 */
int pdae_conv_tc2_create_s2_ex(pdae_conv_tc2_plan** plan, const void* in_bf16, const void* w_bf16, const float* bias, void* out,
                               int out_dtype, float* ch_stats, int B, int H, int W, int Cin, int Cout);
/* Split-K Linear (bf16 autocast latent training): out[B][Cout] (fp32) += in[B][Cin] (bf16) * w[Cout][Cin]^T (bf16) + bias.
 * Each output tile's k range is split so that about one wave of (tile, k range) items covers the SMs; the partial tiles are
 * added with fp32 reductions, so `out` must be zeroed before every run.  Cin, Cout multiples of 64.                     */
int pdae_conv_tc2_create_splitk(pdae_conv_tc2_plan** plan, const void* in_bf16, const void* w_bf16, const float* bias, float* out,
                                int B, int Cin, int Cout);
int pdae_conv_tc2_run(const pdae_conv_tc2_plan* plan, pdae_stream_t stream);
/* Deterministic plans: switch a forward conv (stride 1 or 2, with or without fused skip), a plain batched GEMM or a split-K
 * Linear plan to the DET kernels (no float atomics).  Statistics as pdae_conv_tc3_set_deterministic, a slot per (image, tile)
 * also when a tile holds several images.  Split-K: each (tile, k
 * range) stores its partial tile in its own slot and the run adds the ranges in order, then the bias, into `out`, which no
 * longer needs zeroing; the number of k ranges follows Cin and Cout only.  Call once, after create and before the first run;
 * workspace: caller-owned, pdae_conv_tc2_det_workspace_bytes(plan) bytes (may be 0).  Other modes: PDAE_EINVAL.              */
int64_t pdae_conv_tc2_det_workspace_bytes(const pdae_conv_tc2_plan* plan);
int pdae_conv_tc2_set_deterministic(pdae_conv_tc2_plan* plan, float* workspace, int64_t workspace_bytes);
/* Image-head plans (cout_valid > 0): fuse the per-step sampling update into the head's epilogue, x_t updated in place.
 * fuse_desc_device: 10 x int64 in DEVICE memory, read at run time, flags = enabled | use_grad<<1 | eps_only<<2 | ddpm<<3 |
 * interp<<4 | C<<8 | C_eps<<16; flags == 0 -> plain head.
 *  DDIM (diffusion/ddim.py:43-55,66-79,91-107,123-138): { flags, eps*, x_t*, t*, tab_A*, tab_Bm*, tab_s1m*, tab_ab*, g1*, a };
 *    arithmetic identical to pdae_ddim_step.  interp (ddim.py:149-174, on the second shift head, with use_grad): the gradient is
 *    a1*g1 + a2*head with a = fp32 bits of a1 = 1 - alpha in the low and of a2 = alpha in the high 32 bits (pdae_grad_blend).
 *  ddpm (gaussian_diffusion.py:112-126): { flags, eps*, x_t*, t*, tab_cx*, tab_ce*, tab_shift*, tab_logvar*, noise*, 0 };
 *    arithmetic identical to pdae_noise_p_sample_shift (use_grad: eps + shift[t] * head) or pdae_noise_p_sample.               */
int pdae_conv_tc2_set_head_fuse(pdae_conv_tc2_plan* plan, const int64_t* fuse_desc_device);
/* P = softmax(alpha * S) per row, fp32 in -> bf16 out.  vT[b*heads+h][c][t] = V part of qkv (bf16 [B][T][3C]).        */
int pdae_softmax_bf16(const float* S, void* P_bf16, int64_t rows, int cols, float alpha, pdae_stream_t stream);
int pdae_transpose_v(const void* qkv_bf16, void* vT_bf16, int B, int T, int C, int heads, int legacy, pdae_stream_t stream);
/* Split-operand ("bf16x3") attention: re-lay the fp32 qkv rows as bf16 blocks Q3 = [q_hi|q_lo|q_hi], K3 = [k_hi|k_hi|k_lo]
 * ([B*heads][T][3*ch]) and VT3 = [vT_hi|vT_hi|vT_lo] ([B*heads][ch][3*T]) so that QK^T and PV (model/module.py:452-456,
 * 483-487) run as batched wgmma GEMMs with fp32-grade products; pdae_softmax_split3 turns the fp32 scores into
 * P3 = [p_hi|p_lo|p_hi] with p = softmax(alpha * S) evaluated in fp32.                                                  */
int pdae_qkv_split3(const float* qkv, void* Q3, void* K3, void* VT3, int B, int T, int C, int heads, int legacy,
                    pdae_stream_t stream);
int pdae_softmax_split3(const float* S, void* P3_bf16, int64_t rows, int cols, float alpha, pdae_stream_t stream);
void pdae_conv_tc2_destroy(pdae_conv_tc2_plan* plan);

/* Stem: nn.Conv2d(input_channel, base, 3, padding=1) on the NCHW fp32 image (unet.py:62-64, shift_unet.py:64-66), written
 * straight into the bf16 NHWC residual stream; ch_stats (optional, [B][Cout][2] fp32, zero it first) accumulates the
 * per-channel (sum, sum^2) of the stored values for the GroupNorms that read it.  w_packed fp32 [9][Cin][Cout].
 * Cin <= 4, Cout % 8 == 0, Cout <= 256.                                                                                */
int pdae_stem_conv_bf16(const float* x_nchw, const float* w_packed, const float* bias, void* out_bf16_nhwc, float* ch_stats,
                        int B, int H, int W, int Cin, int Cout, pdae_stream_t stream);
/* The semantic encoder's stem, nn.Conv2d(3, 64, 3, stride 2, padding 1) (model/representation_learning/encoder/ffhq.py), the
 * same way: H, W the input size (H even, W % 8 == 0), out_bf16_nhwc [B][H/2][W/2][Cout], arguments otherwise as above.  */
int pdae_stem_conv_s2_bf16(const float* x_nchw, const float* w_packed, const float* bias, void* out_bf16_nhwc, float* ch_stats,
                           int B, int H, int W, int Cin, int Cout, pdae_stream_t stream);
/* Deterministic stems (stride 1: pdae_stem_conv_bf16, stride 2: pdae_stem_conv_s2_bf16): the same output, the statistics
 * written (not added) to ch_stats through per-CTA slots summed in order.  workspace: pdae_stem_conv_det_workspace_bytes(B, H,
 * W, Cout, stride) bytes (H, W: the input size).  Needs (9 Cin + 2 + 2 (256 / (Cout / 8))) Cout floats <= 48 KiB of shared
 * memory.                                                                                                                    */
int64_t pdae_stem_conv_det_workspace_bytes(int B, int H, int W, int Cout, int stride);
int pdae_stem_conv_bf16_det(const float* x_nchw, const float* w_packed, const float* bias, void* out_bf16_nhwc, float* ch_stats,
                            int B, int H, int W, int Cin, int Cout, int stride, float* workspace, int64_t workspace_bytes,
                            pdae_stream_t stream);

/* ---- callers either side of the hot path (SURVEY.md 8(f)) -------------------------------------------------------------
 * Fused multi-tensor Adam + EMA: replaces torch.optim.Adam.step() as configured at
 * trainer/train_representation_learning.py:54-69 plus the per-parameter python EMA loop of :192-212
 * (`ema.mul_(decay).add_(p, alpha=1-decay)`, run after the optimizer step).  `table` is a DEVICE array of n tensors;
 * `block_map` a DEVICE array of n_blocks (tensor index, chunk index) int32 pairs covering every tensor in `chunk`-element
 * pieces (chunk % 4 == 0).  g is multiplied by grad_scale first (1/world_size after a sum all-reduce, or 1/loss_scale).
 * `step` is the 1-based Adam step count (bias corrections are evaluated in fp64 on the host like torch does).
 * ema_decay < 0 or ema == NULL skips the EMA update.                                                                    */
typedef struct pdae_adam_tensor {
  float* p;        /* parameter, updated in place        */
  const float* g;  /* gradient                           */
  float* m;        /* exp_avg                            */
  float* v;        /* exp_avg_sq                         */
  float* ema;      /* EMA copy of p, or NULL             */
  int64_t n;       /* elements                           */
} pdae_adam_tensor;
int pdae_adam_ema_step(const pdae_adam_tensor* table, const int32_t* block_map, int n_blocks, int chunk, float lr,
                       float beta1, float beta2, float eps, float weight_decay, int64_t step, float grad_scale,
                       float ema_decay, pdae_stream_t stream);
/* Hand the weight gradients of a backward plan to autograd in the parameters' own layouts (what loss.backward() leaves in
 * p.grad, trainer/train_representation_learning.py:112): item i copies a <= 4-D strided fp32 view (element strides; e.g. the
 * packed conv accumulator [k*k][Cin][Cout] viewed as [Cout][Cin][k*k]) to g[dst_off ...] contiguously, or adds to it (`add`,
 * a parameter that received a second contribution -- such items must be in a LATER launch than the first write).
 * `items`, `block_map` ((item, chunk) int32 pairs, `chunk` elements each) are DEVICE arrays.                              */
typedef struct pdae_unpack_item {
  const float* src;
  int64_t dst_off;
  int32_t shape[4];
  int64_t stride[4];
  int32_t add;
  int32_t pad_;
} pdae_unpack_item;
int pdae_unpack_grads(const pdae_unpack_item* items, const int32_t* block_map, int n_blocks, int chunk, float* g,
                      pdae_stream_t stream);
/* ---- launch plans (SURVEY.md 8(b): plan_create / destroy / run_step) ---------------------------------------------------
 * An ordered list of recorded calls of the entry points above, replayed from native code: what one `forward()` of a
 * reference module (model/unet.py:178-202, model/shift_unet.py:251-310) or one autograd backward pass amounts to here.
 * `pdae_plan_add(plan, "pdae_gn_apply", args, nargs, stream_slot)` records one call: `args` holds the argument values in the
 * entry point's order (pointers in .p, int / int64 in .i, float in .f), `stream_slot` is the index of its pdae_stream_t
 * argument (patched at every run) or -1.  Every entry point that returns int and takes only pointers / int / int64 / float
 * is recordable (incl. the `*_run` functions of the tensor-core kernel plans).  `pdae_plan_run_step` issues the calls in order
 * on `stream` and stops at the first failure (returns its code; pdae_last_error() describes it).  The caller owns every
 * buffer; one plan per stream (not thread-safe).                                                                          */
typedef union pdae_arg {
  void* p;
  int64_t i;
  double f;
} pdae_arg;
typedef struct pdae_plan pdae_plan;
int pdae_plan_create(pdae_plan** plan);
int pdae_plan_add(pdae_plan* plan, const char* entry, const pdae_arg* args, int nargs, int stream_slot);
int pdae_plan_run_step(pdae_plan* plan, pdae_stream_t stream);
int pdae_plan_size(const pdae_plan* plan);
const char* pdae_plan_op_name(const pdae_plan* plan, int index);
void pdae_plan_destroy(pdae_plan* plan);

/* Wire formats.  fp32 NCHW in [-1,1] -> uint8 NHWC with the reference's exact op sequence
 * `x.mul(0.5).add(0.5).mul(255).add(0.5).clamp(0,255).permute(0,2,3,1).to(uint8)`
 * (trainer/train_representation_learning.py:173-174, sampler/autoencoding_example.py:53 ...): bit-exact.
 * uint8 NHWC -> fp32 NCHW `(x/255 - 0.5)/0.5` = torchvision ToTensor + Normalize(0.5,0.5) (dataset/ffhq.py:27-31).      */
int pdae_images_to_u8_nhwc(const float* x_nchw, uint8_t* out_nhwc, int B, int C, int H, int W, pdae_stream_t stream);
int pdae_u8_nhwc_to_images(const uint8_t* in_nhwc, float* out_nchw, int B, int C, int H, int W, pdae_stream_t stream);
/* Per-image metrics over fp32 NCHW batches: calculate_mse (metric/utils.py:62-63) and calculate_ssim
 * (metric/utils.py:35-60; `window_11x11` = the fp32 11x11 Gaussian window of :25-33, device memory).
 * workspace: B doubles (device); out: B floats.                                                                        */
int pdae_mse_per_image(const float* a, const float* b, int B, int64_t per_image, double* workspace, float* out,
                       pdae_stream_t stream);
int pdae_ssim_per_image(const float* img1, const float* img2, const float* window_11x11, int B, int C, int H, int W,
                        double* workspace, float* out, pdae_stream_t stream);
/* Deterministic per-image MSE / SSIM: every block's fp64 sum in its own workspace slot, an image's slots added in order.
 * workspace: pdae_mse_det_workspace_bytes(B, per_image) / pdae_ssim_det_workspace_bytes(B, C, H, W) bytes.              */
int64_t pdae_mse_det_workspace_bytes(int B, int64_t per_image);
int pdae_mse_per_image_det(const float* a, const float* b, int B, int64_t per_image, double* workspace, int64_t workspace_bytes,
                           float* out, pdae_stream_t stream);
int64_t pdae_ssim_det_workspace_bytes(int B, int C, int H, int W);
int pdae_ssim_per_image_det(const float* img1, const float* img2, const float* window_11x11, int B, int C, int H, int W,
                            double* workspace, int64_t workspace_bytes, float* out, pdae_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* PDAE_B200_H */
