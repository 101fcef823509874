/*
 * rave_b200 -- C ABI of the H100-native (sm_90a) waveform hot path of acids-ircam/RAVE.
 *
 * The reference has no FFI: its hot path is issued through ATen library calls
 * (F.pad + F.conv1d / F.conv_transpose1d / nn.Conv2d -> cuDNN).  Each entry point below
 * replaces one of those call sites; the reference-side binding a maintainer would add is the
 * ctypes stub in rave_b200/_lib.py (see INTEGRATION.md).
 *
 * Conventions
 *   - every pointer is a DEVICE pointer borrowed for the duration of the stream-ordered call;
 *     the library owns no tensors and never synchronises the host;
 *   - tensors are dense row-major fp32 "NCL": x[b][c][t] at (b*C + c)*L + t, unless stated;
 *   - `stream` is a cudaStream_t passed as void*;
 *   - return value 0 = success, non-zero = failure, message via rave_b200_last_error();
 *   - re-entrant across streams (no global mutable state except the last-error string).
 *
 * Activation codes (the `activation(dim)` module that precedes almost every conv,
 * rave/blocks.py:56,90,528,614): 0 = none, 1 = LeakyReLU(slope), 2 = Snake(alpha[C]).
 */
#ifndef RAVE_B200_H
#define RAVE_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RAVE_ACT_NONE 0
#define RAVE_ACT_LEAKY 1
#define RAVE_ACT_SNAKE 2

/* precision modes of the tensor-core conv engine */
#define RAVE_PREC_FP32 0 /* CUDA-core fp32 FMA: parity mode (<=1e-5 rel-L2 vs the fp32 CPU oracle) */
#define RAVE_PREC_BF16 1 /* wgmma, bf16 operands, fp32 accumulate in registers */
#define RAVE_PREC_TF32 2 /* fp32 operands read as tf32 (no kernel on this path) */

int rave_b200_version(void);
const char *rave_b200_last_error(void);
/* number of kernels launched by this library since load (bench.py's gpu_launches) */
unsigned long long rave_b200_launch_count(void);

/* ---------------------------------------------------------------------------------------------
 * PQMF (replaces CachedPQMF.forward / .inverse, rave/pqmf.py:279-294, and their autograd).
 *
 * analysis:  y[b][k][n] = sgn(k,n) * sum_{j<ntaps} taps[k][j] * x[b][16 n + j - pad_l]
 *            x: [B][T], taps: [16][ntaps] (ntaps <= 528), y: [B][16][Lout];
 *            sgn = -1 for odd k and even n when flip_sign != 0 (reverse_half, pqmf.py:13-17).
 * synthesis: out[b][16 t + 15 - m] = scale * sum_{c<16} sum_{j<K} w[m][c][j] * sgn(c,tau) * x[b][c][tau],
 *            tau = t + j - pad_l;  x: [B][16][L], w: [16][16][K] (K <= 33), out: [B][16 L].
 *            (conv 16->16, *M, channel flip and channel->time interleave of pqmf.py:288-294 fused.)
 * The backward of each is the other with re-indexed taps (done by the host wrapper).
 * Only n_band == 16 (every shipped config, configs/v1.gin:15) has a device kernel.
 * ------------------------------------------------------------------------------------------- */
int rave_pqmf_analysis_fwd(const float *x, const float *taps, float *y, int B, int T, int Lout,
                           int ntaps, int pad_l, int flip_sign, void *stream);
int rave_pqmf_synthesis_fwd(const float *x, const float *w, float *out, int B, int L, int K,
                            int pad_l, float scale, int flip_sign, void *stream);
/* The same two operators for a COSINE-MODULATED bank (rave/pqmf.py:32-52 builds nothing else): every table is rank
 * one per tap residue mod 32, T[k][32 i + r] = C[k][r] * Q[r][i], so the FIR splits into a polyphase prototype
 * filter (Qt: [17][32], Qt[i][r] = Q[r][i]) and a 16 x 32 (de)modulation (analysis: Ct [32 r][16 k]; synthesis:
 * Cc [16 c][32 r]) -- 66 instead of 512 / 528 multiply-adds per sample.  Same index conventions as above with
 * taps[k][j] = Ct[j%32][k] Qt[j/32][j%32] and w[m][c][j] = Cc[c][(16j+m)%32] Qt[(16j+m)/32][(16j+m)%32].
 * Results agree with the dense form to fp32 rounding (different summation order). */
int rave_pqmf_analysis_fast(const float *x, const float *Ct, const float *Qt, float *y, int B, int T, int Lout,
                            int pad_l, int flip_sign, void *stream);
int rave_pqmf_synthesis_fast(const float *x, const float *Cc, const float *Qt, float *out, int B, int L,
                             int pad_l, float scale, int flip_sign, void *stream);

/* ---------------------------------------------------------------------------------------------
 * conv1d family, fp32 CUDA-core path (replaces cc.Conv1d.forward = F.pad + F.conv1d,
 * cached_conv [EXT] via rave/blocks.py:96-108,538-592,637-692 and nn.Conv1d/Conv2d(k,1) in
 * rave/discriminator.py:99-111, plus the autograd of those calls).
 *
 * gather ("conv forward" form; also the input-gradient of a transposed conv):
 *   out[b][m][l] = bias[m] + res[b][m][l]
 *                + sum_{c<Cs} sum_{k<K} W(m,c,k) * act(src[b][c][l*stride + k*dil - pad_l])
 *   then, if post_act != 0:  out *= act'(post_x[b][m][l])      (chain rule through a pre-activation)
 *   W(m,c,k) = w[m*ws_m + c*ws_c + k];  src: [B][Cs][Ls];  out: [B][Cm][Lo].
 *
 * scatter ("transposed" form: conv input-gradient, ConvTranspose1d forward):
 *   out[b][m][t] = bias[m] + res[b][m][t]
 *                + sum_{c<Cs} sum_{k<K} W(m,c,k) * act(src[b][c][q/stride]),  q = t + pad_l - k*dil,
 *                  terms kept only where q >= 0, q % stride == 0 and q/stride < Ls
 *   then the same optional post factor.
 *
 * act codes: see top.  `alpha` is the Snake alpha of the source channels (act == 2).
 * ------------------------------------------------------------------------------------------- */
int rave_conv1d_gather_f32(const float *src, const float *w, const float *bias, const float *res,
                           float *out, int B, int Cs, int Ls, int Cm, int Lo, int K, int stride,
                           int dil, int pad_l, long ws_m, long ws_c, int act, float slope,
                           const float *alpha, int post_act, float post_slope, const float *post_x,
                           const float *post_alpha, void *stream);
int rave_conv1d_scatter_f32(const float *src, const float *w, const float *bias, const float *res,
                            float *out, int B, int Cs, int Ls, int Cm, int Lo, int K, int stride,
                            int dil, int pad_l, long ws_m, long ws_c, int act, float slope,
                            const float *alpha, int post_act, float post_slope, const float *post_x,
                            const float *post_alpha, void *stream);

/* weight gradient:
 *   dw[a*os_a + c*os_c + k] = sum_b sum_{l<Lp} actP(P[b][a][l]) * actQ(Q[b][c][l*stride + k*dil - pad_l])
 *   P: [B][Ca][Lp] (indexed at l), Q: [B][Cc][Lq] (indexed at the shifted position).
 *   For Conv1d: P = dy, Q = x (act on Q).  For ConvTranspose1d: P = x (act on P), Q = dy.
 *   `workspace` must hold rave_conv1d_wgrad_workspace_bytes(...) bytes; the split-K partials are
 *   reduced in a fixed order (deterministic). */
size_t rave_conv1d_wgrad_workspace_bytes(int B, int Ca, int Cc, int Lp, int K);
int rave_conv1d_wgrad_f32(const float *P, const float *Q, float *dw, int B, int Ca, int Lp, int Cc,
                          int Lq, int K, int stride, int dil, int pad_l, long os_a, long os_c,
                          int act_p, int act_q, float slope, const float *alpha, void *workspace,
                          void *stream);

/* ---------------------------------------------------------------------------------------------
 * weight norm (replaces torch._weight_norm, rave/blocks.py:15-22): w = g * v / ||v||, the norm
 * over all dims but 0.  v: [C0][R], g: [C0], w: [C0][R], norm_out: [C0] (saved for backward).
 * backward: dv = (g/n) * (dw - v * <dw,v>/n^2),  dg = <dw,v>/n.
 * ------------------------------------------------------------------------------------------- */
int rave_weight_norm_fwd(const float *v, const float *g, float *w, float *norm_out, int C0, int R,
                         void *stream);
int rave_weight_norm_bwd(const float *dw, const float *v, const float *g, const float *norm,
                         float *dv, float *dg, int C0, int R, void *stream);

/* ---------------------------------------------------------------------------------------------
 * elementwise pieces that are not absorbed by a conv prologue/epilogue
 * ------------------------------------------------------------------------------------------- */
/* y = act(x); x,y: [B][C][L] */
int rave_act_fwd(const float *x, float *y, int B, int C, int L, int act, float slope,
                 const float *alpha, void *stream);
/* dx = dy * act'(x); for Snake also dalpha[c] = sum_{b,t} dy * d act/d alpha (dalpha: [C], overwritten) */
int rave_act_bwd(const float *dy, const float *x, float *dx, float *dalpha, int B, int C, int L,
                 int act, float slope, const float *alpha, void *stream);
/* GeneratorV2 tail (rave/blocks.py:704-711): y[b][c][t] = tanh(x[b][c][t] * sigmoid(x[b][C+c][t])); x: [B][2C][L] */
int rave_am_tanh_fwd(const float *x, float *y, int B, int C, int L, void *stream);
int rave_am_tanh_bwd(const float *dy, const float *x, float *dx, int B, int C, int L, void *stream);
/* VariationalEncoder.reparametrize (rave/blocks.py:725-737) in one pass: z [B][2C][L] = (mean | scale);
 * zs[b][c][t] = eps * (softplus(scale) + 1e-4) + mean;  *kl_sum += sum (mean^2 + var - log var - 1)  (zero it first) */
int rave_reparam_fwd(const float *z, const float *eps, float *zs, float *kl_sum, int B, int C, int L, void *stream);
/* WasserteinEncoder.reparametrize's regulariser (rave/blocks.py:761-774), fp32, fixed-order sums.  Rows: x_i = z[b][:][t]
 * of z [B][D][L] (i = b * L + t, read in place), y_i = prior[i][:] of prior [N][D], N = B * L <= 65536, D <= 64.
 *   fwd: means = (mean_ij k(x_i, x_j), mean_ij k(y_i, y_j), mean_ij k(x_i, y_j)), k(a, b) = exp(-|a - b|^2 / D^2);
 *        *mmd = means[0] + means[1] - 2 means[2]
 *   bwd: dz [B][D][L] = g[0] * (-4 / (D^2 N^2)) * (sum_j k(x_i, x_j) (x_i - x_j) - sum_j k(x_i, y_j) (x_i - y_j)),
 *        g = the device scalar gradient of *mmd */
int rave_mmd_fwd(const float *z, const float *prior, float *means, float *mmd, int B, int D, int L, void *stream);
int rave_mmd_bwd(const float *z, const float *prior, const float *g, float *dz, int B, int D, int L, void *stream);
/* SphericalEncoder.reparametrize (rave/blocks.py:839-842): out = z / |z|_2 over C per (b, t) of z [B][C][L], norm [B][L];
 * bwd: dz = (g - out (out . g)) / norm */
int rave_sphere_norm_fwd(const float *z, float *out, float *norm, int B, int C, int L, void *stream);
/* Validation PCA (rave/model.py:464-488): accumulates the count, mean and centred scatter matrix of the rows
 * x_(b,t) = z[b][0:D][t] of z [B][C][L] fp32 (D <= C: the posterior mean is the first half of the encoder output, read in
 * place) into state = [n | mean[D] | M2[D*D]] (fp64, updated in place; all zero to start).  Per-block moments, then
 * Chan's pairwise merge in block order.  Fixed-order sums: bit-identical across runs, no host read, graph-capturable.
 * 1 <= D <= 256; `work` holds rave_latent_moments_workspace_bytes(B, L, D) bytes. */
int  rave_latent_moments(const float *z, int B, int C, int L, int D, double *state, double *work, void *stream);
long rave_latent_moments_workspace_bytes(int B, int L, int D);
int rave_sphere_norm_bwd(const float *g, const float *out, const float *norm, float *dz, int B, int C, int L,
                         void *stream);

/* ---------------------------------------------------------------------------------------------
 * tensor-core conv engine (wgmma + TMA, register accumulators), implicit GEMM, time on the MMA M axis:
 *   D[(b,l)][co] = sum_k sum_ci A_k[(b,l)][ci] * W_k[co][ci],   A_k = row-shifted view of the input.
 * See DESIGN.md section "wgmma conv engine".  Tensors on this path are CHANNEL-LAST:
 *   xa      [B][Lin][Cin]  bf16 : the ALREADY ACTIVATED operand (written by the previous kernel's epilogue)
 *   wt      [K][Cout][Cin] bf16 : tap-major effective weights (rave_weight_to_tapmajor_bf16)
 *   res     [B][out_rows][Cout] fp32 or NULL (res_bf16: the same in bf16), bias [Cout] or NULL
 *   res_act [B][out_rows][Cout] bf16 or NULL : residual skip taken from an ACTIVATED operand tensor
 *             a = LeakyReLU_{res_slope}(h): adds h = a > 0 ? a : a / res_slope (no separate fp32 stream)
 *   dact_src[B][out_rows][Cout] bf16 or NULL : result *= LeakyReLU'(dact_src) before the residual add
 *             (backward use: the activated operand saved by the forward pass carries the sign)
 *   fm_d    2 device floats (d0, d1) or NULL  : fused feature-matching gradient (needs dact_src): the batch is
 *             [real; fake] with fm_bh rows per half; after the LeakyReLU' mask the epilogue adds, with
 *             h = LeakyReLU^-1(dact_src), d0 sgn(h_r-h_f) + d1 sgn(h_r) to real rows and -d0 sgn(h_r-h_f) to fake
 *             rows (rave/model.py:355-361 with core.mean_difference L1, rave/core.py:236-252).  fm_bh < 0: the
 *             launch covers ONLY the fake half (B = -fm_bh rows; generator step: the real half's input gradient is
 *             never used), the real partner rows lie |fm_bh| batches before dact_src in the same allocation
 *   out_f32 [B][out_rows][Cout] fp32 or NULL : pre-activation stream (residual / features)
 *   out_act [B][out_rows][Cout] bf16 or NULL : act(out), the next conv's operand
 * Output row of (b,l) is l*out_row_stride + out_row_offset (phases of a transposed conv interleave);
 * pass out_rows = 0, stride = 0, offset = 0 for a plain conv.  `in_pitch` = allocated rows per batch
 * of xa (0 = Lin); it must be >= Lin rounded up to `stride`, with rows [Lin, in_pitch) zero.
 * Requirements: Cin % 16 == 0, Cout % 16 == 0.
 * ------------------------------------------------------------------------------------------- */
int rave_conv1d_tc_supported(int Cin, int Cout, int K, int stride, int dil);
/* Fused Residual(DilatedUnit) forward (rave/blocks.py:31-45, 83-112):  out = x + Conv1x1(LeakyReLU(Conv3_dil(LeakyReLU(x))))
 * in one wgmma kernel; the intermediate operand stays in shared memory as the A operand of the second GEMM.
 *   xa      [B][pitch][C] bf16 : a = LeakyReLU_{slope_in}(x), the unit's input operand (the skip x is recovered from it)
 *   w3t     [3][C][C] bf16, w1t [1][C][C] bf16 : tap-major effective weights (rave_weight_prep_tc_multi)
 *   a1_out  [B][pitch][C] bf16 or NULL : LeakyReLU_{slope_mid}(conv3) kept for the backward (training)
 *   out_f32 / out_act [B][pitch][C] or NULL : the unit's output, fp32 and / or act_out(out) as bf16 operand
 * conv3 reads rows l + k*dil - pad_l (zero outside [0, L)).  C in {96, 192, 384} (the v2 / v3 / discrete widths below
 * the 768-channel stage, whose [128 x 768] intermediate does not fit on one SM).  Backward: the per-layer kernels. */
int rave_dilated_unit_tc_supported(int C, int L);
int rave_dilated_unit_tc_fwd(const void *xa_bf16, const void *w3t_bf16, const void *w1t_bf16, void *a1_out,
                             float *out_f32, void *out_act, int B, int C, int L, int pitch, int dil, int pad_l,
                             float slope_in, float slope_mid, int act_out, float slope_out, void *stream);
/* kernel instance rave_conv1d_tc_fwd selects for a shape (a launch that writes out_act): BLOCK_N | BLOCK_K << 12 |
 * (accumulator buffers - 1) << 24 | (bf16 output staged in shared memory, written by TMA) << 25 | ring stages << 26;
 * 0 = none (bench.py names the dominant kernel with it) */
int rave_conv1d_tc_plan(int B, int Cin, int Cout, int Lout, int K);
/* ring stages of the ping-pong kernel for an input-gradient launch of this shape (dact_src set, bf16 output only; fm:
 * with fm_d, res_bf16: with the gradient skip); 0 = the launch runs the single-warpgroup kernel */
int rave_conv1d_tc_pp_stages(int B, int Cin, int Cout, int Lout, int K, int fm, int res_bf16);
/* ring stages of the ping-pong kernel for a forward launch of this shape (bias and / or LeakyReLU, bf16 output only:
 * no res, res_bf16, res_act, dact_src or out_f32); 0 = the launch runs the single-warpgroup kernel */
int rave_conv1d_tc_pp_fwd_stages(int B, int Cin, int Cout, int Lout, int K);
int rave_conv1d_tc_fwd(const void *xa_bf16, const void *wt_bf16, const float *bias, const float *res,
                       const void *res_bf16, const void *dact_src_bf16, const void *res_act_bf16, float res_slope,
                       float *out_f32, void *out_act_bf16,
                       int B, int Cin, int Lin, int in_pitch, int Cout, int Lout,
                       int K, int stride, int dil, int pad_l, int act, float slope, int out_rows,
                       int out_row_stride, int out_row_offset, const float *fm_d, int fm_bh, void *stream);
/* Split-operand ("bf16x3") forward: the accurate fast mode (<= 1e-4 rel-L2 end to end; reference arithmetic is fp32,
 * scripts/train.py:135-136 allow TF32).  xa [B][in_pitch][2*Cin] bf16 rows [hi | lo] (x = hi + lo), wt [2][K][Cout][Cin]
 * (rave_weight_prep_tc_multi_x3); the tensor cores accumulate hi*hi + lo*hi + hi*lo in fp32.  out_act / res_act are
 * [hi | lo] rows of 2*Cout; bias / res / out_f32 as in rave_conv1d_tc_fwd.  act_cs (0 = Cout): channels per POSITION
 * when an output row holds several positions side by side (phase-fused transposed conv) -- each position is its own
 * [hi | lo] pair of 2*act_cs channels.  No gradient epilogues (forward path). */
int rave_conv1d_tc_fwd_x3(const void *xa_bf16, const void *wt_bf16, const float *bias, const float *res,
                          const void *res_act, float res_slope, float *out_f32, void *out_act, int B, int Cin, int Lin,
                          int in_pitch, int Cout, int Lout, int K, int stride, int dil, int pad_l, int act, float slope,
                          int out_rows, int out_row_stride, int out_row_offset, int act_cs, void *stream);
/* weight gradient on the same engine (split-K over row slices; each slice writes its own partial):
 *   sum_s dwt[s][k][m][n] = sum_{b,l} P[b][l][m] * Q[b][l*stride + k*dil - pad_l][n]
 * P [B][Lp][Cm] bf16 (conv: dy), Q [B][Lq][Cn] bf16 (conv: activated input);
 * dwt [splits][K][Cm][Cn] fp32 with splits = rave_conv1d_tc_wgrad_splits(...) (every element written once;
 * the slices are summed, in order, by rave_weight_norm_bwd_tapmajor / rave_tapmajor_to_weight_f32).
 * For ConvTranspose1d swap the roles (P = activated input, Q = dy).  Cm, Cn multiples of 8.
 * dbias [Cm] fp32, pre-zeroed, or NULL: += sum_{b,l} P[b][l][m] (the conv bias gradient when P = dy), reduced by the
 * tap-0 CTAs from the tiles they stream anyway (fp32 atomics across row slices). */
int rave_conv1d_tc_wgrad_splits(int B, int Cm, int Lp, int Cn, int K);
/* Operand of a (kt, kf) Conv2d evaluated as a conv along frequency (Descript MRD, rave/descript_discriminator.py:118-184):
 * x [B][C][T][F] fp32 -> out [(b,t)][Fp][Cp] bf16 with out[.][f][dt*C + c] = x[b][c][t + dt - pt][f] (zero elsewhere), and
 * the adjoint gx [B][C][T][F] += (written once) from g [(b,t)][Fp][Cp]. */
int rave_time_stack_cl(const float *x, void *out_bf16, int B, int C, int T, int F, int Fp, int Cp, int kt, int pt,
                       void *stream);
int rave_time_stack_cl_bwd(const void *g_bf16, float *gx, int B, int C, int T, int F, int Fp, int Cp, int kt, int pt,
                           void *stream);
/* The same operand from a CHANNEL-LAST source x[b][t][f][c] (element strides sb, st; f-stride C): the MRD keeps its
 * activations channel-last between layers, so no NCHW copy exists (rave/descript_discriminator.py:118-184). */
int rave_time_stack_nhwc(const float *x, void *out_bf16, int B, int C, int T, int F, long sb, long st, int Fp, int Cp, int kt,
                         int pt, void *stream);
int rave_time_stack_nhwc_bwd(const void *g_bf16, float *gx, int B, int C, int T, int F, int Fp, int Cp, int kt, int pt,
                             void *stream);
/* The same with time dilation dil (EncodecConvNet of the multi-scale spectral discriminator, rave/discriminator.py:54-74):
 * out[(b,t)][f][dt*C + c] = x[b][t + dt*dil - pt][f][c]; dil = 1 is rave_time_stack_nhwc. */
int rave_time_stack_nhwc_dil(const float *x, void *out_bf16, int B, int C, int T, int F, long sb, long st, int Fp, int Cp,
                             int kt, int pt, int dil, void *stream);
int rave_time_stack_nhwc_dil_bwd(const void *g_bf16, float *gx, int B, int C, int T, int F, int Fp, int Cp, int kt, int pt,
                                 int dil, void *stream);
/* L1 feature matching on fp32 features (core.mean_difference, rave/core.py:236-252): stats[0] += sum|t - v|,
 * stats[1] += sum|t| (stats zeroed by the caller); gradient of d[0] * stats[0] + d[1] * stats[1]: gt = d0 sgn(t - v) +
 * d1 sgn(t), gv = -d0 sgn(t - v) (either may be null). */
int rave_l1_stats_f32(const float *t, const float *v, float *stats, long n, void *stream);
int rave_l1_grad_f32(const float *t, const float *v, const float *d, float *gt, float *gv, long n, void *stream);
/* Post-activation feature tap of the Descript discriminator with its L1 feature matching (rave/descript_discriminator.py:
 * 59-61, rave/model.py:353-361): x = [real; fake] halves of H elements each (one contiguous buffer, identical zero padding).
 * fwd: a = LeakyReLU(x), stats[0] += sum|a_r - a_f|, stats[1] += sum|a_r| (stats zeroed by the caller).
 * bwd: gx_r = (g_r + d0 sgn(a_r - a_f) + d1 sgn(a_r)) leaky'(a_r), gx_f = (g_f - d0 sgn(a_r - a_f)) leaky'(a_f);
 * g (gradient from the feature's other consumers) or d (gradient of the two sums) may be null, not both. */
int rave_leaky_fm_fwd(const float *x, float *a, float *stats, long H, float slope, void *stream);
int rave_leaky_fm_bwd(const float *a, const float *g, const float *d, float *gx, long H, float slope, void *stream);
/* the same tap that also writes the NEXT MRD conv's operand: x rows are (b, t) pairs [2 Rh][F][C] (first Rh rows real);
 * xs [2 Rh][Fp][3 C] bf16 = rave_time_stack_nhwc(a, kt = 3, pt = 1) incl. the zero borders / pad columns f >= F */
int rave_leaky_fm_stack_fwd(const float *x, float *a, float *stats, void *xs_bf16, long Rh, int T, int F, int C, int Fp,
                            float slope, void *stream);
/* its backward in one pass: gx = (adjoint of the time stack applied to gxs [2 Rh][Fp][3 C] bf16 (+ ga, nullable) + the
 * feature-matching terms d (nullable)) * LeakyReLU'(a) */
int rave_leaky_fm_stack_bwd(const float *a, const void *gxs_bf16, const float *ga, const float *d, float *gx, long Rh, int T,
                            int F, int C, int Fp, float slope, void *stream);
/* the same tap and backward for a next conv with time dilation dil (kt = 3, pt = dil):
 * xs = rave_time_stack_nhwc_dil(a, kt = 3, pt = dil, dil); dil = 1 is rave_leaky_fm_stack_fwd / _bwd. */
int rave_leaky_fm_stack_dil_fwd(const float *x, float *a, float *stats, void *xs_bf16, long Rh, int T, int F, int C, int Fp,
                                int dil, float slope, void *stream);
int rave_leaky_fm_stack_dil_bwd(const float *a, const void *gxs_bf16, const float *ga, const float *d, float *gx, long Rh,
                                int T, int F, int C, int Fp, int dil, float slope, void *stream);
/* Snake (rave/blocks.py:852-860) on the engine's channel-last bf16 streams [rows][C] (v3 chains on the wgmma kernels):
 * a = h + sin^2(alpha h) / (alpha + 1e-9);  backward: gh = ga * da/dh + add (add may be null), dalpha[c] += sum_rows
 * ga * da/dalpha (dalpha zeroed by the caller). */
int rave_snake_cl_fwd(const void *h_bf16, const float *alpha, void *a_bf16, long rows, int C, void *stream);
int rave_snake_cl_bwd(const void *ga_bf16, const void *h_bf16, const float *alpha, const void *add_bf16, void *gh_bf16,
                      float *dalpha, long rows, int C, void *stream);
/* AdaptiveInstanceNormalization (rave/blocks.py:863-926) in eval mode on a channel-last bf16 stream h [B][pitch][C]
 * (csrc/adain.cu).  The statistics buffers are the module's own, fp32: mean_* / std_* [max_batch][C], learn_* and
 * num_update_* [1]; every flag and counter is read on the device.
 *   adain_cl_stats   : per (b, c), the mean and unbiased std of the L valid rows (fixed-order fp32 sums; NaN for L = 1);
 *                      learn_y set -> mean_y / std_y += (stat - old) / (num_update_y + 1), num_update_y += 1 (learn_x
 *                      ignored); else learn_x set -> the same on the x buffers.  Then scale / shift [B][C] of the
 *                      transfer from the updated buffers: scale = std_y / (std_x + 1e-5), shift = mean_y - mean_x scale
 *                      when learn_y is clear and both counters are non-zero, else exactly 1 / 0.  B <= max_batch.
 *   adain_snake_cl_fwd: rows l < L: h = h scale + shift in place (the residual's skip stream), a = Snake(h) as the next
 *                      conv's operand (rave_snake_cl_fwd's arithmetic); rows [L, pitch) of a are zeroed.  C % 8 == 0. */
int rave_adain_cl_stats(const void *h_bf16, int B, int L, int pitch, int C, float *mean_x, float *std_x, float *mean_y,
                        float *std_y, const float *learn_x, const float *learn_y, float *num_update_x,
                        float *num_update_y, int max_batch, float *scale, float *shift, void *stream);
int rave_adain_snake_cl_fwd(void *h_bf16, const float *alpha, const float *scale, const float *shift, void *a_bf16,
                            int B, int L, int pitch, int C, void *stream);
int rave_conv1d_tc_wgrad(const void *P_bf16, const void *Q_bf16, float *dwt, float *dbias, int B, int Cm, int Lp,
                         int p_pitch, int Cn, int Lq, int q_pitch, int K, int stride, int dil, int pad_l,
                         void *stream);
/* sum_s dwt[s][K][Cm][Cn] -> dw[Cm][Cn][K] (transpose=0) or dw[Cn][Cm][K] (transpose=1), fp32 */
int rave_tapmajor_to_weight_f32(const float *dwt, float *dw, int Cm, int Cn, int K, int transpose, int splits,
                                void *stream);
/* ---------------------------------------------------------------------------------------------
 * small-channel kernels of the discriminators (csrc/conv_small.cu)
 *   c1_fwd  : first conv of a ConvNet (Cin = 1; rave/discriminator.py:99-111 with in_size = 1):
 *             out[r][l][co] = bias[co] + sum_k w[co][k] x[r][l*stride + k - pad_l];  x [R][x_pitch] fp32,
 *             outputs channel-last [R][out_pitch][Cout] (fp32 stream and/or bf16 act(out)); Cout % 8 == 0.
 *   c1_wgrad: dwt[s][k][co] with s < rave_conv1d_c1_wgrad_splits(R, Lout) (= 1: CTA partials are combined
 *             with fp32 atomics); g bf16 channel-last [R][g_pitch][Cg] (first Cout channels), K <= 16.
 *   fm_stats: feature-matching sums of rave/model.py:360-368 + core.mean_difference (rave/core.py:236-252)
 *             on the bf16 operand stream a = LeakyReLU_slope(h), [2*Bh][pitch][C] (first Bh = real):
 *             stats[0] += sum |h_r - h_f|, stats[1] += sum |h_r|  (l < L); stats must be pre-zeroed.
 *   fm_grad : gradient of d0*S_diff + d1*S_abs w.r.t. h as a bf16 stream (slack rows zero). C % 8 == 0.
 * ------------------------------------------------------------------------------------------- */
int rave_conv1d_c1_fwd(const float *x, const float *w, const float *bias, float *out_f32, void *out_act_bf16,
                       int R, int x_pitch, int Lin, int Cout, int Lout, int out_pitch, int K, int stride,
                       int pad_l, int act, float slope, void *stream);
int rave_conv1d_c1_wgrad_splits(int R, int Lout);
int rave_conv1d_c1_wgrad(const void *g_bf16, const float *x, float *dwt, int R, int x_pitch, int Lin, int Cout,
                         int Cg, int Lout, int g_pitch, int K, int stride, int pad_l, void *stream);
/* c1_dgrad: dx[r][t] = sum_k sum_co g[r][(t+pad-k)/stride][co] w[co][k]  (fp32 rows [R][x_pitch]);
 * colsum : out[c] = sum_{r, l<L} g[r][l][c]  (bias gradient of a channel-last bf16 gradient stream). */
int rave_conv1d_c1_dgrad(const void *g_bf16, const float *w, float *dx, int R, int x_pitch, int Lin, int Cout,
                         int Cg, int Lout, int g_pitch, int K, int stride, int pad_l, void *stream);
int rave_colsum_bf16(const void *g_bf16, float *out, int R, int L, int pitch, int Cg, int C, void *stream);
/* Cin = 1 first layer on the tensor-core kernels: im2col of the K (<= 16) taps into 16 bf16 "channels"
 *   X[r][l][k] = bf16(row_r[l*stride + k - pad_l])        (X [R][out_pitch][16], zero elsewhere)
 * where the R rows are read straight from a signal tensor src [Bs][src_pitch] (src_len valid samples):
 *   row r = b*period + w, position i -> (1/pool) * sum_{j<pool} src[b][(i*pool + j)*period + w]
 * (period > 1 = MultiPeriodDiscriminator.fold, rave/discriminator.py:187-195; pool = 2^scale = the avg_pool1d
 * chain of MultiScaleDiscriminator, rave/discriminator.py:150-171; period = pool = 1: src already holds the rows),
 * and the adjoint: dsrc (pre-zeroed or accumulating) += scatter-free gather of P [R][p_pitch][16] fp32 back through
 * the taps, the pooling and the fold. */
int rave_im2col_c1(const float *src, void *X_bf16, int R, int src_pitch, int src_len, int Lin, int Lout,
                   int out_pitch, int K, int stride, int pad_l, int period, int pool, void *stream);
int rave_gather_c1(const float *P, float *dsrc, int R, int src_pitch, int src_len, int Lin, int Lout, int p_pitch,
                   int K, int stride, int pad_l, int period, int pool, void *stream);
/* The same for a first layer with cin input channels (multichannel models): src [Bs][cin][src_pitch], the fold /
 * pooling applied per channel (R = Bs*period rows, independent of cin), X rows of W = 16 or 32 bf16 columns
 *   X[r][l][c*K + k] = bf16(row_{r,c}[l*stride + k - pad_l])   (cin*K <= W: the [c][k] order of
 *                                                                weight.reshape(Cout, Cin*K); zero beyond cin*K)
 * and the adjoint from P [R][p_pitch][W] fp32 into dsrc [Bs][cin][src_pitch].  rave_im2col_c1 / rave_gather_c1 are
 * the cin = 1, W = 16 instances. */
int rave_im2col_cin(const float *src, void *X_bf16, int R, int cin, int src_pitch, int src_len, int Lin, int Lout,
                    int out_pitch, int W, int K, int stride, int pad_l, int period, int pool, void *stream);
int rave_gather_cin(const float *P, float *dsrc, int R, int cin, int src_pitch, int src_len, int Lin, int Lout,
                    int p_pitch, int W, int K, int stride, int pad_l, int period, int pool, void *stream);
int rave_fm_stats(const void *a_bf16, float *stats, int Bh, int L, int pitch, int C, float slope, void *stream);
int rave_fm_grad(const void *a_bf16, const float *dstats, void *gout_bf16, int Bh, int L, int pitch, int C,
                 float slope, void *stream);
/* Discriminator score tail (replaces, per ConvNet, the scalar arithmetic of rave/model.py:348-379 with
 * core.hinge_gan, rave/core.py:151-155, and core.mean_difference, 236-252, on the score map).
 * score: channel-last fp32 [2*Bh][pitch][C], channel 0 = the score, real half first.
 * stats (pre-zeroed) += { sum|s_r-s_f|, sum|s_r|, sum relu(1-s_r), sum relu(1+s_f), sum s_r, sum s_f }.
 * rave_score_grad writes d(sum_i dstats[i]*stats[i])/ds as the bf16 gradient stream [2*Bh][pitch][C]. */
int rave_score_stats(const float *score, float *stats, int Bh, int L, int pitch, int C, void *stream);
int rave_score_grad(const float *score, const float *dstats, void *gout_bf16, int Bh, int L, int pitch, int C,
                    void *stream);

/* ---------------------------------------------------------------------------------------------
 * fused spectral distance (replaces the elementwise tail of core.AudioDistanceV1, rave/core.py:322-344,
 * and mean_difference, 236-252, for one STFT scale).  X, Y: complex64 spectrograms (interleaved re/im), n
 * complex elements.  stats: 5 pre-zeroed floats; [0..2] += { sum(|X|-|Y|)^2, sum|X|^2,
 * sum|log(|X|+eps)-log(|Y|+eps)| }, [3] is a block ticket, [4] = the distance s0/s1 + s2/n (written by the last
 * block).  grad: dY = (c_lin*-2(|X|-|Y|) - c_log*sgn(logX-logY)/(|Y|+eps)) * Y/|Y| with c_lin = g/stats[1],
 * c_log = g/n and g = *gup the upstream gradient of the distance (device float).
 * ------------------------------------------------------------------------------------------- */
int rave_spectral_stats(const void *X_c64, const void *Y_c64, float *stats, long n, float eps, void *stream);
int rave_spectral_grad(const void *X_c64, const void *Y_c64, void *dY_c64, const float *stats, const float *gup,
                       long n, float eps, void *stream);
/* STFT framing of torch.stft(center=True, pad_mode="reflect", hop | n_fft) without the FFT (rave/core.py:286-306):
 * frames[n][f][t] = window[t] * x[n][reflect(f*hop + t - n_fft/2)], F = 1 + T/hop frames; and its adjoint
 * dx[n][j] (window, overlap-add, fold of the reflected borders). */
int rave_stft_frames(const float *x, const float *window, float *frames, int N, int T, int n_fft, int hop,
                     void *stream);
int rave_stft_frames_bwd(const float *dframes, const float *window, float *dx, int N, int T, int n_fft, int hop,
                         void *stream);
/* Uncentred framing of torchaudio Spectrogram(center=False, normalized=True) (rave/discriminator.py:12-20):
 * frames[n][f][t] = scale * window[t] * x[n][f*hop + t], F = 1 + (T - n_fft)/hop frames, no padding (scale = 1/||w||_2
 * for normalized=True); and its adjoint dx[n][j] (overlap-add as a gather, zero past the last frame). */
int rave_stft_frames_valid(const float *x, const float *window, float *frames, int N, int T, int n_fft, int hop,
                           float scale, void *stream);
int rave_stft_frames_valid_bwd(const float *dframes, const float *window, float *dx, int N, int T, int n_fft, int hop,
                               float scale, void *stream);
/* gradient of rfft (last axis, n = 2*(bins-1)) prepared for ONE c2r transform: Z[k] = G[k]*n*(1 | 1/2 | ... | 1/2 | 1)
 * with the imaginary parts of the DC / Nyquist bins dropped; dx = irfft(Z, n).  G [N][F][bins] complex64 with element
 * strides (sN, sF, sB); Z contiguous. */
int rave_rfft_bwd_scale(const void *G_c64, void *Z_c64, long N, int F, int bins, long sN, long sF, long sB,
                        void *stream);

/* fused weight preparation for the engine: v [C0][C1][K] fp32 (+ weight-norm g [C0]; norm [C0] is written)
 *   outA[t][c0][c1] = bf16(w[c0][c1][tapsA[t]]), dims [nA][C0p][C1p]  (padded region zero)
 *   outB[t][c1][c0] = bf16(w[c0][c1][tapsB[t]]), dims [nB][C1p][C0p]
 * tapsA / tapsB are HOST int arrays (<= 32 entries); either output may be NULL.  w = g v / ||v|| (or v). */
int rave_weight_prep_tc(const float *v, const float *g, float *norm, void *outA_bf16, const int *tapsA, int nA,
                        void *outB_bf16, const int *tapsB, int nB, int C0, int C1, int K, int C0p, int C1p,
                        void *stream);
/* tap-major fp32 weight gradient dwt [K][C0p][C1p] -> dv [C0][C1][K] (+ dg [C0]) through the weight norm
 * (g == NULL: plain re-layout). */
int rave_weight_norm_bwd_tapmajor(const float *dwt, const float *v, const float *g, const float *norm, float *dv,
                                  float *dg, int C0, int C1, int K, int C0p, int C1p, int splits, void *stream);
/* multi-tensor forms of the two calls above: one launch pair for up to 64 layers (a whole chain). */
typedef struct rave_wprep_layer {
  const float *v, *g;          /* parameter [C0][C1][K] and its weight-norm gain (or NULL)            */
  float *norm;                 /* [C0] row norms: written by prep, read by the backward                */
  void *outA, *outB;           /* bf16 outputs as in rave_weight_prep_tc (either may be NULL)         */
  const float *dwt;            /* backward: [splits][K][C0p][C1p] fp32 partial weight gradients; or, when nA > 1,
                                  the phase-wide form [splits][nB][C0p][nA*C1p] (strided layers: the wgrad ran on
                                  the operand viewed with nA positions per row) with tap k in slot tapsA[k] = j*nA+p */
  float *dv, *dg;              /* backward: gradients of v and g                                      */
  int C0, C1, K, C0p, C1p, nA, nB, splits;
  int tapsA[32], tapsB[32];    /* tap index, or -1 for an all-zero slab (phase-fused layouts)          */
} rave_wprep_layer;
int rave_weight_prep_tc_multi(int n, const rave_wprep_layer *layers, void *stream);
/* split-operand ("bf16x3") layouts: outA [2][nA][C0p][C1p], outB [2][nB][C1p][C0p] with part 0 = bf16(w) and
 * part 1 = bf16(w - part 0) (operands of rave_conv1d_tc_fwd_x3) */
int rave_weight_prep_tc_multi_x3(int n, const rave_wprep_layer *layers, void *stream);
int rave_weight_norm_bwd_multi(int n, const rave_wprep_layer *layers, void *stream);
/* layout converters between the module-boundary layout [B][C][L] fp32 and the engine's channel-last:
 *   to_cl:   y_bf16[b][l][c] = bf16(act(x[b][c][l])), optionally also y_f32[b][l][c] = x[b][c][l]
 *   from_cl: y[b][c][l] = x_f32[b][l][c] */
int rave_ncl_to_cl(const float *x, void *y_bf16, float *y_f32, int B, int C, int L, int act, float slope,
                   const float *alpha, void *stream);
int rave_cl_to_ncl(const float *x_cl, float *y, int B, int C, int L, void *stream);
/* split-operand entry: y[b][l][0..C) = hi = bf16(x[b][c][l]), y[b][l][C..2C) = bf16(x - hi) */
int rave_ncl_to_cl_x3(const float *x, void *y_bf16, int B, int C, int L, void *stream);
/* fp32 -> bf16 operand preparation: y = bf16(act(x)) */
int rave_act_to_bf16(const float *x, void *y_bf16, int B, int C, int L, int act, float slope,
                     const float *alpha, void *stream);
/* weight re-layout: w[Cout][Cin][K] fp32 (or transposed-conv [Cin][Cout][K] with transpose=1)
 * -> wt[K][Cout][Cin] bf16 */
int rave_weight_to_tapmajor_bf16(const float *w, void *wt_bf16, int Cout, int Cin, int K, int transpose,
                                 int flip, void *stream);

/* ---------------------------------------------------------------------------------------------
 * NoiseGeneratorV2 tail (rave/blocks.py:284-292 + mod_sigmoid / amp_to_impulse_response / fft_convolve,
 * rave/core.py:20-21,48-81) as ONE kernel:  amp = 2 sigmoid(h - 5)^2.3 + 1e-7;  ir = M amp (M [TS][NB]: the linear
 * irfft -> roll -> hann -> crop/pad -> roll pipeline applied to the identity, built by the host);
 * out[b][c][t*TS + i] = sum_{j<=i} noise[b][t][c][j] ir[i-j].  h [B][C*NB][T], noise [B][T][C][TS], out [B][C][T*TS].
 * TS <= 16, NB <= 64.  bwd: gradient with respect to h (noise is a constant).
 * ------------------------------------------------------------------------------------------- */
int rave_noise_fir_fwd(const float *h, const float *M, const float *noise, float *out, int B, int C, int NB, int T,
                       int TS, void *stream);
int rave_noise_fir_bwd(const float *h, const float *M, const float *noise, const float *dout, float *dh, int B, int C,
                       int NB, int T, int TS, void *stream);

/* ---------------------------------------------------------------------------------------------
 * Mel front end of the hybrid encoder (rave/model.py:238-242, torchaudio MelSpectrogram(normalized=True)):
 *   out[n][m][f] = log1p(scale * sum_{k in [lo_m, hi_m)} w[off_m + k - lo_m] |X[n][f][k]|^2),  f < F - 1
 * X: [N][F][bins] complex64 (rfft of centred frames), band: [M][3] ints (lo, hi, off), weights: the nnz packed
 * nonzero filter-bank entries, out: [N][M][F-1] (= [B][C*M][F-1] for n = b*C + c), scale = 1 / sum(window^2).
 * ------------------------------------------------------------------------------------------- */
int rave_mel_log1p_fwd(const void *X_c64, const int *band, const float *weights, float *out, int N, int F, int bins,
                       int M, int nnz, float scale, void *stream);
/* its gradient with respect to X: dX[n][f][k] = 2 scale X[n][f][k] sum_m w_m[k] dy[n][m][f] / (1 + mel[n][m][f]) for
 * f < F - 1, zero for the dropped last frame; dy [N][M][F-1], dX [N][F][bins] complex64. */
int rave_mel_log1p_bwd(const void *X_c64, const int *band, const float *weights, const float *dy, void *dX_c64, int N,
                       int F, int bins, int M, int nnz, float scale, void *stream);

/* ---------------------------------------------------------------------------------------------
 * GRU layer (rave/blocks.py:295-319: nn.GRU, gate order r, z, n), fp32, H = 128, one persistent launch per layer:
 *   fwd: gi [B][T][3H] = W_ih x_t + b_ih (precomputed), w_hh [3H][H], b_hh [3H] -> h_out [B][T][H] (h0 = 0);
 *        save [B][T][5][H] = (r, z, n, W_hn h + b_hn, h_prev) for the backward (NULL: not written)
 *   bwd: dy [B][T][H] (gradient of h_out) -> gate gradients dgi [B][T][3H] (of gi) and dgh [B][T][3H] (of W_hh h + b_hh)
 * ------------------------------------------------------------------------------------------- */
int rave_gru_fwd(const float *gi, const float *w_hh, const float *b_hh, float *h_out, float *save, int B, int T, int H,
                 void *stream);
int rave_gru_bwd(const float *dy, const float *save, const float *w_hh, float *dgi, float *dgh, int B, int T, int H,
                 void *stream);
/* C[m][n] = sum_k A[m*sam + k*sak] B[k*sbk + n*sbn] (+ bias[n]), row pitch ldc; rowsum[m] = sum_k A(m, k) if non-NULL.
 * Fixed-order split-K over `splits` (rave_gemm_f32_splits) with workspace ws of splits*(M*N + M) floats. */
int rave_gemm_f32_splits(int M, int N, int K);
int rave_gemm_f32(const float *A, long sam, long sak, const float *B, long sbk, long sbn, const float *bias, float *C,
                  long ldc, float *rowsum, int M, int N, int K, float *ws, int splits, void *stream);

/* ---------------------------------------------------------------------------------------------
 * Multi-tensor Adam, torch.optim.Adam arithmetic without weight decay / amsgrad (rave/model.py:226-236):
 *   step += 1;  m = lerp(m, g, 1-b1);  v = b2 v + (1-b2) g^2;  p -= lr/(1-b1^step) * m / (sqrt(v)/sqrt(1-b2^step) + eps)
 * n fp32 tensors given by host arrays of device pointers; lr and step are single device floats (graph-replayable).
 * ------------------------------------------------------------------------------------------- */
int rave_adam_multi(int n, float *const *params, const float *const *grads, float *const *exp_avg,
                    float *const *exp_avg_sq, const long *numel, const float *lr, float *step, float beta1, float beta2,
                    float eps, void *stream);

/* ---------------------------------------------------------------------------------------------
 * Latent prior (rave/prior/{core,residual_block,model}.py: VariationalPrior.training_step), fp32 CUDA-core arithmetic,
 * fixed-order sums.  Streams [B][T][C] follow `cl_bf16`: 1 = channel-last with bf16 operands (wgmma engine), 0 = [B][C][T]
 * fp32 (parity path); fp32 gradient inputs (dout, dg) use the same layout.
 *   latent_classes: z [B][2L][T] encoder output (mean | scale), eps [B][L][T] ->
 *                   classes [B][T-D+1][D] int32 = clamp(floor(R Phi(y_d(b, t + D-1-d))), 0, R-1),
 *                   y = latent_pca[:D] (eps (softplus(scale) + 1e-4) + mean - latent_mean)   (post_process_latent,
 *                   DiagonalShift and QuantizedNormal.encode without the one-hot)
 *   embed_fwd:      pre_net on class indices, w [Cout][R][K], group d = o / (Cout/D):
 *                   out[b][t][o] = LeakyReLU(bias[o] + sum_{k: t+k-(K-1) >= 0} w[o][c_d(b, t+k-(K-1))][k]) as the fp32
 *                   stream out_f32 and (cl_bf16) the bf16 operand out_op [B][T][Cout]
 *   embed_wgrad:    dw [Cout][R][K], dbias [Cout] (nullable) of it from dout (gradient of out) and x (out_op, or out_f32
 *                   when cl_bf16 = 0, for LeakyReLU'); K <= 8
 *   gate:           g [B][T][C] = sigmoid(h[.., c]) tanh(h[.., C + c]) of h [B][T][2C]; bwd: dh from dg (fp32)
 *   head_ce:        x = LeakyReLU(p), p [B][Tp][Cin] post_net.0 output; logits of group d: w [D R][Cin/D] x[d Cin/D ..]
 *                   + bias; *loss = mean over B D (Tp-1) of the cross-entropy against classes[b][t+1][d];
 *                   bwd: dx = d loss / d p (times *gloss, a device float) in p's type, dw [D R][Cin/D], dbias [D R]
 * ------------------------------------------------------------------------------------------- */
int rave_prior_latent_classes(const float *z, const float *eps, const float *latent_mean, const float *latent_pca,
                              int *classes, int B, int L, int T, int D, int R, void *stream);
int rave_prior_embed_fwd(const int *classes, const float *w, const float *bias, float *out_f32, void *out_op_bf16, int B,
                         int Tp, int D, int R, int Cout, int K, int cl_bf16, float slope, void *stream);
int rave_prior_embed_wgrad(const int *classes, const float *dout, const void *x, float *dw, float *dbias, int B, int Tp,
                           int D, int R, int Cout, int K, int cl_bf16, float slope, void *stream);
int rave_gate_fwd(const void *h, void *g, int B, int C, int T, int cl_bf16, void *stream);
int rave_gate_bwd(const float *dg, const void *h, void *dh, int B, int C, int T, int cl_bf16, void *stream);
int rave_prior_head_ce_fwd(const void *x, const float *w, const float *bias, const int *classes, float *loss, int B,
                           int Tp, int D, int R, int Cin, int cl_bf16, float slope, void *stream);
int rave_prior_head_ce_bwd(const void *x, const float *w, const float *bias, const int *classes, const float *gloss,
                           void *dx, float *dw, float *dbias, int B, int Tp, int D, int R, int Cin, int cl_bf16,
                           float slope, void *stream);

/* ---------------------------------------------------------------------------------------------
 * Sampling from the latent prior (Prior.generate / validation_epoch_end), fp32 CUDA-core arithmetic, fixed-order sums.
 *   prior_sample:   `params` = host array of the 2 + 6 n_layers + 4 device pointers of Prior._trained_parameters()
 *                   (pre_net.0 w/b, per block dconv w/b, rconv w/b, sconv w/b, post_net.0 w/b, post_net.2 w/b); block i
 *                   has dilation 2^(i mod cycle_size).  prefix [B][P][D] int32, uniform [B][T][D] (frames < P unused;
 *                   may be NULL with argmax), classes [B][T][D] int32 out (frames < P copied from the prefix), logits
 *                   [B][T-1][D][R] out or NULL.  Step i consumes frame i and produces frame i + 1 (the prefix's while
 *                   i + 1 < P); a class is the first argmax, or the first r whose running softmax probability exceeds u
 *                   (the last r of non-zero probability if none does).  State lives in `work`
 *                   (rave_prior_sample_workspace_bytes, -1 for a bad shape) and is reset by every call.  The call
 *                   captures and replays its own CUDA graph, so it refuses to run inside a stream capture.
 *                   1 <= B <= 64, D divides res_size and skp_size, K <= 8, R <= 1024, 1 <= P <= T.
 *   classes_to_latent: classes [B][T][D], dither [B][T][D], noise [B][L-D][T-D+1] (NULL when L = D), latent_pca [L][L],
 *                   latent_mean [L] -> z [B][L][T-D+1] = latent_pca^T [y ; noise] + latent_mean, y[d][t] =
 *                   clamp(erfinv(2 x - 1) sqrt 2, -4, 4) of x = k / R + dither / R, k = classes[b][t + d][d]
 *                   (QuantizedNormal.decode, DiagonalShift.inverse, VariationalPrior.pre_process_latent)
 * ------------------------------------------------------------------------------------------- */
long rave_prior_sample_workspace_bytes(int B, int n_layers, int cycle_size, int res_size, int skp_size, int K, int D);
int rave_prior_sample(const float *const *params, int n_layers, int cycle_size, int res_size, int skp_size, int K, int R,
                      int D, const int *prefix, int P, const float *uniform, int T, int B, int argmax, int *classes,
                      float *logits, void *work, long work_bytes, void *stream);
int rave_prior_classes_to_latent(const int *classes, const float *dither, const float *noise, const float *latent_pca,
                                 const float *latent_mean, float *z, int B, int T, int D, int L, int R, void *stream);

/* ---------------------------------------------------------------------------------------------
 * Training-batch transforms (get_dataset's transform list, rave/dataset.py:207-262), per example b of raw [B][C][L]
 * (int16 when raw_int16, else float32; C channels share every draw) -> out [B][C][N] float32:
 *   decode float32(int16) / 32767; crop [off, off + N); when apply, the allpass lfilter(b, a) of
 *   pole_to_z_filter(omega, .99) from zero state, in float64; + U[0, 1) / 2^16; with normalize, normalize_signal over
 *   the example; with derivative, lfilter([.5, -.5], [1]); times keep; float32.
 *   draws [B][4] float64 = (off, apply, omega, keep), off clamped to [0, L - N]; key [2] int64 = (Philox seed,
 *   counter offset) of the dequantisation uniforms, keyed by (b, c, n); noise [B][C][N] float64 replaces them (or
 *   NULL).  One launch, two with normalize; graph-capturable (stream-ordered workspace, no host synchronisation).
 * ------------------------------------------------------------------------------------------- */
int rave_augment(const void *raw, int raw_int16, int B, int C, int L, int N, const double *draws, const long long *key,
                 const double *noise, float *out, int normalize, int derivative, void *stream);

/* ---------------------------------------------------------------------------------------------
 * Exponential moving average of parameters (the reference's EMA callback, scripts/train.py:81-119), multi-tensor.
 *   table [4T + 1] int64 = [ p[T] | ema[T] | numel[T] | chunk0[T + 1] ]: float32 pointers, element counts and the
 *   prefix sum of each tensor's chunk count, ceil(numel / rave_ema_chunk_elems()); n_chunks = chunk0[T].
 *   update: ema = rn(rn(ema * factor) + rn(p * one_minus_factor)) element by element (no FMA: torch's float32
 *   `w * factor + p * (1 - factor)` bit for bit), or ema = p for a tensor t whose state[t] is 0; the launch then sets
 *   state[0 .. T) to 1.  state [T + 1] int32 = [ initialised flags | completion ticket, 0 between launches ].
 *   swap: exchange p and ema in place.  One launch each, graph-capturable.
 * ------------------------------------------------------------------------------------------- */
long long rave_ema_chunk_elems(void);
int rave_ema_update(const long long *table, int n_tensors, long long n_chunks, int *state, float factor,
                    float one_minus_factor, void *stream);
int rave_ema_swap(const long long *table, int n_tensors, long long n_chunks, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* RAVE_B200_H */
