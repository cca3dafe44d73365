/* byol_b200.h — C ABI of libbyol_b200.so: the sm_100a kernels behind the BYOL training-step hot path.
 *
 * The reference (jramapuram/BYOL) is pure Python and has no FFI / operator registry of its own; its hot path
 * reaches cuDNN / cuBLAS / ATen / NCCL through torch.  This header is therefore the boundary a maintainer binds
 * from Python (ctypes stub in byol_b200/_lib.py; see INTEGRATION.md): plain pointers and sizes, one CUDA stream,
 * no torch types, no allocation, no implicit synchronisation, no global mutable state.
 *
 * Conventions
 *   - every function returns 0 on success, < 0 on error; byol_last_error() gives the thread-local message
 *   - all pointers are device pointers unless stated otherwise; `stream` is the caller's cudaStream_t
 *   - activations are NHWC bf16 with the channel count padded to a multiple of 8; "[M, C]" means M = N*H*W rows
 *   - fp32 parameter / gradient tensors use the reference's layouts ([Cout, Cin, KH, KW], [out, in], [C])
 *   - launches are asynchronous; errors detected at launch time are reported, device faults surface at the
 *     caller's next synchronisation
 *
 * Reference lines cited below are relative to /root/reference (jramapuram/BYOL @ 5ea487e).
 */
#ifndef BYOL_B200_H
#define BYOL_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct CUstream_st* byol_stream_t; /* == cudaStream_t */

const char* byol_last_error(void);
int byol_abi_version(void);
int byol_device_sm_count(void);

/* ---- tensor-core convolution / linear: replaces the cuDNN conv fwd/dgrad and cuBLAS Linear calls under
 *      main.py:229-240 (BYOL.prediction -> base_network, head, predictor) and main.py:250-252 (classifier) ----
 * out[M = Nimg*Ho*Wo, Ndim] = gather(src) x Wt^T (+bias) (+resid) (relu); optional fused per-column
 * sum / sum-of-squares of the stored values (BatchNorm statistics).
 *   mode 0 (fprop): src = x [Nimg,Hs,Ws,C], src coordinate = o*stride - pad + k
 *   mode 1 (dgrad): src = dY [Nimg,Hs,Ws,C=Cout], (Ho,Wo) = spatial size of dX, coordinate = (o + pad - k)/stride
 * wt: bf16 [Ndim, ldw] K-major with k = (kh*KW + kw)*C + c (made by byol_prep_weight).
 * resid_mask (optional, uint8 [M*ldc/8], written by byol_bn_apply): resid is added only where its bit is set, i.e.
 * the epilogue applies the ReLU mask of the residual branch (block backward, torchvision resnet.py Bottleneck.forward).
 * resid_up = 1: resid is the COMPACT [Nimg, Ho/2, Wo/2, ldc] gradient of a stride-2 1x1 branch and is added to the
 * even (h, w) pixels only (the dense, 3/4-zero gradient map of the downsample branch is never written). */
int byol_conv_igemm(const void* src, const void* wt, void* dst, const void* resid, const void* resid_mask,
                    int resid_up, const float* bias, float* col_sum, float* col_sqsum, int Nimg, int Hs, int Ws, int C, int Ho, int Wo, int Ndim,
                    int KH, int KW, int stride, int pad, int mode, int ldw, int ldc, int out_fp32, int relu,
                    int force_gather, byol_stream_t stream);

/* dW[Cout][Cin_real][KH][KW] (fp32, accumulated) += dY^T x im2col(x): replaces cuDNN wgrad / cuBLAS in the
 * autograd of main.py:617 (loss.backward()). */
int byol_conv_wgrad(const void* src, const void* dy, float* dw, int Nimg, int Hs, int Ws, int C, int Cin_real,
                    int Ho, int Wo, int Cout, int ldy /* row pitch of dy, 0 = Cout */, int KH, int KW, int stride,
                    int pad, int force_gather, byol_stream_t stream);

/* ---- stem (7x7 / stride 2 / pad 3, <= 4 input channels, 64 output channels, W <= 256): the torchvision ResNet
 *      conv1 reached from main.py:237.  The image is converted once to zero-padded NHWC4 bf16
 *      ([N][H+6][264][4]); the kernel forms the im2col rows with overlapping no-swizzle UMMA descriptors. ---- */
int byol_stem4_supported(int Cin, int Cout, int H, int W, int k, int stride, int pad);
int byol_stem4_row_pixels(void); /* Wp of the padded image tensor [N][H+6][Wp][4] */
int byol_nchw_to_stem4(const float* x, void* xs, int N, int Cin, int H, int W, byol_stream_t stream);
/* w fp32 [64][Cin][7][7] -> ws bf16 [7][4][64][8] (14336 elements) */
int byol_prep_weight_stem4(const float* w, void* ws, int Cin, byol_stream_t stream);
/* y [N, H/2, W/2, 64] bf16; col_sum / col_sqsum (both or none): += per-channel sum / sum of squares of y */
int byol_stem_conv_fprop(const void* xs, const void* ws, void* y, float* col_sum, float* col_sqsum, int N, int H, int W,
                         byol_stream_t stream);

/* dw [64][Cin][7][7] fp32 += dY^T x im2col(xs); dy [N, H/2, W/2, 64] bf16 (autograd of main.py:617 for the stem) */
int byol_stem_conv_wgrad(const void* xs, const void* dy, float* dw, int N, int Cin, int H, int W, byol_stream_t stream);

/* ---- BatchNorm (train / eval, optionally cross-rank): replaces ATen batch_norm and SyncBatchNorm
 *      (main.py:196,202,237,433; torch/nn/modules/_functions.py:10-205) ---- */
int byol_bn_stats(const void* x, float* stats /* zeroed [2C] */, int M, int C, byol_stream_t stream);
/* statistics -> coefficients for L <= 4 lock-step lanes in one launch: stats [L][2C], coeffs [L][4][C] = scale, shift, mean, invstd;
 * running statistics are updated lane after lane (the order of the reference's four forward passes) */
int byol_bn_finalize_lanes(const float* stats, double count, int L, const float* gamma0, const float* beta0,
                           const float* gamma1, const float* beta1, const float* gamma2, const float* beta2,
                           const float* gamma3, const float* beta3, float* running_mean, float* running_var,
                           float momentum, float eps, float* coeffs, int C, byol_stream_t stream);
int byol_bn_eval_coeffs(const float* gamma, const float* beta, const float* running_mean, const float* running_var,
                        float eps, float* scale, float* shift, int C, byol_stream_t stream);
/* y = act(x*scale + shift + (resid | resid*rscale + rshift)); mask_out (optional, uint8 [M*C/8]): bit e of byte i =
 * (y[8*i + e] > 0), the ReLU mask the backward kernels read instead of the activation (mask_mode 3) */
int byol_bn_apply(const void* x, const float* scale, const float* shift, const void* resid, const float* rscale,
                  const float* rshift, void* y, float* y_f32, void* mask_out, int M, int C, int relu,
                  byol_stream_t stream);
/* s12 (zeroed [2C]) += [sum dz, sum dz*xhat]; mask_mode 0 none / 1 relu(x*scale+shift) / 2 act > 0 (act = bf16
 * activation) / 3 mask bits (act = uint8 mask written by byol_bn_apply) */
int byol_bn_bwd_reduce(const void* g, const void* x, const void* act, const float* scale, const float* shift,
                       const float* mean, const float* invstd, float* s12, int M, int C, int mask_mode,
                       byol_stream_t stream);
/* dy = gamma*invstd*(dz - s1/n - xhat*s2/n); dgamma/dbeta (optional) += rank-local sums */
int byol_bn_bwd_apply(const void* g, const void* x, const void* act, const float* scale, const float* shift,
                      const float* mean, const float* invstd, const float* gamma, const float* s12, double count,
                      void* dy, void* dz_out, int M, int C, int mask_mode, const float* s12_local, float* dgamma,
                      float* dbeta, byol_stream_t stream);
int byol_col_sum(const void* x, float* out, int M, int C, int ld, int is_f32, byol_stream_t stream);

/* ---- GroupNorm (32 groups) and weight standardisation: BYOL(norm="group_ws") ---- */
/* desc: device int64 [num_units][5] = {src offset in flat, offset in w_out / dwhat, Cout, fan-in, first row}, rows in
 * unit order.  w_out[row] = (w - mean) / sqrt(var + 1e-5) (biased variance, fp64, rounded once); stats [rows][2] =
 * fp32 (mean, rstd) */
int byol_ws_fwd(const float* flat, const int64_t* desc, int num_units, int64_t num_rows, float* w_out, float* stats,
                byol_stream_t stream);
/* grad[row] += rstd * (dw^ - mean(dw^) - w^ * mean(dw^ * w^)) with w^ = w_out and stats of byol_ws_fwd */
int byol_ws_bwd(const float* dwhat, const float* what, const float* stats, const int64_t* desc, int num_units,
                int64_t num_rows, float* grad, byol_stream_t stream);
/* y [N, HW, C] bf16 (C % 32 == 0, C % 8 == 0) -> stats [N][32][2] = fp32 (mean, rstd) per (image, group); sums64
 * (optional, fp64 [N][32][2]) receives the sum and sum of squares */
int byol_gn_stats(const void* y, float* stats, double* sums64, int N, int HW, int C, float eps, byol_stream_t stream);
/* y = act(x*scale + shift (+ resid | + resid*rscale + rshift)), scale[n,c] = gamma[c]*rstd[n,g], shift[n,c] =
 * beta[c] - mean[n,g]*scale[n,c]; the residual's (rscale, rshift) come from (rgamma, rbeta, rstats) when given;
 * mask_out (optional, uint8 [N*HW*C/8]) as byol_bn_apply */
int byol_gn_apply(const void* x, const float* gamma, const float* beta, const float* stats, const void* resid,
                  const float* rgamma, const float* rbeta, const float* rstats, void* y, void* mask_out, int N, int HW,
                  int C, int relu, byol_stream_t stream);
/* stem fusion: y = maxpool(relu(gn(x))); values and argmax indices equal byol_gn_apply + byol_maxpool_fwd */
int byol_gn_relu_maxpool_fwd(const void* x, const float* gamma, const float* beta, const float* stats, void* y,
                             void* idx, int N, int H, int W, int C, int k, int s, int p, byol_stream_t stream);
/* s12 (zeroed fp32 [N][32][2]) += per (image, group) (sum gamma*dz, sum gamma*dz*xhat); dgamma / dbeta (required)
 * += per-channel sum dz*xhat / sum dz; mask_mode as byol_bn_bwd_reduce */
int byol_gn_bwd_reduce(const void* g, const void* x, const void* act, const float* gamma, const float* beta,
                       const float* stats, float* s12, float* dgamma, float* dbeta, int N, int HW, int C, int mask_mode,
                       byol_stream_t stream);
/* dy = rstd*(gamma*dz - s1/m - xhat*s2/m), m = HW*C/32; dz_out (optional) receives dz */
int byol_gn_bwd_apply(const void* g, const void* x, const void* act, const float* gamma, const float* beta,
                      const float* stats, const float* s12, void* dy, void* dz_out, int N, int HW, int C, int mask_mode,
                      byol_stream_t stream);

/* ---- layout / pooling: torchvision ResNet stem and tail reached from main.py:237 ---- */
int byol_nchw_to_nhwc8(const float* x, void* y, int N, int Cin, int H, int W, byol_stream_t stream);
int byol_prep_weight(const float* w, void* w_fprop, void* w_dgrad, int Cout, int Cin, int Cpad, int KH, int KW,
                     byol_stream_t stream);
/* stem layout ([Cout][KH*64], column = kh*64 + kw*8 + c) selected by byol_conv_igemm when C == 8 and ldw == KH*64 */
int byol_prep_weight_fold(const float* w, void* w_fprop, int Cout, int Cin, int KH, int KW, byol_stream_t stream);
/* every conv / linear weight of one parameter set in one launch; desc: device int64 [num_units][8] =
 * {src offset in flat, fprop offset in pool_f, dgrad offset in pool_d or -1, Cout, Cin, Cpad, taps, fold (KH*16+KW or 0)} */
int byol_prep_unit_blocks(int Cout, int Cin, int Cpad, int taps, int fold);   /* blocks one unit needs */
int byol_prep_weights_multi(const float* flat, void* pool_f, void* pool_d, const int64_t* desc, int num_units,
                            int num_blocks /* sum of byol_prep_unit_blocks over the units */, byol_stream_t stream);
/* ---- grouped 3x3 convolutions (ResNeXt conv2, torchvision Bottleneck with groups > 1): Cin == Cout == C with
 *      C % 64 == 0, Cg = C / groups dividing 64, 3x3, pad 1, stride 1 or 2.  A 64-channel output tile only meets its
 *      own 64 input channels, so the weights are kept as block-diagonal tiles [C / 64][64][9 * 64]; each tile runs
 *      9 k-blocks of 64 channels (64 / Cg times the algorithmic FLOPs).  Arguments are validated before any launch. */
/* desc: device int64 [num_units][5] = {src offset in flat (fp32 [C][Cg][3][3]), fprop offset in pool_f,
 * dgrad offset in pool_d or -1, C, Cg}; max_c: the largest C.  fprop column tap*64 + (ci - n0) for row co,
 * dgrad column tap*64 + (co - n0) for row ci (n0 = the row's 64-aligned tile start); off-group entries are 0. */
int byol_prep_weights_grouped(const float* flat, void* pool_f, void* pool_d, const int64_t* desc, int num_units,
                              int max_c, byol_stream_t stream);
/* y [Nimg, Ho, Wo, C] bf16; col_sum / col_sqsum (both or none): += per-channel sum / sum of squares of y */
int byol_conv_fprop_grouped(const void* x, const void* wt, void* y, float* col_sum, float* col_sqsum, int Nimg, int H,
                            int W, int C, int Ho, int Wo, int KH, int KW, int stride, int pad, byol_stream_t stream);
/* dx [Nimg, H, W, C] bf16 from dy [Nimg, Ho, Wo, C] and the dgrad tiles */
int byol_conv_dgrad_grouped(const void* dy, const void* wd, void* dx, int Nimg, int Ho, int Wo, int C, int H, int W,
                            int KH, int KW, int stride, int pad, byol_stream_t stream);
/* dw (fp32 [C][Cg][KH][KW], the parameter itself) += its in-group entries of dY^T x im2col(x); nothing else is written */
int byol_conv_wgrad_grouped(const void* x, const void* dy, float* dw, int Nimg, int H, int W, int C, int Cg, int Ho,
                            int Wo, int KH, int KW, int stride, int pad, byol_stream_t stream);
/* y[n,i,j,:] = x[n,2i,2j,:] (input of a 1x1 / stride-2 downsample conv, compacted for the TMA-fed GEMM) */
int byol_subsample2(const void* x, void* y, int N, int H, int W, int C, byol_stream_t stream);
int byol_cast_f32_bf16(const float* x, void* y, int64_t n, byol_stream_t stream);
/* y[r, c] = bf16(x[r, c]) for c < cols and 0 for cols <= c < ldy (pitched copy, e.g. classifier gradients) */
int byol_cast_f32_bf16_2d(const float* x, void* y, int rows, int cols, int ldx, int ldy, byol_stream_t stream);
int byol_maxpool_fwd(const void* x, void* y, void* idx, int N, int H, int W, int C, int k, int s, int p,
                     byol_stream_t stream);
/* stem fusion: y = maxpool(relu(x*scale + shift)); values and argmax indices equal bn_apply + maxpool_fwd exactly */
int byol_bn_relu_maxpool_fwd(const void* x, const float* scale, const float* shift, void* y, void* idx, int N, int H,
                             int W, int C, int k, int s, int p, byol_stream_t stream);
int byol_maxpool_bwd(const void* dy, const void* idx, void* dx, int N, int H, int W, int C, int k, int s, int p,
                     byol_stream_t stream);
int byol_avgpool_fwd(const void* x, float* y_f32, void* y_bf16, int N, int HW, int C, byol_stream_t stream);
int byol_avgpool_bwd(const void* g_bf16, const float* g_f32, void* dx, int N, int HW, int C, byol_stream_t stream);

/* ---- objective: replaces objective.py:6-25 (regression_loss / loss_function; Frobenius-normalised, rank-local) ----
 * workspace: 6 doubles; loss: 1 float; saved: 6 floats consumed by byol_loss_bwd. */
int byol_loss_fwd(const float* q1, const float* q2, const float* z1, const float* z2, int rows, int dim,
                  double* workspace, float* loss, float* saved, byol_stream_t stream);
int byol_loss_bwd(const float* q1, const float* q2, const float* z1, const float* z2, const float* saved,
                  const float* grad_out, float* dq1, float* dq2, int rows, int dim, byol_stream_t stream);

/* ---- the BYOL paper's loss: per-row L2-normalised predictions and targets, one warp per sample ----
 * r(x) = max(sum x^2, 1e-12)^(-1/2), x^ = r(x) x; loss = (1/rows) sum_i |q1^_i - z2^_i|^2 + |q2^_i - z1^_i|^2.
 * q1, q2, z1, z2: [rows, dim] fp32 contiguous and 16-byte aligned, dim a positive multiple of 4.  loss: 1 float;
 * saved: [rows, 8] floats (16-byte aligned) = r(q1), r(z2), c12, l12, r(q2), r(z1), c21, l21 per row (c = q^.u, or
 * 0 for a clamped row; l the row's pair loss), consumed by byol_loss_rows_bwd.  A row with a NaN or inf element, or
 * whose sum of squares overflows, has r = NaN.  Deterministic: the grid depends on rows only.
 * dq = grad_out * 2/rows * r(q) * (u - c q^), u = q^ - z^ (grad_out may be null: 1).  No gradient reaches z. */
int byol_loss_rows_fwd(const float* q1, const float* q2, const float* z1, const float* z2, int rows, int dim,
                       float* loss, float* saved, byol_stream_t stream);
int byol_loss_rows_bwd(const float* q1, const float* q2, const float* z1, const float* z2, const float* saved,
                       const float* grad_out, float* dq1, float* dq2, int rows, int dim, byol_stream_t stream);

/* ---- target network: replaces CosEMA.forward, main.py:159-162.  mean = fl(fl(a*x) + fl(d*mean)), bit-exact ---- */
int byol_ema_update(const float* x, float* mean, float one_minus_decay, float decay, int64_t n,
                    byol_stream_t stream);

/* ---- optimizer: replaces LARS.apply_adaptive_lrs + SGD(momentum).step, optimizers/lars.py:84-127 ----
 * p_ptrs / g_ptrs / m_ptrs: device arrays of num_tensors fp32 pointers (m_ptrs may be NULL: no momentum);
 * chunk tables split the tensors into work items (chunks of one tensor are contiguous:
 * [tensor_first_chunk[t], tensor_first_chunk[t+1])); partial: 2*num_chunks doubles of scratch.  No atomics: the
 * per-tensor norms are bit-reproducible, so data-parallel replicas stay bit-identical (main.py:440). */
int byol_lars_sgd_step(const void* p_ptrs, const void* g_ptrs, const void* m_ptrs, const int64_t* chunk_start,
                       const int* chunk_len, const int* chunk_tensor, int num_chunks, const int* tensor_first_chunk,
                       const float* wd, const float* lr, const int* ignore, int num_tensors, double* partial,
                       float trust_coef, float eps, float momentum, int first_step, byol_stream_t stream);

/* One Nesterov-SGD step over the chunk tables of byol_lars_sgd_step (fine-tuning, byol_b200/finetune.py), in
 * torch.optim.SGD(nesterov=True)'s order with each fp32 operation rounded on its own: g = dW + wd*w;
 * buf = momentum*buf + g; d = g + momentum*buf; w = w - lr*d, with lr = fp32(lr[t] * lr_scale) and wd[t] per tensor
 * (fp32 device arrays).  m_ptrs is required; the gradients are zeroed.  Any range length and alignment (float4 accesses
 * where p / g / momentum share a 16-byte phase). */
int byol_sgd_nesterov_step(const void* p_ptrs, const void* g_ptrs, const void* m_ptrs, const int64_t* chunk_start,
                           const int* chunk_len, const int* chunk_tensor, int num_chunks, const float* wd,
                           const float* lr, float lr_scale, float momentum, byol_stream_t stream);

/* ---- linear-probe objective: replaces F.cross_entropy + helpers.metrics.topk, main.py:596-598 ----
 * logits fp32 [R, C] (row pitch ld), labels int64 [label_rows] (row r uses labels[r % label_rows]: the two views
 * of a sample share its label, main.py:591); scratch: row_lse / row_loss [R] floats, row_rank [R] ints,
 * ticket: one zeroed uint32.  out = [mean loss, top-1 %, top-5 %] (deterministic row-order reduction). */
int byol_ce_topk_fwd(const float* logits, const int64_t* labels, int label_rows, int R, int C, int ld, float* row_lse,
                     float* row_loss, int* row_rank, unsigned int* ticket, float* out, byol_stream_t stream);
/* dlogits[r, c] = grad_out / R * (softmax(logits[r])[c] - [c == labels[r]]) */
int byol_ce_bwd(const float* logits, const int64_t* labels, int label_rows, const float* row_lse, const float* grad_out, int R, int C,
                int ld, float* dlogits, int ldd, byol_stream_t stream);

/* ---- fp32-accurate forward path ("split-bf16", BASELINE.json configs[1]): the reference runs main.py:229-276 in
 *      fp32; here every fp32 operand is split exactly into T bf16 planes (T = 3: ~16 bits, T = 6: 24 bits) that feed
 *      the SAME tensor-core kernels as one GEMM over T*C channels (byol_conv_igemm with C := T*C, out_fp32 = 1);
 *      BatchNorm statistics are accumulated in fp64.  See csrc/split.cu. ---- */
int byol_split_planes(const float* x /* [M, C], pitch ldx */, void* planes /* bf16 [M, T*Cpad] */,
                      void* copy_bf16 /* optional [M, C] */, int64_t M, int C, int Cpad, int ldx, int T,
                      byol_stream_t stream);
int byol_nchw_to_planes(const float* x /* NCHW */, void* planes /* bf16 NHWC [N,H,W,T*Cpad] */, int N, int Cin, int H,
                        int W, int Cpad, int T, byol_stream_t stream);
int byol_prep_weight_planes(const float* w /* [Cout, Cin, taps] */, void* out /* bf16 [Cout, taps*T*Cpad] */, int Cout,
                            int Cin, int Cpad, int taps, int T, byol_stream_t stream);
int byol_stats_f32(const float* y, double* stats /* zeroed [2C] */, int64_t M, int C, byol_stream_t stream);
int byol_bn_finalize_lanes_f64(const double* stats, double count, int L, const float* gamma0, const float* beta0,
                               const float* gamma1, const float* beta1, const float* gamma2, const float* beta2,
                               const float* gamma3, const float* beta3, float* running_mean, float* running_var,
                               float momentum, float eps, float* coeffs, int C, byol_stream_t stream);
int byol_bn_apply_f32(const float* y, const float* scale, const float* shift, const float* resid, const float* rscale,
                      const float* rshift, float* out32, void* planes, void* copy_bf16, void* mask, int64_t M, int C,
                      int relu, int T, byol_stream_t stream);
int byol_maxpool_f32(const float* x, float* y, void* idx, int N, int H, int W, int C, int k, int s, int p,
                     byol_stream_t stream);
int byol_avgpool_f32(const float* x, float* y, int N, int HW, int C, byol_stream_t stream);

/* ---- fp32-accurate backward path (BYOL(backward_precision="fp32")): the same exact splits on the backward GEMMs,
 *      fp32 gradients between layers, fp64 BatchNorm-backward sums (csrc/split.cu, csrc/conv_igemm.cu). ---- */
int byol_prep_weight_dgrad_planes(const float* w /* [Cout, Cin, taps] */, void* out /* bf16 [Cin, taps*T*Cout] */,
                                  int Cout, int Cin, int taps, int T, byol_stream_t stream);
/* dx (fp32 [Nimg, H, W, Cin]) = conv_transpose(dy planes [Nimg, Hs, Ws, T*Cout], wd) (+ resid_f32, optional) */
int byol_conv_dgrad_planes(const void* dy, const void* wd, float* dx, const float* resid_f32, int Nimg, int Hs, int Ws,
                           int Cout, int H, int W, int Cin, int KH, int KW, int stride, int pad, int T,
                           byol_stream_t stream);
/* dw (fp32 [Cout, Cin_real, KH, KW]) += sum of the T terms dY-plane^T x im2col(src-plane);
 * src planes [Nimg, Hs, Ws, T*C], dy planes [Nimg, Ho, Wo, T*ldy] */
int byol_conv_wgrad_planes(const void* src, const void* dy, float* dw, int Nimg, int Hs, int Ws, int C, int Cin_real,
                           int Ho, int Wo, int Cout, int ldy, int KH, int KW, int stride, int pad, int T,
                           byol_stream_t stream);
/* s12 (fp64 [2C]) += [sum dz, sum dz*xhat]; mask_mode 0 none / 1 relu(y*scale+shift) / 3 mask bits */
int byol_bn_bwd_reduce_f32(const float* g, const float* y, const void* mask, const float* scale, const float* shift,
                           const float* mean, const float* invstd, double* s12, int64_t M, int C, int mask_mode,
                           byol_stream_t stream);
/* dy = gamma*invstd*(dz - s1/n - xhat*s2/n) -> planes bf16 [M, T*C] and / or fp32 [M, C]; dz_out optional fp32;
 * dgamma / dbeta (optional) += the rank-local sums s12_local (default s12) */
int byol_bn_bwd_apply_f32(const float* g, const float* y, const void* mask, const float* scale, const float* shift,
                          const float* mean, const float* invstd, const float* gamma, const double* s12,
                          const double* s12_local, double count, void* planes, float* dy32, float* dz_out,
                          float* dgamma, float* dbeta, int64_t M, int C, int mask_mode, int T, byol_stream_t stream);
int byol_maxpool_bwd_f32(const float* dy, const void* idx, float* dx, int N, int H, int W, int C, int k, int s, int p,
                         byol_stream_t stream);
int byol_avgpool_bwd_f32(const float* ga, const float* gb, float* dx, int N, int HW, int C, byol_stream_t stream);

/* ---- projector / predictor MLP forward as ONE cooperative kernel (main.py:194-205, 238-239):
 *      Linear -> BatchNorm1d (batch statistics, grid barrier, optional cross-rank exchange) -> ReLU -> Linear.
 *      x [B, K1] bf16, w1 [H, ldw1], w2 [O, ldw2] bf16 (fprop layouts); stats [2H] and out [B, O] fp32 ZEROED by the
 *      caller; coeffs [4, H]; h_save / a_save optional bf16 [B, H] (for the backward pass); grid_bar: 2 zeroed uint32.
 *      See csrc/mlp_fused.cu. ---- */
int byol_mlp_fused_supported(int B, int K1, int H, int O);
int byol_mlp_fused_fwd(const void* x, const void* w1, const float* b1, const float* gamma, const float* beta,
                       const void* w2, const float* b2, float* stats, float* running_mean, float* running_var,
                       float momentum, float eps, double count, float* coeffs, float* out, void* h_save, void* a_save,
                       void* grid_bar, int B, int K1, int H, int O, int ldw1, int ldw2, int train,
                       const uint64_t* peer_ptrs, int world, int rank, int64_t cap_bytes, void* counter,
                       byol_stream_t stream);

/* ---- SyncBatchNorm statistic exchange over NVLink peer memory (main.py:433; replaces the per-layer all_gather /
 *      all_reduce of torch/nn/modules/_functions.py:49-74,158-159): one single-CTA kernel per exchange — publish into
 *      this rank's symmetric buffer, flag every peer, wait, add all peers' values in rank order.  See csrc/xchg.cu. */
int byol_xchg_layout(int* slots, int* max_world, int* flag_bytes);
int byol_xchg_sum(void* vals, void* local_copy, int n, int is_f64, const uint64_t* peer_ptrs /* host, [world] */,
                  int world, int rank, int64_t cap_bytes, void* counter /* device uint32 */, byol_stream_t stream);

/* ---- on-device two-view augmentation (main.py:386-397: RandomResizedCrop, flip, ColorJitter p = 0.8, grayscale
 *      p = 0.2, Gaussian blur p = 0.5) for decoded fp32 NCHW images resident in HBM.  params: fp32 [2, N, 16] records
 *      (view-major; byol_augment_record_floats() floats each: crop top / left / h / w, flip, jitter on, op order x 4,
 *      brightness, contrast, saturation, hue, flag word (bit 0 gray), blur sigma).  See csrc/augment.cu. ---- */
int byol_augment_record_floats(void);
int byol_augment_params(float* params, int N, int Hs, int Ws, uint64_t seed, uint64_t step, float strength,
                        float p_flip, float p_jitter, float p_gray, float p_blur, byol_stream_t stream);
int byol_augment_apply(const float* src, const float* params, float* out /* [2, N, 3, R, R] */, float* tmp,
                       double* gray_sum /* [2N] */, int N, int Hs, int Ws, int R, int ksize, byol_stream_t stream);
/* mixed-size batches: hw is a device int32 [n, 2] table of image heights and widths.  The sampler draws the records of
 * samples [n0, n0 + n) of an N-image batch (chunks of one batch give the records of one call; equal sizes with n0 = 0,
 * n = N give byol_augment_params' records).  The apply reads a device table of N uint8 CHW [3, H_i, W_i] images as
 * v / 255 and otherwise computes exactly what byol_augment_apply does. */
int byol_augment_params_ragged(float* params /* [2, n, 16] */, const int* hw, int n, int n0, int N, uint64_t seed,
                               uint64_t step, float strength, float p_flip, float p_jitter, float p_gray, float p_blur,
                               byol_stream_t stream);
int byol_augment_apply_ragged(const uint8_t* const* srcs, const int* hw, const float* params,
                              float* out /* [2, N, 3, R, R] */, float* tmp, int N, int R, int ksize,
                              byol_stream_t stream);
/* The samplers with the recipe spelled out: the BYOL paper's (Grill et al. 2020, Appendix B) is jitter {0.4, 0.4,
 * 0.2, 0.1}, p_blur {1.0, 0.1}, p_solarize {0.0, 0.2}, bicubic; the reference's is jitter {0.8, 0.8, 0.8, 0.2},
 * p_blur {0.5, 0.5}, p_solarize {0, 0}, bilinear, and gives byol_augment_params' records.  Record float 14 is a flag
 * word: bit 0 grayscale, bit 1 solarize (x >= 0.5 -> 1 - x, after the blur), bit 2 bicubic resampling (clamped to
 * [0, 1]); the apply entries above run records of either recipe.  A probability outside [0, 1] is rejected. */
typedef struct {
  float jitter[4];      /* brightness, contrast, saturation, hue factors; the kernel multiplies them by strength */
  float p_flip, p_jitter, p_gray;
  float p_blur[2];      /* view 1, view 2 */
  float p_solarize[2];  /* view 1, view 2 */
  int bicubic;          /* 1: antialiased bicubic crop resize, 0: antialiased bilinear */
} byol_augment_recipe_t;
int byol_augment_params_recipe(float* params /* [2, N, 16] */, int N, int Hs, int Ws, uint64_t seed, uint64_t step,
                               float strength, const byol_augment_recipe_t* recipe /* host */, byol_stream_t stream);
int byol_augment_params_ragged_recipe(float* params /* [2, n, 16] */, const int* hw, int n, int n0, int N,
                                      uint64_t seed, uint64_t step, float strength,
                                      const byol_augment_recipe_t* recipe /* host */, byol_stream_t stream);

/* ---- weighted k-NN evaluation of frozen features (csrc/knn.cu; the similarity chunks come from byol_conv_igemm as a
 *      linear layer over bf16 rows).  Entries rank by similarity descending, then bank index ascending (-0 as +0, NaN
 *      last): a total order, so the selection is exactly the first k entries of a full sort of each row. ---- */
/* y bf16 [R, D] = x / ||x||_2 per row of fp32 x [R, D] (row pitch ldx); the norm is a fixed-order fp32 sum; a zero row
 * stays zero */
int byol_l2_normalize_rows(const float* x, void* y, int64_t R, int D, int64_t ldx, byol_stream_t stream);
/* sim fp32 [Q, Nc] (row pitch ld): similarities of Q queries against bank rows n0 .. n0 + Nc - 1.  top_vals fp32 /
 * top_idx int32 [Q, k] (1 <= k <= 256): per query the k best entries, best first, of the chunk merged with the list
 * already there (merge = 1) or of the chunk alone (merge = 0); slots beyond the entries seen hold -inf / -1 */
int byol_knn_topk(const float* sim, int Q, int Nc, int64_t ld, int n0, int k, int merge, float* top_vals,
                  int* top_idx, byol_stream_t stream);
/* pred int32 [Q, 5]: the 5 best classes by score = sum over the class's neighbours (rank order, fp64) of the fp32
 * weight expf(s / temperature), then class index ascending; bank_labels int64 in [0, num_classes); slots beyond
 * num_classes hold -1; pred_scores (optional) fp32 [Q, 5]: the scores of pred */
int byol_knn_vote(const float* top_vals, const int* top_idx, const int64_t* bank_labels, int Q, int k, int num_classes,
                  float temperature, int* pred, float* pred_scores, byol_stream_t stream);

/* ---- linear evaluation of frozen features (csrc/linear_eval.cu): H linear heads over one feature matrix, stored as
 *      one [H * Cp, D] weight matrix (Cp = C rounded up to a multiple of 8, rows c >= C of each head are padding) and
 *      [H, Cp] biases, so that one byol_conv_igemm computes the logits of every head. ---- */
/* logits fp32 [B, >= H * Cp] (row pitch ld, a multiple of 4; 16-byte aligned): per row r and head h the softmax
 * cross-entropy of columns h * Cp .. h * Cp + C - 1 against labels[r] (int64; 2 <= C; a row whose label is outside
 * [0, C) is ignored: no loss, no hit, zero gradient).  Outputs (each
 * optional, at least one given): dlogits bf16 [B, H * Cp] (16-byte aligned) = (softmax - onehot) / B, 0 in the padding
 * columns; loss_sum fp32 [H] += the per-head sum of the row losses; hits int64 [H, 2] += the rows whose label has
 * rank < 1 / rank < 5 (rank = the number of other logits not <= the label's: strictly larger ones and NaNs; a NaN label
 * logit is a miss).  Deterministic (fixed-point / integer sums). */
int byol_linprobe_ce(const float* logits, int64_t ld, const int64_t* labels, int B, int H, int C, int Cp,
                     void* dlogits, float* loss_sum, long long* hits, byol_stream_t stream);
/* One Nesterov-SGD step of every head, in torch.optim.SGD's order with each fp32 operation rounded on its own:
 * g = dW + wd*w; buf = momentum*buf + g; d = g + momentum*buf; w = w - lr*d with lr = fp32(lr[h] * lr_scale).
 * params / grads / momentum_buf: fp32 [H * Cp * D] weights followed by [H * Cp] biases (16-byte aligned); lr, wd: fp32
 * [H] on the device.  Writes weight_bf16 [H * Cp, D] = bf16(w) (round to nearest even) and zeroes grads; the padding
 * rows c >= C are not touched. */
int byol_linprobe_sgd(float* params, float* grads, float* momentum_buf, void* weight_bf16, const float* lr,
                      const float* wd, float lr_scale, float momentum, int H, int C, int Cp, int D,
                      byol_stream_t stream);

/* ---- transfer linear evaluation (csrc/logreg.cu): H L2-regularised multinomial logistic regressions fitted together
 *      by full-batch L-BFGS.  Parameters: one fp32 buffer of [H * Cp, D] weights followed by [H, Cp] biases (the layout
 *      of the linear-evaluation heads); head h's vector is its Cp weight rows and its Cp biases.  Fixed-point
 *      accumulators (loss_acc [H], bias_acc [H * Cp]) are 24-byte records, zeroed by the caller.  mode: int32 [H] per-head
 *      state (0 stopped, 1 line search, 2 accept + new direction, 3 starting point, 4 accept + stop); a vector kernel acts
 *      on the heads whose mode bit is set in mask.  part: fp64 scratch of at least 8 * H * byol_logreg_vec_blocks(Cp, D)
 *      entries.  Every reduction has a fixed order that depends on Cp and D only. ---- */
/* blocks per head of the vector kernels (slices of 16384 elements of a head's Cp * D + Cp parameters) */
int byol_logreg_vec_blocks(int Cp, int D);
/* logits fp32 [B, >= H * Cp] (pitch ld, 16-byte aligned), labels int64 [B].  Fit: planes bf16 [B, 6 * H * Cp] = the
 * six activation-pattern split planes of (softmax - onehot) / n_total (0 in padding columns and rows whose label is
 * outside [0, C)); loss_acc += the per-head row losses; bias_acc += the column sums of the same fp32 gradient.
 * Evaluation: class_hits int64 [H, Cp] += top-1 hits per label (a NaN label logit is a miss); class_count int64 [Cp]
 * += the rows per label. */
int byol_logreg_ce(const float* logits, int64_t ld, const int64_t* labels, int B, int H, int C, int Cp,
                   double n_total, void* planes, void* loss_acc, void* bias_acc, long long* class_hits,
                   long long* class_count, byol_stream_t stream);
/* gt (weights: the data term's gradient at xt) += l2[h] * W; gt biases = bias_acc; out[h * ldo + 0..2] = (loss sum,
 * max |gt|, ||W||^2) in fp64 */
int byol_logreg_grad(const float* xt, float* gt, const void* loss_acc, const void* bias_acc, const double* l2,
                     const int* mode, int mask, int H, int C, int Cp, int D, double* part, double* out, int ldo,
                     byol_stream_t stream);
/* out[h * ldo + k] = fp64 dot product of head h's parts of u[k] and v[k], k < K <= 8 (host arrays of device pointers) */
int byol_logreg_dots(const void* const* u, const void* const* v, int K, const int* mode, int mask, int H, int C, int Cp,
                     int D, double* part, double* out, int ldo, byol_stream_t stream);
/* modes 2 / 4: s = xt - x and y = gt - g into the free history slot, x = xt, g = gt; mode 3: x = xt, g = gt.  Mode 2
 * keeps the pair when s.y > 1e-10 y.y (rho = 1 / s.y, gamma = s.y / y.y; hist int32 [H, 2] = (oldest slot, count) of
 * a ring of m + 1 slots in S, Y [m + 1, buffer]). */
int byol_logreg_accept(float* x, const float* xt, float* g, const float* gt, float* S, float* Y, int* hist,
                       double* rho, double* gamma, const int* mode, int m, int H, int C, int Cp, int D, double* part,
                       byol_stream_t stream);
/* d = -H g by the two-loop recursion over the stored pairs (scaled by gamma; -g / ||g||_2 without pairs); alpha fp64
 * [H, m + 1] scratch */
int byol_logreg_twoloop(const float* g, float* d, const float* S, const float* Y, const int* hist, const double* rho,
                        const double* gamma, double* alpha, double* part, const int* mode, int mask, int m, int H,
                        int C, int Cp, int D, byol_stream_t stream);
/* xt = x + fp32(t[h]) * d */
int byol_logreg_trial(const float* x, const float* d, float* xt, const double* t, const int* mode, int mask, int H,
                      int C, int Cp, int D, byol_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* BYOL_B200_H */
