/*
 * simclr_b200 -- C-ABI of the H100-native SimCLR pretrain step.
 *
 * The reference (google-research/simclr) has no FFI layer: its hot path is
 * Python calling TensorFlow ops.  This header is therefore the *new* boundary
 * a maintainer binds with ctypes (see INTEGRATION.md); every entry point cites
 * the reference call site whose arithmetic it replaces (paths relative to the
 * reference repository root).
 *
 * Conventions (SURVEY.md section 8b):
 *   - plain C, no torch types; all tensor pointers are DEVICE pointers owned by
 *     the caller; the library never allocates or frees device memory and keeps
 *     no reference after return.
 *   - every call only enqueues work on `stream` (a cudaStream_t passed as
 *     void*); no hidden synchronisation, no default-stream use => capturable in
 *     a CUDA graph.
 *   - return value: 0 on success, negative simclr_status for argument errors
 *     (checked before launch), positive = cudaError_t.  simclr_last_error()
 *     returns thread-local text for the last failure.
 *   - activations are NHWC, conv kernels HWIO, dense kernels [in,out], exactly
 *     the layouts of the reference's variables (tf2/resnet.py:196-208,
 *     tf2/model.py:143-147).  `dtype` selects the activation storage type.
 */
#ifndef SIMCLR_B200_H_
#define SIMCLR_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SIMCLR_API __attribute__((visibility("default")))

enum simclr_status {
  SIMCLR_OK = 0,
  SIMCLR_ERR_INVALID_ARG = -1,
  SIMCLR_ERR_UNSUPPORTED = -2,
  SIMCLR_ERR_WORKSPACE = -3,
  SIMCLR_ERR_DRIVER = -4
};

enum simclr_dtype { SIMCLR_F32 = 0, SIMCLR_BF16 = 1 };

SIMCLR_API int simclr_version(void);
SIMCLR_API const char* simclr_last_error(void);

/* ------------------------------------------------------------------------- *
 * NT-Xent objective  (tf2/objective.py:35-89)
 * ------------------------------------------------------------------------- */

/* l2-normalise rows (tf2/objective.py:53-54; tf.math.l2_normalize eps 1e-12).
 * hidden [rows,dim] -> z [rows,dim], inv_norm [rows].  hidden_norm==0 copies. */
SIMCLR_API int simclr_ntxent_normalize(const float* hidden, int64_t rows, int64_t dim, int hidden_norm,
                                       float* z, float* inv_norm, void* stream);

SIMCLR_API size_t simclr_ntxent_workspace_bytes(int64_t B, int64_t R, int64_t D);

/* Forward for the local 2B rows against all 2*R*B gathered rows.
 * z_all is the all-gather of every replica's z, layout [R][2][B][D]
 * (replaces tpu_cross_replica_concat, tf2/objective.py:92-127; R==1: local z).
 * Outputs: logits_ab [B][R*B] (tf2/objective.py:80, nullable), lse [2][B],
 * row_loss [2][B], loss [1] = mean_i(loss_a_i + loss_b_i) (tf2/objective.py:83-87). */
SIMCLR_API int simclr_ntxent_forward(const float* z_all, int64_t B, int64_t R, int64_t D, int64_t replica_id,
                                     float temperature, float* logits_ab, float* lse, float* row_loss,
                                     float* loss, void* workspace, size_t workspace_bytes, void* stream);

/* Integer index / one-hot construction (tf2/objective.py:64-69), bit-exact:
 * labels_idx[i] = i + replica_id*B; labels [B][2*R*B]; masks [B][R*B]. Any may be NULL. */
SIMCLR_API int simclr_ntxent_labels(int64_t B, int64_t R, int64_t replica_id, int64_t* labels_idx,
                                    float* labels, float* masks, void* stream);

/* Backward of the job loss (sum_r loss_r / R) w.r.t. this replica's `hidden`
 * [2B][D].  lse_all is the all-gather of lse, layout [R][2][B].  Includes the
 * key-side terms TF obtains through the backward of the all-reduce (SURVEY 8e)
 * and the l2-normalise backward.  grad_scale = dL/d(row loss) (1/(B*R) in the step). */
SIMCLR_API int simclr_ntxent_backward(const float* z_all, const float* lse_all, const float* inv_norm,
                                      int hidden_norm, int64_t B, int64_t R, int64_t D, int64_t replica_id,
                                      float temperature, float grad_scale, float* dhidden,
                                      void* workspace, size_t workspace_bytes, void* stream);

/* Contrastive accuracy / entropy (tf2/metrics.py:23-36) from logits_ab [B][G]
 * with label column i + replica_id*B.  out [2 + 2*B] floats: out[0] = accuracy,
 * out[1] = entropy, the rest is per-row scratch. */
SIMCLR_API int simclr_contrast_metrics(const float* logits_ab, int64_t B, int64_t G, int64_t replica_id,
                                       float* out, void* stream);

/* ------------------------------------------------------------------------- *
 * Supervised head loss  (tf2/objective.py:27-32) and small dense helpers
 * ------------------------------------------------------------------------- */

/* logits [rows][classes]; labels one-hot [label_rows][classes], row r uses
 * labels[r % label_rows] (tf2/run.py:600-602 concat([l,l])).  loss [1] = mean CE;
 * dlogits = (softmax - labels) * grad_scale (nullable).
 * loss must have room for 1 + rows floats (loss[1..] holds the per-row losses). */
SIMCLR_API int simclr_softmax_xent(const float* logits, const float* labels, int64_t rows, int64_t label_rows,
                                   int64_t classes, float grad_scale, float* loss, float* dlogits,
                                   void* stream);
SIMCLR_API int simclr_bias_add(float* y, const float* bias, int64_t rows, int64_t C, void* stream);
SIMCLR_API int simclr_bias_grad(const float* dy, float* dbias, int64_t rows, int64_t C, void* stream);
/* y += a*x  (weight-decay gradient of the supervised head, tf2/model.py:47-60). */
SIMCLR_API int simclr_axpy(float a, const float* x, float* y, int64_t n, void* stream);
/* out[0] = sum(x^2)/2  (tf.nn.l2_loss); out must have room for 257 floats (scratch). */
SIMCLR_API int simclr_l2_loss(const float* x, int64_t n, float* out, void* stream);
SIMCLR_API int simclr_cast(const void* src, int src_dtype, void* dst, int dst_dtype, int64_t n, void* stream);
/* a += b (gradient fan-in of the residual branches, tf2/resnet.py:382,487 backward). */
SIMCLR_API int simclr_add_inplace(void* a, const void* b, int dtype, int64_t n, void* stream);

/* ------------------------------------------------------------------------- *
 * LARS  (tf2/lars_optimizer.py:83-137), multi-tensor, two launches per step
 * ------------------------------------------------------------------------- */

/* Device tables (built once by the host): per tensor w/g/v pointers, numel,
 * flags (bit0: weight decay applies, bit1: layer adaptation applies -- the
 * name filters of tf2/lars_optimizer.py:139-157 evaluated by the host);
 * per chunk (chunk_elems elements): tensor index and element offset;
 * tensor_chunk_begin [n_tensors+1].  lr is a device scalar (lr_t).
 * partials: scratch [n_chunks][2] floats.  Deterministic reduction order, so
 * every replica applies bit-identical updates. */
SIMCLR_API int simclr_lars_apply(int64_t n_tensors, int64_t n_chunks, const void* w_ptrs, const void* g_ptrs,
                                 const void* v_ptrs, const int64_t* numels, const int32_t* flags,
                                 const int32_t* chunk_tensor, const int64_t* chunk_offset,
                                 const int64_t* tensor_chunk_begin, int64_t chunk_elems, const float* lr,
                                 float momentum, float weight_decay, float eeta, float* partials,
                                 void* stream);

/* ------------------------------------------------------------------------- *
 * BatchNorm family  (tf2/resnet.py:31-78; formulas SURVEY.md A4)
 * All tensors are [rows][C] views of NHWC activations (rows = N*H*W).
 * ------------------------------------------------------------------------- */

/* sums [2][C] doubles: sum x, sum x^2 over rows (zeroed by the call). */
SIMCLR_API int simclr_bn_stats(const void* x, int dtype, int64_t rows, int64_t C, double* sums, void* stream);

/* From (all-reduced) sums and the global element count: mean, rstd, fused
 * scale = gamma*rstd and shift = beta - mean*scale; moving statistics update
 * m <- m - (m - batch)*(1-momentum) with the biased variance.
 * gamma/beta may be NULL (scale=False / center=False, tf2/model.py:135). */
SIMCLR_API int simclr_bn_finalize(const double* sums, double count, const float* gamma, const float* beta,
                                  float eps, float momentum, float* moving_mean, float* moving_var,
                                  float* mean, float* rstd, float* scale, float* shift, int64_t C,
                                  void* stream);

/* z = act(y*scale + shift (+ residual)); relu: tf2/resnet.py:76-77,382,487. */
SIMCLR_API int simclr_bn_apply(const void* y, int y_dtype, const void* residual, void* z, int z_dtype,
                               int64_t rows, int64_t C, const float* scale, const float* shift, int relu,
                               void* stream);

/* Backward, phase 1.  dz <- (dz (+ dz2)) * [z > 0 if relu_mask_z != NULL] in
 * place; sums [2][C] doubles: sum dz, sum dz*xhat with xhat=(y-mean)*rstd. */
SIMCLR_API int simclr_bn_bwd_reduce(void* dz, const void* dz2, const void* relu_mask_z, int dtype,
                                    const void* y, int y_dtype, int64_t rows, int64_t C, const float* mean,
                                    const float* rstd, double* sums, void* stream);

/* Backward, phase 1 of a BN + ReLU without residual (tf2/resnet.py:75-77): the ReLU
 * mask [scale*y + shift > 0] is recomputed from the saved conv output y, so dz is read
 * once and never rewritten.  sums as above, over dz*mask. */
SIMCLR_API int simclr_bn_bwd_relu_reduce(const void* dz, int dtype, const void* y, int y_dtype,
                                         int64_t rows, int64_t C, const float* mean, const float* rstd,
                                         const float* scale, const float* shift, double* sums,
                                         void* stream);

/* Backward, phase 2.  dy = gamma*rstd*(dz - S0/count - xhat*S1/count) with
 * the (all-reduced) sums; dgamma/dbeta (nullable) are written from
 * sums_local (this replica's contribution, summed later with the other grads).
 * mask_scale / mask_shift (nullable, together): dz is masked on the fly with
 * [mask_scale*y + mask_shift > 0] (pairs with simclr_bn_bwd_relu_reduce). */
/* Block tail (tf2/resnet.py:382,487: relu(bn(y) + shortcut)) with the ReLU mask kept as ONE BIT per element:
 * `relu_mask_bits` [rows*C/8] bytes, bit k of byte i = [z > 0] of channel k of 16-byte vector i.  The backward
 * reduction then reads 1/16 of the bytes it would read from z: dz <- (dz + dz2) * mask in place,
 * sums [2][C] = (sum dz, sum dz*xhat), as simclr_bn_bwd_reduce. */
SIMCLR_API int simclr_bn_apply_relu_mask(const void* y, int y_dtype, const void* residual, void* z, int z_dtype,
                                         int64_t rows, int64_t C, const float* scale, const float* shift,
                                         uint8_t* relu_mask_bits, void* stream);
SIMCLR_API int simclr_bn_bwd_reduce_bits(void* dz, const void* dz2, const uint8_t* relu_mask_bits, int dtype,
                                         const void* y, int y_dtype, int64_t rows, int64_t C, const float* mean,
                                         const float* rstd, double* sums, void* stream);
SIMCLR_API int simclr_bn_bwd_apply(const void* dz, int dtype, const void* y, int y_dtype, void* dy,
                                   int dy_dtype, int64_t rows, int64_t C, const float* mean,
                                   const float* rstd, const float* gamma, const double* sums,
                                   const double* sums_local, double count, float* dgamma, float* dbeta,
                                   float* coef_ws /* scratch [3][C] */, const float* mask_scale,
                                   const float* mask_shift, void* stream);
/* The element-wise pass of simclr_bn_bwd_apply alone, with coef [3][C] already computed
 * (by simclr_comm_bn_bwd_coef: SyncBN statistics exchanged over peer memory). */
SIMCLR_API int simclr_bn_bwd_apply_coef(const void* dz, int dtype, const void* y, int y_dtype, void* dy,
                                        int dy_dtype, int64_t rows, int64_t C, const float* coef,
                                        const float* mask_scale, const float* mask_shift, void* stream);

/* Tail of a PROJECTION block (tf2/resnet.py:342-353,415-423 + :382,:487) with the shortcut's BatchNorm folded in:
 *   forward  z = relu(scale*y + shift + round(scale2*y2 + shift2))   (y2: the shortcut conv's output; its BN output
 *            is rounded to the activation type as the separate kernel would have stored it, but never stored),
 *            one ReLU bit per element like simclr_bn_apply_relu_mask;
 *   backward dz <- (dz + dz2) * mask in place, sums of both BatchNorms in the same pass (sums2 [2][C] w.r.t. y2,
 *            mean2, rstd2), then dy = coef*(dz, y, 1) and dy2 = coef2*(dz, y2, 1) in one pass over dz.
 * fp32/fp32 or bf16/bf16 tensors. */
SIMCLR_API int simclr_bn_apply2_relu_mask(const void* y, const void* y2, int y_dtype, void* z, int z_dtype,
                                          int64_t rows, int64_t C, const float* scale, const float* shift,
                                          const float* scale2, const float* shift2, uint8_t* relu_mask_bits,
                                          void* stream);
SIMCLR_API int simclr_bn_bwd_reduce2_bits(void* dz, const void* dz2, const uint8_t* relu_mask_bits, int dtype,
                                          const void* y, const void* y2, int y_dtype, int64_t rows, int64_t C,
                                          const float* mean, const float* rstd, const float* mean2,
                                          const float* rstd2, double* sums, double* sums2, void* stream);
SIMCLR_API int simclr_bn_bwd_apply2_coef(const void* dz, int dtype, const void* y, const void* y2, int y_dtype,
                                         void* dy, void* dy2, int dy_dtype, int64_t rows, int64_t C,
                                         const float* coef, const float* coef2, void* stream);

/* The stem's BatchNorm + ReLU + MaxPooling2D (tf2/resnet.py:593-611) without materialising the BN output:
 * forward pools relu(scale*y + shift) of the conv output y directly (same rounding as the unfused chain);
 * backward forms dz = maxpool_bwd(d [+ d2]) * [scale*y + shift > 0] on the fly, first for the BatchNorm
 * reduction (sums [2][C] = (sum dz, sum dz*xhat)), then for dy = coef0*dz + coef1*y + coef2.
 * C/8 (bf16; C/4 fp32) must divide 256.  bf16 only, optional: `ysel` [N,Ho,Wo,C] = y at each window's argmax,
 * written by the forward; given to the reduction it replaces the pass over y by one over the pooled tensors. */
SIMCLR_API int simclr_bn_relu_maxpool_fwd(const void* y, int dtype, const float* scale, const float* shift,
                                          void* out, uint8_t* argmax, void* ysel, int64_t N, int64_t H, int64_t W,
                                          int64_t C, void* stream);
SIMCLR_API int simclr_maxpool_bn_bwd_reduce(const void* d, const void* d2, const uint8_t* argmax, const void* y,
                                            const void* ysel, int dtype, int64_t N, int64_t H, int64_t W, int64_t C,
                                            const float* mean, const float* rstd, const float* scale,
                                            const float* shift, double* sums, void* stream);
SIMCLR_API int simclr_maxpool_bn_bwd_apply(const void* d, const void* d2, const uint8_t* argmax, const void* y,
                                           int dtype, void* dy, int64_t N, int64_t H, int64_t W, int64_t C,
                                           const float* coef, const float* scale, const float* shift, void* stream);
/* coef [3][C] of dy = coef0*dz + coef1*y + coef2 (+ dgamma, dbeta from sums_local) alone: the first launch of
 * simclr_bn_bwd_apply. */
SIMCLR_API int simclr_bn_bwd_coef(const float* mean, const float* rstd, const float* gamma, const double* sums,
                                  const double* sums_local, double count, float* coef, float* dgamma,
                                  float* dbeta, int64_t C, void* stream);
/* ------------------------------------------------------------------------- *
 * Pooling  (tf2/resnet.py:605-611 MaxPooling2D(3,2,'SAME'); :693-696 mean)
 * ------------------------------------------------------------------------- */
SIMCLR_API int simclr_maxpool3x3s2_fwd(const void* x, void* y, uint8_t* argmax, int dtype, int64_t N,
                                       int64_t H, int64_t W, int64_t C, void* stream);
SIMCLR_API int simclr_maxpool3x3s2_bwd(const void* dy, const uint8_t* argmax, void* dx, int dtype, int64_t N,
                                       int64_t H, int64_t W, int64_t C, void* stream);
SIMCLR_API int simclr_global_avgpool_fwd(const void* x, int dtype, void* y, int y_dtype, int64_t N,
                                         int64_t HW, int64_t C, void* stream);
SIMCLR_API int simclr_global_avgpool_bwd(const void* dy, int dy_dtype, void* dx, int dtype, int64_t N,
                                         int64_t HW, int64_t C, void* stream);

/* ------------------------------------------------------------------------- *
 * Convolution / dense as implicit GEMM  (tf2/resnet.py:183-208 Conv2dFixedPadding,
 * tf2/model.py:143-151 Dense = 1x1 conv on [rows,1,1,Cin])
 *   x  [N,H,W,Cs]   Cs = stored channels (Cin, or 4 for the 3-channel stem)
 *   y  [N,Ho,Wo,Cout], Ho = H (stride 1) or (H-1)/stride+1 with pad (k-1)/2
 * ------------------------------------------------------------------------- */

/* tensor-core engine operands: K-major packed copies of the fp32 HWIO master.
 *   wf [Cout][Kp]       k = (r*S+s)*Cs + c,   Kp = round_up(R*S*Cs, 128B/elt)
 *                       bf16 with Cs == 4 (the stem: 3 image channels + 1 zero):
 *                       k = (r*(S+1) + s+1)*4 + c, Kp = round_up(R*(S+1)*4, 64); slot 0 of each
 *                       filter row is zero, so a row is a whole number of 16-byte pixel pairs
 *   wd [Cin ][Kdp]      k = (r*S+s)*Cout + co, Kdp = round_up(R*S*Cout, 128B/elt)
 *                       (NULL: not needed, e.g. the stem) */
SIMCLR_API int simclr_pack_conv_weight(const float* w_hwio, void* wf, void* wd, int dtype, int64_t R,
                                       int64_t S, int64_t Cin, int64_t Cs, int64_t Cout, int64_t Kp,
                                       void* stream);
/* Every layer's packed bf16 operands in ONE launch (the per-step refresh after the optimizer update):
 * `table_dev` is a device array of n_layers rows of 10 int64 {w_hwio, wf, wd (0: none), R, S, Cin, Cs,
 * Cout, Kp, Kdp}, same layouts as simclr_pack_conv_weight with dtype bf16. */
SIMCLR_API int simclr_pack_conv_weights_multi(const void* table_dev, int64_t n_layers, void* stream);
/* Accumulation outputs -- the BatchNorm sums of simclr_conv2d_fprop_tc / simclr_bn_stats /
 * simclr_bn_bwd_*reduce and dW of simclr_conv2d_wgrad_tc -- are zeroed by the call that fills them.  A caller
 * that keeps them in pooled buffers and zeroes those once per step (simclr_memset_zero) switches the per-call
 * memsets off with on = 1; returns the previous setting.  Process-wide, not thread-safe. */
SIMCLR_API int simclr_set_accumulate_prezeroed(int on);
SIMCLR_API int simclr_memset_zero(void* p, int64_t bytes, void* stream);
/* bn_sums (nullable): [2][Cout] doubles receiving sum y / sum y^2 of the stored outputs -- the
 * BatchNorm statistics of tf2/resnet.py:50-72 fused into the conv epilogue (zeroed by the call). */
SIMCLR_API int simclr_conv2d_fprop_tc(const void* x, const void* wf, void* y, int dtype, int y_dtype,
                                      int64_t N, int64_t H, int64_t W, int64_t Cs, int64_t Cout, int64_t R,
                                      int64_t S, int64_t stride, double* bn_sums, void* stream);
SIMCLR_API int simclr_conv2d_dgrad_tc(const void* dy, const void* wd, void* dx, int dtype, int dx_dtype,
                                      int64_t N, int64_t H, int64_t W, int64_t Cin, int64_t Cout, int64_t R,
                                      int64_t S, int64_t stride, void* stream);
/* dw: fp32 HWIO [R][S][Cin][Cout], overwritten. */
SIMCLR_API int simclr_conv2d_wgrad_tc(const void* x, const void* dy, float* dw, int dtype, int64_t N,
                                      int64_t H, int64_t W, int64_t Cs, int64_t Cin, int64_t Cout, int64_t R,
                                      int64_t S, int64_t stride, void* stream);

/* Split-bf16 products -- the tensor-core VERIFICATION mode (`--b200_conv_engine=tc3`: fp32 storage,
 * 1e-3 step parity with the fp32 reference of tf2/run.py:557-622 on the tensor-core pipe).  Every fp32
 * operand v is split three ways, v = v0 + v1 + v2 with v0 = bf16(v), v1 = bf16(v - v0),
 * v2 = bf16(v - v0 - v1) (`simclr_split_bf16x3`; `simclr_pack_conv_weight_part` writes part 0 / 1 / 2
 * of the packed weights in the layouts of `simclr_pack_conv_weight`), and a product is taken as
 * a0*b0 + a0*b1 + a1*b0 + a1*b1 + a0*b2 + a2*b0: six exact-product / fp32-accumulate GEMMs summed in
 * fp32 (TMA reduce-add); the dropped terms are 2^-24 relative.  Outputs are fp32 and overwritten. */
SIMCLR_API int simclr_split_bf16x3(const float* x, void* v0, void* v1, void* v2, int64_t n, void* stream);
SIMCLR_API int simclr_pack_conv_weight_part(const float* w_hwio, void* wf, void* wd, int part, int64_t R,
                                            int64_t S, int64_t Cin, int64_t Cs, int64_t Cout, int64_t Kp,
                                            void* stream);
SIMCLR_API int simclr_conv2d_fprop_tc3(const void* x0, const void* x1, const void* x2, const void* wf0,
                                       const void* wf1, const void* wf2, float* y, int64_t N, int64_t H,
                                       int64_t W, int64_t Cs, int64_t Cout, int64_t R, int64_t S,
                                       int64_t stride, void* stream);
SIMCLR_API int simclr_conv2d_dgrad_tc3(const void* dy0, const void* dy1, const void* dy2, const void* wd0,
                                       const void* wd1, const void* wd2, float* dx, int64_t N, int64_t H,
                                       int64_t W, int64_t Cin, int64_t Cout, int64_t R, int64_t S,
                                       int64_t stride, void* stream);
SIMCLR_API int simclr_conv2d_wgrad_tc3(const void* x0, const void* x1, const void* x2, const void* dy0,
                                       const void* dy1, const void* dy2, float* dw, int64_t N, int64_t H,
                                       int64_t W, int64_t Cs, int64_t Cin, int64_t Cout, int64_t R, int64_t S,
                                       int64_t stride, void* stream);

/* CUDA-core fp32 engine reading the fp32 HWIO master directly (verification
 * engine for the tensor-core path; not the default). */
SIMCLR_API int simclr_conv2d_fprop_simt(const void* x, const float* w_hwio, void* y, int dtype, int y_dtype,
                                        int64_t N, int64_t H, int64_t W, int64_t Cs, int64_t Cin,
                                        int64_t Cout, int64_t R, int64_t S, int64_t stride, void* stream);
SIMCLR_API int simclr_conv2d_dgrad_simt(const void* dy, const float* w_hwio, void* dx, int dtype,
                                        int dx_dtype, int64_t N, int64_t H, int64_t W, int64_t Cin,
                                        int64_t Cout, int64_t R, int64_t S, int64_t stride, void* stream);
SIMCLR_API int simclr_conv2d_wgrad_simt(const void* x, const void* dy, float* dw, int dtype, int64_t N,
                                        int64_t H, int64_t W, int64_t Cs, int64_t Cin, int64_t Cout,
                                        int64_t R, int64_t S, int64_t stride, void* stream);

/* ------------------------------------------------------------------------- *
 * Selective-kernel block (tf2/resnet.py:217-277 SK_Conv2D) and ResNet-D shortcut
 * pooling (tf2/resnet.py:333-340,401-408).  x is the BN+ReLU output of the 3x3 conv,
 * [N][HW][2f]; stream s occupies channels [s*f, (s+1)*f).
 * ------------------------------------------------------------------------- */
/* g[n,c] = mean_hw(x[n,hw,c] + x[n,hw,f+c])                       (tf2/resnet.py:265-266) */
SIMCLR_API int simclr_sk_pool(const void* x, int dtype, float* g, int64_t N, int64_t HW, int64_t f, void* stream);
/* mixing = softmax over the two streams of logits [N][2f]; out[n,hw,c] = x0*m0 + x1*m1  (:270-275) */
SIMCLR_API int simclr_sk_mix_fwd(const void* x, const float* logits, float* mixing, void* out, int dtype,
                                 int64_t N, int64_t HW, int64_t f, void* stream);
/* dlogits [N][2f] = softmax backward of dmix_s[n,c] = sum_hw dout*x_s */
SIMCLR_API int simclr_sk_mix_bwd_reduce(const void* dout, const void* x, const float* mixing, float* dlogits,
                                        int dtype, int64_t N, int64_t HW, int64_t f, void* stream);
/* dx[n,hw,s*f+c] = dout[n,hw,c]*m_s[n,c] + dg[n,c]/HW  (dg: gradient w.r.t. the pooled features) */
SIMCLR_API int simclr_sk_mix_bwd_apply(const void* dout, const float* mixing, const float* dg, void* dx, int dtype,
                                       int64_t N, int64_t HW, int64_t f, void* stream);
/* Squeeze-and-excitation (tf2/resnet.py:280-311): out = sigmoid(l[n,c]) * x[n,hw,c]; backward
 * dl = sigma'(l) * sum_hw dout*x and dx = dout*sigmoid(l) + dmean[n,c]/HW.  The two tiny
 * "1x1 convs" of the gate run on the dense path (simclr_conv2d_*_simt with H=W=1, any width). */
SIMCLR_API int simclr_se_scale_fwd(const void* x, const float* logits, void* out, int dtype, int64_t N,
                                   int64_t HW, int64_t C, void* stream);
SIMCLR_API int simclr_se_scale_bwd_reduce(const void* dout, const void* x, const float* logits, float* dlogits,
                                          int dtype, int64_t N, int64_t HW, int64_t C, void* stream);
SIMCLR_API int simclr_se_scale_bwd_apply(const void* dout, const float* logits, const float* dmean, void* dx,
                                         int dtype, int64_t N, int64_t HW, int64_t C, void* stream);
/* mask_src == NULL: x = max(x, 0); else x = x * [mask_src > 0]   (fp32, in place) */
SIMCLR_API int simclr_relu_inplace(float* x, const float* mask_src, int64_t n, void* stream);
/* AveragePooling2D(2, stride): stride 2 = FixedPadding(2) + 'VALID'; stride 1 = 'SAME' with the
 * divisor counting valid elements only (SURVEY.md A3).  x [N,H,W,C]. */
SIMCLR_API int simclr_avgpool2x2_fwd(const void* x, void* y, int dtype, int64_t N, int64_t H, int64_t W, int64_t C,
                                     int64_t stride, void* stream);
SIMCLR_API int simclr_avgpool2x2_bwd(const void* dy, void* dx, int dtype, int64_t N, int64_t H, int64_t W,
                                     int64_t C, int64_t stride, void* stream);

/* ------------------------------------------------------------------------- *
 * Input preparation: split views, batch_random_blur, cast, pad 3->4 channels
 * (tf2/model.py:250-259, tf2/data_util.py:323-361,393-440)
 *   features [B,H,W,3*T] fp32 in [0,1]  ->  out [T*B,H,W,4] (view-major)
 *   sigma [T] device floats; selector [T][B] device bytes; tmp [T*B,H,W,3] fp32.
 * ------------------------------------------------------------------------- */
SIMCLR_API int simclr_input_prep(const float* features, void* out, int dtype, int64_t B, int64_t H,
                                 int64_t W, int64_t T, int use_blur, int64_t blur_kernel_size,
                                 const float* sigma, const uint8_t* selector, float* tmp, void* stream);

/* ------------------------------------------------------------------------- *
 * Train-time augmentation on device (tf2/data_util.py:443-475 preprocess_for_train):
 * crop (box from sample_distorted_bounding_box, supplied by the caller) + bicubic
 * resize (tf.image.resize BICUBIC semantics), random_flip_left_right, random_color_jitter
 * (brightness / contrast / saturation / hue in a drawn order, clip after each),
 * grayscale, final clip.  Every tf.random draw is an input.
 *   src        uint8 images [Hs,Ws,3] packed back to back; image i starts at src + src_offset[i]
 *   src_hw     [n][2] int32 {Hs, Ws};  box [n][4] int32 {y, x, h, w};  flip [n] bytes
 *   colour     [n][8] floats {apply_jitter, perm code (op_t = (code >> 2t) & 3; 0 brightness,
 *              1 contrast, 2 saturation, 3 hue), brightness factor, contrast factor,
 *              saturation factor, hue delta, apply_gray, unused}
 *   out        fp32; pixel (i, y, x) channel c at out[((i*height + y)*width + x)*out_pixel_stride
 *              + out_channel_offset + c]  (stride 6 / offsets 0 and 3 write the two views of
 *              tf2/data.py:55-58 straight into the [B,H,W,6] feature tensor)
 * ------------------------------------------------------------------------- */
SIMCLR_API int simclr_augment(const uint8_t* src, const int64_t* src_offset, const int32_t* src_hw,
                              const int32_t* box, const uint8_t* flip, const float* colour, float* out,
                              int64_t n, int64_t height, int64_t width, int64_t out_pixel_stride,
                              int64_t out_channel_offset, void* stream);

/* The other optimizers of build_optimizer (tf2/model.py:29-44), element-wise over flat buffers of n floats.
 * hyper_dev: device float[1] staged by the caller (stream-ordered): SGD {lr}; Adam
 * {lr * sqrt(1 - beta2^t) / (1 - beta1^t)} with t the 1-based step. */
SIMCLR_API int simclr_sgd_momentum_apply(float* w, const float* g, float* v, int64_t n, const float* hyper_dev,
                                         float momentum, int nesterov, void* stream);
SIMCLR_API int simclr_adam_apply(float* w, const float* g, float* m, float* v, int64_t n, const float* hyper_dev,
                                 float beta1, float beta2, float eps, void* stream);

/* ---------------------------------------------------------------------------
 * Collectives over NVLink peer memory, fused into the kernels that consume them (no NCCL on these
 * paths; SURVEY.md 8e).  Every rank owns one allocation of identical layout that all peers have
 * mapped ("symmetric memory"); `peer_bufs_dev` is a DEVICE array of `world` base pointers (entry
 * `rank` is the local one), the remaining arguments are byte offsets into that allocation, the
 * same on every rank.  `seq_dev` points to TWO device uint64: [0] the sequence number (initialised to 1,
 * identical on every rank) that the kernel advances by one per call, [1] a counter (initialise to 0) to which
 * the kernel adds the nanoseconds this rank spent waiting for its peers -- per-rank slack, reported by
 * bench.py.  The calls are CUDA-graph capturable and must be issued in the same order on every rank.  A peer that does not show up within 20 s traps the kernel.
 *
 * SyncBatchNormalization (tf2/resnet.py:54-60): sums [2][C] doubles of THIS replica ->
 * one-shot exchange (region data_off + ((seq % nslot)*world + rank)*slot_bytes of every peer,
 * flags u64 [nslot][world] at flag_off) -> global statistics, summed in rank order, then the
 * arithmetic of simclr_bn_finalize / the coefficient kernel of simclr_bn_bwd_apply. */
SIMCLR_API int simclr_comm_bn_finalize(const double* sums_local, double count_local, const float* gamma,
                                       const float* beta, float eps, float momentum, float* moving_mean,
                                       float* moving_var, float* mean, float* rstd, float* scale,
                                       float* shift, int64_t C, const void* peer_bufs_dev, int rank,
                                       int world, int64_t data_off, int64_t flag_off, int nslot,
                                       int64_t slot_bytes, void* seq_dev, void* stream);
/* coef [3][C]: dy = coef0*dz + coef1*y + coef2 from the GLOBAL (sum dz, sum dz*xhat); dgamma / dbeta
 * receive this replica's sums (the gradient all-reduce adds the replicas). */
SIMCLR_API int simclr_comm_bn_bwd_coef(const double* sums_local, double count_local, const float* mean,
                                       const float* rstd, const float* gamma, float* coef, float* dgamma,
                                       float* dbeta, int64_t C, const void* peer_bufs_dev, int rank,
                                       int world, int64_t data_off, int64_t flag_off, int nslot,
                                       int64_t slot_bytes, void* seq_dev, void* stream);
/* tpu_cross_replica_concat (tf2/objective.py:92-127) as pushes: `nbytes` of `src` land in region
 * data_off + rank*chunk_stride_bytes of every peer; on return (stream order) the `world` regions at
 * data_off of the LOCAL allocation hold all ranks' rows, rank-major.  flags u64 [world] at flag_off;
 * `arrive_dev`: a zeroed device uint32 private to this channel.  One region per channel: the caller
 * must not start gather t+1 of a channel before every rank has consumed gather t (in the training
 * step the gradient collective that ends every step guarantees it). */
SIMCLR_API int simclr_comm_all_gather(const void* src, int64_t nbytes, const void* peer_bufs_dev, int rank,
                                      int world, int64_t data_off, int64_t flag_off,
                                      int64_t chunk_stride_bytes, void* seq_dev, void* arrive_dev,
                                      void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SIMCLR_B200_H_ */
