/* vjepa_b200.h - C ABI of the H100-native V-JEPA pre-training hot path (libvjepa_b200.so).
 *
 * The reference (facebookresearch/jepa) is pure Python: it has no FFI layer, its hot path is the
 * set of torch library calls listed in SURVEY.md section 2.3 (K1..K15).  Every entry point below
 * replaces one of those call sites; the comment on each declaration cites the reference file:line
 * it stands in for.  Conventions (SURVEY.md section 8b):
 *   - plain pointers and sizes only; all pointers are DEVICE pointers unless stated otherwise;
 *     the caller owns every buffer; nothing is retained past the call;
 *   - `stream` is a cudaStream_t passed as void*; every call only ENQUEUES work on it;
 *   - return 0 = enqueued, <0 = argument / shape / alignment violation (nothing launched),
 *     >0 = cudaError_t; vj_last_error_string() gives the thread-local detail;
 *   - bf16 activations are row-major [tokens, features]; "ld" is a row stride in ELEMENTS.
 */
#ifndef VJEPA_B200_H_
#define VJEPA_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VJ_VERSION 100

/* GEMM epilogues */
#define VJ_EPI_NONE 0  /* D = alpha*acc + bias                                             */
#define VJ_EPI_GELU 1  /* D = gelu_erf(alpha*acc + bias); aux_out (bf16, optional) = pre-activation */
#define VJ_EPI_ADD 2   /* D = alpha*acc + bias + aux[rowmap(r), c]   (residual / pos-embed) */
#define VJ_EPI_DGELU 3 /* D = (alpha*acc + bias) * gelu_erf'(aux[r, c])                     */
#define VJ_EPI_MUL 4   /* D = (alpha*acc + bias) * aux[r, c]                                */
#define VJ_EPI_GELU_GRAD 5 /* like GELU, but aux_out (bf16) = gelu_erf'(pre-activation): the fc2 dgrad then
                              only needs VJ_EPI_MUL (one erf per element per step instead of two)      */

const char* vj_last_error_string(void);
int vj_version(void);
/* Number of kernels this library has launched so far in this process (monotonic). */
long long vj_launch_count(void);
/* Cap the grid of the PERSISTENT kernels (GEMM, second-generation attention) at n SMs (n <= 0: all SMs).  Data-parallel
 * training leaves a few SMs to NCCL's CTAs while gradient buckets are in flight (jepa_b200/distributed.py). */
int vj_set_sm_limit(int n);
/* CUtensorMap cache statistics: which = 0 -> hits, 1 -> misses (driver encode calls) since the library was loaded. */
long long vj_tmap_cache_stats(int which);

/* D[M,N] = epi(alpha * A[M,K] . B[N,K]^T), bf16 operands, fp32 accumulate (wgmma).
 * a_mn = 0: A stored [M,K] (K contiguous, ld = lda);  a_mn = 1: A stored [K,M] (M contiguous).
 * b_mn = 0: B stored [N,K];                            b_mn = 1: B stored [K,N].
 * Supported (a_mn,b_mn): (0,0) forward / nn.Linear, (0,1) dgrad, (1,1) wgrad.
 * d_f32: D is fp32 (else bf16).  accumulate!=0 or split_k>1 reduce-add into fp32 D.  split_k < 0 (with accumulate,
 * no epilogue): stream-K - the (tile, k-block) space is cut into one equal contiguous range per SM (weight gradients).
 * bias: fp32 [N] or NULL.  aux: bf16 or fp32 (aux_f32) tile source for ADD / MUL / DGELU.  An fp32 aux may be
 * row-mapped: row r reads aux row aux_rowmap[r] if given, else r % aux_period if aux_period > 0, else r (pos-embed
 * add of the patch-embed GEMM); a bf16 aux is a plain [M,N] matrix (residual stream / saved gelu').  No aux epilogue
 * combines with split-K (every piece runs the epilogue).  aux_out (bf16 [M,N], optional) is the second output of the GELU epilogues.
 * Replaces F.linear / Conv3d-as-GEMM and their backward:
 *   src/models/utils/modules.py:31-34,63,76; src/models/predictor.py:194,237;
 *   src/models/utils/patch_embed.py:54-57. */
int vj_gemm(const void* A, long long lda, int a_mn, const void* B, long long ldb, int b_mn,
            void* D, long long ldd, int d_f32, int M, int N, int K, const float* bias, float alpha,
            int epi, const void* aux, long long ldaux, int aux_f32, const int* aux_rowmap,
            int aux_period, void* aux_out, long long ldauxout, int split_k, int accumulate,
            void* stream);
/* vj_gemm with fp16 operands: A, B and every 16-bit D / aux / aux_out are fp16 (d_f32 = 0 / aux_f32 = 0), fp32 D and
 * fp32 aux as above.  Frozen evaluation under torch.cuda.amp.autocast(dtype=torch.float16)
 * (evals/video_classification_frozen/eval.py:323, evals/image_classification_frozen/eval.py:284), where F.linear and
 * the Conv3d of the patch embedding run in fp16.  Instantiated: forward (0,0) with NONE / GELU / GELU_GRAD / ADD (fp16
 * or row-mapped / periodic fp32 aux), dgrad (0,1) plain and MUL, wgrad (1,1) into fp32. */
int vj_gemm_f16(const void* A, long long lda, int a_mn, const void* B, long long ldb, int b_mn,
                void* D, long long ldd, int d_f32, int M, int N, int K, const float* bias, float alpha,
                int epi, const void* aux, long long ldaux, int aux_f32, const int* aux_rowmap,
                int aux_period, void* aux_out, long long ldauxout, int split_k, int accumulate,
                void* stream);

/* Dense var-len flash attention forward (wgmma).  qkv bf16 [T, 3*H*HD] (q|k|v thirds, head-major),
 * out bf16 [T, H*HD], lse2 fp32 [H, T] (log2 domain).  Sequences are the row ranges
 * [cu_seqlens[s], cu_seqlens[s+1]) (device int32 [nseq+1]); max_len = longest sequence.
 * HD in {32, 64, 128} (hd=24 heads are zero-padded to 32 by the weight layout).
 * Replaces F.scaled_dot_product_attention, src/models/utils/modules.py:66-69. */
int vj_attn_fwd(const void* qkv, void* out, float* lse2, const int* cu_seqlens, int nseq, int max_len,
                int H, int HD, int T, float scale, void* stream);
/* vj_attn_fwd with fp16 qkv and out (P rounded to fp16 for P V): the SDPA of modules.py:66-69 under the evals'
 * autocast(float16) (evals/video_classification_frozen/eval.py:323). */
int vj_attn_fwd_f16(const void* qkv, void* out, float* lse2, const int* cu_seqlens, int nseq, int max_len,
                    int H, int HD, int T, float scale, void* stream);

/* Backward of the above: dqkv bf16 [T, 3*H*HD] from dout bf16 [T, H*HD]; delta_ws fp32 [H*T] scratch.
 * dq_acc_ws: unused (may be NULL); kept so callers built against earlier versions of this header still link.
 * (autograd of modules.py:66-69). */
int vj_attn_bwd(const void* qkv, const void* out, const void* dout, const float* lse2, float* delta_ws,
                void* dqkv, float* dq_acc_ws, const int* cu_seqlens, int nseq, int max_len, int H, int HD, int T,
                float scale, void* stream);

/* LayerNorm over the last dim, one warp per row.  x bf16|fp32 [T,D] -> y bf16|fp32; mean/rstd fp32 [T]
 * (nullable) are saved for the backward.  x_f32 / y_f32 = 2: fp16, paired with fp16 or fp32 (LayerNorm under the
 * evals' autocast(float16), evals/video_classification_frozen/eval.py:323: fp16 in, fp32 out, or fused with the
 * following Linear's cast to fp16).  nn.LayerNorm(eps=1e-6) at modules.py:115,119,
 * vision_transformer.py:192-193, predictor.py:233. */
int vj_layernorm_fwd(const void* x, int x_f32, void* y, int y_f32, const float* gamma, const float* beta,
                     float* mean, float* rstd, int T, int D, float eps, void* stream);
size_t vj_layernorm_bwd_workspace(int T, int D);
/* dx = dres + LN'(dy) (dres nullable, same dtype as x/dx); dgamma/dbeta fp32 [D] are ACCUMULATED (+=). */
int vj_layernorm_bwd(const void* dy, const void* x, int x_f32, const float* gamma, const float* mean,
                     const float* rstd, const void* dres, void* dx, float* dgamma, float* dbeta,
                     void* workspace, size_t ws_bytes, int T, int D, void* stream);
/* vj_layernorm_bwd with an fp16 dy [T,D] and fp32 x / dres / dx (workspace as vj_layernorm_bwd_workspace): the
 * backward of the attentive probe's norm1 / norm2 (modules.py:172,174) under the evals' autocast(float16)
 * (evals/video_classification_frozen/eval.py:323): LayerNorm reads the fp32 features / residual, and its gradient comes
 * from the next fp16 Linear.  dgamma / dbeta fp32 [D] are accumulated (+=) in fp32. */
int vj_layernorm_bwd_f16(const void* dy, const float* x, const float* gamma, const float* mean, const float* rstd,
                         const float* dres, float* dx, float* dgamma, float* dbeta, void* workspace, size_t ws_bytes,
                         int T, int D, void* stream);

/* out[N] += column sums of in[T,N] (bf16|fp32) over rows r with lo <= r % period < hi (period<=0: all).
 * Bias gradients of every nn.Linear; mask-token gradient (predictor.py:207-210 backward). */
int vj_colsum(const void* in, int in_f32, float* out, long long T, int N, long long ld, int period, int lo,
              int hi, void* stream);
/* vj_colsum of fp16 rows (in fp16 [T,N], out fp32 [N] +=): the bias gradients of the attentive probe's kv, q, fc1 and
 * fc2 Linears when the probe trains under the evals' autocast(float16) (evals/video_classification_frozen/eval.py:323,
 * evals/image_classification_frozen/eval.py:284; backward of modules.py:31-34,138-153). */
int vj_colsum_f16(const void* in, float* out, long long T, int N, long long ld, int period, int lo, int hi,
                  void* stream);

/* Tubelet im2col: clips fp32 [B,C,T,H,W] -> patches bf16 [B*K', C*tub*ps*ps] in Conv3d weight order
 * (c,dt,dh,dw); idx (int64 [B,K], nullable) gathers tokens first (context path), else K' = all tokens.
 * PatchEmbed3D, src/models/utils/patch_embed.py:47-57 (+ apply_masks, vision_transformer.py:178-180). */
int vj_im2col_tubelets(const float* clips, void* patches, const long long* idx, int B, int C, int T, int H,
                       int W, int tubelet, int patch, int K, void* stream);
/* The same with fp16 patches: the Conv3d input cast of PatchEmbed3D under the evals' autocast(float16)
 * (evals/video_classification_frozen/eval.py:323). */
int vj_im2col_tubelets_f16(const float* clips, void* patches, const long long* idx, int B, int C, int T, int H,
                           int W, int tubelet, int patch, int K, void* stream);

/* Positional-embedding resampling for off-size encoder inputs (interpolate_pos_encoding,
 * src/models/vision_transformer.py:197-246): fp32 in [Nt,Nh,Nw,D] -> fp32 out [T,H,W,D], bit-exact with torch's CPU
 * F.interpolate(scale_factor=..., align_corners=False).  mode 3: trilinear with per-axis scale factors; mode 2:
 * bicubic (A = -0.75) over a 2-D grid (Nt = T = 1, scale_t ignored).  Each output extent must be
 * floor(in * scale); D a multiple of 4, both pointers 16-byte aligned. */
int vj_pos_interp(const float* in, float* out, int Nt, int Nh, int Nw, int T, int H, int W, int D, double scale_t,
                  double scale_h, double scale_w, int mode, void* stream);

/* out[b,k,:] = x[b, idx[b,k], :], rows of row_bytes (multiple of 16).  apply_masks, src/masks/utils.py:11-23. */
int vj_gather_rows(const void* x, void* out, const long long* idx, int B, int N, int K, int row_bytes,
                   void* stream);
/* dx[b, idx[b,k], :] += dy[b,k,:]  (backward of the gather; indices unique per row). */
int vj_scatter_rows_add(const void* dy, void* dx, const long long* idx, int B, int N, int K, int D, int f32,
                        void* stream);

/* Targets: out fp32 [B,K,D] = layer_norm(LN_affine(x[b, idx[b,k]]; eps_norm), eps_target, no affine).
 * vision_transformer.py:192-193 + app/vjepa/train.py:426-428 fused, gathered rows only. */
int vj_target_ln_gather(const void* x, float* out, const long long* idx, const float* gamma, const float* beta,
                        int B, int N, int K, int D, float eps_norm, float eps_target, void* stream);

/* Predictor input for one mask: x[b,:Ke] = emb[b] + pos[idx_ctx[b]]; x[b,Ke:] = mask_token + pos[idx_tgt[b]].
 * emb bf16 [B*Ke,Dp], pos fp32 [N,Dp], x bf16|fp32 [B,Ke+Kp,Dp].  src/models/predictor.py:194-221. */
int vj_pred_assemble_fwd(const void* emb, const float* pos, const float* mask_token, const long long* idx_ctx,
                         const long long* idx_tgt, void* x, int x_f32, int B, int Ke, int Kp, int Dp, void* stream);
/* demb bf16 [B*Ke,Dp] = dx[:, :Ke];  dmask_token fp32 [Dp] += sum of dx[:, Ke:]. */
int vj_pred_assemble_bwd(const void* dx, int dx_f32, void* demb, float* dmask_token, int B, int Ke, int Kp,
                         int Dp, void* stream);
/* scatter=0: dst[B*Kp,D] = src[B,Ke+Kp,D][:, Ke:]  (predictor.py:236);  scatter=1: the reverse
 * (zero_ctx: also zero the first Ke rows of every sequence). */
int vj_seq_slice(const void* src, void* dst, int f32, int B, int Ke, int Kp, int D, int scatter, int zero_ctx,
                 void* stream);

/* loss_sum[0] += weight * sum |z - h|   (z bf16, h fp32, n elements; weight = 1/(M*n) gives the
 * per-mask mean averaged over M masks).  app/vjepa/train.py:440-446. */
int vj_l1_loss_fwd(const void* z, const float* h, float* loss_sum, long long n, float weight, void* stream);
/* dz bf16 = sign(z - h) * scale * (grad_scale_dev ? *grad_scale_dev : 1). */
int vj_l1_loss_bwd(const void* z, const float* h, const float* grad_scale_dev, float scale, void* dz,
                   long long n, void* stream);
/* General exponent of loss_fn (app/vjepa/train.py:440-446, loss_exp != 1): *loss_sum += weight * sum |z - h|^p;
 * dz bf16 = sign(z - h) |z - h|^(p-1) * scale * (grad_scale_dev ? *grad_scale_dev : 1). */
int vj_lp_loss_fwd(const void* z, const float* h, float* loss_sum, long long n, float weight, float p, void* stream);
int vj_lp_loss_bwd(const void* z, const float* h, const float* grad_scale_dev, float scale, void* dz, long long n, float p,
                   void* stream);
/* Backward of the variance regulariser (reg_fn + relu-mean, app/vjepa/train.py:448-449,458-459, reg_coeff != 0) for one
 * mask: dz[b,k,d] = -[pstd_total[b,d] < 1] / (B D) * weight * (z - mean_k z) / ((K-1) sqrt(var_k + eps)) * scale * *grad_scale_dev. */
int vj_token_std_bwd(const void* z, const float* pstd_total, const float* grad_scale_dev, float scale, void* dz, int B, int K,
                     int D, float eps, float weight, void* stream);
/* pstd[b,d] += weight * sqrt(var_unbiased_k(z[b,k,d]) + eps).  reg_fn, app/vjepa/train.py:448-449. */
int vj_token_std_accum(const void* z, float* pstd, int B, int K, int D, float eps, float weight, void* stream);

/* ---- attentive probe (frozen-encoder evaluation, SURVEY section 8 row f4) ----------------------- */
/* out bf16 [B*nq, H*HD] = softmax(q k^T * scale) v per (clip, head, query): CrossAttention.forward's SDPA
 * (src/models/utils/modules.py:138-153) for the nq learned query tokens of AttentivePooler
 * (src/models/attentive_pooler.py:96-102).  q bf16 [B*nq, H*HD]; kv bf16 [B*S, 2*H*HD] = the kv Linear's output
 * (k | v halves, head-major).  HD in {32, 64, 80, 128}. */
int vj_cross_attn_fwd(const void* q, const void* kv, void* out, int B, int nq, int S, int H, int HD, float scale,
                      void* stream);
/* Same as vj_cross_attn_fwd (out bitwise identical), and also writes the softmax statistics lse2 fp32 [B*nq, H]
 * (row b*nq + j, column head; log2 domain: lse2 = log2 sum_k exp2(scale log2e q.k)) for the backward. */
int vj_cross_attn_fwd_lse(const void* q, const void* kv, void* out, float* lse2, int B, int nq, int S, int H, int HD,
                          float scale, void* stream);
/* Bytes of fp32 workspace vj_cross_attn_bwd needs (per-key-chunk dq partials). */
size_t vj_cross_attn_bwd_workspace(int B, int nq, int S, int H, int HD);
/* Backward of the above (autograd of modules.py:138-153 for training the attentive probe).  From q, kv, out, dout
 * (bf16, layouts as in the forward) and lse2: dq fp32 [B*nq, H*HD], dkv bf16 [B*S, 2*H*HD] (dk | dv halves).
 * dk / dv sum over the clip's nq queries.  Deterministic: no atomics, every dkv element is written once and dq is
 * reduced over key chunks in a fixed order.  HD in {32, 64, 80, 128}. */
int vj_cross_attn_bwd(const void* q, const void* kv, const void* out, const void* dout, const float* lse2, float* dq,
                      void* dkv, void* workspace, size_t ws_bytes, int B, int nq, int S, int H, int HD, float scale,
                      void* stream);
/* The three above with fp16 q / kv / out / dout / dkv (lse2, dq and the workspace stay fp32; same workspace query,
 * same key chunks and reduction order, still no atomics): CrossAttention's SDPA and its autograd under the evals'
 * autocast(float16) (evals/video_classification_frozen/eval.py:323, evals/image_classification_frozen/eval.py:284),
 * where the q / kv Linears emit fp16 and SDPA runs in fp16.  Every fp16 store rounds to nearest; a value past 65504
 * becomes +-inf. */
int vj_cross_attn_fwd_f16(const void* q, const void* kv, void* out, int B, int nq, int S, int H, int HD, float scale,
                          void* stream);
int vj_cross_attn_fwd_lse_f16(const void* q, const void* kv, void* out, float* lse2, int B, int nq, int S, int H, int HD,
                              float scale, void* stream);
int vj_cross_attn_bwd_f16(const void* q, const void* kv, const void* out, const void* dout, const float* lse2, float* dq,
                          void* dkv, void* workspace, size_t ws_bytes, int B, int nq, int S, int H, int HD, float scale,
                          void* stream);

/* ---- flat-buffer parameter kernels ------------------------------------------------------------ */
/* dst bf16[n] = src fp32[n]: the per-step bf16 shadow of the fp32 master weights (what autocast's
 * weight cast does for every F.linear under torch.cuda.amp.autocast, app/vjepa/train.py:453). */
int vj_cast_f32_bf16(const float* src, void* dst, long long n, void* stream);
/* dst fp16[n] = src fp32[n]: the fp16 shadow, autocast(float16)'s weight cast in the eval loops
 * (evals/video_classification_frozen/eval.py:323, evals/image_classification_frozen/eval.py:284). */
int vj_cast_f32_f16(const float* src, void* dst, long long n, void* stream);
/* Tensors viewed as [outer, G, hd, inner] <-> [outer, G, hdp, inner]: zero-pad heads (unpad_add=0) or
 * accumulate the padded fp32 gradient back into the unpadded one (unpad_add=1).  dst_f32 = 2: an fp16 destination
 * from an fp32 source (head-padded weights of an fp16 forward, ViT-H's hd 80 -> 128).  Predictor heads are
 * hd = 384/16 = 24 (app/vjepa/utils.py:119) and run as 32-wide wgmma tiles. */
int vj_head_pad(const void* src, int src_f32, void* dst, int dst_f32, long long outer, int G, int hd, int hdp,
                long long inner, int unpad_add, void* stream);
/* k = k*m + one_minus_m*q over a flat fp32 buffer, rounding op-for-op like
 * param_k.mul_(m).add_((1.-m)*param_q)  (app/vjepa/train.py:484-487). */
int vj_ema_update(float* k, const float* q, long long n, float m, float one_minus_m, void* stream);
/* One AdamW step over a flat fp32 segment (torch.optim.AdamW rule; app/vjepa/utils.py:173-194).
 * inv_scale_dev / found_inf_dev (device scalars, nullable) implement GradScaler unscale + skip. */
int vj_adamw_step(float* p, const float* g, float* m, float* v, long long n, float lr, float beta1, float beta2,
                  float eps, float weight_decay, int step, const float* inv_scale_dev, const float* found_inf_dev,
                  void* stream);
/* AdamW over a whole flat parameter buffer in one launch: group_ids (device uint8 per 64-element block)
 * select lr / weight decay from the 4-entry HOST tables lr4 / wd4; id 255 = frozen or padding (skipped). */
/* step_dev (device fp32 scalar, nullable): when given the step count is read from (and, unless found_inf, advanced on) the
 * device, so a GradScaler-skipped step does not advance the bias correction (torch's fused/capturable AdamW semantics;
 * `step` is then ignored).  shadow_bf16 (nullable, n elements): bf16 copy of the updated parameters written in the same
 * pass - the tensor-core operands of the next step (replaces the separate vj_cast_f32_bf16 pass). */
int vj_adamw_flat(float* p, const float* g, float* m, float* v, const unsigned char* group_ids, long long n,
                  const float* lr4, const float* wd4, float beta1, float beta2, float eps, int step,
                  const float* inv_scale_dev, const float* found_inf_dev, float* step_dev, void* shadow_bf16, void* stream);
/* vj_ema_update that also writes the bf16 shadow of the updated k (target-encoder weights of the next step). */
int vj_ema_update_shadow(float* k, const float* q, long long n, float m, float one_minus_m, void* shadow_bf16, void* stream);

/* ---- segmented statistics over flat gradient / moment buffers (logging + clipping without host syncs) ------------
 * seg: device uint16 per 64-element block of the flat buffer = parameter-tensor id, 0xFFFF = skip (frozen / padding).
 * vj_grad_unscale_stats: one pass over the flat gradient buffer: g *= *inv_scale_dev (if given; written back iff
 * write_back), *found_inf_dev = 1 if any value is non-finite, sumsq_out[id] += sum of squares of tensor id.
 * Replaces torch._amp_foreach_non_finite_check_and_unscale_ behind scaler.unscale_ (app/vjepa/train.py:463) and the
 * per-tensor torch.norm loop of grad_logger (src/utils/logging.py:91-105). */
int vj_grad_unscale_stats(float* g, const unsigned short* seg, long long n, const float* inv_scale_dev,
                          float* found_inf_dev, float* sumsq_out, int write_back, void* stream);
/* out[id] += sum |x| over tensor id  (adamw_logger's exp_avg.abs().mean() / exp_avg_sq.abs().mean(), logging.py:108-118). */
int vj_seg_abs_sum(const float* x, const unsigned short* seg, long long n, float* out, void* stream);
/* total_norm = sqrt(sum sumsq[0..n_seg)), coef = min(1, max_norm / (total_norm + 1e-6)), both device scalars
 * (torch.nn.utils.clip_grad_norm_, app/vjepa/train.py:468-471). */
int vj_clip_coef(const float* sumsq, int n_seg, float max_norm, float* total_norm_out, float* coef_out, void* stream);
/* x *= *coef_dev when *coef_dev < 1 (no memory traffic otherwise). */
int vj_scale_flat(float* x, long long n, const float* coef_dev, void* stream);
/* out[0] += sum(x^2) over a flat fp32 buffer (grad-norm statistics, src/utils/logging.py:91-105). */
int vj_sumsq(const float* x, long long n, float* out, void* stream);

/* ---- GPU input pipeline (SURVEY 8f-3) -------------------------------------------------------------------------
 * Decoded uint8 frames -> random-resized crop (bilinear, align_corners = False) -> horizontal flip -> (x - 255 mean) /
 * (255 std) -> out [B, 3, T, S, S] (fp32 or bf16), one launch per batch.  src_u8: device buffer holding every clip's
 * frames [T, H_b, W_b, 3]; params: device table, one 40-byte record per clip = {int64 byte offset into src_u8,
 * int32 H, W, i, j, h, w (crop box), flip, pad}.  mean3 / std3: HOST arrays of 3 floats (0..1 scale).
 * Replaces VideoTransform.__call__ (app/vjepa/transforms.py:86-117: float conversion, random_resized_crop,
 * horizontal_flip, _tensor_normalize_inplace :140-153) for the non-auto-augment path; the random decisions are drawn
 * on the host in the reference's RNG order (jepa_b200/transforms.py). */
int vj_clip_preprocess(const void* src_u8, const void* params, void* out, int out_f32, int B, int T, int S,
                       const float* mean3, const float* std3, void* stream);

/* Deterministic evaluation views: uint8 frames -> OpenCV INTER_LINEAR short-side resize (bit-exact fixed point) ->
 * S x S window -> / 255 -> (x - mean) / std -> fp32 or bf16 [3, T, S, S] per view, one launch for every (clip, segment,
 * view).  jobs: device table, one 32-byte record per view = {int64 byte offset of the clip in src_u8, int64 element
 * offset of the view in out, int32 H, W, ytab, xtab}; tab: device int4 table (source index 0, source index 1, weight 0,
 * weight 1) per resized row / column, OpenCV's 11-bit weights, S consecutive entries from ytab (rows) and xtab
 * (columns) per view.  mean3 / std3: HOST arrays of 3 floats.  Replaces EvalVideoTransform and
 * VideoTransform(training=False) of evals/video_classification_frozen/utils.py; the geometry and the tables come from
 * jepa_b200/transforms.py. */
int vj_clip_views(const void* src_u8, const void* jobs, const void* tab, void* out, int out_f32, int n_jobs, int T, int S,
                  const float* mean3, const float* std3, void* stream);

/* Training transform with RandAugment and random erasing: uint8 frames -> n_layers RandAugment layers (PIL 12
 * arithmetic, bit-exact) -> random-resized crop (bilinear) -> flip -> (x - 255 mean) / (255 std) -> erase box filled
 * with N(0, 1) (Philox keyed by the clip's seed) -> fp32 or bf16 [B, 3, T, S, S].
 * buf0 / buf1: two device uint8 work buffers of equal size; buf0 holds the frames on entry, both are overwritten.
 * clips: device table, one 64-byte record per clip = {int64 byte offset of the clip [T, H, W, 3] in each buffer, int32 H,
 * W, i, j, h, w (crop box), flip, final_buf (buffer holding the clip after the last layer), erase top, left, h, w (h 0:
 * no erase), uint64 seed}.  ops: device table [n_layers, B] of 64-byte records = {double inverse affine matrix[6],
 * int32 op (index in jepa_b200.transforms.RA_OPS, -1 skipped), float factor, int32 argument, int32 input buffer}.
 * hist: device int32 scratch of n_layers * B * T * 1024.  layer_flags: HOST int[n_layers], bit 0: some op applied,
 * bit 1: some op reads the frame histogram.  mean3 / std3: HOST arrays of 3 floats.  At most 2 launches per layer + 1.
 * Replaces src/datasets/utils/video/randaugment.py:51-180 / :324-465 (RandAugment on PIL frames),
 * src/datasets/utils/video/randerase.py:116-156 (RandomErasing._erase_cube, mode 'pixel') and the training paths of
 * app/vjepa/transforms.py:86-115 and evals/video_classification_frozen/utils.py:251-283; the decisions come from
 * jepa_b200/transforms.py. */
int vj_clip_augment(void* buf0, void* buf1, const void* clips, const void* ops, void* hist, const int* layer_flags,
                    int n_layers, void* out, int out_f32, int B, int T, int S, const float* mean3, const float* std3,
                    void* stream);

/* Frozen image evaluation, validation: uint8 RGB images of mixed sizes -> PIL 12's Image.resize (BILINEAR / BICUBIC,
 * Resample.c 8-bit fixed point, bit-exact) -> S x S window -> torchvision ToTensor + Normalize in fp32 ((v / 255 - mean) /
 * std, each step rounded) -> out [B, 3, S, S] fp32 or bf16.  2 launches.  src_u8: device buffer of every image [H, W, 3];
 * jobs: device table, one 64-byte record per image = {int64 byte offset of the image in src_u8, int64 byte offset of its
 * rows in tmp, int32 W, first source row r0, row count nrows, first source column c0, xtab, ytab, xk, yk, flip, pad[3]};
 * coefs: device int32 table; S entries of xk ints from xtab (output columns) and S entries of yk ints from ytab (output
 * rows), each {first tap (columns: from c0; rows: from r0), tap count, int32 weights at 22 fractional bits}.  tmp: device
 * uint8 scratch of nrows * S * 3 bytes per image at its tmp offset.  mean3 / std3: HOST arrays of 3 floats.  Replaces
 * Resize(int(S * 256 / 224)) / CenterCrop(S) / ToTensor / Normalize of evals/image_classification_frozen/eval.py:405-409;
 * the tables come from jepa_b200/image_transforms.py. */
int vj_image_views(const void* src_u8, const void* jobs, const void* coefs, void* tmp, void* out, int out_f32, int B, int S,
                   const float* mean3, const float* std3, void* stream);

/* Frozen image evaluation, training: the resample of vj_image_views over each image's random-resized-crop box (jobs /
 * coefs / tmp as there; flip mirrors the result) into buf0 [B, S, S, 3] -> n_layers AutoAugment layers through the
 * RandAugment kernels of vj_clip_augment (T = 1, clips / ops / hist / layer_flags as there; geometric ops fill with the
 * HOST RGB fill3) -> ToTensor + Normalize (as vj_image_views) -> erase box copied from noise (device fp32; a clip record's
 * seed field is the element offset of its [3, eh, ew] block; may be NULL when no image erases) -> out [B, 3, S, S] fp32
 * or bf16.  At most 2 + 2 * n_layers + 1 launches.  Replaces timm's create_transform(is_training=True,
 * auto_augment='original', interpolation='bicubic', re_prob=0.25, re_mode='pixel', re_count=1) of
 * evals/image_classification_frozen/eval.py:392-403; the decisions come from jepa_b200/image_transforms.py. */
int vj_image_augment(const void* src_u8, const void* jobs, const void* coefs, void* tmp, void* buf0, void* buf1,
                     const void* clips, const void* ops, void* hist, const int* layer_flags, int n_layers,
                     const float* noise, void* out, int out_f32, int B, int S, const float* mean3, const float* std3,
                     const unsigned char* fill3, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* VJEPA_B200_H_ */
