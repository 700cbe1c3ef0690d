/* b200vq.h -- C ABI of libb200vq.so: the H100 (sm_90a) kernels behind the ViT-VQGAN hot path of
 * thuanz123/enhancing-transformers.
 *
 * Boundary (SURVEY.md section 8b).  The reference has no FFI of its own on this path: its
 * ViTEncoder / ViTDecoder / VectorQuantizer are nn.Modules whose arithmetic lives in ATen.  The
 * drop-in boundary is therefore the nn.Module surface (enhancing_transformers_b200/layers.py,
 * quantizers.py) and *this* header is what those modules bind with ctypes -- each entry point
 * names the reference line(s) whose ATen calls it replaces.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer to fp32 unless typed otherwise; nothing is allocated or
 *     freed inside the library, workspaces are sized by the *_workspace_bytes queries and owned
 *     by the caller (PyTorch's caching allocator on the Python side);
 *   - every call is asynchronous on `stream` (a cudaStream_t passed as void*), never
 *     synchronises the device, and returns 0 on success or a negative code; the message is
 *     available from b200vq_last_error() (thread local);
 *   - matrices are row-major with an explicit leading dimension in elements;
 *   - `round_out != 0` stores values rounded to tf32 (round-to-nearest, fp32 container) because
 *     the tensor is only ever consumed as a tf32 tensor-core operand, which would otherwise
 *     truncate the low 13 mantissa bits;
 *   - fp16 buffers (void*) are plain IEEE binary16 arrays; they only ever hold GEMM operands.
 */
#ifndef B200VQ_H_
#define B200VQ_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200VQ_VERSION 202 /* 0.2.2 */

int b200vq_version(void);
const char* b200vq_last_error(void);
/* compiled-for architecture string, e.g. "sm_90a" */
const char* b200vq_arch(void);
/* number of kernel launches issued through this library since load (bench.py's gpu_launches) */
long long b200vq_launch_count(void);
/* cap the grid of the persistent (one CTA per SM) GEMM / attention kernels at n CTAs, 0 = no cap.  Leaves SMs to a
 * concurrently running NCCL all-reduce (reference main.py:54-57 strategy="ddp").  Also read once from the environment
 * variable B200VQ_SM_LIMIT. */
int b200vq_set_sm_limit(int n);

/* ---- GEMM: C[M,N] = epi( alpha * A . B^T ) on mma.sync tensor cores, fp32 accumulate ------------------
 * Replaces nn.Linear / Conv2d(k=s) / ConvTranspose2d(k=s) forward, dgrad and wgrad:
 *   layers.py:99-101 (FeedForward), :118,:120 (to_qkv, to_out), :169 (patch embed), :204 (to_pixel),
 *   vitvqgan.py:38-39 (pre_quant / post_quant).
 * a_major/b_major: 0 = operand stored [rows, K] (K contiguous); 1 = stored [K_total, rows]
 * (rows contiguous).  splits > 1 contracts K_total = K*splits in `splits` slices and writes
 * slice z to C + z*c_split_stride (reduce with b200vq_splitk_reduce).
 * Epilogue, in this order: * alpha; + bias[N]; act (0 none, 1 tanh -- layers.py:100);
 * * (1 - aux^2) (tanh backward); + res[row % res_row_mod or row] (residual add layers.py:147-148
 * or positional table :179,:210); tf32 rounding / fp16 conversion.
 * colsum_part (nullable, [ceil(M/16)][N], splits must be 1): receives the column sums of every 16-row group of
 * the stored C -- summed over the groups (b200vq_colsum) they are the bias gradient of the Linear whose
 * pre-activation gradient this GEMM produced (net.0, layers.py:99), without another pass over C.
 * cta_group: accepted and ignored (one CTA per tile).  bn in {0=auto,64,128,192,256} picks the tile width of the tf32
 * kinds (64 or 128 columns); the fp16 kind always runs on 128 x 256 tiles.
 *
 * Three operand flavours:
 *   gemm_tf32   A, B fp32, tf32 MMA (10-bit mantissa; the hardware truncates, so producers round to nearest).
 *   gemm_3xtf32 A, B fp32 plus their truncation residues A_lo, B_lo (b200vq_split_tf32_lo): the
 *               error-compensated product A_lo.B + A.B_lo + A.B -- fp32-grade, used by precision="parity".
 *   gemm_f16    A, B fp16 (f16 MMA: the same 11-bit significand as tf32 at twice the tensor rate and half the
 *               operand bytes); C fp32, or fp16 when out_half (then aux is fp16 too; no residual / split-K).
 *               alpha (device scalar, nullable) undoes the power-of-two scale fp16 gradient operands carry. */
int b200vq_gemm_tf32(const float* A, long long lda, int a_major, const float* B, long long ldb, int b_major,
                     float* C, long long ldc, int M, int N, int K, int splits, long long c_split_stride,
                     const float* bias, const float* res, long long ldres, int res_row_mod,
                     const float* aux, long long ldaux, float* colsum_part, int act, int round_out, int cta_group,
                     int bn, void* stream);
int b200vq_gemm_3xtf32(const float* A, const float* A_lo, long long lda, int a_major, const float* B, const float* B_lo,
                       long long ldb, int b_major, float* C, long long ldc, int M, int N, int K, int splits,
                       long long c_split_stride, const float* bias, const float* res, long long ldres, int res_row_mod,
                       const float* aux, long long ldaux, float* colsum_part, int act, int cta_group, int bn, void* stream);
int b200vq_gemm_f16(const void* A, long long lda, int a_major, const void* B, long long ldb, int b_major, void* C,
                    long long ldc, int out_half, int M, int N, int K, int splits, long long c_split_stride,
                    const float* bias, const float* res, long long ldres, int res_row_mod, const void* aux,
                    long long ldaux, float* colsum_part, int act, int round_out, const float* alpha, int cta_group,
                    int bn, void* stream);
/* out = alpha * sum_z part[z] (alpha: device scalar or NULL) */
int b200vq_splitk_reduce(const float* part, int splits, long long n, long long split_stride, const float* alpha,
                         float* out, void* stream);

/* ---- LayerNorm (nn.LayerNorm(dim), eps 1e-5: layers.py:88,143) ---------------------------------
 * y (fp32, optionally tf32-rounded) and/or y16 (fp16) receive the normalised rows; either may be NULL. */
int b200vq_layernorm_fwd(const float* x, const float* gamma, const float* beta, float* y, void* y16, float* mean,
                         float* rstd, int M, int D, int round_out, void* stream);
size_t b200vq_layernorm_bwd_workspace_bytes(int D);
/* dx = LN'(dy) (+ dres, the skip-connection gradient of layers.py:147-148).  dxsum (nullable, [D]) receives the
 * column sums of dx: dx is also the gradient at the bias of the Linear that wrote this residual stream
 * (to_out layers.py:118, net.2 layers.py:101), so that bias gradient costs no extra pass over dx.
 * dx16 (nullable): fp16 copy of dx multiplied by *dx16_scale, the operand of the next block's fp16 GEMMs.
 * dy: fp32, or (dy_half = 1) fp16 carrying a gradient scale -- the fp16 output of a dgrad GEMM -- multiplied by
 * *dy_scale (device scalar 1/S, or NULL) as it is read. */
int b200vq_layernorm_bwd(const void* dy, int dy_half, const float* dy_scale, const float* x, const float* mean,
                         const float* rstd, const float* gamma, const float* dres, float* dx, void* dx16,
                         const float* dx16_scale, float* dgamma, float* dbeta, float* dxsum, int M, int D, int round_out,
                         void* workspace, size_t ws_bytes, void* stream);

/* ---- attention core (layers.py:124-130): softmax(q k^T * scale) v, no mask -----------------------
 * qkv is the [B*N, 3*heads*dh] output of to_qkv (q | k | v thirds, head h at columns h*dh);
 * out is [B*N, heads*dh] (fp32, or fp16 when out_half); lse [B*heads*N] holds log-sum-exp of the scaled scores
 * (saved for backward instead of the [B,h,N,N] probabilities the reference keeps).  dh must be 64 or 32. */
int b200vq_attention_fwd(const float* qkv, void* out, int out_half, float* lse, int B, int N, int heads, int dh,
                         float scale, int round_out, void* stream);
/* dqkv [B*N, 3*heads*dh] from dout (fp32); `out` as the forward stored it; delta [B*heads*N] is scratch
 * (rowsum(dout*out)).  dqkv_half: store fp16, multiplied by *dqkv_scale (nullable). */
int b200vq_attention_bwd(const float* qkv, const void* out, int out_half, const float* lse, const float* dout,
                         void* dqkv, int dqkv_half, const float* dqkv_scale, float* delta, int B, int N, int heads,
                         int dh, float scale, int round_out, void* stream);
/* fp16-operand core (dh == 64): qkv16 / out16 / dout16 / dqkv16 are fp16 matrices of the shapes above; tensor-core
 * operands fp16, scores / softmax / accumulation fp32.  dout16 carries the power-of-two gradient scale of
 * the backward segment and dqkv16 comes out with the same scale (everything is linear in dout). */
int b200vq_attention_f16_fwd(const void* qkv16, void* out16, float* lse, int B, int N, int heads, int dh, float scale,
                             void* stream);
int b200vq_attention_f16_bwd(const void* qkv16, const void* out16, const float* lse, const void* dout16, void* dqkv16,
                             float* delta, int B, int N, int heads, int dh, float scale, void* stream);
/* the same contract with every product in error-compensated 3xTF32 (fp32-grade; precision="parity") */
int b200vq_attention_exact_fwd(const float* qkv, float* out, float* lse, int B, int N, int heads, int dh, float scale,
                               void* stream);
int b200vq_attention_exact_bwd(const float* qkv, const float* out, const float* lse, const float* dout, float* dqkv,
                               float* delta, int B, int N, int heads, int dh, float scale, void* stream);

/* ---- vector quantiser (quantizers.py:38-92) ------------------------------------------------------
 * z [M,D], codebook E [K,D] (un-normalised nn.Embedding weight); out [M,D] = straight-through
 * value z + (z_q - z); idx int64 [M, depth]; loss: device scalar.  depth = 1 for the plain
 * quantiser, num_quantizers for use_residual=True.  use_norm: quantizers.py:24 (1 = l2-normalise).
 * Every VQ entry point takes embed_dim D = any multiple of 32 from 32 to 256 and rejects other widths.
 * b200vq_vq_fwd_workspace_bytes: the forward workspace at width D (0 for an unsupported D); at D = 32 it equals
 * b200vq_vq_workspace_bytes, the D = 32 query kept for existing callers. */
size_t b200vq_vq_workspace_bytes(int M, int K, int depth);
size_t b200vq_vq_fwd_workspace_bytes(int M, int K, int D, int depth);
int b200vq_vq_fwd(const float* z, const float* E, float* out, long long* idx, float* loss, int M, int K, int D,
                  int depth, float beta, int use_norm, void* workspace, size_t ws_bytes, void* stream);
/* g_out [M,D] or NULL, g_loss device scalar or NULL; gz [M,D] written, gE [K,D] zero-filled then
 * accumulated (nn.Embedding dense backward). */
int b200vq_vq_bwd(const float* z, const float* E, const long long* idx, const float* g_out, const float* g_loss,
                  float* gz, float* gE, int M, int K, int D, int depth, int residual, float beta, int use_norm,
                  void* stream);
/* bit-reproducible variant of b200vq_vq_bwd: the same gz (same arithmetic, bit for bit) and a gE whose summation order
 * depends only on idx and the shape -- not on the SM count, b200vq_set_sm_limit or timing.  Each entry m*depth + t of
 * idx (m for the plain quantiser) stores its codebook contribution in the workspace; a stable radix sort of the
 * entries by code and a segmented sum in ascending entry order (fixed runs of entries, then the runs in order) make gE.
 * No float atomics.  Same constraints as b200vq_vq_bwd plus n_embed % 4 == 0; workspace from the query below. */
size_t b200vq_vq_bwd_deterministic_workspace_bytes(int M, int K, int D, int depth);
int b200vq_vq_bwd_deterministic(const float* z, const float* E, const long long* idx, const float* g_out, const float* g_loss,
                                float* gz, float* gE, int M, int K, int D, int depth, int residual, float beta, int use_norm,
                                void* workspace, size_t ws_bytes, void* stream);
/* decode_codes (vitvqgan.py:81-86): out[m] = sum_t norm(E[codes[m,t]]) */
int b200vq_vq_embed(const float* E, const long long* codes, float* out, int M, int K, int D, int depth, int use_norm,
                    void* stream);
/* EMA codebook (EMAVectorQuantizer; van den Oord et al. 2017 appendix A.1 as in Taming Transformers' EMAVectorQuantizer).
 * vq_fwd_ema: the lookup of b200vq_vq_fwd (same out and idx, bit for bit) with the EMA loss beta * mean((q - x)^2), averaged
 *   over the depths -- no codebook term.  counts [K] and sums [K,D] (both NULL: no statistics, e.g. in eval mode) are
 *   overwritten with n_k = #{(m,t) : idx[m,t] = k} (exact integers in fp32) and s_k = sum of the vectors the lookup compared
 *   for those entries (norm(residual_t[m]), or the raw residual when use_norm == 0).  deterministic == 0: s is summed with
 *   float atomics (per-CTA shared-memory tables, then one global atomic per CTA, code and column); != 0: s is summed in
 *   the fixed order of b200vq_vq_bwd_deterministic, the same bits on every run.  M * depth < 2^24; workspace from the query.
 * vq_ema_update: in place, with no host synchronisation:
 *   cluster_size = decay * cluster_size + (1 - decay) * counts;  embed_avg = decay * embed_avg + (1 - decay) * sums;
 *   N = sum_k cluster_size_k (fixed order);  weight_k = embed_avg_k / ((cluster_size_k + eps) / (N + K * eps) * N). */
size_t b200vq_vq_fwd_ema_workspace_bytes(int M, int K, int D, int depth, int deterministic);
int b200vq_vq_fwd_ema(const float* z, const float* E, float* out, long long* idx, float* loss, float* counts, float* sums, int M, int K,
                      int D, int depth, float beta, int use_norm, int deterministic, void* workspace, size_t ws_bytes, void* stream);
int b200vq_vq_ema_update(const float* counts, const float* sums, float* cluster_size, float* embed_avg, float* weight, int K, int D,
                         float decay, float eps, void* stream);

/* ---- re-layout / reductions ------------------------------------------------------------------------*/
/* [B,C,H,W] -> [B*(H/ph)*(W/pw), C*ph*pw], patch vector ordered (c,row,col) (layers.py:157-171); pw % 4 == 0 */
int b200vq_patchify(const float* img, float* patches, int B, int C, int H, int W, int ph, int pw, int round_out,
                    void* stream);
/* inverse, adding bias[c] if non-NULL (ConvTranspose2d bias, layers.py:204) */
int b200vq_unpatchify(const float* tokens, const float* bias, float* img, int B, int C, int H, int W, int ph, int pw,
                      void* stream);
size_t b200vq_colsum_workspace_bytes(int N);
/* out[n] = sum_m X[m,n] (bias gradients) */
int b200vq_colsum(const float* X, long long ld, int M, int N, float* out, void* workspace, size_t ws_bytes, void* stream);
/* out = tf32-rounded copy of in (weights shadow for the tensor-core path): round to nearest, ties away from zero, as
 * cvt.rna.tf32.f32 does, kept in an fp32 container with the low 13 bits clear (values past the largest tf32 become
 * inf).  NaN stays NaN with its sign: the quiet bit is set, so it is still NaN after a tensor core truncates it.  Every
 * round_out of this header rounds the same way. */
int b200vq_round_tf32(const float* in, float* out, long long n, void* stream);

/* out[m,:] = x[m,:] + table[m % R,:]  (token + de_pos_embedding, layers.py:210) */
int b200vq_add_rows_mod(const float* x, const float* table, float* out, long long M, int D, int R, void* stream);


/* ---- operand preparation for the 3xTF32 and fp16 data paths --------------------------------------*/
/* lo = in - trunc_tf32(in): the bits a tf32 MMA drops (exact in fp32) */
int b200vq_split_tf32_lo(const float* in, float* lo, long long n, void* stream);
/* out16 = fp16(in * *scale), saturating at +-65504 (scale: device scalar or NULL) */
int b200vq_to_half(const float* in, void* out16, long long n, const float* scale, void* stream);
/* scale2 = {S, 1/S}, S = 2^(target_log2 - ceil(log2(max|g|))): the power-of-two gradient scale of one backward
 * segment, chosen on the device from the incoming gradient (no host synchronisation), so max|g| * S lies in
 * (2^(target_log2-1), 2^target_log2].  The exponent is clamped to [-100, 100] (a subnormal or huge max|g|), and a
 * gradient whose max|g| is zero, inf or NaN gets S = 1. */
size_t b200vq_grad_scale_workspace_bytes(void);
int b200vq_grad_scale(const float* g, long long n, int target_log2, float* scale2, void* workspace, size_t ws_bytes,
                      void* stream);

/* ---- the loss stage's two native ops (SURVEY.md section 8f-2) ------------------------------------------
 * bias_act: out = act'(x + bias[(i / step_b) % size_b], ref) * scale -- losses/op/fused_bias_act_kernel.cu:18-65.
 *   act 1 linear / 3 leaky ReLU (slope alpha); grad 0 value, 1 first derivative applied to x (ref = forward output),
 *   2 second derivative (zero).  bias / ref nullable.
 * upfirdn2d: per plane [in_h, in_w]: zero-insert upsample (up), pad / crop, FIR with `kernel` [kh, kw] (true
 *   convolution), decimate (down) -- losses/op/upfirdn2d_kernel.cu:107-207, upfirdn2d.py:168-206.
 *   out_h = (in_h*up_y + pad_y0 + pad_y1 - kh + down_y) / down_y, likewise out_w. */
int b200vq_bias_act(const float* x, const float* bias, const float* ref, float* out, long long n, int step_b, int size_b,
                    int act, int grad, float alpha, float scale, void* stream);
int b200vq_upfirdn2d(const float* in, const float* kernel, float* out, long long planes, int in_h, int in_w, int kh, int kw,
                     int up_x, int up_y, int down_x, int down_y, int pad_x0, int pad_x1, int pad_y0, int pad_y1,
                     void* stream);

/* ---- stage-2 transformer (SURVEY.md section 8f-3; reference enhancing/modules/stage2/layers.py) --------------------
 * attention_causal: the stage-1 attention contract (same packed qkv / out / lse / delta layouts, fp32) with the stage-2
 *   mask of layers.py:43-48,83-85: query q attends to key k iff k <= max(q, cond_len - 1) -- causal, the cond_len
 *   condition tokens fully visible to each other.  exact != 0: error-compensated 3xTF32 (precision="parity");
 *   otherwise the single-pass tf32 kernels (round_out as in b200vq_attention_fwd).  dh (the head size
 *   embed_dim / n_heads) must be 32, 64, 96 or 128; 96 and 128 run on wide-head kernels that read their resident operand
 *   from shared memory, with the same mask, LSE, round_out and bit-reproducibility (no atomics).  The stage-1 entry
 *   points above keep their head sizes.
 * time_mix: y = x * w + shift(x) * (1 - w), shift = one step along T with a zero first row (layers.py:50-58), bit-identical
 *   to the reference's four fp32 tensor ops.  x, y [M = B*T, C]; w [C].
 *   bwd: gx likewise; gw_part [ceil(M / 64), C] holds per-64-row partial sums of g * (x - shift(x)) -- b200vq_colsum over
 *   it is the gradient of w.
 * sqrelu: grad 0: y = relu(x)^2 (layers.py:108); grad 1: y = g * 2 relu(x), x the pre-activation.
 * token_embed: x[b] = cat(Wc[conds[b]] + pos_c, Wi[codes[b]] + pos_i) (layers.py:199-206); conds int64 [B, Tc], codes
 *   int64 [B, Ti], x [B, Tc + Ti, C].  bwd: gWc / gWi are zero-filled then accumulated, gpos_* = sum over the batch.
 *   bwd_deterministic: the same results with gWc / gWi summed in a fixed order (ids clamped as in bwd; the stable sort
 *   and segmented sum of b200vq_vq_bwd_deterministic, no float atomics), gpos_* bit-identical to bwd's; Vc, Vi > 0;
 *   workspace from its query.
 * copy_rows: dst[b, t] = src[b, t - off_dst + off_src] for off_dst <= t < off_dst + n, else 0 (the window
 *   x[:, cond-1:-1] of layers.py:210 and its zero-padded gradient).
 * decode_attention: one sampling step of layers.py:66-81 (use_cache with layer_past): appends the k / v thirds of
 *   qkv [B, 3*C] to cache_k / cache_v [B, Tmax, C] at row `pos` and writes softmax(q K^T * scale) V over rows 0..pos
 *   to out [B, C].  hs 32, 64, 96 or 128. */
int b200vq_attention_causal_fwd(const float* qkv, float* out, float* lse, int B, int N, int heads, int dh, float scale,
                                int cond_len, int exact, int round_out, void* stream);
int b200vq_attention_causal_bwd(const float* qkv, const float* out, const float* lse, const float* dout, float* dqkv,
                                float* delta, int B, int N, int heads, int dh, float scale, int cond_len, int exact,
                                int round_out, void* stream);
int b200vq_time_mix_fwd(const float* x, const float* w, float* y, long long M, int T, int C, int round_out, void* stream);
size_t b200vq_time_mix_bwd_workspace_bytes(long long M, int C);
int b200vq_time_mix_bwd(const float* g, const float* x, const float* w, float* gx, float* gw_part, long long M, int T, int C,
                        void* stream);
int b200vq_sqrelu(const float* x, const float* g, float* y, long long n, int grad, int round_out, void* stream);
int b200vq_token_embed_fwd(const long long* conds, const long long* codes, const float* Wc, const float* pos_c, const float* Wi,
                           const float* pos_i, float* x, int B, int Tc, int Ti, int C, int Vc, int Vi, void* stream);
int b200vq_token_embed_bwd(const long long* conds, const long long* codes, const float* g, float* gWc, float* gpos_c, float* gWi,
                           float* gpos_i, int B, int Tc, int Ti, int C, int Vc, int Vi, void* stream);
size_t b200vq_token_embed_bwd_deterministic_workspace_bytes(int B, int Tc, int Ti, int C, int Vc, int Vi);
int b200vq_token_embed_bwd_deterministic(const long long* conds, const long long* codes, const float* g, float* gWc, float* gpos_c,
                                         float* gWi, float* gpos_i, int B, int Tc, int Ti, int C, int Vc, int Vi, void* workspace,
                                         size_t ws_bytes, void* stream);
int b200vq_copy_rows(const float* src, float* dst, int B, int T_src, int T_dst, int off_src, int off_dst, int n, int C,
                     void* stream);
int b200vq_decode_attention(const float* qkv, float* cache_k, float* cache_v, float* out, int B, int heads, int hs, int Tmax,
                            int pos, float scale, void* stream);

/* ---- stage-2 RQTransformer (reference enhancing/modules/stage2/layers.py:306-547) ---------------------------------------
 * short_attention: the depth transformer's attention core -- nseq independent sequences of D tokens (1 <= D <= 16), the
 *   packed qkv [nseq*D, 3*heads*hs] of b200vq_attention_causal_fwd (q | k | v thirds, head h at columns h*hs) -> out
 *   [nseq*D, heads*hs]; the mask of b200vq_attention_causal_fwd (k <= max(q, cond_len - 1)); hs 32, 64, 96 or 128, heads*hs <= 2048.
 *   fp32 FMA arithmetic and an fp32 softmax on every data path.  bwd recomputes the scores from qkv and writes every
 *   element of dqkv [nseq*D, 3*heads*hs] (no lse / out / delta needed, no atomics: the same bits on every run).  Both
 *   are persistent grid-stride kernels: b200vq_set_sm_limit caps their grid at that many CTAs (the results do not
 *   depend on the grid).
 * rq_embed: the spatial input x [B, Tc + T, C] of layers.py:374-384: rows t < Tc are Wc[conds[b, t]] + pos_c[t]; row Tc + t is
 *   cumsum over the channels of Wi[codes[b, t, D-1]] (scanned in fp64, rounded once: torch's CPU cumsum bit for bit) +
 *   pos_i[t].  conds int64 [B, Tc], codes int64 [B, T, D].  bwd: gWc / gWi zero-filled then accumulated with float
 *   atomics (gWi as the reverse channel scan of the scattered rows; with Tc == 0 a non-NULL gWc comes out all zero),
 *   gpos_c [Tc, C] / gpos_i [T, C] = sums over the batch in a fixed order.  bwd_deterministic: the same with gWc / gWi summed in a fixed order (the sort and segmented sum of
 *   b200vq_token_embed_bwd_deterministic) -- bit-reproducible whatever the SM count; workspace from its query.
 * rq_depth_input: the depth input v [nseq*D, C] of layers.py:388-391 (nseq = B*T): v[s, 0] = h[s] (h [nseq, C]);
 *   v[s, d] = cumsum over the channels of Wi[codes[s, d-1]] + pos_d[d-1] for d >= 1 (codes int64 [nseq, D], pos_d
 *   [D-1, C]).  bwd: gh [nseq, C] = the row-0 gradients, gWi as in rq_embed_bwd, gpos_d [D-1, C] = sums over the sequences
 *   in a fixed order.  bwd_deterministic as for rq_embed.
 * code_sum_embed: out[b] = sum_{j < n} Wi[codes[b*ld + j]] + pos (pos one [C] row): the inputs of the sampling steps,
 *   layers.py:501-502 (the previous position's D codes) and :534-535 (this position's codes so far). */
int b200vq_short_attention_fwd(const float* qkv, float* out, long long nseq, int D, int heads, int hs, int cond_len, float scale,
                               void* stream);
int b200vq_short_attention_bwd(const float* qkv, const float* dout, float* dqkv, long long nseq, int D, int heads, int hs, int cond_len,
                               float scale, void* stream);
int b200vq_rq_embed_fwd(const long long* conds, const long long* codes, const float* Wc, const float* pos_c, const float* Wi,
                        const float* pos_i, float* x, int B, int Tc, int T, int D, int C, int Vc, int Vi, void* stream);
int b200vq_rq_embed_bwd(const long long* conds, const long long* codes, const float* g, float* gWc, float* gpos_c, float* gWi,
                        float* gpos_i, int B, int Tc, int T, int D, int C, int Vc, int Vi, void* stream);
size_t b200vq_rq_embed_bwd_deterministic_workspace_bytes(int B, int Tc, int T, int D, int C, int Vc, int Vi);
int b200vq_rq_embed_bwd_deterministic(const long long* conds, const long long* codes, const float* g, float* gWc, float* gpos_c,
                                      float* gWi, float* gpos_i, int B, int Tc, int T, int D, int C, int Vc, int Vi, void* workspace,
                                      size_t ws_bytes, void* stream);
int b200vq_rq_depth_input_fwd(const float* h, const long long* codes, const float* Wi, const float* pos_d, float* v, long long nseq,
                              int D, int C, int Vi, void* stream);
int b200vq_rq_depth_input_bwd(const long long* codes, const float* g, float* gh, float* gWi, float* gpos_d, long long nseq, int D, int C,
                              int Vi, void* stream);
size_t b200vq_rq_depth_input_bwd_deterministic_workspace_bytes(long long nseq, int D, int C, int Vi);
int b200vq_rq_depth_input_bwd_deterministic(const long long* codes, const float* g, float* gh, float* gWi, float* gpos_d, long long nseq,
                                            int D, int C, int Vi, void* workspace, size_t ws_bytes, void* stream);
int b200vq_code_sum_embed(const long long* codes, long long ld, int n, const float* Wi, const float* pos, float* out, int B, int C, int Vi,
                          void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200VQ_H_ */
