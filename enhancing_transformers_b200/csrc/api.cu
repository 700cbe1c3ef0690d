// extern "C" surface of libb200vq.so (see include/b200vq.h).  Thin: argument forwarding,
// error text, launch accounting.  No allocation, no synchronisation.
#include "../../include/b200vq.h"

#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>

#include "common.cuh"

namespace b200 {

static thread_local char g_err[512] = "";
std::atomic<long long> g_launches{0};

int set_error(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }

int current_device() {
  int dev = -1;
  return cudaGetDevice(&dev) == cudaSuccess ? dev : -1;
}

int num_sms() {
  static PerDevice cache;
  const int dev = current_device();
  if (dev < 0 || dev >= kMaxDevices) return 132;
  if (!cache.done[dev]) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    cache.value[dev] = n;
    cache.done[dev] = true;
  }
  return cache.value[dev];
}

static std::atomic<int> g_sm_limit{-1};
int sm_limit() {
  int v = g_sm_limit.load(std::memory_order_relaxed);
  if (v < 0) {
    const char* e = getenv("B200VQ_SM_LIMIT");
    v = e ? atoi(e) : 0;
    if (v < 0) v = 0;
    g_sm_limit.store(v);
  }
  return v;
}

// implemented in the other translation units
int gemm_tf32(const float*, long long, int, const float*, long long, int, float*, long long, int, int, int, int, long long,
              const float*, const float*, long long, int, const float*, long long, float*, int, int, int, int, cudaStream_t);
int gemm_3xtf32(const float*, const float*, long long, int, const float*, const float*, long long, int, float*, long long, int, int,
                int, int, long long, const float*, const float*, long long, int, const float*, long long, float*, int, int, int,
                cudaStream_t);
int gemm_f16(const void*, long long, int, const void*, long long, int, void*, long long, int, int, int, int, int, long long,
             const float*, const float*, long long, int, const void*, long long, float*, int, int, const float*, int, int,
             cudaStream_t);
int splitk_reduce(const float*, int, long long, long long, const float*, float*, cudaStream_t);
int layernorm_forward(const float*, const float*, const float*, float*, void*, float*, float*, int, int, int, cudaStream_t);
size_t layernorm_bwd_workspace_bytes(int);
int layernorm_backward(const void*, int, const float*, const float*, const float*, const float*, const float*, const float*, float*, void*,
                       const float*, float*, float*, float*, int, int, int, void*, size_t, cudaStream_t);
int attention_forward(const float*, void*, int, float*, int, int, int, int, float, int, cudaStream_t);
int attention_backward(const float*, const void*, int, const float*, const float*, void*, int, const float*, float*, int, int,
                       int, int, float, int, cudaStream_t);
int attention_f16_forward(const void*, void*, float*, int, int, int, int, float, cudaStream_t);
int attention_f16_backward(const void*, const void*, const float*, const void*, void*, float*, int, int, int, int, float, cudaStream_t);
int attention_exact_forward(const float*, float*, float*, int, int, int, int, float, int, cudaStream_t);
int attention_exact_backward(const float*, const float*, const float*, const float*, float*, float*, int, int, int, int, float, int,
                             cudaStream_t);
int attention_causal_forward(const float*, float*, float*, int, int, int, int, float, int, int, int, cudaStream_t);
int attention_causal_backward(const float*, const float*, const float*, const float*, float*, float*, int, int, int, int, float, int,
                              int, int, cudaStream_t);
size_t vq_workspace_bytes(int, int, int);
int vq_forward(const float*, const float*, float*, long long*, float*, int, int, int, int, float, int, void*, size_t, cudaStream_t);
int vq_backward(const float*, const float*, const long long*, const float*, const float*, float*, float*, int, int, int, int,
                int, float, int, cudaStream_t);
int vq_embed(const float*, const long long*, float*, int, int, int, int, int, cudaStream_t);
size_t vq_bwd_deterministic_workspace_bytes(int, int, int, int);
int vq_backward_deterministic(const float*, const float*, const long long*, const float*, const float*, float*, float*, int, int, int,
                              int, int, float, int, void*, size_t, cudaStream_t);
size_t vq_fwd_ema_workspace_bytes(int, int, int, int, int);
int vq_forward_ema(const float*, const float*, float*, long long*, float*, float*, float*, int, int, int, int, float, int, int, void*,
                   size_t, cudaStream_t);
int vq_ema_update(const float*, const float*, float*, float*, float*, int, int, float, float, cudaStream_t);
int patchify(const float*, float*, int, int, int, int, int, int, int, cudaStream_t);
int unpatchify(const float*, const float*, float*, int, int, int, int, int, int, cudaStream_t);
size_t colsum_workspace_bytes(int);
int colsum(const float*, long long, int, int, float*, void*, size_t, cudaStream_t);
int round_tf32_copy(const float*, float*, long long, cudaStream_t);
int add_rows_mod(const float*, const float*, float*, long long, int, int, cudaStream_t);
int split_tf32_lo(const float*, float*, long long, cudaStream_t);
int to_half(const float*, void*, long long, const float*, cudaStream_t);
size_t grad_scale_workspace_bytes();
int bias_act(const float*, const float*, const float*, float*, long long, int, int, int, int, float, float, cudaStream_t);
int upfirdn2d(const float*, const float*, float*, long long, int, int, int, int, int, int, int, int, int, int, int, int, cudaStream_t);
int grad_scale(const float*, long long, int, float*, void*, size_t, cudaStream_t);
int time_mix_forward(const float*, const float*, float*, long long, int, int, int, cudaStream_t);
size_t time_mix_bwd_workspace_bytes(long long, int);
int time_mix_backward(const float*, const float*, const float*, float*, float*, long long, int, int, cudaStream_t);
int sqrelu(const float*, const float*, float*, long long, int, int, cudaStream_t);
int token_embed_forward(const long long*, const long long*, const float*, const float*, const float*, const float*, float*, int, int,
                        int, int, int, int, cudaStream_t);
int token_embed_backward(const long long*, const long long*, const float*, float*, float*, float*, float*, int, int, int, int, int,
                         int, cudaStream_t);
size_t token_embed_bwd_deterministic_workspace_bytes(int, int, int, int, int, int);
int token_embed_backward_deterministic(const long long*, const long long*, const float*, float*, float*, float*, float*, int, int, int,
                                       int, int, int, void*, size_t, cudaStream_t);
int copy_rows(const float*, float*, int, int, int, int, int, int, int, cudaStream_t);
int decode_attention(const float*, float*, float*, float*, int, int, int, int, int, float, cudaStream_t);
int short_attention_forward(const float*, float*, long long, int, int, int, int, float, cudaStream_t);
int short_attention_backward(const float*, const float*, float*, long long, int, int, int, int, float, cudaStream_t);
int rq_embed_forward(const long long*, const long long*, const float*, const float*, const float*, const float*, float*, int, int, int,
                     int, int, int, int, cudaStream_t);
int rq_embed_backward(const long long*, const long long*, const float*, float*, float*, float*, float*, int, int, int, int, int, int,
                      int, cudaStream_t);
size_t rq_embed_bwd_deterministic_workspace_bytes(int, int, int, int, int, int, int);
int rq_embed_backward_deterministic(const long long*, const long long*, const float*, float*, float*, float*, float*, int, int, int, int,
                                    int, int, int, void*, size_t, cudaStream_t);
int rq_depth_input_forward(const float*, const long long*, const float*, const float*, float*, long long, int, int, int, cudaStream_t);
int rq_depth_input_backward(const long long*, const float*, float*, float*, float*, long long, int, int, int, cudaStream_t);
size_t rq_depth_input_bwd_deterministic_workspace_bytes(long long, int, int, int);
int rq_depth_input_backward_deterministic(const long long*, const float*, float*, float*, float*, long long, int, int, int, void*, size_t,
                                          cudaStream_t);
int code_sum_embed(const long long*, long long, int, const float*, const float*, float*, int, int, int, cudaStream_t);

}  // namespace b200

using namespace b200;
#define S(stream) static_cast<cudaStream_t>(stream)

extern "C" {

int b200vq_version(void) { return B200VQ_VERSION; }
const char* b200vq_last_error(void) { return g_err; }
const char* b200vq_arch(void) { return "sm_90a"; }
long long b200vq_launch_count(void) { return g_launches.load(); }

int b200vq_set_sm_limit(int n) { g_sm_limit.store(n < 0 ? 0 : n); return 0; }

int b200vq_gemm_tf32(const float* A, long long lda, int a_major, const float* B, long long ldb, int b_major, float* C,
                     long long ldc, int M, int N, int K, int splits, long long c_split_stride, const float* bias,
                     const float* res, long long ldres, int res_row_mod, const float* aux, long long ldaux,
                     float* colsum_part, int act, int round_out, int cta_group, int bn, void* stream) {
  return gemm_tf32(A, lda, a_major, B, ldb, b_major, C, ldc, M, N, K, splits, c_split_stride, bias, res, ldres, res_row_mod,
                   aux, ldaux, colsum_part, act, round_out, cta_group, bn, S(stream));
}
int b200vq_gemm_3xtf32(const float* A, const float* A_lo, long long lda, int a_major, const float* B, const float* B_lo,
                       long long ldb, int b_major, float* C, long long ldc, int M, int N, int K, int splits,
                       long long c_split_stride, const float* bias, const float* res, long long ldres, int res_row_mod,
                       const float* aux, long long ldaux, float* colsum_part, int act, int cta_group, int bn, void* stream) {
  return gemm_3xtf32(A, A_lo, lda, a_major, B, B_lo, ldb, b_major, C, ldc, M, N, K, splits, c_split_stride, bias, res, ldres,
                     res_row_mod, aux, ldaux, colsum_part, act, cta_group, bn, S(stream));
}
int b200vq_gemm_f16(const void* A, long long lda, int a_major, const void* B, long long ldb, int b_major, void* C, long long ldc,
                    int out_half, int M, int N, int K, int splits, long long c_split_stride, const float* bias,
                    const float* res, long long ldres, int res_row_mod, const void* aux, long long ldaux, float* colsum_part,
                    int act, int round_out, const float* alpha, int cta_group, int bn, void* stream) {
  return gemm_f16(A, lda, a_major, B, ldb, b_major, C, ldc, out_half, M, N, K, splits, c_split_stride, bias, res, ldres,
                  res_row_mod, aux, ldaux, colsum_part, act, round_out, alpha, cta_group, bn, S(stream));
}
int b200vq_splitk_reduce(const float* part, int splits, long long n, long long split_stride, const float* alpha, float* out,
                         void* stream) {
  return splitk_reduce(part, splits, n, split_stride, alpha, out, S(stream));
}
int b200vq_layernorm_fwd(const float* x, const float* gamma, const float* beta, float* y, void* y16, float* mean, float* rstd,
                         int M, int D, int round_out, void* stream) {
  return layernorm_forward(x, gamma, beta, y, y16, mean, rstd, M, D, round_out, S(stream));
}
size_t b200vq_layernorm_bwd_workspace_bytes(int D) { return layernorm_bwd_workspace_bytes(D); }
int b200vq_layernorm_bwd(const void* dy, int dy_half, const float* dy_scale, const float* x, const float* mean, const float* rstd,
                         const float* gamma, const float* dres, float* dx, void* dx16, const float* dx16_scale, float* dgamma,
                         float* dbeta, float* dxsum, int M, int D, int round_out, void* workspace, size_t ws_bytes, void* stream) {
  return layernorm_backward(dy, dy_half, dy_scale, x, mean, rstd, gamma, dres, dx, dx16, dx16_scale, dgamma, dbeta, dxsum, M, D, round_out,
                            workspace, ws_bytes, S(stream));
}
int b200vq_attention_fwd(const float* qkv, void* out, int out_half, float* lse, int B, int N, int heads, int dh, float scale,
                         int round_out, void* stream) {
  return attention_forward(qkv, out, out_half, lse, B, N, heads, dh, scale, round_out, S(stream));
}
int b200vq_attention_bwd(const float* qkv, const void* out, int out_half, const float* lse, const float* dout, void* dqkv,
                         int dqkv_half, const float* dqkv_scale, float* delta, int B, int N, int heads, int dh, float scale,
                         int round_out, void* stream) {
  return attention_backward(qkv, out, out_half, lse, dout, dqkv, dqkv_half, dqkv_scale, delta, B, N, heads, dh, scale,
                            round_out, S(stream));
}
int b200vq_attention_f16_fwd(const void* qkv16, void* out16, float* lse, int B, int N, int heads, int dh, float scale, void* stream) {
  return attention_f16_forward(qkv16, out16, lse, B, N, heads, dh, scale, S(stream));
}
int b200vq_attention_f16_bwd(const void* qkv16, const void* out16, const float* lse, const void* dout16, void* dqkv16, float* delta,
                             int B, int N, int heads, int dh, float scale, void* stream) {
  return attention_f16_backward(qkv16, out16, lse, dout16, dqkv16, delta, B, N, heads, dh, scale, S(stream));
}
int b200vq_attention_exact_fwd(const float* qkv, float* out, float* lse, int B, int N, int heads, int dh, float scale,
                               void* stream) {
  return attention_exact_forward(qkv, out, lse, B, N, heads, dh, scale, -1, S(stream));
}
int b200vq_attention_exact_bwd(const float* qkv, const float* out, const float* lse, const float* dout, float* dqkv,
                               float* delta, int B, int N, int heads, int dh, float scale, void* stream) {
  return attention_exact_backward(qkv, out, lse, dout, dqkv, delta, B, N, heads, dh, scale, -1, S(stream));
}
int b200vq_attention_causal_fwd(const float* qkv, float* out, float* lse, int B, int N, int heads, int dh, float scale,
                                int cond_len, int exact, int round_out, void* stream) {
  return attention_causal_forward(qkv, out, lse, B, N, heads, dh, scale, cond_len, exact, round_out, S(stream));
}
int b200vq_attention_causal_bwd(const float* qkv, const float* out, const float* lse, const float* dout, float* dqkv,
                                float* delta, int B, int N, int heads, int dh, float scale, int cond_len, int exact,
                                int round_out, void* stream) {
  return attention_causal_backward(qkv, out, lse, dout, dqkv, delta, B, N, heads, dh, scale, cond_len, exact, round_out,
                                   S(stream));
}
size_t b200vq_vq_workspace_bytes(int M, int K, int depth) { return vq_workspace_bytes(M, K, depth); }
int b200vq_vq_fwd(const float* z, const float* E, float* out, long long* idx, float* loss, int M, int K, int D, int depth,
                  float beta, int use_norm, void* workspace, size_t ws_bytes, void* stream) {
  return vq_forward(z, E, out, idx, loss, M, K, D, depth, beta, use_norm, workspace, ws_bytes, S(stream));
}
int b200vq_vq_bwd(const float* z, const float* E, const long long* idx, const float* g_out, const float* g_loss, float* gz,
                  float* gE, int M, int K, int D, int depth, int residual, float beta, int use_norm, void* stream) {
  return vq_backward(z, E, idx, g_out, g_loss, gz, gE, M, K, D, depth, residual, beta, use_norm, S(stream));
}
size_t b200vq_vq_bwd_deterministic_workspace_bytes(int M, int K, int D, int depth) {
  return vq_bwd_deterministic_workspace_bytes(M, K, D, depth);
}
int b200vq_vq_bwd_deterministic(const float* z, const float* E, const long long* idx, const float* g_out, const float* g_loss,
                                float* gz, float* gE, int M, int K, int D, int depth, int residual, float beta, int use_norm,
                                void* workspace, size_t ws_bytes, void* stream) {
  return vq_backward_deterministic(z, E, idx, g_out, g_loss, gz, gE, M, K, D, depth, residual, beta, use_norm, workspace, ws_bytes,
                                   S(stream));
}
int b200vq_vq_embed(const float* E, const long long* codes, float* out, int M, int K, int D, int depth, int use_norm,
                    void* stream) {
  return vq_embed(E, codes, out, M, K, D, depth, use_norm, S(stream));
}
size_t b200vq_vq_fwd_ema_workspace_bytes(int M, int K, int D, int depth, int deterministic) {
  return vq_fwd_ema_workspace_bytes(M, K, D, depth, deterministic);
}
int b200vq_vq_fwd_ema(const float* z, const float* E, float* out, long long* idx, float* loss, float* counts, float* sums, int M, int K,
                      int D, int depth, float beta, int use_norm, int deterministic, void* workspace, size_t ws_bytes, void* stream) {
  return vq_forward_ema(z, E, out, idx, loss, counts, sums, M, K, D, depth, beta, use_norm, deterministic, workspace, ws_bytes,
                        S(stream));
}
int b200vq_vq_ema_update(const float* counts, const float* sums, float* cluster_size, float* embed_avg, float* weight, int K, int D,
                         float decay, float eps, void* stream) {
  return vq_ema_update(counts, sums, cluster_size, embed_avg, weight, K, D, decay, eps, S(stream));
}
int b200vq_patchify(const float* img, float* patches, int B, int C, int H, int W, int ph, int pw, int round_out, void* stream) {
  return patchify(img, patches, B, C, H, W, ph, pw, round_out, S(stream));
}
int b200vq_unpatchify(const float* tokens, const float* bias, float* img, int B, int C, int H, int W, int ph, int pw, void* stream) {
  return unpatchify(tokens, bias, img, B, C, H, W, ph, pw, S(stream));
}
size_t b200vq_colsum_workspace_bytes(int N) { return colsum_workspace_bytes(N); }
int b200vq_colsum(const float* X, long long ld, int M, int N, float* out, void* workspace, size_t ws_bytes, void* stream) {
  return colsum(X, ld, M, N, out, workspace, ws_bytes, S(stream));
}
int b200vq_round_tf32(const float* in, float* out, long long n, void* stream) { return round_tf32_copy(in, out, n, S(stream)); }

int b200vq_add_rows_mod(const float* x, const float* table, float* out, long long M, int D, int R, void* stream) {
  return add_rows_mod(x, table, out, M, D, R, S(stream));
}

int b200vq_split_tf32_lo(const float* in, float* lo, long long n, void* stream) { return split_tf32_lo(in, lo, n, S(stream)); }
int b200vq_to_half(const float* in, void* out, long long n, const float* scale, void* stream) {
  return to_half(in, out, n, scale, S(stream));
}
size_t b200vq_grad_scale_workspace_bytes(void) { return grad_scale_workspace_bytes(); }
int b200vq_grad_scale(const float* g, long long n, int target_log2, float* scale2, void* workspace, size_t ws_bytes,
                      void* stream) {
  return grad_scale(g, n, target_log2, scale2, workspace, ws_bytes, S(stream));
}

int b200vq_bias_act(const float* x, const float* bias, const float* ref, float* out, long long n, int step_b, int size_b, int act,
                    int grad, float alpha, float scale, void* stream) {
  return bias_act(x, bias, ref, out, n, step_b, size_b, act, grad, alpha, scale, S(stream));
}
int b200vq_upfirdn2d(const float* in, const float* kernel, float* out, long long planes, int in_h, int in_w, int kh, int kw, int up_x,
                     int up_y, int down_x, int down_y, int pad_x0, int pad_x1, int pad_y0, int pad_y1, void* stream) {
  return upfirdn2d(in, kernel, out, planes, in_h, in_w, kh, kw, up_x, up_y, down_x, down_y, pad_x0, pad_x1, pad_y0, pad_y1, S(stream));
}

int b200vq_time_mix_fwd(const float* x, const float* w, float* y, long long M, int T, int C, int round_out, void* stream) {
  return time_mix_forward(x, w, y, M, T, C, round_out, S(stream));
}
size_t b200vq_time_mix_bwd_workspace_bytes(long long M, int C) { return time_mix_bwd_workspace_bytes(M, C); }
int b200vq_time_mix_bwd(const float* g, const float* x, const float* w, float* gx, float* gw_part, long long M, int T, int C,
                        void* stream) {
  return time_mix_backward(g, x, w, gx, gw_part, M, T, C, S(stream));
}
int b200vq_sqrelu(const float* x, const float* g, float* y, long long n, int grad, int round_out, void* stream) {
  return sqrelu(x, g, y, n, grad, round_out, S(stream));
}
int b200vq_token_embed_fwd(const long long* conds, const long long* codes, const float* Wc, const float* pos_c, const float* Wi,
                           const float* pos_i, float* x, int B, int Tc, int Ti, int C, int Vc, int Vi, void* stream) {
  return token_embed_forward(conds, codes, Wc, pos_c, Wi, pos_i, x, B, Tc, Ti, C, Vc, Vi, S(stream));
}
int b200vq_token_embed_bwd(const long long* conds, const long long* codes, const float* g, float* gWc, float* gpos_c, float* gWi,
                           float* gpos_i, int B, int Tc, int Ti, int C, int Vc, int Vi, void* stream) {
  return token_embed_backward(conds, codes, g, gWc, gpos_c, gWi, gpos_i, B, Tc, Ti, C, Vc, Vi, S(stream));
}
size_t b200vq_token_embed_bwd_deterministic_workspace_bytes(int B, int Tc, int Ti, int C, int Vc, int Vi) {
  return token_embed_bwd_deterministic_workspace_bytes(B, Tc, Ti, C, Vc, Vi);
}
int b200vq_token_embed_bwd_deterministic(const long long* conds, const long long* codes, const float* g, float* gWc, float* gpos_c,
                                         float* gWi, float* gpos_i, int B, int Tc, int Ti, int C, int Vc, int Vi, void* workspace,
                                         size_t ws_bytes, void* stream) {
  return token_embed_backward_deterministic(conds, codes, g, gWc, gpos_c, gWi, gpos_i, B, Tc, Ti, C, Vc, Vi, workspace, ws_bytes,
                                            S(stream));
}
int b200vq_copy_rows(const float* src, float* dst, int B, int T_src, int T_dst, int off_src, int off_dst, int n, int C,
                     void* stream) {
  return copy_rows(src, dst, B, T_src, T_dst, off_src, off_dst, n, C, S(stream));
}
int b200vq_decode_attention(const float* qkv, float* cache_k, float* cache_v, float* out, int B, int heads, int hs, int Tmax,
                            int pos, float scale, void* stream) {
  return decode_attention(qkv, cache_k, cache_v, out, B, heads, hs, Tmax, pos, scale, S(stream));
}

int b200vq_short_attention_fwd(const float* qkv, float* out, long long nseq, int D, int heads, int hs, int cond_len, float scale,
                               void* stream) {
  return short_attention_forward(qkv, out, nseq, D, heads, hs, cond_len, scale, S(stream));
}
int b200vq_short_attention_bwd(const float* qkv, const float* dout, float* dqkv, long long nseq, int D, int heads, int hs, int cond_len,
                               float scale, void* stream) {
  return short_attention_backward(qkv, dout, dqkv, nseq, D, heads, hs, cond_len, scale, S(stream));
}
int b200vq_rq_embed_fwd(const long long* conds, const long long* codes, const float* Wc, const float* pos_c, const float* Wi,
                        const float* pos_i, float* x, int B, int Tc, int T, int D, int C, int Vc, int Vi, void* stream) {
  return rq_embed_forward(conds, codes, Wc, pos_c, Wi, pos_i, x, B, Tc, T, D, C, Vc, Vi, S(stream));
}
int b200vq_rq_embed_bwd(const long long* conds, const long long* codes, const float* g, float* gWc, float* gpos_c, float* gWi,
                        float* gpos_i, int B, int Tc, int T, int D, int C, int Vc, int Vi, void* stream) {
  return rq_embed_backward(conds, codes, g, gWc, gpos_c, gWi, gpos_i, B, Tc, T, D, C, Vc, Vi, S(stream));
}
size_t b200vq_rq_embed_bwd_deterministic_workspace_bytes(int B, int Tc, int T, int D, int C, int Vc, int Vi) {
  return rq_embed_bwd_deterministic_workspace_bytes(B, Tc, T, D, C, Vc, Vi);
}
int b200vq_rq_embed_bwd_deterministic(const long long* conds, const long long* codes, const float* g, float* gWc, float* gpos_c,
                                      float* gWi, float* gpos_i, int B, int Tc, int T, int D, int C, int Vc, int Vi, void* workspace,
                                      size_t ws_bytes, void* stream) {
  return rq_embed_backward_deterministic(conds, codes, g, gWc, gpos_c, gWi, gpos_i, B, Tc, T, D, C, Vc, Vi, workspace, ws_bytes,
                                         S(stream));
}
int b200vq_rq_depth_input_fwd(const float* h, const long long* codes, const float* Wi, const float* pos_d, float* v, long long nseq,
                              int D, int C, int Vi, void* stream) {
  return rq_depth_input_forward(h, codes, Wi, pos_d, v, nseq, D, C, Vi, S(stream));
}
int b200vq_rq_depth_input_bwd(const long long* codes, const float* g, float* gh, float* gWi, float* gpos_d, long long nseq, int D, int C,
                              int Vi, void* stream) {
  return rq_depth_input_backward(codes, g, gh, gWi, gpos_d, nseq, D, C, Vi, S(stream));
}
size_t b200vq_rq_depth_input_bwd_deterministic_workspace_bytes(long long nseq, int D, int C, int Vi) {
  return rq_depth_input_bwd_deterministic_workspace_bytes(nseq, D, C, Vi);
}
int b200vq_rq_depth_input_bwd_deterministic(const long long* codes, const float* g, float* gh, float* gWi, float* gpos_d, long long nseq,
                                            int D, int C, int Vi, void* workspace, size_t ws_bytes, void* stream) {
  return rq_depth_input_backward_deterministic(codes, g, gh, gWi, gpos_d, nseq, D, C, Vi, workspace, ws_bytes, S(stream));
}
int b200vq_code_sum_embed(const long long* codes, long long ld, int n, const float* Wi, const float* pos, float* out, int B, int C, int Vi,
                          void* stream) {
  return code_sum_embed(codes, ld, n, Wi, pos, out, B, C, Vi, S(stream));
}

}  // extern "C"
