// Stage-2 (class-conditional GPT over the code grid: reference enhancing/modules/stage2/layers.py) -- the pieces its
// blocks need beyond the stage-1 kernels.  The seven Linear layers of a block run on the tensor-core GEMMs of gemm_tc.cu, the
// masked attention core on attention_exact.cu (attention_causal_*), LayerNorm on rowwise.cu.  Here:
//   time_mix     x * w + shift(x) * (1 - w), shift = one step along T with a zero first row   (layers.py:50-58)
//   sqrelu       square(relu(x)) and its derivative                                           (layers.py:108)
//   token_embed  cat(tok_emb_cond(conds) + pos_emb_cond, tok_emb_code(codes) + pos_emb_code)  (layers.py:199-206)
//   copy_rows    x[:, a:b] row windows (logits are taken at positions cond-1 .. T-2)          (layers.py:210)
//   decode_attention  one query per (batch, head) against the KV cache                        (layers.py:76-81, sampling)
// All HBM-bound streams: float4 grid-stride loops, no shared-memory staging needed (every element is read once).
// token_embed's backward scatters the table gradients with float atomics, or, on request, sums them in a fixed order
// through scatter_det.cu (bit-reproducible).
#include "../../include/b200vq.h"
#include "common.cuh"
#include "scatter_det.cuh"

namespace b200 {

static inline int s2_grid(long long work_items, int threads) {
  long long blocks = (work_items + threads - 1) / threads;
  const long long cap = (long long)num_sms() * 8;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return (int)blocks;
}

// The reference evaluates (x * w) + (shift(x) * (1 - w)) as four separately rounded fp32 tensor ops; the round-to-nearest
// intrinsics keep the compiler from contracting them into FMAs, so the result is bit-identical to the reference's.
__device__ __forceinline__ float mix1(float x, float xp, float w) {
  return __fadd_rn(__fmul_rn(x, w), __fmul_rn(xp, __fsub_rn(1.0f, w)));
}

__global__ void __launch_bounds__(256)
time_mix_fwd_kernel(const float* __restrict__ x, const float* __restrict__ w, float* __restrict__ y, long long M, int T, int C4,
                    int round_out) {
  const long long total = M * C4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long m = i / C4;
    const int c = (int)(i - m * C4);
    const int t = (int)(m % T);
    const float4 xv = reinterpret_cast<const float4*>(x)[i];
    const float4 xp = t > 0 ? reinterpret_cast<const float4*>(x)[i - C4] : make_float4(0.f, 0.f, 0.f, 0.f);
    const float4 wv = __ldg(reinterpret_cast<const float4*>(w) + c);
    float4 r = make_float4(mix1(xv.x, xp.x, wv.x), mix1(xv.y, xp.y, wv.y), mix1(xv.z, xp.z, wv.z), mix1(xv.w, xp.w, wv.w));
    if (round_out) { r.x = round_tf32(r.x); r.y = round_tf32(r.y); r.z = round_tf32(r.z); r.w = round_tf32(r.w); }
    reinterpret_cast<float4*>(y)[i] = r;
  }
}

// gx[b,t] = g[b,t] * w + g[b,t+1] * (1 - w);  gw_part[chunk] = sum over the chunk's rows of g * (x - shift(x)).
// One thread owns a float4 column over `rows` consecutive rows: coalesced across the block, deterministic.
__global__ void __launch_bounds__(256)
time_mix_bwd_kernel(const float* __restrict__ g, const float* __restrict__ x, const float* __restrict__ w, float* __restrict__ gx,
                    float* __restrict__ gw_part, long long M, int T, int C4, int rows) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C4) return;
  const long long m0 = (long long)blockIdx.y * rows;
  const long long m1 = min(M, m0 + rows);
  const float4 wv = __ldg(reinterpret_cast<const float4*>(w) + c);
  const float4 ow = make_float4(1.f - wv.x, 1.f - wv.y, 1.f - wv.z, 1.f - wv.w);
  const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
  float4 acc = zero;
  for (long long m = m0; m < m1; ++m) {
    const int t = (int)(m % T);
    const long long i = m * C4 + c;
    const float4 gv = reinterpret_cast<const float4*>(g)[i];
    const float4 gn = t + 1 < T ? reinterpret_cast<const float4*>(g)[i + C4] : zero;
    const float4 xv = reinterpret_cast<const float4*>(x)[i];
    const float4 xp = t > 0 ? reinterpret_cast<const float4*>(x)[i - C4] : zero;
    reinterpret_cast<float4*>(gx)[i] = make_float4(fmaf(gv.x, wv.x, gn.x * ow.x), fmaf(gv.y, wv.y, gn.y * ow.y),
                                                   fmaf(gv.z, wv.z, gn.z * ow.z), fmaf(gv.w, wv.w, gn.w * ow.w));
    acc.x = fmaf(gv.x, xv.x - xp.x, acc.x); acc.y = fmaf(gv.y, xv.y - xp.y, acc.y);
    acc.z = fmaf(gv.z, xv.z - xp.z, acc.z); acc.w = fmaf(gv.w, xv.w - xp.w, acc.w);
  }
  reinterpret_cast<float4*>(gw_part)[(long long)blockIdx.y * C4 + c] = acc;
}

// torch.relu's threshold rule, x <= 0 ? 0 : x: NaN passes through (fmaxf(NaN, 0) would give 0) and -0 becomes +0
__device__ __forceinline__ float relu_nan(float v) { return v <= 0.f ? 0.f : v; }

// grad 0: y = relu(x)^2 ; grad 1: y = g * 2 * relu(x)   (x = the pre-activation in both cases)
__global__ void __launch_bounds__(256)
sqrelu_kernel(const float* __restrict__ x, const float* __restrict__ g, float* __restrict__ y, long long n4, int grad, int round_out) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const float4 v = reinterpret_cast<const float4*>(x)[i];
    const float4 r = make_float4(relu_nan(v.x), relu_nan(v.y), relu_nan(v.z), relu_nan(v.w));
    float4 o;
    if (grad) {
      const float4 gv = reinterpret_cast<const float4*>(g)[i];
      o = make_float4(gv.x * (2.f * r.x), gv.y * (2.f * r.y), gv.z * (2.f * r.z), gv.w * (2.f * r.w));
    } else {
      o = make_float4(r.x * r.x, r.y * r.y, r.z * r.z, r.w * r.w);
    }
    if (round_out) { o.x = round_tf32(o.x); o.y = round_tf32(o.y); o.z = round_tf32(o.z); o.w = round_tf32(o.w); }
    reinterpret_cast<float4*>(y)[i] = o;
  }
}

// x[b, t] = t < Tc ? Wc[conds[b, t]] + pos_c[t] : Wi[codes[b, t - Tc]] + pos_i[t - Tc]
__global__ void __launch_bounds__(256)
token_embed_fwd_kernel(const long long* __restrict__ conds, const long long* __restrict__ codes, const float* __restrict__ Wc,
                       const float* __restrict__ pos_c, const float* __restrict__ Wi, const float* __restrict__ pos_i,
                       float* __restrict__ x, int B, int Tc, int Ti, int C4, int Vc, int Vi) {
  const int T = Tc + Ti;
  const long long total = (long long)B * T * C4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long m = i / C4;
    const int c = (int)(i - m * C4);
    const int b = (int)(m / T), t = (int)(m - (long long)b * T);
    float4 e, p;
    if (t < Tc) {
      long long id = conds[(long long)b * Tc + t];
      id = id < 0 ? 0 : (id >= Vc ? Vc - 1 : id);          // nn.Embedding device-asserts on such ids; never read out of bounds
      e = __ldg(reinterpret_cast<const float4*>(Wc) + id * C4 + c);
      p = __ldg(reinterpret_cast<const float4*>(pos_c) + (long long)t * C4 + c);
    } else {
      long long id = codes[(long long)b * Ti + (t - Tc)];
      id = id < 0 ? 0 : (id >= Vi ? Vi - 1 : id);
      e = __ldg(reinterpret_cast<const float4*>(Wi) + id * C4 + c);
      p = __ldg(reinterpret_cast<const float4*>(pos_i) + (long long)(t - Tc) * C4 + c);
    }
    reinterpret_cast<float4*>(x)[i] = make_float4(e.x + p.x, e.y + p.y, e.z + p.z, e.w + p.w);
  }
}

// gWc / gWi (zero-filled by the host wrapper) += scattered rows of g (nn.Embedding dense backward);
// gpos_c[t] / gpos_i[t] = sum over the batch of g[b, t] (deterministic: one thread walks the batch)
__global__ void __launch_bounds__(256)
token_embed_bwd_kernel(const long long* __restrict__ conds, const long long* __restrict__ codes, const float* __restrict__ g,
                       float* __restrict__ gWc, float* __restrict__ gpos_c, float* __restrict__ gWi, float* __restrict__ gpos_i,
                       int B, int Tc, int Ti, int C, int Vc, int Vi) {
  const int T = Tc + Ti;
  const long long total = (long long)T * C;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int t = (int)(i / C), c = (int)(i - (long long)t * C);
    float acc = 0.f;
    for (int b = 0; b < B; ++b) {
      const float v = g[((long long)b * T + t) * C + c];
      acc += v;
      if (t < Tc) {
        long long id = conds[(long long)b * Tc + t];
        id = id < 0 ? 0 : (id >= Vc ? Vc - 1 : id);
        atomicAdd(gWc + id * C + c, v);
      } else {
        long long id = codes[(long long)b * Ti + (t - Tc)];
        id = id < 0 ? 0 : (id >= Vi ? Vi - 1 : id);
        atomicAdd(gWi + id * C + c, v);
      }
    }
    if (t < Tc) gpos_c[(long long)t * C + c] = acc;
    else        gpos_i[(long long)(t - Tc) * C + c] = acc;
  }
}

// gpos_c / gpos_i alone, with token_embed_bwd_kernel's arithmetic (one thread walks the batch); the deterministic backward
// takes gWc / gWi from scatter_rows_det.  Grid from the shape: one thread per (t, c).
__global__ void __launch_bounds__(256)
token_embed_pos_bwd_kernel(const float* __restrict__ g, float* __restrict__ gpos_c, float* __restrict__ gpos_i, int B, int Tc, int Ti,
                           int C) {
  const int T = Tc + Ti;
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= (long long)T * C) return;
  const int t = (int)(i / C), c = (int)(i - (long long)t * C);
  float acc = 0.f;
  for (int b = 0; b < B; ++b) acc += g[((long long)b * T + t) * C + c];
  if (t < Tc) gpos_c[(long long)t * C + c] = acc;
  else        gpos_i[(long long)(t - Tc) * C + c] = acc;
}

// dst[b, t] = (off_dst <= t < off_dst + n) ? src[b, t - off_dst + off_src] : 0      (dst [B, T_dst, C], src [B, T_src, C])
__global__ void __launch_bounds__(256)
copy_rows_kernel(const float* __restrict__ src, float* __restrict__ dst, int B, int T_src, int T_dst, int off_src, int off_dst, int n,
                 int C4) {
  const long long total = (long long)B * T_dst * C4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long m = i / C4;
    const int c = (int)(i - m * C4);
    const int b = (int)(m / T_dst), t = (int)(m - (long long)b * T_dst);
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (t >= off_dst && t < off_dst + n)
      v = reinterpret_cast<const float4*>(src)[((long long)b * T_src + (t - off_dst + off_src)) * C4 + c];
    reinterpret_cast<float4*>(dst)[i] = v;
  }
}

// Sampling step (layers.py:66-81 with use_cache and layer_past): block (h, b) appends this step's key / value rows of its head
// to the cache at position `pos`, then attends its single query to cache rows 0 .. pos (no mask):
// scores -> shared memory, block-wide max / sum, out[d] = sum_j p_j V[j, d] with one thread per head dim (HS <= 128 = the
// block size).
// qkv [B, 3*C] (q | k | v thirds), cache_k / cache_v [B, Tmax, C], out [B, C].
template <int HS>
__global__ void __launch_bounds__(128)
decode_attention_kernel(const float* __restrict__ qkv, float* __restrict__ cache_k, float* __restrict__ cache_v,
                        float* __restrict__ out, int C, int Tmax, int pos, float scale) {
  extern __shared__ float sc[];                    // [pos + 1] scores, then 4 warp partials
  __shared__ float qs[HS];
  __shared__ float red[4];
  const int h = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
  const float* row = qkv + (long long)b * 3 * C + h * HS;
  float* kc = cache_k + (long long)b * Tmax * C + h * HS;
  float* vc = cache_v + (long long)b * Tmax * C + h * HS;
  if (tid < HS) {
    qs[tid] = row[tid];
    kc[(long long)pos * C + tid] = row[C + tid];
    vc[(long long)pos * C + tid] = row[2 * C + tid];
  }
  __syncthreads();                                  // the appended row is read below by other threads of this block
  const int n = pos + 1;
  float mx = -INFINITY;
  for (int j = tid; j < n; j += 128) {
    const float4* kr = reinterpret_cast<const float4*>(kc + (long long)j * C);
    float s = 0.f;
#pragma unroll
    for (int d = 0; d < HS / 4; ++d) {
      const float4 kv = kr[d];
      s = fmaf(qs[4 * d], kv.x, s); s = fmaf(qs[4 * d + 1], kv.y, s); s = fmaf(qs[4 * d + 2], kv.z, s); s = fmaf(qs[4 * d + 3], kv.w, s);
    }
    s *= scale;
    sc[j] = s;
    mx = fmaxf(mx, s);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if ((tid & 31) == 0) red[tid >> 5] = mx;
  __syncthreads();
  mx = fmaxf(fmaxf(red[0], red[1]), fmaxf(red[2], red[3]));
  __syncthreads();
  float sum = 0.f;
  for (int j = tid; j < n; j += 128) {
    const float e = expf(sc[j] - mx);
    sc[j] = e;
    sum += e;
  }
  sum = warp_sum(sum);
  if ((tid & 31) == 0) red[tid >> 5] = sum;
  __syncthreads();
  const float inv = 1.f / (red[0] + red[1] + red[2] + red[3]);
  if (tid < HS) {
    float acc = 0.f;
    for (int j = 0; j < n; ++j) acc = fmaf(sc[j], vc[(long long)j * C + tid], acc);
    out[(long long)b * C + h * HS + tid] = acc * inv;
  }
}

}  // namespace b200

// ---------------------------------------------------------------------------------------------
using namespace b200;

extern "C" int b200vq_time_mix_fwd(const float* x, const float* w, float* y, long long M, int T, int C, int round_out,
                                   void* streamv) {
  const cudaStream_t stream = static_cast<cudaStream_t>(streamv);
  B200_CHECK_ARG(M > 0 && T > 0 && C > 0 && C % 4 == 0 && M % T == 0, "time_mix: need C %% 4 == 0 and M %% T == 0 (M=%lld T=%d C=%d)", M, T, C);
  time_mix_fwd_kernel<<<s2_grid(M * (C / 4), 256), 256, 0, stream>>>(x, w, y, M, T, C / 4, round_out);
  B200_LAUNCH_OK("time_mix_fwd_kernel");
  return 0;
}

constexpr int kTimeMixRows = 64;
extern "C" size_t b200vq_time_mix_bwd_workspace_bytes(long long M, int C) {
  return (size_t)((M + kTimeMixRows - 1) / kTimeMixRows) * C * sizeof(float);
}

// gw_part [ceil(M/64), C]: summed over its rows (b200vq_colsum) it is the gradient of time_mix
extern "C" int b200vq_time_mix_bwd(const float* g, const float* x, const float* w, float* gx, float* gw_part, long long M, int T,
                                   int C, void* streamv) {
  const cudaStream_t stream = static_cast<cudaStream_t>(streamv);
  B200_CHECK_ARG(M > 0 && T > 0 && C > 0 && C % 4 == 0 && M % T == 0, "time_mix: need C %% 4 == 0 and M %% T == 0 (M=%lld T=%d C=%d)", M, T, C);
  const long long chunks = (M + kTimeMixRows - 1) / kTimeMixRows;
  B200_CHECK_ARG(chunks <= 65535, "time_mix_backward: too many rows (%lld)", M);
  const int C4 = C / 4;
  time_mix_bwd_kernel<<<dim3((C4 + 255) / 256, (unsigned)chunks), 256, 0, stream>>>(g, x, w, gx, gw_part, M, T, C4, kTimeMixRows);
  B200_LAUNCH_OK("time_mix_bwd_kernel");
  return 0;
}

extern "C" int b200vq_sqrelu(const float* x, const float* g, float* y, long long n, int grad, int round_out, void* streamv) {
  const cudaStream_t stream = static_cast<cudaStream_t>(streamv);
  B200_CHECK_ARG(n > 0 && n % 4 == 0, "sqrelu: n %% 4");
  B200_CHECK_ARG(!grad || g, "sqrelu: the derivative form needs the incoming gradient");
  sqrelu_kernel<<<s2_grid(n / 4, 256), 256, 0, stream>>>(x, g, y, n / 4, grad, round_out);
  B200_LAUNCH_OK("sqrelu_kernel");
  return 0;
}

extern "C" int b200vq_token_embed_fwd(const long long* conds, const long long* codes, const float* Wc, const float* pos_c,
                                      const float* Wi, const float* pos_i, float* x, int B, int Tc, int Ti, int C, int Vc, int Vi,
                                      void* streamv) {
  const cudaStream_t stream = static_cast<cudaStream_t>(streamv);
  B200_CHECK_ARG(B > 0 && Tc >= 0 && Ti >= 0 && Tc + Ti > 0 && C > 0 && C % 4 == 0, "token_embed: bad shape B=%d Tc=%d Ti=%d C=%d", B, Tc, Ti, C);
  token_embed_fwd_kernel<<<s2_grid((long long)B * (Tc + Ti) * (C / 4), 256), 256, 0, stream>>>(conds, codes, Wc, pos_c, Wi, pos_i, x, B,
                                                                                              Tc, Ti, C / 4, Vc, Vi);
  B200_LAUNCH_OK("token_embed_fwd_kernel");
  return 0;
}

extern "C" int b200vq_token_embed_bwd(const long long* conds, const long long* codes, const float* g, float* gWc, float* gpos_c,
                                      float* gWi, float* gpos_i, int B, int Tc, int Ti, int C, int Vc, int Vi, void* streamv) {
  const cudaStream_t stream = static_cast<cudaStream_t>(streamv);
  B200_CHECK_ARG(B > 0 && Tc >= 0 && Ti >= 0 && Tc + Ti > 0 && C > 0, "token_embed: bad shape B=%d Tc=%d Ti=%d C=%d", B, Tc, Ti, C);
  B200_CUDA_OK(cudaMemsetAsync(gWc, 0, (size_t)Vc * C * sizeof(float), stream));
  B200_CUDA_OK(cudaMemsetAsync(gWi, 0, (size_t)Vi * C * sizeof(float), stream));
  token_embed_bwd_kernel<<<s2_grid((long long)(Tc + Ti) * C, 256), 256, 0, stream>>>(conds, codes, g, gWc, gpos_c, gWi, gpos_i, B, Tc,
                                                                                    Ti, C, Vc, Vi);
  B200_LAUNCH_OK("token_embed_bwd_kernel");
  return 0;
}

// one scatter workspace, reused by the two tables in turn
extern "C" size_t b200vq_token_embed_bwd_deterministic_workspace_bytes(int B, int Tc, int Ti, int C, int Vc, int Vi) {
  if (B <= 0 || Tc < 0 || Ti < 0 || C <= 0) return 0;
  const size_t wc = Vc > 0 ? scatter_det_workspace_bytes((long long)B * Tc, Vc, C, kScatterRunToken) : 0;
  const size_t wi = Vi > 0 ? scatter_det_workspace_bytes((long long)B * Ti, Vi, C, kScatterRunToken) : 0;
  return wc > wi ? wc : wi;
}

extern "C" int b200vq_token_embed_bwd_deterministic(const long long* conds, const long long* codes, const float* g, float* gWc,
                                                    float* gpos_c, float* gWi, float* gpos_i, int B, int Tc, int Ti, int C, int Vc,
                                                    int Vi, void* workspace, size_t ws_bytes, void* streamv) {
  const cudaStream_t stream = static_cast<cudaStream_t>(streamv);
  B200_CHECK_ARG(B > 0 && Tc >= 0 && Ti >= 0 && Tc + Ti > 0 && C > 0, "token_embed: bad shape B=%d Tc=%d Ti=%d C=%d", B, Tc, Ti, C);
  B200_CHECK_ARG(Vc > 0 && Vi > 0, "token_embed: vocabulary sizes must be positive (Vc=%d Vi=%d)", Vc, Vi);
  B200_CHECK_ARG((long long)B * (Tc + Ti) <= (1LL << 30), "token_embed: too many tokens");
  B200_CHECK_ARG(g && gWc && gWi && (Tc == 0 || (conds && gpos_c)) && (Ti == 0 || (codes && gpos_i)) && workspace,
                 "token_embed_bwd_deterministic: null pointer argument");
  B200_CHECK_ARG(ws_bytes >= b200vq_token_embed_bwd_deterministic_workspace_bytes(B, Tc, Ti, C, Vc, Vi),
                 "token_embed_bwd_deterministic: workspace too small");
  const long long T = Tc + Ti;
  int rc = scatter_rows_det<kScatterRunToken>(conds, (long long)B * Tc, Vc, g, Tc, T, 0, C, gWc, workspace, ws_bytes, stream);
  if (rc) return rc;
  rc = scatter_rows_det<kScatterRunToken>(codes, (long long)B * Ti, Vi, g, Ti, T, Tc, C, gWi, workspace, ws_bytes, stream);
  if (rc) return rc;
  token_embed_pos_bwd_kernel<<<(unsigned)((T * C + 255) / 256), 256, 0, stream>>>(g, gpos_c, gpos_i, B, Tc, Ti, C);
  B200_LAUNCH_OK("token_embed_pos_bwd_kernel");
  return 0;
}

extern "C" int b200vq_copy_rows(const float* src, float* dst, int B, int T_src, int T_dst, int off_src, int off_dst, int n, int C,
                                void* streamv) {
  const cudaStream_t stream = static_cast<cudaStream_t>(streamv);
  B200_CHECK_ARG(B > 0 && T_src > 0 && T_dst > 0 && C > 0 && C % 4 == 0, "copy_rows: bad shape");
  B200_CHECK_ARG(n >= 0 && off_src >= 0 && off_dst >= 0 && off_src + n <= T_src && off_dst + n <= T_dst,
                 "copy_rows: window [%d, %d) / [%d, %d) outside the tensors", off_src, off_src + n, off_dst, off_dst + n);
  copy_rows_kernel<<<s2_grid((long long)B * T_dst * (C / 4), 256), 256, 0, stream>>>(src, dst, B, T_src, T_dst, off_src, off_dst, n, C / 4);
  B200_LAUNCH_OK("copy_rows_kernel");
  return 0;
}

extern "C" int b200vq_decode_attention(const float* qkv, float* cache_k, float* cache_v, float* out, int B, int heads, int hs,
                                       int Tmax, int pos, float scale, void* streamv) {
  const cudaStream_t stream = static_cast<cudaStream_t>(streamv);
  B200_CHECK_ARG(B > 0 && heads > 0 && (hs == 32 || hs == 64 || hs == 96 || hs == 128),
                 "decode_attention: head size must be 32, 64, 96 or 128 (got %d)", hs);
  B200_CHECK_ARG(pos >= 0 && pos < Tmax, "decode_attention: position %d outside the cache (%d rows)", pos, Tmax);
  B200_CHECK_ARG(B <= 65535, "decode_attention: batch too large");
  const int C = heads * hs;
  const size_t smem = (size_t)(pos + 1) * sizeof(float);
  B200_CHECK_ARG(smem <= 40 * 1024, "decode_attention: context of %d keys exceeds the score buffer", pos + 1);
  if (hs == 128)     decode_attention_kernel<128><<<dim3(heads, B), 128, smem, stream>>>(qkv, cache_k, cache_v, out, C, Tmax, pos, scale);
  else if (hs == 96) decode_attention_kernel<96><<<dim3(heads, B), 128, smem, stream>>>(qkv, cache_k, cache_v, out, C, Tmax, pos, scale);
  else if (hs == 64) decode_attention_kernel<64><<<dim3(heads, B), 128, smem, stream>>>(qkv, cache_k, cache_v, out, C, Tmax, pos, scale);
  else               decode_attention_kernel<32><<<dim3(heads, B), 128, smem, stream>>>(qkv, cache_k, cache_v, out, C, Tmax, pos, scale);
  B200_LAUNCH_OK("decode_attention_kernel");
  return 0;
}
