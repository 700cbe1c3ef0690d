// Attention core entry points (reference enhancing/modules/stage1/layers.py:124-130:
// q k^T * scale -> softmax -> . v) and the row-wise helper of its backward.
//
// The reference materialises and saves a [B, heads, N, N] fp32 probability tensor per layer
// (6.4 GB at B=128, base).  Here the scores live in registers only (attention_f16.cu: wgmma
// kernels of the fp16 data path; attention_exact.cu: mma.sync tf32 / 3xTF32 kernels and the
// stage-2 mask); backward recomputes them from the saved log-sum-exp and needs
// delta = rowsum(dO * O), computed below.
#include "../../include/b200vq.h"
#include "attention.cuh"
#include "common.cuh"

namespace b200 {

// delta[b,h,n] = sum_d dO[b,n,h,d] * O[b,n,h,d].  HBM-bound: one float4 of O and dO per thread, dh/4 adjacent
// lanes per (row, head) reduced with shuffles, so a warp streams 512 contiguous bytes of each tensor.
// O is fp32, or fp16 (OHALF) when the forward stored it for an fp16 to_out GEMM.
template <int LANES, int OHALF, int DHALF>   // lanes per (row, head) = dh / 4: 16 (dh 64) or 8 (dh 32)
__global__ void __launch_bounds__(256)
attn_delta_kernel(const void* __restrict__ o, const void* __restrict__ dout, float* __restrict__ delta, long long groups,
                  int N, int heads) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  const long long total = groups * LANES;          // one thread per float4
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < ((total + 31) / 32) * 32; i += stride) {
    float s = 0.f;
    if (i < total) {
      auto load4 = [i](const void* ptr, bool half) {
        if (half) {
          const uint2 h = reinterpret_cast<const uint2*>(ptr)[i];
          const float2 lo = __half22float2(*reinterpret_cast<const __half2*>(&h.x)), hi = __half22float2(*reinterpret_cast<const __half2*>(&h.y));
          return make_float4(lo.x, lo.y, hi.x, hi.y);
        }
        return reinterpret_cast<const float4*>(ptr)[i];
      };
      const float4 a = load4(o, OHALF != 0);
      const float4 b = load4(dout, DHALF != 0);
      s = a.x * b.x + a.y * b.y + a.z * b.z + a.w * b.w;
    }
#pragma unroll
    for (int off = LANES / 2; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
    if (i < total && (i & (LANES - 1)) == 0) {
      const long long g = i / LANES;                // (b*N + n) * heads + h
      const int h = (int)(g % heads);
      const long long bn = g / heads;
      const long long b = bn / N, n = bn % N;
      delta[(b * heads + h) * N + n] = s;
    }
  }
}

// The same sum for dh 96 / 128 (fp32 only): dh / 4 lanes per row would be 24 at dh 96, not a power of two, so a row group is
// 8 lanes, lane l summing float4s l, l + 8, ... (VEC = dh / 32 of them).  Each step of the 8 lanes reads 128 contiguous bytes.
template <int VEC>
__global__ void __launch_bounds__(256)
attn_delta_wide_kernel(const float* __restrict__ o, const float* __restrict__ dout, float* __restrict__ delta, long long groups, int N,
                       int heads) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  const long long total = groups * 8;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < ((total + 31) / 32) * 32; i += stride) {
    float s = 0.f;
    if (i < total) {
      const long long base = (i >> 3) * (8 * VEC) + (i & 7);
      const float4* a = reinterpret_cast<const float4*>(o) + base;
      const float4* b = reinterpret_cast<const float4*>(dout) + base;
#pragma unroll
      for (int v = 0; v < VEC; ++v) {
        const float4 x = a[8 * v], y = b[8 * v];
        s += x.x * y.x + x.y * y.y + x.z * y.z + x.w * y.w;
      }
    }
#pragma unroll
    for (int off = 4; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
    if (i < total && (i & 7) == 0) {
      const long long g = i >> 3;                   // (b*N + n) * heads + h
      const int h = (int)(g % heads);
      const long long bn = g / heads;
      const long long b = bn / N, n = bn % N;
      delta[(b * heads + h) * N + n] = s;
    }
  }
}

int attention_delta(const void* out, int out_half, const void* dout, int dout_half, float* delta, int B, int N, int heads, int dh,
                    cudaStream_t stream) {
  const long long groups = (long long)B * N * heads;
  if (dh == 96 || dh == 128) {
    B200_CHECK_ARG(!out_half && !dout_half, "attention: head size %d takes fp32 O and dO", dh);
    long long blocks = (groups * 8 + 255) / 256;
    const long long cap = (long long)num_sms() * 16;
    if (blocks > cap) blocks = cap;
    const float* o = static_cast<const float*>(out);
    const float* d = static_cast<const float*>(dout);
    if (dh == 128) attn_delta_wide_kernel<4><<<(unsigned)blocks, 256, 0, stream>>>(o, d, delta, groups, N, heads);
    else           attn_delta_wide_kernel<3><<<(unsigned)blocks, 256, 0, stream>>>(o, d, delta, groups, N, heads);
    B200_LAUNCH_OK("attn_delta_wide_kernel");
    return 0;
  }
  const long long threads = groups * (dh / 4);
  long long blocks = (threads + 255) / 256;
  const long long cap = (long long)num_sms() * 16;
  if (blocks > cap) blocks = cap;
  const unsigned g = (unsigned)blocks;
#define B200_DELTA(L, OH, DHF) attn_delta_kernel<L, OH, DHF><<<g, 256, 0, stream>>>(out, dout, delta, groups, N, heads)
  if (dh == 64) {
    if (out_half && dout_half) B200_DELTA(16, 1, 1);
    else if (out_half)         B200_DELTA(16, 1, 0);
    else if (dout_half)        B200_DELTA(16, 0, 1);
    else                       B200_DELTA(16, 0, 0);
  } else {
    if (out_half && dout_half) B200_DELTA(8, 1, 1);
    else if (out_half)         B200_DELTA(8, 1, 0);
    else if (dout_half)        B200_DELTA(8, 0, 1);
    else                       B200_DELTA(8, 0, 0);
  }
#undef B200_DELTA
  B200_LAUNCH_OK("attn_delta_kernel");
  return 0;
}

}  // namespace b200

using namespace b200;

extern "C" int b200vq_attention_fwd(const float* qkv, void* out, int out_half, float* lse, int B, int N, int heads, int dh,
                                    float scale, int round_out, void* streamv) {
  const cudaStream_t stream = static_cast<cudaStream_t>(streamv);
  B200_CHECK_ARG(B > 0 && N > 0 && heads > 0, "attention: empty problem");
  B200_CHECK_ARG(dh == 64 || dh == 32, "attention: dim_head must be 32 or 64 (got %d)", dh);
  return attention_forward_tc(qkv, out, out_half, lse, B, N, heads, dh, scale, round_out, -1, stream);
}

extern "C" int b200vq_attention_bwd(const float* qkv, const void* out, int out_half, const float* lse, const float* dout, void* dqkv,
                                    int dqkv_half, const float* dqkv_scale, float* delta, int B, int N, int heads, int dh,
                                    float scale, int round_out, void* streamv) {
  const cudaStream_t stream = static_cast<cudaStream_t>(streamv);
  B200_CHECK_ARG(B > 0 && N > 0 && heads > 0, "attention: empty problem");
  B200_CHECK_ARG(dh == 64 || dh == 32, "attention: dim_head must be 32 or 64 (got %d)", dh);
  int rc = attention_delta(out, out_half, dout, 0, delta, B, N, heads, dh, stream);
  if (rc) return rc;
  return attention_backward_tc(qkv, dout, lse, delta, dqkv, dqkv_half, dqkv_scale, B, N, heads, dh, scale, round_out, -1, stream);
}

// Stage-2 attention (reference enhancing/modules/stage2/layers.py:76-89): causal mask whose first cond_len tokens (the
// condition prefix) see each other fully -- query q attends to key k iff k <= max(q, cond_len - 1).  Same packed qkv layout
// as the stage-1 core (the reference's (T, B*nh, hs) views are that layout transposed).  exact != 0: 3xTF32 mma.sync kernels
// (precision="parity"); otherwise the single-pass tf32 kernels with the same mask.  Head sizes 96 and 128 run on the wide-head
// kernels of attention_exact.cu, which read their resident operand from shared memory.
extern "C" int b200vq_attention_causal_fwd(const float* qkv, float* out, float* lse, int B, int N, int heads, int dh, float scale,
                                           int cond_len, int exact, int round_out, void* streamv) {
  const cudaStream_t stream = static_cast<cudaStream_t>(streamv);
  B200_CHECK_ARG(B > 0 && N > 0 && heads > 0, "attention: empty problem");
  B200_CHECK_ARG(dh == 64 || dh == 32 || dh == 96 || dh == 128, "attention: head size must be 32 or 64, or 96 or 128 (got %d)", dh);
  B200_CHECK_ARG(cond_len >= 0 && cond_len <= N, "attention: cond_len %d outside [0, %d]", cond_len, N);
  if (dh > 64) return attention_wide_forward(qkv, out, lse, B, N, heads, dh, scale, cond_len, exact, round_out, stream);
  if (exact) return attention_exact_forward(qkv, out, lse, B, N, heads, dh, scale, cond_len, stream);
  return attention_forward_tc(qkv, out, 0, lse, B, N, heads, dh, scale, round_out, cond_len, stream);
}

extern "C" int b200vq_attention_causal_bwd(const float* qkv, const float* out, const float* lse, const float* dout, float* dqkv,
                                           float* delta, int B, int N, int heads, int dh, float scale, int cond_len, int exact,
                                           int round_out, void* streamv) {
  const cudaStream_t stream = static_cast<cudaStream_t>(streamv);
  B200_CHECK_ARG(B > 0 && N > 0 && heads > 0, "attention: empty problem");
  B200_CHECK_ARG(dh == 64 || dh == 32 || dh == 96 || dh == 128, "attention: head size must be 32 or 64, or 96 or 128 (got %d)", dh);
  B200_CHECK_ARG(cond_len >= 0 && cond_len <= N, "attention: cond_len %d outside [0, %d]", cond_len, N);
  if (dh > 64) return attention_wide_backward(qkv, out, lse, dout, dqkv, delta, B, N, heads, dh, scale, cond_len, exact, round_out, stream);
  if (exact) return attention_exact_backward(qkv, out, lse, dout, dqkv, delta, B, N, heads, dh, scale, cond_len, stream);
  int rc = attention_delta(out, 0, dout, 0, delta, B, N, heads, dh, stream);
  if (rc) return rc;
  return attention_backward_tc(qkv, dout, lse, delta, dqkv, 0, nullptr, B, N, heads, dh, scale, round_out, cond_len, stream);
}
