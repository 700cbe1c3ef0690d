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

// delta[b,h,n] = sum_d dO[b,n,h,d] * O[b,n,h,d].  HBM-bound: LANES adjacent lanes per (row, head), reduced with shuffles.
//   VEC == 1 (dh 32 / 64): LANES = dh / 4, one float4 of O and dO per lane, so a warp streams 512 contiguous bytes of each
//     tensor.  O is fp32, or fp16 (OHALF) when the forward stored it for an fp16 to_out GEMM; dO is fp16 (DHALF) on the
//     fp16 data path.
//   VEC > 1 (dh 96 / 128, fp32): dh / 4 lanes would be 24 at dh 96, not a power of two, so LANES = 8, lane l summing
//     float4s l, l + 8, ... (VEC = dh / 32 of them).  Each step of the 8 lanes reads 128 contiguous bytes.
template <int LANES, int VEC, int OHALF, int DHALF>
__global__ void __launch_bounds__(256)
attn_delta_kernel(const void* __restrict__ o, const void* __restrict__ dout, float* __restrict__ delta, long long groups,
                  int N, int heads) {
  static_assert(VEC == 1 || (!OHALF && !DHALF), "the multi-float4 form reads fp32 O and dO");
  const long long stride = (long long)gridDim.x * blockDim.x;
  const long long total = groups * LANES;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < ((total + 31) / 32) * 32; i += stride) {
    float s = 0.f;
    if (i < total) {
      if constexpr (VEC == 1) {
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
      } else {
        const long long base = (i / LANES) * (LANES * VEC) + (i & (LANES - 1));
        const float4* a = reinterpret_cast<const float4*>(o) + base;
        const float4* b = reinterpret_cast<const float4*>(dout) + base;
#pragma unroll
        for (int v = 0; v < VEC; ++v) {
          const float4 x = a[LANES * v], y = b[LANES * v];
          s += x.x * y.x + x.y * y.y + x.z * y.z + x.w * y.w;
        }
      }
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

int attention_delta(const void* out, int out_half, const void* dout, int dout_half, float* delta, int B, int N, int heads, int dh,
                    cudaStream_t stream) {
  B200_CHECK_ARG(dh <= 64 || (!out_half && !dout_half), "attention: head size %d takes fp32 O and dO", dh);
  B200_CHECK_ARG(!dout_half || (out_half && dh == 64), "attention: fp16 dO takes fp16 O and head size 64");
  const long long groups = (long long)B * N * heads;
  long long blocks = (groups * (dh > 64 ? 8 : dh / 4) + 255) / 256;
  const long long cap = (long long)num_sms() * 16;
  if (blocks > cap) blocks = cap;
  const unsigned g = (unsigned)blocks;
#define B200_DELTA(L, V, OH, DHF) attn_delta_kernel<L, V, OH, DHF><<<g, 256, 0, stream>>>(out, dout, delta, groups, N, heads)
  if (dh == 128)                     B200_DELTA(8, 4, 0, 0);
  else if (dh == 96)                 B200_DELTA(8, 3, 0, 0);
  else if (dh == 64 && dout_half)    B200_DELTA(16, 1, 1, 1);
  else if (dh == 64 && out_half)     B200_DELTA(16, 1, 1, 0);
  else if (dh == 64)                 B200_DELTA(16, 1, 0, 0);
  else if (out_half)                 B200_DELTA(8, 1, 1, 0);
  else                               B200_DELTA(8, 1, 0, 0);
#undef B200_DELTA
  B200_LAUNCH_OK("attn_delta_kernel");
  return 0;
}

}  // namespace b200

using namespace b200;

extern "C" int b200vq_attention_fwd(const float* qkv, void* out, int out_half, float* lse, int B, int N, int heads, int dh,
                                    float scale, int round_out, void* streamv) {
  B200_CHECK_ARG(B > 0 && N > 0 && heads > 0, "attention: empty problem");
  B200_CHECK_ARG(dh == 64 || dh == 32, "attention: dim_head must be 32 or 64 (got %d)", dh);
  return attention_forward(dh, 1, out_half, -1, round_out, qkv, out, lse, B, N, heads, scale, static_cast<cudaStream_t>(streamv));
}

extern "C" int b200vq_attention_bwd(const float* qkv, const void* out, int out_half, const float* lse, const float* dout, void* dqkv,
                                    int dqkv_half, const float* dqkv_scale, float* delta, int B, int N, int heads, int dh,
                                    float scale, int round_out, void* streamv) {
  B200_CHECK_ARG(B > 0 && N > 0 && heads > 0, "attention: empty problem");
  B200_CHECK_ARG(dh == 64 || dh == 32, "attention: dim_head must be 32 or 64 (got %d)", dh);
  return attention_backward(dh, 1, dqkv_half, -1, round_out, qkv, out, out_half, lse, dout, delta, dqkv, dqkv_scale, B, N, heads,
                            scale, static_cast<cudaStream_t>(streamv));
}

// Stage-2 attention (reference enhancing/modules/stage2/layers.py:76-89): causal mask whose first cond_len tokens (the
// condition prefix) see each other fully -- query q attends to key k iff k <= max(q, cond_len - 1).  Same packed qkv layout
// as the stage-1 core (the reference's (T, B*nh, hs) views are that layout transposed).  exact != 0: 3xTF32 mma.sync kernels
// (precision="parity"); otherwise the single-pass tf32 kernels with the same mask.
extern "C" int b200vq_attention_causal_fwd(const float* qkv, float* out, float* lse, int B, int N, int heads, int dh, float scale,
                                           int cond_len, int exact, int round_out, void* streamv) {
  B200_CHECK_ARG(B > 0 && N > 0 && heads > 0, "attention: empty problem");
  B200_CHECK_ARG(dh == 64 || dh == 32 || dh == 96 || dh == 128, "attention: head size must be 32 or 64, or 96 or 128 (got %d)", dh);
  B200_CHECK_ARG(cond_len >= 0 && cond_len <= N, "attention: cond_len %d outside [0, %d]", cond_len, N);
  return attention_forward(dh, exact ? 3 : 1, 0, cond_len, round_out, qkv, out, lse, B, N, heads, scale,
                           static_cast<cudaStream_t>(streamv));
}

extern "C" int b200vq_attention_causal_bwd(const float* qkv, const float* out, const float* lse, const float* dout, float* dqkv,
                                           float* delta, int B, int N, int heads, int dh, float scale, int cond_len, int exact,
                                           int round_out, void* streamv) {
  B200_CHECK_ARG(B > 0 && N > 0 && heads > 0, "attention: empty problem");
  B200_CHECK_ARG(dh == 64 || dh == 32 || dh == 96 || dh == 128, "attention: head size must be 32 or 64, or 96 or 128 (got %d)", dh);
  B200_CHECK_ARG(cond_len >= 0 && cond_len <= N, "attention: cond_len %d outside [0, %d]", cond_len, N);
  return attention_backward(dh, exact ? 3 : 1, 0, cond_len, round_out, qkv, out, 0, lse, dout, delta, dqkv, nullptr, B, N, heads,
                            scale, static_cast<cudaStream_t>(streamv));
}
