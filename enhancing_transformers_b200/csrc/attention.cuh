// Host functions shared by the attention files (attention.cu, attention_exact.cu, attention_f16.cu).  Their public entry
// points are declared in include/b200vq.h.
#pragma once
#include <cuda_runtime.h>

namespace b200 {

// delta[b,h,n] = rowsum(dO * O) of one (row, head); O and dO fp32, or fp16 where out_half / dout_half (attention.cu)
int attention_delta(const void* out, int out_half, const void* dout, int dout_half, float* delta, int B, int N, int heads, int dh,
                    cudaStream_t stream);

// attention_exact.cu.  cond_len < 0: no mask (stage 1); cond_len >= 0: the stage-2 mask, causal with a fully visible
// prefix of cond_len tokens.
// tf32 core: fp32 q/k/v (tf32-rounded by the GEMM that wrote them); O in fp32 (optionally tf32-rounded) or fp16
int attention_forward_tc(const float* qkv, void* out, int out_half, float* lse, int B, int N, int heads, int dh, float scale,
                         int round_out, int cond_len, cudaStream_t stream);
// delta must already hold rowsum(dO * O).  dqkv fp32 (optionally tf32-rounded) or, with out_half, fp16(dqkv * out_scale[0]).
int attention_backward_tc(const float* qkv, const float* dout, const float* lse, const float* delta, void* dqkv, int out_half,
                          const float* out_scale, int B, int N, int heads, int dh, float scale, int round_out, int cond_len,
                          cudaStream_t stream);
// 3xTF32 core (fp32-grade)
int attention_exact_forward(const float* qkv, float* out, float* lse, int B, int N, int heads, int dh, float scale,
                            int cond_len, cudaStream_t stream);
int attention_exact_backward(const float* qkv, const float* out, const float* lse, const float* dout, float* dqkv, float* delta,
                             int B, int N, int heads, int dh, float scale, int cond_len, cudaStream_t stream);
// Wide heads (dh 96 / 128), stage-2 mask only (cond_len >= 0), fp32 in and out: exact != 0 -> 3xTF32, otherwise one tf32
// pass with round_out.  The backward computes delta itself.
int attention_wide_forward(const float* qkv, float* out, float* lse, int B, int N, int heads, int dh, float scale, int cond_len,
                           int exact, int round_out, cudaStream_t stream);
int attention_wide_backward(const float* qkv, const float* out, const float* lse, const float* dout, float* dqkv, float* delta,
                            int B, int N, int heads, int dh, float scale, int cond_len, int exact, int round_out,
                            cudaStream_t stream);

}  // namespace b200
