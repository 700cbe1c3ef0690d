// Host functions shared by the attention files (attention.cu, attention_exact.cu, attention_f16.cu).  Their public entry
// points are declared in include/b200vq.h.
#pragma once
#include <cuda_runtime.h>

namespace b200 {

// delta[b,h,n] = rowsum(dO * O) of one (row, head) (attention.cu).  O and dO fp32; at dh 32 and 64 O may be fp16
// (out_half), and at dh 64 with fp16 O so may dO (dout_half).
int attention_delta(const void* out, int out_half, const void* dout, int dout_half, float* delta, int B, int N, int heads, int dh,
                    cudaStream_t stream);

// The mma.sync core (attention_exact.cu) on packed fp32 qkv [B*N, 3*heads*dh].
//   dh: 32 or 64; 96 or 128 only with cond_len >= 0 and fp32 output.
//   passes: 1 (tf32; outputs tf32-rounded if round_out) or 3 (3xTF32, fp32-grade; round_out ignored).
//   out_half / dqkv_half: fp16 output (passes 1, dh 32 / 64): O of the forward, fp16(dqkv * out_scale[0]) of the
//   backward.
//   cond_len < 0: no mask (stage 1); cond_len >= 0: the stage-2 mask, causal with a fully visible prefix of cond_len
//   tokens.
int attention_forward(int dh, int passes, int out_half, int cond_len, int round_out, const float* qkv, void* out, float* lse, int B,
                      int N, int heads, float scale, cudaStream_t stream);
// Computes delta from the forward's output o (fp16 if o_half) and dout into `delta` [B*heads*N], then dqkv.
int attention_backward(int dh, int passes, int dqkv_half, int cond_len, int round_out, const float* qkv, const void* o, int o_half,
                       const float* lse, const float* dout, float* delta, void* dqkv, const float* out_scale, int B, int N,
                       int heads, float scale, cudaStream_t stream);

}  // namespace b200
