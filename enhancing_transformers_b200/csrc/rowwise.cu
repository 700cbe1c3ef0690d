// HBM-bound row-wise kernels around the GEMMs: LayerNorm forward/backward
// (reference layers.py:85-92,143,150), patch <-> image re-layout for the kernel==stride
// convolutions (layers.py:168-171,202-205), column sums (bias gradients), split-K reduction
// and tf32 rounding of GEMM operands.  All are coalesced float4 streams sized to the SM count.
#include "../../include/b200vq.h"
#include "common.cuh"

namespace b200 {

constexpr float kLnEps = 1e-5f;

// ---------------------------------------------------------------------------------------------
// LayerNorm forward: one warp per row, row held in registers (NV float4 per lane, D <= 128*NV)
// ---------------------------------------------------------------------------------------------
template <int NV>
__global__ void __launch_bounds__(256)
ln_fwd_kernel(const float* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta,
              float* __restrict__ y, __half* __restrict__ y16, float* __restrict__ mean_out, float* __restrict__ rstd_out,
              int M, int D, int round_out) {
  const int warps_per_block = blockDim.x >> 5;
  const int lane = threadIdx.x & 31;
  const int nv = D >> 2;
  for (int row = blockIdx.x * warps_per_block + (threadIdx.x >> 5); row < M; row += gridDim.x * warps_per_block) {
    const float4* xr = reinterpret_cast<const float4*>(x + (size_t)row * D);
    float4 v[NV];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c = lane + i * 32;
      v[i] = c < nv ? xr[c] : make_float4(0.f, 0.f, 0.f, 0.f);
      s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
    }
    const float mu = warp_sum(s) / (float)D;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c = lane + i * 32;
      if (c < nv) {
        const float a = v[i].x - mu, b = v[i].y - mu, cc = v[i].z - mu, d = v[i].w - mu;
        q += (a * a + b * b) + (cc * cc + d * d);
      }
    }
    const float rstd = rsqrtf(warp_sum(q) / (float)D + kLnEps);
    float4* yr = reinterpret_cast<float4*>(y + (size_t)row * D);
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c = lane + i * 32;
      if (c < nv) {
        const float4 g = __ldg(reinterpret_cast<const float4*>(gamma) + c);
        const float4 b = __ldg(reinterpret_cast<const float4*>(beta) + c);
        float4 o;
        o.x = (v[i].x - mu) * rstd * g.x + b.x;
        o.y = (v[i].y - mu) * rstd * g.y + b.y;
        o.z = (v[i].z - mu) * rstd * g.z + b.z;
        o.w = (v[i].w - mu) * rstd * g.w + b.w;
        if (y16) {   // the normalised row only feeds an fp16 GEMM: 8 bytes per 4 values
          uint2 pk;
          pk.x = pack_half2_sat(o.x, o.y); pk.y = pack_half2_sat(o.z, o.w);
          reinterpret_cast<uint2*>(y16 + (size_t)row * D)[c] = pk;
        }
        if (y) {
          if (round_out) { o.x = round_tf32(o.x); o.y = round_tf32(o.y); o.z = round_tf32(o.z); o.w = round_tf32(o.w); }
          yr[c] = o;
        }
      }
    }
    if (lane == 0) {
      if (mean_out) mean_out[row] = mu;
      if (rstd_out) rstd_out[row] = rstd;
    }
  }
}

// LayerNorm backward.  dx = rstd * (dy*g - mean(dy*g) - xh * mean(dy*g*xh)) [+ dres];
// per-CTA partial sums of dgamma = sum dy*xh and dbeta = sum dy go to part[blk][NACC][D]; with NACC == 3 the
// column sums of the *output* dx are produced too (dx is the gradient arriving at the bias of the Linear that
// fed this residual stream, reference layers.py:118 / :99-101, so its bias gradient needs no pass of its own).
// HBM-bound (reads dy, x, dres; writes dx).  One warp per row; what limits the stream is how many bytes a
// warp keeps in flight, i.e. registers: the column accumulators therefore live in the warp's private
// shared-memory slab (conflict-free float4 read-modify-write per row), which leaves the register file to
// the row being loaded, and the dres row is requested together with x and dy so a row costs one HBM
// round trip, not two.
// DYH: dy arrives as fp16 carrying a gradient scale (the output of an fp16 dgrad GEMM) and is multiplied by *dy_scale (1/S)
// on the way in: the GEMM writes, and this kernel reads, half the bytes of the fp32 hand-off.
template <int NV, int NACC, int DYH>
__global__ void __launch_bounds__(256, NV <= 6 ? 2 : 1)
ln_bwd_kernel(const void* __restrict__ dyv, const float* __restrict__ dy_scale, const float* __restrict__ x,
              const float* __restrict__ mean, const float* __restrict__ rstd, const float* __restrict__ gamma,
              const float* __restrict__ dres, float* __restrict__ dx, __half* __restrict__ dx16,
              const float* __restrict__ scale_ptr, float* __restrict__ part, int M, int D, int round_out) {
  extern __shared__ float sm[];   // [warps][NACC][D]
  const float gscale = (dx16 && scale_ptr) ? __ldg(scale_ptr) : 1.f;   // gradient scale of the fp16 copy
  const float dys = (DYH && dy_scale) ? __ldg(dy_scale) : 1.f;
  const float* dy = static_cast<const float*>(dyv);
  const __half* dyh = static_cast<const __half*>(dyv);
  const int warps_per_block = blockDim.x >> 5;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nv = D >> 2;
  float4* acc_g = reinterpret_cast<float4*>(sm + (size_t)warp * NACC * D);
  float4* acc_b = reinterpret_cast<float4*>(sm + (size_t)warp * NACC * D + D);
  float4* acc_o = reinterpret_cast<float4*>(sm + (size_t)warp * NACC * D + 2 * D);   // used when NACC == 3
  // fp16 dy: a lane's four columns are 8 bytes, and 8-byte loads halve the bytes each load instruction keeps in flight
  // (measured: the fp16 row read was SLOWER than the fp32 one, 296 vs 272 us).  With D % 8 == 0 the warp therefore fetches the
  // row as 16-byte loads (lane l: halfs 8l..8l+7 of each 256-column block), parks it in a private shared-memory slab and
  // every lane picks up its own 8 bytes per chunk from there.
  const bool wide16 = DYH && (D & 7) == 0;
  uint4* stage = reinterpret_cast<uint4*>(sm + (size_t)warps_per_block * NACC * D) + (size_t)warp * (D >> 3);
  const float4 zero4 = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int c = lane + i * 32;
    if (c < nv) {
      acc_g[c] = zero4; acc_b[c] = zero4;
      if (NACC == 3) acc_o[c] = zero4;
    }
  }
  for (int row = blockIdx.x * warps_per_block + warp; row < M; row += gridDim.x * warps_per_block) {
    const float4* xr = reinterpret_cast<const float4*>(x + (size_t)row * D);
    const float4* gr = reinterpret_cast<const float4*>(dy + (size_t)row * D);
    const uint2* gh = reinterpret_cast<const uint2*>(dyh + (size_t)row * D);
    const float4* rr = dres ? reinterpret_cast<const float4*>(dres + (size_t)row * D) : nullptr;
    float4 xh[NV], g[NV], r[NV];
    constexpr int NV16 = (NV + 1) / 2;
    uint4 wide[NV16];
    if (wide16) {
#pragma unroll
      for (int i = 0; i < NV16; ++i) {
        const int c = lane + i * 32;
        if (c < (D >> 3)) wide[i] = reinterpret_cast<const uint4*>(gh)[c];
      }
    }
#pragma unroll
    for (int i = 0; i < NV; ++i) {          // all of the row's HBM requests go out back to back
      const int c = lane + i * 32;
      xh[i] = zero4; r[i] = zero4;
      if (c < nv) {
        xh[i] = xr[c];
        if (rr) r[i] = rr[c];
      }
    }
    if (wide16) {
#pragma unroll
      for (int i = 0; i < NV16; ++i) {
        const int c = lane + i * 32;
        if (c < (D >> 3)) stage[c] = wide[i];
      }
      __syncwarp();
    }
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c = lane + i * 32;
      g[i] = zero4;
      if (c < nv) {
        if (DYH) {
          const uint2 pk = wide16 ? reinterpret_cast<const uint2*>(stage)[c] : gh[c];
          const float2 lo = __half22float2(*reinterpret_cast<const __half2*>(&pk.x));
          const float2 hi = __half22float2(*reinterpret_cast<const __half2*>(&pk.y));
          g[i] = make_float4(lo.x * dys, lo.y * dys, hi.x * dys, hi.y * dys);
        } else {
          g[i] = gr[c];
        }
      }
    }
    const float mu = mean[row], rs = rstd[row];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c = lane + i * 32;
      if (c < nv) {
        const float4 gm = __ldg(reinterpret_cast<const float4*>(gamma) + c);
        const float4 d = g[i];
        const float4 h = make_float4((xh[i].x - mu) * rs, (xh[i].y - mu) * rs, (xh[i].z - mu) * rs, (xh[i].w - mu) * rs);
        float4 ag = acc_g[c], ab = acc_b[c];
        ag.x += d.x * h.x; ag.y += d.y * h.y; ag.z += d.z * h.z; ag.w += d.w * h.w;
        ab.x += d.x; ab.y += d.y; ab.z += d.z; ab.w += d.w;
        acc_g[c] = ag; acc_b[c] = ab;
        const float4 t = make_float4(d.x * gm.x, d.y * gm.y, d.z * gm.z, d.w * gm.w);
        s1 += (t.x + t.y) + (t.z + t.w);
        s2 += (t.x * h.x + t.y * h.y) + (t.z * h.z + t.w * h.w);
        xh[i] = h; g[i] = t;
      }
    }
    const float m1 = warp_sum(s1) / (float)D, m2 = warp_sum(s2) / (float)D;
    float4* outr = reinterpret_cast<float4*>(dx + (size_t)row * D);
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c = lane + i * 32;
      if (c < nv) {
        float4 o;
        o.x = rs * (g[i].x - m1 - xh[i].x * m2) + r[i].x;
        o.y = rs * (g[i].y - m1 - xh[i].y * m2) + r[i].y;
        o.z = rs * (g[i].z - m1 - xh[i].z * m2) + r[i].z;
        o.w = rs * (g[i].w - m1 - xh[i].w * m2) + r[i].w;
        if (dx16) {   // the same gradient, scaled, as the fp16 operand of the next dgrad / wgrad GEMMs
          uint2 pk;
          pk.x = pack_half2_sat(o.x * gscale, o.y * gscale); pk.y = pack_half2_sat(o.z * gscale, o.w * gscale);
          reinterpret_cast<uint2*>(dx16 + (size_t)row * D)[c] = pk;
        }
        if (round_out) { o.x = round_tf32(o.x); o.y = round_tf32(o.y); o.z = round_tf32(o.z); o.w = round_tf32(o.w); }
        outr[c] = o;
        if (NACC == 3) {
          float4 ao = acc_o[c];
          ao.x += o.x; ao.y += o.y; ao.z += o.z; ao.w += o.w;
          acc_o[c] = ao;
        }
      }
    }
  }
  // CTA-level reduction of the per-warp column partials
  __syncthreads();
  for (int j = threadIdx.x; j < NACC * D; j += blockDim.x) {
    float a = 0.f;
    for (int w = 0; w < warps_per_block; ++w) a += sm[(size_t)w * NACC * D + j];
    part[(size_t)blockIdx.x * NACC * D + j] = a;
  }
}

// out[j] = sum_i part[i][j], j < n  (deterministic second stage)
__global__ void colpart_reduce_kernel(const float* __restrict__ part, int nparts, int n, float* __restrict__ out) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  float a = 0.f;
  for (int i = 0; i < nparts; ++i) a += part[(size_t)i * n + j];
  out[j] = a;
}

// part is [nparts][nacc][D] -> dgamma[D], dbeta[D] (, dxsum[D]).  A CTA owns 32 columns; its 8 warps take every 8th
// partial (independent, coalesced 128-byte loads) and meet in shared memory: a chain of nparts / 8 loads per thread
// instead of nparts.
__global__ void __launch_bounds__(256)
ln_param_reduce_kernel(const float* __restrict__ part, int nparts, int D, int nacc, float* __restrict__ dgamma,
                       float* __restrict__ dbeta, float* __restrict__ dxsum) {
  __shared__ float sm[8][32];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int j = blockIdx.x * 32 + tx;
  const int total = nacc * D;
  float a0 = 0.f, a1 = 0.f;
  if (j < total) {
    int i = ty;
    for (; i + 8 < nparts; i += 16) {
      a0 += part[(size_t)i * total + j];
      a1 += part[(size_t)(i + 8) * total + j];
    }
    if (i < nparts) a0 += part[(size_t)i * total + j];
  }
  sm[ty][tx] = a0 + a1;
  __syncthreads();
  if (ty == 0 && j < total) {
    float a = sm[0][tx];
#pragma unroll
    for (int w = 1; w < 8; ++w) a += sm[w][tx];
    if (j < D) dgamma[j] = a;
    else if (j < 2 * D) dbeta[j - D] = a;
    else dxsum[j - 2 * D] = a;
  }
}

// column sums of X[M, N] (bias gradients): stage 1 writes part[blockIdx.y][N].
// grid = (ceil(N/128), R): a CTA owns 128 columns (32 float4 lanes) and every R-th group of 8 rows,
// accumulates in registers over its rows (4 independent 16-byte loads in flight per thread) and
// reduces across its 8 row-lanes once at the end.
__global__ void __launch_bounds__(256)
colsum_kernel(const float* __restrict__ X, long long ld, int M, int N, float* __restrict__ part) {
  __shared__ float4 sm[8][32];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + tx;          // float4 column
  const int nv = N >> 2;
  float4 a0 = make_float4(0.f, 0.f, 0.f, 0.f), a1 = a0, a2 = a0, a3 = a0;
  if (c < nv) {
    const long long stride = 8ll * gridDim.y;
    long long r = (long long)blockIdx.y * 8 + ty;
    const float* base = X + c * 4;
    for (; r + 3 * stride < M; r += 4 * stride) {
      const float4 v0 = *reinterpret_cast<const float4*>(base + r * ld);
      const float4 v1 = *reinterpret_cast<const float4*>(base + (r + stride) * ld);
      const float4 v2 = *reinterpret_cast<const float4*>(base + (r + 2 * stride) * ld);
      const float4 v3 = *reinterpret_cast<const float4*>(base + (r + 3 * stride) * ld);
      a0.x += v0.x; a0.y += v0.y; a0.z += v0.z; a0.w += v0.w;
      a1.x += v1.x; a1.y += v1.y; a1.z += v1.z; a1.w += v1.w;
      a2.x += v2.x; a2.y += v2.y; a2.z += v2.z; a2.w += v2.w;
      a3.x += v3.x; a3.y += v3.y; a3.z += v3.z; a3.w += v3.w;
    }
    for (; r < M; r += stride) {
      const float4 v0 = *reinterpret_cast<const float4*>(base + r * ld);
      a0.x += v0.x; a0.y += v0.y; a0.z += v0.z; a0.w += v0.w;
    }
  }
  a0.x += a1.x + a2.x + a3.x; a0.y += a1.y + a2.y + a3.y; a0.z += a1.z + a2.z + a3.z; a0.w += a1.w + a2.w + a3.w;
  sm[ty][tx] = a0;
  __syncthreads();
  if (ty == 0 && c < nv) {
    float4 t = sm[0][tx];
    for (int w = 1; w < 8; ++w) { t.x += sm[w][tx].x; t.y += sm[w][tx].y; t.z += sm[w][tx].z; t.w += sm[w][tx].w; }
    *reinterpret_cast<float4*>(part + (size_t)blockIdx.y * N + c * 4) = t;
  }
}

// out[i] = sum_z part[z][i] (+ bias-free), used after split-K wgrad
__global__ void splitk_reduce_kernel(const float* __restrict__ part, int splits, long long n4, long long stride4,
                                     const float* __restrict__ alpha_ptr, float* __restrict__ out) {
  const float alpha = alpha_ptr ? __ldg(alpha_ptr) : 1.f;   // undoes the gradient scale of fp16 wgrad operands
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    float4 a = reinterpret_cast<const float4*>(part)[i];
    for (int z = 1; z < splits; ++z) {
      const float4 v = reinterpret_cast<const float4*>(part)[i + z * stride4];
      a.x += v.x; a.y += v.y; a.z += v.z; a.w += v.w;
    }
    a.x *= alpha; a.y *= alpha; a.z *= alpha; a.w *= alpha;
    reinterpret_cast<float4*>(out)[i] = a;
  }
}

__global__ void round_tf32_kernel(const float* __restrict__ in, float* __restrict__ out, long long n4) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    float4 v = reinterpret_cast<const float4*>(in)[i];
    v.x = round_tf32(v.x); v.y = round_tf32(v.y); v.z = round_tf32(v.z); v.w = round_tf32(v.w);
    reinterpret_cast<float4*>(out)[i] = v;
  }
}

// lo = x - trunc_tf32(x): the part of an fp32 operand the tensor core drops (a tf32 MMA truncates to 10 mantissa
// bits); exact in fp32.  The 3xTF32 product adds A_lo.B + A.B_lo to A.B.
__global__ void split_tf32_lo_kernel(const float* __restrict__ in, float* __restrict__ lo, long long n4) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const float4 v = reinterpret_cast<const float4*>(in)[i];
    float4 o;
    o.x = v.x - __uint_as_float(__float_as_uint(v.x) & 0xFFFFE000u);
    o.y = v.y - __uint_as_float(__float_as_uint(v.y) & 0xFFFFE000u);
    o.z = v.z - __uint_as_float(__float_as_uint(v.z) & 0xFFFFE000u);
    o.w = v.w - __uint_as_float(__float_as_uint(v.w) & 0xFFFFE000u);
    reinterpret_cast<float4*>(lo)[i] = o;
  }
}

// out16 = fp16(in * scale), saturating (scale: device scalar or null)
__global__ void to_half_kernel(const float* __restrict__ in, __half* __restrict__ out, long long n4,
                               const float* __restrict__ scale_ptr) {
  const float sc = scale_ptr ? __ldg(scale_ptr) : 1.f;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const float4 v = reinterpret_cast<const float4*>(in)[i];
    uint2 pk;
    pk.x = pack_half2_sat(v.x * sc, v.y * sc); pk.y = pack_half2_sat(v.z * sc, v.w * sc);
    reinterpret_cast<uint2*>(out)[i] = pk;
  }
}

// Gradient scale of one backward segment: S = 2^(target_log2 - ceil(log2(max|g|))), the power of two that puts the
// largest entry of the incoming gradient at ~2^target_log2, so that everything derived from it sits in fp16's
// normal range (65504 = 2^16 at the top, 2^-14 at the bottom).  Stage 1: per-block |max| (bit pattern of a
// non-negative float orders like an unsigned int); stage 2: one block -> scale2 = {S, 1/S}.
__global__ void __launch_bounds__(256)
absmax_part_kernel(const float* __restrict__ g, long long n4, unsigned* __restrict__ part) {
  unsigned m = 0;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const float4 v = reinterpret_cast<const float4*>(g)[i];
    m = max(max(m, __float_as_uint(fabsf(v.x))), max(__float_as_uint(fabsf(v.y)), max(__float_as_uint(fabsf(v.z)), __float_as_uint(fabsf(v.w)))));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
  __shared__ unsigned red[8];
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < 8; ++w) m = max(m, red[w]);
    part[blockIdx.x] = m;
  }
}
__global__ void grad_scale_kernel(const unsigned* __restrict__ part, int nparts, int target_log2, float* __restrict__ scale2) {
  unsigned m = 0;
  for (int i = threadIdx.x; i < nparts; i += 32) m = max(m, part[i]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
  if (threadIdx.x == 0) {
    const float amax = __uint_as_float(m);
    float S = 1.f;
    if (amax > 0.f && amax < INFINITY) {          // zero / inf / nan gradients: leave unscaled
      int e;
      const float f = frexpf(amax, &e);          // amax = f * 2^e, f in [0.5, 1)  ->  amax <= 2^e
      if (f == 0.5f) --e;                        // amax = 2^(e-1) exactly: ceil(log2(amax)) = e - 1
      int sh = target_log2 - e;
      sh = sh > 100 ? 100 : (sh < -100 ? -100 : sh);
      S = ldexpf(1.f, sh);
    }
    scale2[0] = S;
    scale2[1] = 1.f / S;
  }
}

// out[m,:] = x[m,:] + table[m % R,:]  (decoder positional add, layers.py:210)
__global__ void add_rows_mod_kernel(const float* __restrict__ x, const float* __restrict__ table, float* __restrict__ out,
                                    long long M, int D4, int R) {
  const long long total = M * D4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long m = i / D4;
    const int c = (int)(i - m * D4);
    float4 v = reinterpret_cast<const float4*>(x)[i];
    const float4 t = __ldg(reinterpret_cast<const float4*>(table) + (m % R) * D4 + c);
    v.x += t.x; v.y += t.y; v.z += t.z; v.w += t.w;
    reinterpret_cast<float4*>(out)[i] = v;
  }
}

// img [B,C,H,W] -> patches [B*gh*gw, C*ph*pw] with the patch vector ordered (c, row, col): the
// im2col of Conv2d(kernel=stride=(ph,pw)) followed by 'b c h w -> b (h w) c' (layers.py:157-171).
// pw % 4 == 0 so that one float4 stays inside a patch row.
__global__ void patchify_kernel(const float* __restrict__ img, float* __restrict__ out, int B, int C, int H, int W, int ph_, int pw_,
                                int round_out) {
  const int gh = H / ph_, gw = W / pw_;
  const int pd = C * ph_ * pw_;
  const long long total4 = (long long)B * gh * gw * pd / 4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total4; i += (long long)gridDim.x * blockDim.x) {
    // iterate in *image* order so that global reads are fully coalesced; writes are 16-byte pieces
    const long long e = i * 4;
    const int w = (int)(e % W);
    long long r = e / W;
    const int h = (int)(r % H); r /= H;
    const int c = (int)(r % C);
    const int b = (int)(r / C);
    float4 v = reinterpret_cast<const float4*>(img)[i];
    if (round_out) { v.x = round_tf32(v.x); v.y = round_tf32(v.y); v.z = round_tf32(v.z); v.w = round_tf32(v.w); }
    const int hp = h / ph_, ph = h % ph_, wp = w / pw_, pw = w % pw_;
    const long long row = ((long long)b * gh + hp) * gw + wp;
    *reinterpret_cast<float4*>(out + row * pd + (c * ph_ + ph) * pw_ + pw) = v;
  }
}

// tokens [B*gh*gw, C*p*p] (+ bias[c]) -> img [B,C,H,W]: the pixel-shuffle store of
// ConvTranspose2d(kernel=stride=p) after 'b (h w) c -> b c h w' (layers.py:202-205).
// With bias == nullptr and the roles swapped it is also the backward of patchify.
__global__ void unpatchify_kernel(const float* __restrict__ tok, const float* __restrict__ bias, float* __restrict__ img,
                                  int B, int C, int H, int W, int ph_, int pw_) {
  const int gh = H / ph_, gw = W / pw_;
  const int pd = C * ph_ * pw_;
  const long long total4 = (long long)B * C * H * W / 4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total4; i += (long long)gridDim.x * blockDim.x) {
    const long long e = i * 4;
    const int w = (int)(e % W);
    long long r = e / W;
    const int h = (int)(r % H); r /= H;
    const int c = (int)(r % C);
    const int b = (int)(r / C);
    const int hp = h / ph_, ph = h % ph_, wp = w / pw_, pw = w % pw_;
    const long long row = ((long long)b * gh + hp) * gw + wp;
    float4 v = *reinterpret_cast<const float4*>(tok + row * pd + (c * ph_ + ph) * pw_ + pw);
    if (bias) { const float bb = __ldg(bias + c); v.x += bb; v.y += bb; v.z += bb; v.w += bb; }
    reinterpret_cast<float4*>(img)[i] = v;
  }
}

// ---------------------------------------------------------------------------------------------
static inline int stream_grid(long long work_items, int threads) {
  long long blocks = (work_items + threads - 1) / threads;
  const long long cap = (long long)num_sms() * 8;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return (int)blocks;
}

}  // namespace b200

using namespace b200;

template <int NV>
static void ln_fwd_launch(const float* x, const float* g, const float* b, float* y, __half* y16, float* mean, float* rstd, int M,
                          int D, int round_out, cudaStream_t s) {
  const int blocks = stream_grid((long long)M * 32, 256);
  ln_fwd_kernel<NV><<<blocks, 256, 0, s>>>(x, g, b, y, y16, mean, rstd, M, D, round_out);
}

extern "C" int b200vq_layernorm_fwd(const float* x, const float* gamma, const float* beta, float* y, void* y16v, float* mean,
                                    float* rstd, int M, int D, int round_out, void* streamv) {
  const cudaStream_t stream = static_cast<cudaStream_t>(streamv);
  B200_CHECK_ARG(M > 0 && D > 0 && D % 4 == 0 && D <= 2048, "layernorm: need D %% 4 == 0 and D <= 2048 (D=%d)", D);
  B200_CHECK_ARG(y || y16v, "layernorm: no output buffer");
  __half* y16 = static_cast<__half*>(y16v);
  const int nv = (D + 127) / 128;
  if (nv <= 1) ln_fwd_launch<1>(x, gamma, beta, y, y16, mean, rstd, M, D, round_out, stream);
  else if (nv <= 2) ln_fwd_launch<2>(x, gamma, beta, y, y16, mean, rstd, M, D, round_out, stream);
  else if (nv <= 4) ln_fwd_launch<4>(x, gamma, beta, y, y16, mean, rstd, M, D, round_out, stream);
  else if (nv <= 6) ln_fwd_launch<6>(x, gamma, beta, y, y16, mean, rstd, M, D, round_out, stream);
  else if (nv <= 10) ln_fwd_launch<10>(x, gamma, beta, y, y16, mean, rstd, M, D, round_out, stream);
  else ln_fwd_launch<16>(x, gamma, beta, y, y16, mean, rstd, M, D, round_out, stream);
  B200_LAUNCH_OK("ln_fwd_kernel");
  return 0;
}

static int layernorm_bwd_blocks() { return num_sms() * 2; }
extern "C" size_t b200vq_layernorm_bwd_workspace_bytes(int D) { return (size_t)layernorm_bwd_blocks() * 3 * D * sizeof(float); }

template <int NV, int NACC>
static int ln_bwd_launch(const void* dy, int dy_half, const float* dy_scale, const float* x, const float* mean, const float* rstd, const float* gamma,
                         const float* dres, float* dx, __half* dx16, const float* scale_ptr, float* part, int M, int D, int round_out,
                         int blocks, cudaStream_t s) {
  const size_t smem = (size_t)8 * NACC * D * sizeof(float) + (dy_half ? (size_t)8 * D * 2 : 0);   // + the fp16 dy staging slabs
  auto kern = dy_half ? ln_bwd_kernel<NV, NACC, 1> : ln_bwd_kernel<NV, NACC, 0>;
  if (smem > 48 * 1024) B200_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  kern<<<blocks, 256, smem, s>>>(dy, dy_scale, x, mean, rstd, gamma, dres, dx, dx16, scale_ptr, part, M, D, round_out);
  return 0;
}

template <int NACC>
static int ln_bwd_dispatch(const void* dy, int dy_half, const float* dy_scale, const float* x, const float* mean, const float* rstd, const float* gamma,
                           const float* dres, float* dx, __half* dx16, const float* scale_ptr, float* part, int M, int D,
                           int round_out, int blocks, cudaStream_t s) {
  const int nv = (D + 127) / 128;
  if (nv <= 1) return ln_bwd_launch<1, NACC>(dy, dy_half, dy_scale, x, mean, rstd, gamma, dres, dx, dx16, scale_ptr, part, M, D, round_out, blocks, s);
  if (nv <= 2) return ln_bwd_launch<2, NACC>(dy, dy_half, dy_scale, x, mean, rstd, gamma, dres, dx, dx16, scale_ptr, part, M, D, round_out, blocks, s);
  if (nv <= 4) return ln_bwd_launch<4, NACC>(dy, dy_half, dy_scale, x, mean, rstd, gamma, dres, dx, dx16, scale_ptr, part, M, D, round_out, blocks, s);
  if (nv <= 6) return ln_bwd_launch<6, NACC>(dy, dy_half, dy_scale, x, mean, rstd, gamma, dres, dx, dx16, scale_ptr, part, M, D, round_out, blocks, s);
  if (nv <= 10) return ln_bwd_launch<10, NACC>(dy, dy_half, dy_scale, x, mean, rstd, gamma, dres, dx, dx16, scale_ptr, part, M, D, round_out, blocks, s);
  return ln_bwd_launch<16, NACC>(dy, dy_half, dy_scale, x, mean, rstd, gamma, dres, dx, dx16, scale_ptr, part, M, D, round_out, blocks, s);
}

extern "C" int b200vq_layernorm_bwd(const void* dy, int dy_half, const float* dy_scale, const float* x, const float* mean,
                                    const float* rstd, const float* gamma, const float* dres, float* dx, void* dx16v,
                                    const float* scale_ptr, float* dgamma, float* dbeta, float* dxsum, int M, int D, int round_out,
                                    void* workspace, size_t ws_bytes, void* streamv) {
  const cudaStream_t stream = static_cast<cudaStream_t>(streamv);
  __half* dx16 = static_cast<__half*>(dx16v);
  B200_CHECK_ARG(M > 0 && D > 0 && D % 4 == 0 && D <= 2048, "layernorm: need D %% 4 == 0 and D <= 2048 (D=%d)", D);
  B200_CHECK_ARG(ws_bytes >= b200vq_layernorm_bwd_workspace_bytes(D), "layernorm_backward: workspace too small");
  int blocks = layernorm_bwd_blocks();
  if (blocks > (M + 7) / 8) blocks = (M + 7) / 8;
  float* part = static_cast<float*>(workspace);
  const int nacc = dxsum ? 3 : 2;
  int rc = dxsum ? ln_bwd_dispatch<3>(dy, dy_half, dy_scale, x, mean, rstd, gamma, dres, dx, dx16, scale_ptr, part, M, D, round_out, blocks, stream)
                 : ln_bwd_dispatch<2>(dy, dy_half, dy_scale, x, mean, rstd, gamma, dres, dx, dx16, scale_ptr, part, M, D, round_out, blocks, stream);
  if (rc) return rc;
  B200_LAUNCH_OK("ln_bwd_kernel");
  ln_param_reduce_kernel<<<(nacc * D + 31) / 32, 256, 0, stream>>>(part, blocks, D, nacc, dgamma, dbeta, dxsum);
  B200_LAUNCH_OK("ln_param_reduce_kernel");
  return 0;
}

constexpr int kColsumMaxSplits = 64;
extern "C" size_t b200vq_colsum_workspace_bytes(int N) { return (size_t)kColsumMaxSplits * N * sizeof(float); }

extern "C" int b200vq_colsum(const float* X, long long ld, int M, int N, float* out, void* workspace, size_t ws_bytes,
                             void* streamv) {
  const cudaStream_t stream = static_cast<cudaStream_t>(streamv);
  B200_CHECK_ARG(M > 0 && N > 0 && N % 4 == 0 && ld % 4 == 0, "colsum: N and ld must be multiples of 4");
  B200_CHECK_ARG(ws_bytes >= b200vq_colsum_workspace_bytes(N), "colsum: workspace too small");
  const int colblocks = (N / 4 + 31) / 32;
  int splits = (num_sms() * 8 + colblocks - 1) / colblocks;
  if (splits > kColsumMaxSplits) splits = kColsumMaxSplits;
  if (splits > (M + 7) / 8) splits = (M + 7) / 8;
  if (splits < 1) splits = 1;
  float* part = static_cast<float*>(workspace);
  colsum_kernel<<<dim3(colblocks, splits), 256, 0, stream>>>(X, ld, M, N, part);
  B200_LAUNCH_OK("colsum_kernel");
  colpart_reduce_kernel<<<(N + 255) / 256, 256, 0, stream>>>(part, splits, N, out);
  B200_LAUNCH_OK("colpart_reduce_kernel");
  return 0;
}

extern "C" int b200vq_splitk_reduce(const float* part, int splits, long long n, long long split_stride, const float* alpha_ptr,
                                    float* out, void* streamv) {
  const cudaStream_t stream = static_cast<cudaStream_t>(streamv);
  B200_CHECK_ARG(n % 4 == 0 && split_stride % 4 == 0, "splitk_reduce: sizes must be multiples of 4");
  splitk_reduce_kernel<<<stream_grid(n / 4, 256), 256, 0, stream>>>(part, splits, n / 4, split_stride / 4, alpha_ptr, out);
  B200_LAUNCH_OK("splitk_reduce_kernel");
  return 0;
}

extern "C" int b200vq_round_tf32(const float* in, float* out, long long n, void* streamv) {
  const cudaStream_t stream = static_cast<cudaStream_t>(streamv);
  B200_CHECK_ARG(n % 4 == 0, "round_tf32: n %% 4");
  round_tf32_kernel<<<stream_grid(n / 4, 256), 256, 0, stream>>>(in, out, n / 4);
  B200_LAUNCH_OK("round_tf32_kernel");
  return 0;
}

extern "C" int b200vq_split_tf32_lo(const float* in, float* lo, long long n, void* streamv) {
  const cudaStream_t stream = static_cast<cudaStream_t>(streamv);
  B200_CHECK_ARG(n % 4 == 0, "split_tf32_lo: n %% 4");
  split_tf32_lo_kernel<<<stream_grid(n / 4, 256), 256, 0, stream>>>(in, lo, n / 4);
  B200_LAUNCH_OK("split_tf32_lo_kernel");
  return 0;
}

extern "C" int b200vq_to_half(const float* in, void* out, long long n, const float* scale_ptr, void* streamv) {
  const cudaStream_t stream = static_cast<cudaStream_t>(streamv);
  B200_CHECK_ARG(n % 4 == 0, "to_half: n %% 4");
  to_half_kernel<<<stream_grid(n / 4, 256), 256, 0, stream>>>(in, static_cast<__half*>(out), n / 4, scale_ptr);
  B200_LAUNCH_OK("to_half_kernel");
  return 0;
}

constexpr int kAbsmaxBlocks = 1056;   // 132 SMs x 8
extern "C" size_t b200vq_grad_scale_workspace_bytes(void) { return kAbsmaxBlocks * sizeof(unsigned); }
extern "C" int b200vq_grad_scale(const float* g, long long n, int target_log2, float* scale2, void* workspace, size_t ws_bytes,
                                 void* streamv) {
  const cudaStream_t stream = static_cast<cudaStream_t>(streamv);
  B200_CHECK_ARG(n > 0 && n % 4 == 0, "grad_scale: n %% 4");
  B200_CHECK_ARG(ws_bytes >= b200vq_grad_scale_workspace_bytes(), "grad_scale: workspace too small");
  B200_CHECK_ARG(target_log2 >= -14 && target_log2 <= 15, "grad_scale: target exponent outside the fp16 range");
  int blocks = stream_grid(n / 4, 256);
  if (blocks > kAbsmaxBlocks) blocks = kAbsmaxBlocks;
  unsigned* part = static_cast<unsigned*>(workspace);
  absmax_part_kernel<<<blocks, 256, 0, stream>>>(g, n / 4, part);
  B200_LAUNCH_OK("absmax_part_kernel");
  grad_scale_kernel<<<1, 32, 0, stream>>>(part, blocks, target_log2, scale2);
  B200_LAUNCH_OK("grad_scale_kernel");
  return 0;
}

extern "C" int b200vq_add_rows_mod(const float* x, const float* table, float* out, long long M, int D, int R, void* streamv) {
  const cudaStream_t stream = static_cast<cudaStream_t>(streamv);
  B200_CHECK_ARG(D % 4 == 0 && R > 0 && M > 0, "add_rows_mod: D %% 4 and R > 0 required");
  add_rows_mod_kernel<<<stream_grid(M * (D / 4), 256), 256, 0, stream>>>(x, table, out, M, D / 4, R);
  B200_LAUNCH_OK("add_rows_mod_kernel");
  return 0;
}

extern "C" int b200vq_patchify(const float* img, float* out, int B, int C, int H, int W, int ph, int pw, int round_out,
                               void* streamv) {
  const cudaStream_t stream = static_cast<cudaStream_t>(streamv);
  B200_CHECK_ARG(ph > 0 && pw > 0 && pw % 4 == 0 && H % ph == 0 && W % pw == 0,
                 "patchify: the patch must divide the image and its width must be a multiple of 4 (got %d x %d)", ph, pw);
  patchify_kernel<<<stream_grid((long long)B * C * H * W / 4, 256), 256, 0, stream>>>(img, out, B, C, H, W, ph, pw, round_out);
  B200_LAUNCH_OK("patchify_kernel");
  return 0;
}

extern "C" int b200vq_unpatchify(const float* tok, const float* bias, float* img, int B, int C, int H, int W, int ph, int pw,
                                 void* streamv) {
  const cudaStream_t stream = static_cast<cudaStream_t>(streamv);
  B200_CHECK_ARG(ph > 0 && pw > 0 && pw % 4 == 0 && H % ph == 0 && W % pw == 0,
                 "unpatchify: the patch must divide the image and its width must be a multiple of 4 (got %d x %d)", ph, pw);
  unpatchify_kernel<<<stream_grid((long long)B * C * H * W / 4, 256), 256, 0, stream>>>(tok, bias, img, B, C, H, W, ph, pw);
  B200_LAUNCH_OK("unpatchify_kernel");
  return 0;
}
