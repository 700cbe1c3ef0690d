// fp16 attention core on wgmma (the default data path; reference enhancing/modules/stage1/layers.py:124-130 and its
// autograd), head size 64.  The scores live in registers only; backward recomputes them from the saved log-sum-exp.
//
// q / k / v are read in place from the packed [B*N, 3*inner] fp16 qkv through one 3-D tensor map {3*inner, N, B}: a
// 64-row box of one head is 64 x 128 B, exactly one SWIZZLE_128B atom wide, and a box that runs past N is zero-filled
// inside its own image.  dO [B*N, inner] has its own map.  Every CTA is two consumer warpgroups of 64 rows each plus one
// producer warp that issues the TMA loads: the CTA's resident tiles once, then 64-row tiles of the streamed operand
// through a ring of mbarrier full / empty pairs (as in gemm_tc.cu).
//
// Every product reads its operands where they are: a K-major operand (rows x 64 contiguous head elements) through the
// swizzled descriptor with 32-byte k steps, an MN-major one (contraction rows x 64 contiguous elements) with 2048-byte
// k steps.  The probabilities and dS re-enter the tensor core from registers: the fp32 accumulator layout of one
// m64n64 wgmma, packed to fp16 pairs, is the register A fragment of the next.
//
//   forward      128 queries per CTA; K / V tiles: S = Q K^T, online softmax in fp32, O += P V
//   key side     128 keys per CTA, K and V resident; Q / dO tiles with their LSE and delta:
//                S^T = K Q^T, dP^T = V dO^T, dV += P^T dO, dK += dS^T Q
//   query side   128 queries per CTA, Q and dO resident; K / V tiles: S = Q K^T, dP = dO V^T, dQ += dS K
// Backward is two kernels so that no atomics are needed: a run is bit-reproducible.
#include "../../include/b200vq.h"
#include "attention.cuh"
#include "common.cuh"

namespace b200 {

namespace {

constexpr float kLog2e = 1.4426950408889634f;
constexpr int kDh = 64;
constexpr int kTileBytes = 64 * 128;                 // 64 rows of one head, fp16
constexpr int kConsumers = 8;                        // warps in the two consumer warpgroups
constexpr int kThreads = 32 * (kConsumers + 1);      // + the producer warp
constexpr int kFwdStages = 4, kDqStages = 4, kDkvStages = 4;

// shared-memory descriptors of a 64-row, 128-byte-pitch swizzled tile for k step ks (16 elements of the contraction)
__device__ __forceinline__ uint64_t desc_k(uint32_t tile, int ks) { return wgmma_desc_sw128(tile + ks * 32, kTileBytes, 1024); }
__device__ __forceinline__ uint64_t desc_mn(uint32_t tile, int ks) { return wgmma_desc_sw128(tile + ks * 2048, kTileBytes, 1024); }

__device__ __forceinline__ void zero(float (&d)[32]) {
#pragma unroll
  for (int i = 0; i < 32; ++i) d[i] = 0.f;
}
// keeps the A fragments of an MMA still in flight alive (and unmodified) until the wait that retires it
__device__ __forceinline__ void keep(uint32_t (&a)[4][4]) {
#pragma unroll
  for (int i = 0; i < 4; ++i) asm volatile("" : "+r"(a[i][0]), "+r"(a[i][1]), "+r"(a[i][2]), "+r"(a[i][3])::"memory");
}
// every warp of the consumer warpgroups releases a ring stage once
__device__ __forceinline__ void release(uint64_t* bar, int lane) {
  __syncwarp();
  if (lane == 0) mbar_arrive(bar);
}

struct Ring {
  int stage = 0;
  uint32_t phase = 0;
  __device__ __forceinline__ void next(int stages) {
    if (++stage == stages) { stage = 0; phase ^= 1; }
  }
};

}  // namespace

// ---------------------------------------------------------------------------------------------
// forward: grid (ceil(N/128), heads, B)
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads, 2)
attn_f16_fwd_kernel(const __grid_constant__ CUtensorMap tm_qkv, __half* __restrict__ out, float* __restrict__ lse, int N,
                    int heads, float scale) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_align1024(smem_raw);
  uint8_t* Qs = smem;                                  // [2][64 rows]
  uint8_t* Ks = Qs + 2 * kTileBytes;                   // [stages][64 keys]
  uint8_t* Vs = Ks + kFwdStages * kTileBytes;
  uint64_t* full = reinterpret_cast<uint64_t*>(Vs + kFwdStages * kTileBytes);
  uint64_t* empty = full + kFwdStages;
  uint64_t* qbar = empty + kFwdStages;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int h = blockIdx.y, b = blockIdx.z;
  const int inner = heads * kDh;
  const int ntiles = (N + 63) / 64;
  if (threadIdx.x == 0) {
    for (int s = 0; s < kFwdStages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], kConsumers); }
    mbar_init(qbar, 1);
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == kConsumers) {
    if (lane == 0) {
      tma_prefetch_desc(&tm_qkv);
      mbar_arrive_expect_tx(qbar, 2 * kTileBytes);
      tma_load_3d(Qs, &tm_qkv, qbar, h * kDh, blockIdx.x * 128, b);
      tma_load_3d(Qs + kTileBytes, &tm_qkv, qbar, h * kDh, blockIdx.x * 128 + 64, b);
      Ring r;
      for (int j = 0; j < ntiles; ++j, r.next(kFwdStages)) {
        mbar_wait(&empty[r.stage], r.phase ^ 1);
        mbar_arrive_expect_tx(&full[r.stage], 2 * kTileBytes);
        tma_load_3d(Ks + r.stage * kTileBytes, &tm_qkv, &full[r.stage], inner + h * kDh, j * 64, b);
        tma_load_3d(Vs + r.stage * kTileBytes, &tm_qkv, &full[r.stage], 2 * inner + h * kDh, j * 64, b);
      }
    }
    return;
  }

  const int wg = warp >> 2, g = lane >> 2, t = lane & 3;
  const float c = scale * kLog2e;
  const uint32_t q_u = smem_u32(Qs + wg * kTileBytes), k_u = smem_u32(Ks), v_u = smem_u32(Vs);
  float o[32], s[32];
  zero(o);
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
  mbar_wait(qbar, 0);
  Ring r;
  for (int j = 0; j < ntiles; ++j, r.next(kFwdStages)) {
    mbar_wait(&full[r.stage], r.phase);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < 4; ++ks)                                    // S = Q K^T
      wgmma_m64n64k16_ss<0>(s, desc_k(q_u, ks), desc_k(k_u + r.stage * kTileBytes, ks), ks);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(s);
    if ((j + 1) * 64 > N) {
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        const int key = j * 64 + nt * 8 + 2 * t;
        if (key >= N) { s[4 * nt] = -INFINITY; s[4 * nt + 2] = -INFINITY; }
        if (key + 1 >= N) { s[4 * nt + 1] = -INFINITY; s[4 * nt + 3] = -INFINITY; }
      }
    }
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      mx0 = fmaxf(mx0, fmaxf(s[4 * nt], s[4 * nt + 1]));
      mx1 = fmaxf(mx1, fmaxf(s[4 * nt + 2], s[4 * nt + 3]));
    }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    const float mn0 = fmaxf(m0, mx0), mn1 = fmaxf(m1, mx1);
    const float al0 = exp2f((m0 - mn0) * c), al1 = exp2f((m1 - mn1) * c);   // exp2(-inf) = 0 on the first tile
    m0 = mn0; m1 = mn1;
    l0 *= al0; l1 *= al1;
#pragma unroll
    for (int i = 0; i < 8; ++i) { o[4 * i] *= al0; o[4 * i + 1] *= al0; o[4 * i + 2] *= al1; o[4 * i + 3] *= al1; }
    uint32_t pf[4][4];
    const float mc0 = m0 * c, mc1 = m1 * c;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      const float p0 = exp2f(s[4 * nt] * c - mc0), p1 = exp2f(s[4 * nt + 1] * c - mc0);
      const float p2 = exp2f(s[4 * nt + 2] * c - mc1), p3 = exp2f(s[4 * nt + 3] * c - mc1);
      l0 += p0 + p1; l1 += p2 + p3;
      pf[nt >> 1][(nt & 1) * 2] = pack_half2_sat(p0, p1);
      pf[nt >> 1][(nt & 1) * 2 + 1] = pack_half2_sat(p2, p3);
    }
    wgmma_fence();
#pragma unroll
    for (int kc = 0; kc < 4; ++kc)                                    // O += P V
      wgmma_m64n64k16_rs<1>(o, pf[kc], desc_mn(v_u + r.stage * kTileBytes, kc));
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(o);
    release(&empty[r.stage], lane);
  }
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const float inv0 = 1.f / l0, inv1 = 1.f / l1;
  const int r0 = blockIdx.x * 128 + warp * 16 + g, r1 = r0 + 8;
  __half* ob = out + (long long)b * N * inner + h * kDh + 2 * t;
#pragma unroll
  for (int dt = 0; dt < 8; ++dt) {
    if (r0 < N) *reinterpret_cast<uint32_t*>(ob + (long long)r0 * inner + dt * 8) = pack_half2_sat(o[4 * dt] * inv0, o[4 * dt + 1] * inv0);
    if (r1 < N) *reinterpret_cast<uint32_t*>(ob + (long long)r1 * inner + dt * 8) = pack_half2_sat(o[4 * dt + 2] * inv1, o[4 * dt + 3] * inv1);
  }
  if (t == 0) {
    float* lb = lse + ((long long)b * heads + h) * N;
    if (r0 < N) lb[r0] = m0 * scale + logf(l0);
    if (r1 < N) lb[r1] = m1 * scale + logf(l1);
  }
}

// ---------------------------------------------------------------------------------------------
// backward, key side: grid (ceil(N/128), heads, B).  Works on transposed score tiles S^T[key, query], so that P^T and
// dS^T come out of the tensor core already in A-operand position for dV += P^T dO and dK += dS^T Q.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads, 1)
attn_f16_bwd_dkv_kernel(const __grid_constant__ CUtensorMap tm_qkv, const __grid_constant__ CUtensorMap tm_do,
                        const float* __restrict__ lse, const float* __restrict__ delta, __half* __restrict__ dqkv, int N,
                        int heads, float scale) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_align1024(smem_raw);
  uint8_t* Ks = smem;                                  // [2][64 keys]
  uint8_t* Vs = Ks + 2 * kTileBytes;                   // [2][64 keys]
  uint8_t* Qs = Vs + 2 * kTileBytes;                   // [stages][64 queries]
  uint8_t* Ds = Qs + kDkvStages * kTileBytes;          // [stages][64 queries] of dO
  float* Ls = reinterpret_cast<float*>(Ds + kDkvStages * kTileBytes);   // [stages][64]: lse * log2(e), +inf past N
  float* Es = Ls + kDkvStages * 64;                                      // [stages][64]: delta, 0 past N
  uint64_t* full = reinterpret_cast<uint64_t*>(Es + kDkvStages * 64);
  uint64_t* empty = full + kDkvStages;
  uint64_t* kvbar = empty + kDkvStages;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int h = blockIdx.y, b = blockIdx.z;
  const int inner = heads * kDh;
  const int ntiles = (N + 63) / 64;
  if (threadIdx.x == 0) {
    // full: the TMA transaction plus one arrival per producer lane once its LSE / delta entries are stored
    for (int s = 0; s < kDkvStages; ++s) { mbar_init(&full[s], 1 + 32); mbar_init(&empty[s], kConsumers); }
    mbar_init(kvbar, 1);
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == kConsumers) {
    const float* lb = lse + ((long long)b * heads + h) * N;
    const float* eb = delta + ((long long)b * heads + h) * N;
    if (lane == 0) {
      tma_prefetch_desc(&tm_qkv);
      tma_prefetch_desc(&tm_do);
      mbar_arrive_expect_tx(kvbar, 4 * kTileBytes);
      for (int i = 0; i < 2; ++i) {
        tma_load_3d(Ks + i * kTileBytes, &tm_qkv, kvbar, inner + h * kDh, blockIdx.x * 128 + i * 64, b);
        tma_load_3d(Vs + i * kTileBytes, &tm_qkv, kvbar, 2 * inner + h * kDh, blockIdx.x * 128 + i * 64, b);
      }
    }
    Ring r;
    for (int j = 0; j < ntiles; ++j, r.next(kDkvStages)) {
      mbar_wait(&empty[r.stage], r.phase ^ 1);
      if (lane == 0) {
        mbar_arrive_expect_tx(&full[r.stage], 2 * kTileBytes);
        tma_load_3d(Qs + r.stage * kTileBytes, &tm_qkv, &full[r.stage], h * kDh, j * 64, b);
        tma_load_3d(Ds + r.stage * kTileBytes, &tm_do, &full[r.stage], h * kDh, j * 64, b);
      }
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int q = j * 64 + i * 32 + lane;
        Ls[r.stage * 64 + i * 32 + lane] = q < N ? lb[q] * kLog2e : INFINITY;   // +inf -> P = 0 for padded queries
        Es[r.stage * 64 + i * 32 + lane] = q < N ? eb[q] : 0.f;
      }
      mbar_arrive(&full[r.stage]);
    }
    return;
  }

  const int wg = warp >> 2, g = lane >> 2, t = lane & 3;
  const float c = scale * kLog2e;
  const uint32_t k_u = smem_u32(Ks + wg * kTileBytes), v_u = smem_u32(Vs + wg * kTileBytes);
  const uint32_t q_u = smem_u32(Qs), d_u = smem_u32(Ds);
  float dk[32], dv[32];
  zero(dk);
  zero(dv);
  mbar_wait(kvbar, 0);
  Ring r;
  for (int j = 0; j < ntiles; ++j, r.next(kDkvStages)) {
    mbar_wait(&full[r.stage], r.phase);
    const uint32_t qt = q_u + r.stage * kTileBytes, dt = d_u + r.stage * kTileBytes;
    float s[32], dp[32];
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) wgmma_m64n64k16_ss<0>(s, desc_k(k_u, ks), desc_k(qt, ks), ks);    // S^T = K Q^T
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) wgmma_m64n64k16_ss<0>(dp, desc_k(v_u, ks), desc_k(dt, ks), ks);   // dP^T = V dO^T
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(s);
    wgmma_fence_regs(dp);
    const float* L = Ls + r.stage * 64;
    const float* E = Es + r.stage * 64;
    uint32_t pf[4][4], sf[4][4];
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      const float2 la = *reinterpret_cast<const float2*>(L + nt * 8 + 2 * t);
      const float2 ea = *reinterpret_cast<const float2*>(E + nt * 8 + 2 * t);
      const float p0 = exp2f(s[4 * nt] * c - la.x), p1 = exp2f(s[4 * nt + 1] * c - la.y);
      const float p2 = exp2f(s[4 * nt + 2] * c - la.x), p3 = exp2f(s[4 * nt + 3] * c - la.y);
      pf[nt >> 1][(nt & 1) * 2] = pack_half2_sat(p0, p1);
      pf[nt >> 1][(nt & 1) * 2 + 1] = pack_half2_sat(p2, p3);
      sf[nt >> 1][(nt & 1) * 2] = pack_half2_sat(p0 * (dp[4 * nt] - ea.x), p1 * (dp[4 * nt + 1] - ea.y));
      sf[nt >> 1][(nt & 1) * 2 + 1] = pack_half2_sat(p2 * (dp[4 * nt + 2] - ea.x), p3 * (dp[4 * nt + 3] - ea.y));
    }
    wgmma_fence();
#pragma unroll
    for (int kc = 0; kc < 4; ++kc) wgmma_m64n64k16_rs<1>(dv, pf[kc], desc_mn(dt, kc));   // dV += P^T dO
#pragma unroll
    for (int kc = 0; kc < 4; ++kc) wgmma_m64n64k16_rs<1>(dk, sf[kc], desc_mn(qt, kc));   // dK += dS^T Q
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(dv);
    wgmma_fence_regs(dk);
    release(&empty[r.stage], lane);
  }
  const int r0 = blockIdx.x * 128 + warp * 16 + g, r1 = r0 + 8;
  const long long ld = 3ll * inner;
  __half* kb = dqkv + (long long)b * N * ld + inner + h * kDh + 2 * t;
  __half* vb = kb + inner;
#pragma unroll
  for (int d = 0; d < 8; ++d) {
    if (r0 < N) {
      *reinterpret_cast<uint32_t*>(kb + r0 * ld + d * 8) = pack_half2_sat(dk[4 * d] * scale, dk[4 * d + 1] * scale);
      *reinterpret_cast<uint32_t*>(vb + r0 * ld + d * 8) = pack_half2_sat(dv[4 * d], dv[4 * d + 1]);
    }
    if (r1 < N) {
      *reinterpret_cast<uint32_t*>(kb + r1 * ld + d * 8) = pack_half2_sat(dk[4 * d + 2] * scale, dk[4 * d + 3] * scale);
      *reinterpret_cast<uint32_t*>(vb + r1 * ld + d * 8) = pack_half2_sat(dv[4 * d + 2], dv[4 * d + 3]);
    }
  }
}

// ---------------------------------------------------------------------------------------------
// backward, query side: grid (ceil(N/128), heads, B)
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads, 1)
attn_f16_bwd_dq_kernel(const __grid_constant__ CUtensorMap tm_qkv, const __grid_constant__ CUtensorMap tm_do,
                       const float* __restrict__ lse, const float* __restrict__ delta, __half* __restrict__ dqkv, int N,
                       int heads, float scale) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_align1024(smem_raw);
  uint8_t* Qs = smem;                                  // [2][64 queries]
  uint8_t* Ds = Qs + 2 * kTileBytes;                   // [2][64 queries] of dO
  uint8_t* Ks = Ds + 2 * kTileBytes;                   // [stages][64 keys]
  uint8_t* Vs = Ks + kDqStages * kTileBytes;
  uint64_t* full = reinterpret_cast<uint64_t*>(Vs + kDqStages * kTileBytes);
  uint64_t* empty = full + kDqStages;
  uint64_t* qbar = empty + kDqStages;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int h = blockIdx.y, b = blockIdx.z;
  const int inner = heads * kDh;
  const int ntiles = (N + 63) / 64;
  if (threadIdx.x == 0) {
    for (int s = 0; s < kDqStages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], kConsumers); }
    mbar_init(qbar, 1);
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == kConsumers) {
    if (lane == 0) {
      tma_prefetch_desc(&tm_qkv);
      tma_prefetch_desc(&tm_do);
      mbar_arrive_expect_tx(qbar, 4 * kTileBytes);
      for (int i = 0; i < 2; ++i) {
        tma_load_3d(Qs + i * kTileBytes, &tm_qkv, qbar, h * kDh, blockIdx.x * 128 + i * 64, b);
        tma_load_3d(Ds + i * kTileBytes, &tm_do, qbar, h * kDh, blockIdx.x * 128 + i * 64, b);
      }
      Ring r;
      for (int j = 0; j < ntiles; ++j, r.next(kDqStages)) {
        mbar_wait(&empty[r.stage], r.phase ^ 1);
        mbar_arrive_expect_tx(&full[r.stage], 2 * kTileBytes);
        tma_load_3d(Ks + r.stage * kTileBytes, &tm_qkv, &full[r.stage], inner + h * kDh, j * 64, b);
        tma_load_3d(Vs + r.stage * kTileBytes, &tm_qkv, &full[r.stage], 2 * inner + h * kDh, j * 64, b);
      }
    }
    return;
  }

  const int wg = warp >> 2, g = lane >> 2, t = lane & 3;
  const float c = scale * kLog2e;
  const int r0 = blockIdx.x * 128 + warp * 16 + g, r1 = r0 + 8;
  const float* lb = lse + ((long long)b * heads + h) * N;
  const float* eb = delta + ((long long)b * heads + h) * N;
  const float lse0 = r0 < N ? lb[r0] * kLog2e : INFINITY, lse1 = r1 < N ? lb[r1] * kLog2e : INFINITY;
  const float e0 = r0 < N ? eb[r0] : 0.f, e1 = r1 < N ? eb[r1] : 0.f;
  const uint32_t q_u = smem_u32(Qs + wg * kTileBytes), d_u = smem_u32(Ds + wg * kTileBytes);
  const uint32_t k_u = smem_u32(Ks), v_u = smem_u32(Vs);
  float dq[32];
  zero(dq);
  mbar_wait(qbar, 0);
  Ring r;
  for (int j = 0; j < ntiles; ++j, r.next(kDqStages)) {
    mbar_wait(&full[r.stage], r.phase);
    const uint32_t kt = k_u + r.stage * kTileBytes, vt = v_u + r.stage * kTileBytes;
    float s[32], dp[32];
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) wgmma_m64n64k16_ss<0>(s, desc_k(q_u, ks), desc_k(kt, ks), ks);    // S = Q K^T
    wgmma_commit();
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) wgmma_m64n64k16_ss<0>(dp, desc_k(d_u, ks), desc_k(vt, ks), ks);   // dP = dO V^T
    wgmma_commit();
    wgmma_wait<1>();                                  // the exponentials of P run while dP is computed
    wgmma_fence_regs(s);
    const bool tail = (j + 1) * 64 > N;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      const int key = j * 64 + nt * 8 + 2 * t;
      const bool ka = !tail || key < N, kb = !tail || key + 1 < N;
      s[4 * nt] = ka ? exp2f(s[4 * nt] * c - lse0) : 0.f; s[4 * nt + 1] = kb ? exp2f(s[4 * nt + 1] * c - lse0) : 0.f;
      s[4 * nt + 2] = ka ? exp2f(s[4 * nt + 2] * c - lse1) : 0.f; s[4 * nt + 3] = kb ? exp2f(s[4 * nt + 3] * c - lse1) : 0.f;
    }
    wgmma_wait<0>();
    wgmma_fence_regs(dp);
    uint32_t sf[4][4];
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      sf[nt >> 1][(nt & 1) * 2] = pack_half2_sat(s[4 * nt] * (dp[4 * nt] - e0), s[4 * nt + 1] * (dp[4 * nt + 1] - e0));
      sf[nt >> 1][(nt & 1) * 2 + 1] = pack_half2_sat(s[4 * nt + 2] * (dp[4 * nt + 2] - e1), s[4 * nt + 3] * (dp[4 * nt + 3] - e1));
    }
    wgmma_fence();
#pragma unroll
    for (int kc = 0; kc < 4; ++kc) wgmma_m64n64k16_rs<1>(dq, sf[kc], desc_mn(kt, kc));   // dQ += dS K
    wgmma_commit();
    wgmma_wait<0>();
    keep(sf);
    wgmma_fence_regs(dq);
    release(&empty[r.stage], lane);
  }
  const long long ld = 3ll * inner;
  __half* qb = dqkv + (long long)b * N * ld + h * kDh + 2 * t;
#pragma unroll
  for (int d = 0; d < 8; ++d) {
    if (r0 < N) *reinterpret_cast<uint32_t*>(qb + r0 * ld + d * 8) = pack_half2_sat(dq[4 * d] * scale, dq[4 * d + 1] * scale);
    if (r1 < N) *reinterpret_cast<uint32_t*>(qb + r1 * ld + d * 8) = pack_half2_sat(dq[4 * d + 2] * scale, dq[4 * d + 3] * scale);
  }
}

}  // namespace b200

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
using namespace b200;

// one image's rows of a packed fp16 [B*N, cols] matrix as {cols, N, B}; 64 x 64 boxes (one head, 64 rows)
static int rows_map(CUtensorMap* m, const void* p, int B, int N, long long cols) {
  const unsigned long long dims[3] = {(unsigned long long)cols, (unsigned long long)N, (unsigned long long)B};
  const unsigned long long strides[2] = {(unsigned long long)cols * 2, (unsigned long long)N * cols * 2};
  const unsigned box[3] = {64, 64, 1};
  return make_tensor_map(m, p, 2, 3, dims, strides, box, 0);
}
constexpr size_t kSmemSlack = 1024 + 256;             // 1024-byte alignment of the base, mbarriers
constexpr size_t kFwdSmem = (2 + 2 * kFwdStages) * kTileBytes + kSmemSlack;
constexpr size_t kDqSmem = (4 + 2 * kDqStages) * kTileBytes + kSmemSlack;
constexpr size_t kDkvSmem = (4 + 2 * kDkvStages) * kTileBytes + kDkvStages * 2 * 64 * sizeof(float) + kSmemSlack;

static int check_problem(const void* qkv, const void* out, int B, int N, int heads, int dh) {
  B200_CHECK_ARG(dh == 64, "attention_f16: dim_head must be 64 (got %d); other head sizes use the tf32 core", dh);
  B200_CHECK_ARG(B > 0 && N > 0 && heads > 0, "attention: empty problem");
  B200_CHECK_ARG(B <= 65535 && heads <= 65535, "attention: grid too large");
  B200_CHECK_ARG((reinterpret_cast<uintptr_t>(qkv) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0,
                 "attention: qkv and out must be 16-byte aligned");
  return 0;
}

// q/k/v fp16 as the to_qkv GEMM stores them, O fp16, LSE fp32 [B, heads, N]
extern "C" int b200vq_attention_f16_fwd(const void* qkv, void* out, float* lse, int B, int N, int heads, int dh, float scale,
                                        void* streamv) {
  const cudaStream_t stream = static_cast<cudaStream_t>(streamv);
  if (int rc = check_problem(qkv, out, B, N, heads, dh)) return rc;
  CUtensorMap tm;
  if (int rc = rows_map(&tm, qkv, B, N, 3ll * heads * kDh)) return rc;
  B200_CONFIGURE_SMEM_ONCE(attn_f16_fwd_kernel, kFwdSmem);
  attn_f16_fwd_kernel<<<dim3((N + 127) / 128, heads, B), kThreads, kFwdSmem, stream>>>(tm, static_cast<__half*>(out), lse, N,
                                                                                      heads, scale);
  B200_LAUNCH_OK("attn_f16_fwd_kernel");
  return 0;
}

// dO fp16 carrying the power-of-two gradient scale S of the backward segment (functional.py); delta, dS and the stored
// fp16 dq / dk / dv carry S too -- everything is linear in dO, nothing is rescaled here.
extern "C" int b200vq_attention_f16_bwd(const void* qkv, const void* out, const float* lse, const void* dout, void* dqkv, float* delta,
                                        int B, int N, int heads, int dh, float scale, void* streamv) {
  const cudaStream_t stream = static_cast<cudaStream_t>(streamv);
  if (int rc = check_problem(qkv, out, B, N, heads, dh)) return rc;
  B200_CHECK_ARG((reinterpret_cast<uintptr_t>(dout) & 15) == 0 && (reinterpret_cast<uintptr_t>(dqkv) & 15) == 0,
                 "attention: dout and dqkv must be 16-byte aligned");
  if (int rc = attention_delta(out, 1, dout, 1, delta, B, N, heads, dh, stream)) return rc;
  CUtensorMap tq, td;
  if (int rc = rows_map(&tq, qkv, B, N, 3ll * heads * kDh)) return rc;
  if (int rc = rows_map(&td, dout, B, N, (long long)heads * kDh)) return rc;
  B200_CONFIGURE_SMEM_ONCE(attn_f16_bwd_dkv_kernel, kDkvSmem);
  B200_CONFIGURE_SMEM_ONCE(attn_f16_bwd_dq_kernel, kDqSmem);
  const dim3 grid((N + 127) / 128, heads, B);
  __half* d = static_cast<__half*>(dqkv);
  attn_f16_bwd_dkv_kernel<<<grid, kThreads, kDkvSmem, stream>>>(tq, td, lse, delta, d, N, heads, scale);
  B200_LAUNCH_OK("attn_f16_bwd_dkv_kernel");
  attn_f16_bwd_dq_kernel<<<grid, kThreads, kDqSmem, stream>>>(tq, td, lse, delta, d, N, heads, scale);
  B200_LAUNCH_OK("attn_f16_bwd_dq_kernel");
  return 0;
}
