// Flash-style attention core on mma.sync tf32 m16n8k8 (reference enhancing/modules/stage1/layers.py:124-130 and its
// autograd): the scores live in registers only, backward recomputes them from the saved log-sum-exp.
//   PASSES == 1: one tf32 product per MMA; the softmax probabilities and dS are rounded to nearest tf32 before they
//                re-enter the tensor core.  Serves the tf32 data path (q/k/v already tf32-rounded by the GEMM that wrote
//                them).
//   PASSES == 3: the error-compensated 3xTF32 form  a.b ~= a_lo.b_hi + a_hi.b_lo + a_hi.b_hi  (hi = the
//                10-bit-mantissa truncation the tensor core applies anyway, lo = x - hi, exact in fp32), split in
//                registers: fp32-grade results (~2^-21 relative) for `precision="parity"`.
// OUT16 selects fp16 storage of the outputs (O, dq/dk/dv).  The fp16 data path runs on wgmma in attention_f16.cu.
// Backward is split in two kernels so that no atomics are needed: one CTA per key tile (dK, dV) and one per
// query tile (dQ).
#include "../../include/b200vq.h"
#include "attention.cuh"
#include "common.cuh"

namespace b200 {

constexpr float kLog2e = 1.4426950408889634f;

constexpr uint32_t kTf32Mask = 0xFFFFE000u;
__device__ __forceinline__ uint32_t tf32_hi(uint32_t x) { return x & kTf32Mask; }
__device__ __forceinline__ uint32_t tf32_lo(uint32_t x) { return __float_as_uint(__uint_as_float(x) - __uint_as_float(x & kTf32Mask)) & kTf32Mask; }
// c += a . b with both operands given as raw fp32 bit patterns (3 passes: small terms first)
template <int PASSES>
__device__ __forceinline__ void mma_x(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  if constexpr (PASSES == 1) {
    mma_tf32(c, a, b0, b1);
  } else {
    const uint32_t ah[4] = {tf32_hi(a[0]), tf32_hi(a[1]), tf32_hi(a[2]), tf32_hi(a[3])};
    const uint32_t al[4] = {tf32_lo(a[0]), tf32_lo(a[1]), tf32_lo(a[2]), tf32_lo(a[3])};
    mma_tf32(c, al, tf32_hi(b0), tf32_hi(b1));
    mma_tf32(c, ah, tf32_lo(b0), tf32_lo(b1));
    mma_tf32(c, ah, tf32_hi(b0), tf32_hi(b1));
  }
}
// one element as fp32 bits
__device__ __forceinline__ uint32_t ldbits(const float* p) { return __float_as_uint(*p); }
// row pitch (elements) of a staged tile: 16 bytes of padding per row
template <typename T, int DH> struct Pitch { static constexpr int LDS = DH + 16 / (int)sizeof(T); };
__device__ __forceinline__ void cpa16(void* dst, const void* src, bool valid) {
  const int sz = valid ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(dst)), "l"(src), "r"(sz) : "memory");
}
__device__ __forceinline__ void cpa_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cpa_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// stage a [ROWS x DH] tile (row stride ld elements in global) into smem with row pitch Pitch::LDS;
// rows >= nvalid are zero-filled
template <int DH, int ROWS, int THREADS, typename T>
__device__ __forceinline__ void load_tile(T* s, const T* g, long long ld, int row0, int nvalid, int tid) {
  constexpr int E = 16 / (int)sizeof(T);   // elements per 16-byte chunk
  constexpr int V = DH / E;
  constexpr int LDS = Pitch<T, DH>::LDS;
#pragma unroll
  for (int i = tid; i < ROWS * V; i += THREADS) {
    const int r = i / V, c = (i % V) * E;
    const bool ok = row0 + r < nvalid;
    cpa16(s + r * LDS + c, g + (long long)(ok ? row0 + r : 0) * ld + c, ok);
  }
}

// A-operand fragments of a 16 x DH row block read straight from global memory (row stride ld)
template <int DH, typename T>
__device__ __forceinline__ void load_a_frags(uint32_t (&f)[DH / 8][4], const T* base, long long ld, int row_lo,
                                             int nvalid, int lane) {
  const int g = lane >> 2, t = lane & 3;
  const int r0 = row_lo + g, r1 = row_lo + g + 8;
  const T* p0 = base + (long long)(r0 < nvalid ? r0 : 0) * ld;
  const T* p1 = base + (long long)(r1 < nvalid ? r1 : 0) * ld;
  const bool ok0 = r0 < nvalid, ok1 = r1 < nvalid;
#pragma unroll
  for (int k = 0; k < DH / 8; ++k) {
    f[k][0] = ok0 ? ldbits(p0 + k * 8 + t) : 0u;
    f[k][1] = ok1 ? ldbits(p1 + k * 8 + t) : 0u;
    f[k][2] = ok0 ? ldbits(p0 + k * 8 + t + 4) : 0u;
    f[k][3] = ok1 ? ldbits(p1 + k * 8 + t + 4) : 0u;
  }
}

// acc[nt] (16 x 8 each, nt over 64/8 column tiles) += A(16 x DH, regs) . T^T where T is a smem
// tile [64][DH+4] whose rows are the output columns ("K-like" read: b = T[n0+g][k0+t])
template <int DH, int PASSES, typename T>
__device__ __forceinline__ void mma_rows_x_tileT(float (&acc)[8][4], const uint32_t (&a)[DH / 8][4], const T* Ts, int lane) {
  constexpr int LDS = Pitch<T, DH>::LDS;
  const int g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int k = 0; k < DH / 8; ++k)
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      const T* p = Ts + (nt * 8 + g) * LDS + k * 8 + t;
      mma_x<PASSES>(acc[nt], a[k], ldbits(p), ldbits(p + 4));
    }
}
// acc[dt] (16 x 8 each, dt over DH/8 column tiles) += P(16 x 64, given as accumulator-layout
// fragments, full fp32) . T where T is a smem tile [64][DH+4] whose rows are the
// contraction index ("V-like" read).  Accumulator columns (2t, 2t+1) of each 8-wide tile serve
// as k-slots (t, t+4), so the tile rows are read in the matching order 2t, 2t+1.
template <int DH, int PASSES, typename T>
__device__ __forceinline__ void mma_p_x_tile(float (&acc)[DH / 8][4], const uint32_t (&p)[8][4], const T* Ts, int lane) {
  constexpr int LDS = Pitch<T, DH>::LDS;
  const int g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int kt = 0; kt < 8; ++kt)
#pragma unroll
    for (int dt = 0; dt < DH / 8; ++dt) {
      const T* q = Ts + (kt * 8 + 2 * t) * LDS + dt * 8 + g;
      mma_x<PASSES>(acc[dt], p[kt], ldbits(q), ldbits(q + LDS));
    }
}
// accumulator (c0,c1,c2,c3) -> A fragment (a0,a1,a2,a3) = (c0,c2,c1,c3): kept in full fp32 for the 3-pass product
// (split at the MMA), rounded to nearest tf32 for the single pass
template <int PASSES>
__device__ __forceinline__ void acc_to_a(uint32_t (&a)[4], float c0, float c1, float c2, float c3) {
  if constexpr (PASSES == 1) { c0 = round_tf32(c0); c1 = round_tf32(c1); c2 = round_tf32(c2); c3 = round_tf32(c3); }
  a[0] = __float_as_uint(c0); a[1] = __float_as_uint(c2); a[2] = __float_as_uint(c1); a[3] = __float_as_uint(c3);
}
// two adjacent output elements: fp32 (optionally tf32-rounded) or fp16 (saturating)
template <int OUT16>
__device__ __forceinline__ void store2(void* base, long long off, float a, float b, int round_out) {
  if constexpr (OUT16) {
    *reinterpret_cast<uint32_t*>(static_cast<__half*>(base) + off) = pack_half2_sat(a, b);
  } else {
    if (round_out) { a = round_tf32(a); b = round_tf32(b); }
    *reinterpret_cast<float2*>(static_cast<float*>(base) + off) = make_float2(a, b);
  }
}

// The operand path of the kernels below: tf32 m16n8k8 (one or three passes), A fragments [DH/8][4], P / dS fragments [8][4].
template <int DH, int PASSES> struct Ops {
  using T = float;
  using QF = uint32_t[DH / 8][4];
  using PF = uint32_t[8][4];
  static __device__ __forceinline__ void load_a(QF& f, const T* base, long long ld, int row_lo, int nvalid, int lane) {
    load_a_frags<DH>(f, base, ld, row_lo, nvalid, lane);
  }
  static __device__ __forceinline__ void rows_x_tileT(float (&acc)[8][4], const QF& a, const T* Ts, int lane) {
    mma_rows_x_tileT<DH, PASSES>(acc, a, Ts, lane);
  }
  static __device__ __forceinline__ void p_x_tile(float (&acc)[DH / 8][4], const PF& pf, const T* Ts, int lane) {
    mma_p_x_tile<DH, PASSES>(acc, pf, Ts, lane);
  }
  static __device__ __forceinline__ void set_p(PF& pf, int nt, float c0, float c1, float c2, float c3) {
    acc_to_a<PASSES>(pf[nt], c0, c1, c2, c3);
  }
};

// ---------------------------------------------------------------------------------------------
// forward: grid (ceil(N/128), heads, B), 256 threads = 8 warps x 16 query rows
// ---------------------------------------------------------------------------------------------
template <int DH, int PASSES, int OUT16>
__global__ void __launch_bounds__(256)
attn_fwd_kernel(const void* __restrict__ qkv_, void* __restrict__ out, float* __restrict__ lse, int N, int heads,
                float scale, int cond, int round_out) {
  using T = float;
  const T* qkv = static_cast<const T*>(qkv_);
  constexpr int LDS = Pitch<T, DH>::LDS;
  constexpr int TILE = 64 * LDS;
  extern __shared__ __align__(16) uint8_t sm_raw[];   // K[2][TILE], V[2][TILE]
  T* Ks = reinterpret_cast<T*>(sm_raw);
  T* Vs = Ks + 2 * TILE;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3;
  const int h = blockIdx.y, b = blockIdx.z;
  const int inner = heads * DH;
  const long long ld = 3ll * inner;
  const T* qbase = qkv + (long long)b * N * ld + h * DH;
  const T* kbase = qbase + inner;
  const T* vbase = qbase + 2 * inner;
  const int q0 = blockIdx.x * 128 + warp * 16;
  const float c = scale * kLog2e;

  using Op = Ops<DH, PASSES>;
  typename Op::QF qf;
  Op::load_a(qf, qbase, ld, q0, N, lane);

  float o[DH / 8][4];
#pragma unroll
  for (int i = 0; i < DH / 8; ++i) { o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f; }
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;

  // cond >= 0: stage-2 mask (reference stage2/layers.py:43-48,83-85): query q sees key k iff k <= max(q, cond - 1)
  // (causal, with the first `cond` condition tokens fully visible to each other).  Key 0 is visible to every row, so the
  // running maximum is finite after the first tile and fully masked tiles contribute exp2(-inf) = 0.
  const bool masked = cond >= 0;
  const int lim0 = masked ? max(q0 + g, cond - 1) : N, lim1 = masked ? max(q0 + g + 8, cond - 1) : N;
  int ntiles = (N + 63) / 64;
  if (masked) ntiles = min(ntiles, max(min(N - 1, (int)blockIdx.x * 128 + 127), cond - 1) / 64 + 1);   // tiles past the CTA's last visible key
  load_tile<DH, 64, 256>(Ks, kbase, ld, 0, N, tid);
  load_tile<DH, 64, 256>(Vs, vbase, ld, 0, N, tid);
  cpa_commit();
  for (int j = 0; j < ntiles; ++j) {
    const int buf = j & 1;
    cpa_wait<0>();
    __syncthreads();
    if (j + 1 < ntiles) {
      load_tile<DH, 64, 256>(Ks + (buf ^ 1) * TILE, kbase, ld, (j + 1) * 64, N, tid);
      load_tile<DH, 64, 256>(Vs + (buf ^ 1) * TILE, vbase, ld, (j + 1) * 64, N, tid);
      cpa_commit();
    }
    float s[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) { s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f; }
    Op::rows_x_tileT(s, qf, Ks + buf * TILE, lane);
    if ((j + 1) * 64 > N) {
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        const int key = j * 64 + nt * 8 + 2 * t;
        if (key >= N) { s[nt][0] = -INFINITY; s[nt][2] = -INFINITY; }
        if (key + 1 >= N) { s[nt][1] = -INFINITY; s[nt][3] = -INFINITY; }
      }
    }
    if (masked && j * 64 + 63 > min(lim0, lim1)) {
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        const int key = j * 64 + nt * 8 + 2 * t;
        if (key > lim0) s[nt][0] = -INFINITY;
        if (key + 1 > lim0) s[nt][1] = -INFINITY;
        if (key > lim1) s[nt][2] = -INFINITY;
        if (key + 1 > lim1) s[nt][3] = -INFINITY;
      }
    }
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      mx0 = fmaxf(mx0, fmaxf(s[nt][0], s[nt][1]));
      mx1 = fmaxf(mx1, fmaxf(s[nt][2], s[nt][3]));
    }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    const float mn0 = fmaxf(m0, mx0), mn1 = fmaxf(m1, mx1);
    const float al0 = exp2f((m0 - mn0) * c), al1 = exp2f((m1 - mn1) * c);   // exp2(-inf) = 0 on the first tile
    m0 = mn0; m1 = mn1;
    l0 *= al0; l1 *= al1;
#pragma unroll
    for (int i = 0; i < DH / 8; ++i) { o[i][0] *= al0; o[i][1] *= al0; o[i][2] *= al1; o[i][3] *= al1; }
    typename Op::PF pf;
    const float mc0 = m0 * c, mc1 = m1 * c;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      const float p0 = exp2f(s[nt][0] * c - mc0), p1 = exp2f(s[nt][1] * c - mc0);
      const float p2 = exp2f(s[nt][2] * c - mc1), p3 = exp2f(s[nt][3] * c - mc1);
      l0 += p0 + p1; l1 += p2 + p3;
      Op::set_p(pf, nt, p0, p1, p2, p3);
    }
    Op::p_x_tile(o, pf, Vs + buf * TILE, lane);
  }
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const float inv0 = 1.f / l0, inv1 = 1.f / l1;
  const int r0 = q0 + g, r1 = q0 + g + 8;
  const long long ob = (long long)b * N * inner + h * DH;
#pragma unroll
  for (int dt = 0; dt < DH / 8; ++dt) {
    if (r0 < N) store2<OUT16>(out, ob + (long long)r0 * inner + dt * 8 + 2 * t, o[dt][0] * inv0, o[dt][1] * inv0, round_out);
    if (r1 < N) store2<OUT16>(out, ob + (long long)r1 * inner + dt * 8 + 2 * t, o[dt][2] * inv1, o[dt][3] * inv1, round_out);
  }
  if (t == 0) {
    float* lb = lse + ((long long)b * heads + h) * N;
    if (r0 < N) lb[r0] = m0 * scale + logf(l0);
    if (r1 < N) lb[r1] = m1 * scale + logf(l1);
  }
}

// ---------------------------------------------------------------------------------------------
// backward, key side: grid (ceil(N/64), heads, B), 128 threads = 4 warps x 16 keys.
// Works on transposed score tiles S^T[key, query] so that P^T / dS^T come out of the tensor
// cores already in A-operand position for dV += P^T dO and dK += dS^T Q.
// ---------------------------------------------------------------------------------------------
template <int DH, int PASSES, int OUT16>
__global__ void __launch_bounds__(128)
attn_bwd_dkv_kernel(const void* __restrict__ qkv_, const void* __restrict__ dout_, const float* __restrict__ lse,
                    const float* __restrict__ delta, void* __restrict__ dqkv, const float* __restrict__ out_scale, int N,
                    int heads, float scale, int cond, int round_out) {
  using T = float;
  const T* qkv = static_cast<const T*>(qkv_);
  const T* dout = static_cast<const T*>(dout_);
  constexpr int LDS = Pitch<T, DH>::LDS;
  constexpr int TILE = 64 * LDS;
  extern __shared__ __align__(16) uint8_t sm_raw[];   // Q[2][TILE], dO[2][TILE], lse[2][64], delta[2][64]
  T* Qs = reinterpret_cast<T*>(sm_raw);
  T* Ds = Qs + 2 * TILE;
  float* Ls = reinterpret_cast<float*>(Ds + 2 * TILE);
  float* Es = Ls + 128;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3;
  const int h = blockIdx.y, b = blockIdx.z;
  const int inner = heads * DH;
  const long long ld = 3ll * inner;
  const T* qbase = qkv + (long long)b * N * ld + h * DH;
  const T* dobase = dout + (long long)b * N * inner + h * DH;
  const float* lb = lse + ((long long)b * heads + h) * N;
  const float* eb = delta + ((long long)b * heads + h) * N;
  const int k0 = blockIdx.x * 64 + warp * 16;
  const float c = scale * kLog2e;

  using Op = Ops<DH, PASSES>;
  typename Op::QF kf, vf;
  Op::load_a(kf, qbase + inner, ld, k0, N, lane);
  Op::load_a(vf, qbase + 2 * inner, ld, k0, N, lane);
  float dk[DH / 8][4], dv[DH / 8][4];
#pragma unroll
  for (int i = 0; i < DH / 8; ++i) { dk[i][0] = dk[i][1] = dk[i][2] = dk[i][3] = 0.f; dv[i][0] = dv[i][1] = dv[i][2] = dv[i][3] = 0.f; }

  auto stage = [&](int j, int buf) {
    load_tile<DH, 64, 128>(Qs + buf * TILE, qbase, ld, j * 64, N, tid);
    load_tile<DH, 64, 128>(Ds + buf * TILE, dobase, inner, j * 64, N, tid);
    if (tid < 64) {
      const int q = j * 64 + tid;
      Ls[buf * 64 + tid] = q < N ? lb[q] * kLog2e : INFINITY;   // +inf -> P = 0 for padded queries
      Es[buf * 64 + tid] = q < N ? eb[q] : 0.f;
    }
    cpa_commit();
  };
  const int ntiles = (N + 63) / 64;
  // stage-2 mask: key k receives from query q iff k <= max(q, cond - 1).  A key tile that starts at or past `cond` is
  // invisible to every query tile before its own.
  const bool masked = cond >= 0;
  const int jbeg = (masked && (int)blockIdx.x * 64 >= cond) ? (int)blockIdx.x : 0;
  const int kr0 = k0 + g, kr1 = k0 + g + 8;
  stage(jbeg, 0);
  for (int j = jbeg; j < ntiles; ++j) {
    const int buf = (j - jbeg) & 1;
    cpa_wait<0>();
    __syncthreads();
    if (j + 1 < ntiles) stage(j + 1, buf ^ 1);
    const T* Q = Qs + buf * TILE;
    const T* dO = Ds + buf * TILE;
    float s[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) { s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f; }
    Op::rows_x_tileT(s, kf, Q, lane);                // S^T = K Q^T
    typename Op::PF pf;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      const float la = Ls[buf * 64 + nt * 8 + 2 * t], lbb = Ls[buf * 64 + nt * 8 + 2 * t + 1];
      s[nt][0] = exp2f(s[nt][0] * c - la);  s[nt][1] = exp2f(s[nt][1] * c - lbb);
      s[nt][2] = exp2f(s[nt][2] * c - la);  s[nt][3] = exp2f(s[nt][3] * c - lbb);
      if (masked) {
        const int va = max(j * 64 + nt * 8 + 2 * t, cond - 1), vb = max(j * 64 + nt * 8 + 2 * t + 1, cond - 1);   // last key each query sees
        if (kr0 > va) s[nt][0] = 0.f;
        if (kr0 > vb) s[nt][1] = 0.f;
        if (kr1 > va) s[nt][2] = 0.f;
        if (kr1 > vb) s[nt][3] = 0.f;
      }
      Op::set_p(pf, nt, s[nt][0], s[nt][1], s[nt][2], s[nt][3]);
    }
    Op::p_x_tile(dv, pf, dO, lane);                  // dV += P^T dO
    float dp[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) { dp[i][0] = dp[i][1] = dp[i][2] = dp[i][3] = 0.f; }
    Op::rows_x_tileT(dp, vf, dO, lane);              // dP^T = V dO^T
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      const float ea = Es[buf * 64 + nt * 8 + 2 * t], ebb = Es[buf * 64 + nt * 8 + 2 * t + 1];
      Op::set_p(pf, nt, s[nt][0] * (dp[nt][0] - ea), s[nt][1] * (dp[nt][1] - ebb), s[nt][2] * (dp[nt][2] - ea),
                s[nt][3] * (dp[nt][3] - ebb));
    }
    Op::p_x_tile(dk, pf, Q, lane);                   // dK += dS^T Q
  }
  const int r0 = k0 + g, r1 = k0 + g + 8;
  const long long dkb = (long long)b * N * ld + inner + h * DH;
  const long long dvb = dkb + inner;
  const float vm = out_scale ? __ldg(out_scale) : 1.f;     // fp16 output: the gradient scale it travels with
  const float km = scale * vm;
#pragma unroll
  for (int dt = 0; dt < DH / 8; ++dt) {
    if (r0 < N) {
      store2<OUT16>(dqkv, dkb + (long long)r0 * ld + dt * 8 + 2 * t, dk[dt][0] * km, dk[dt][1] * km, round_out);
      store2<OUT16>(dqkv, dvb + (long long)r0 * ld + dt * 8 + 2 * t, dv[dt][0] * vm, dv[dt][1] * vm, round_out);
    }
    if (r1 < N) {
      store2<OUT16>(dqkv, dkb + (long long)r1 * ld + dt * 8 + 2 * t, dk[dt][2] * km, dk[dt][3] * km, round_out);
      store2<OUT16>(dqkv, dvb + (long long)r1 * ld + dt * 8 + 2 * t, dv[dt][2] * vm, dv[dt][3] * vm, round_out);
    }
  }
}

// ---------------------------------------------------------------------------------------------
// backward, query side: grid (ceil(N/64), heads, B), 128 threads = 4 warps x 16 queries
// ---------------------------------------------------------------------------------------------
template <int DH, int PASSES, int OUT16>
__global__ void __launch_bounds__(128)
attn_bwd_dq_kernel(const void* __restrict__ qkv_, const void* __restrict__ dout_, const float* __restrict__ lse,
                   const float* __restrict__ delta, void* __restrict__ dqkv, const float* __restrict__ out_scale, int N,
                   int heads, float scale, int cond, int round_out) {
  using T = float;
  const T* qkv = static_cast<const T*>(qkv_);
  const T* dout = static_cast<const T*>(dout_);
  constexpr int LDS = Pitch<T, DH>::LDS;
  constexpr int TILE = 64 * LDS;
  extern __shared__ __align__(16) uint8_t sm_raw[];   // K[2][TILE], V[2][TILE]
  T* Ks = reinterpret_cast<T*>(sm_raw);
  T* Vs = Ks + 2 * TILE;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3;
  const int h = blockIdx.y, b = blockIdx.z;
  const int inner = heads * DH;
  const long long ld = 3ll * inner;
  const T* qbase = qkv + (long long)b * N * ld + h * DH;
  const T* kbase = qbase + inner;
  const T* vbase = qbase + 2 * inner;
  const T* dobase = dout + (long long)b * N * inner + h * DH;
  const int q0 = blockIdx.x * 64 + warp * 16;
  const float c = scale * kLog2e;
  const int r0 = q0 + g, r1 = q0 + g + 8;
  const float* lb = lse + ((long long)b * heads + h) * N;
  const float* eb = delta + ((long long)b * heads + h) * N;
  const float lse0 = r0 < N ? lb[r0] * kLog2e : INFINITY, lse1 = r1 < N ? lb[r1] * kLog2e : INFINITY;
  const float e0 = r0 < N ? eb[r0] : 0.f, e1 = r1 < N ? eb[r1] : 0.f;

  using Op = Ops<DH, PASSES>;
  typename Op::QF qf, dof;
  Op::load_a(qf, qbase, ld, q0, N, lane);
  Op::load_a(dof, dobase, inner, q0, N, lane);
  float dq[DH / 8][4];
#pragma unroll
  for (int i = 0; i < DH / 8; ++i) { dq[i][0] = dq[i][1] = dq[i][2] = dq[i][3] = 0.f; }

  const bool masked = cond >= 0;
  const int lim0 = masked ? max(r0, cond - 1) : N, lim1 = masked ? max(r1, cond - 1) : N;
  int ntiles = (N + 63) / 64;
  if (masked) ntiles = min(ntiles, max(min(N - 1, (int)blockIdx.x * 64 + 63), cond - 1) / 64 + 1);
  load_tile<DH, 64, 128>(Ks, kbase, ld, 0, N, tid);
  load_tile<DH, 64, 128>(Vs, vbase, ld, 0, N, tid);
  cpa_commit();
  for (int j = 0; j < ntiles; ++j) {
    const int buf = j & 1;
    cpa_wait<0>();
    __syncthreads();
    if (j + 1 < ntiles) {
      load_tile<DH, 64, 128>(Ks + (buf ^ 1) * TILE, kbase, ld, (j + 1) * 64, N, tid);
      load_tile<DH, 64, 128>(Vs + (buf ^ 1) * TILE, vbase, ld, (j + 1) * 64, N, tid);
      cpa_commit();
    }
    float s[8][4], dp[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) { s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f; dp[i][0] = dp[i][1] = dp[i][2] = dp[i][3] = 0.f; }
    Op::rows_x_tileT(s, qf, Ks + buf * TILE, lane);     // S = Q K^T
    Op::rows_x_tileT(dp, dof, Vs + buf * TILE, lane);   // dP = dO V^T
    typename Op::PF pf;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      const int key = j * 64 + nt * 8 + 2 * t;
      const bool ka = key < N, kb = key + 1 < N;
      const float p0 = (ka && key <= lim0) ? exp2f(s[nt][0] * c - lse0) : 0.f, p1 = (kb && key + 1 <= lim0) ? exp2f(s[nt][1] * c - lse0) : 0.f;
      const float p2 = (ka && key <= lim1) ? exp2f(s[nt][2] * c - lse1) : 0.f, p3 = (kb && key + 1 <= lim1) ? exp2f(s[nt][3] * c - lse1) : 0.f;
      Op::set_p(pf, nt, p0 * (dp[nt][0] - e0), p1 * (dp[nt][1] - e0), p2 * (dp[nt][2] - e1), p3 * (dp[nt][3] - e1));
    }
    Op::p_x_tile(dq, pf, Ks + buf * TILE, lane);        // dQ += dS K
  }
  const long long dqb = (long long)b * N * ld + h * DH;
  const float qm = scale * (out_scale ? __ldg(out_scale) : 1.f);
#pragma unroll
  for (int dt = 0; dt < DH / 8; ++dt) {
    if (r0 < N) store2<OUT16>(dqkv, dqb + (long long)r0 * ld + dt * 8 + 2 * t, dq[dt][0] * qm, dq[dt][1] * qm, round_out);
    if (r1 < N) store2<OUT16>(dqkv, dqb + (long long)r1 * ld + dt * 8 + 2 * t, dq[dt][2] * qm, dq[dt][3] * qm, round_out);
  }
}

// ---------------------------------------------------------------------------------------------
// Wide heads (DH 96 / 128, stage-2 mask, fp32 in and out).  At these widths a warp's resident operand fragments
// (DH/2 registers each) no longer fit next to its accumulators, so the resident operand of each kernel (forward: Q;
// key side: K, V; query side: Q, dO) is staged once in shared memory and its A fragments are read per k-step, the
// way the streamed tiles' B fragments are.  Registers then hold only the DH/8 x 4 accumulators and the score tiles.
// Every kernel is 8 warps x 16 resident rows = 128 rows per CTA; the streamed tiles are double-buffered, KB rows each
// (forward 64; backward 32, which keeps the score, dP and dS tiles of the key side at 16 registers each beside the
// 2 x DH/2 registers of dK and dV).  Shared memory at DH 128: 384 padded rows of 528 bytes = 198 KB per CTA.
// ---------------------------------------------------------------------------------------------
constexpr int kWideRows = 128;   // resident rows per CTA (8 warps x 16)

// A fragment (k-step k) of the warp's 16-row block `As` of a staged tile (row pitch Pitch::LDS)
template <int DH>
__device__ __forceinline__ void lds_a_frag(uint32_t (&a)[4], const float* As, int k, int lane) {
  constexpr int LDS = Pitch<float, DH>::LDS;
  const float* p = As + (lane >> 2) * LDS + k * 8 + (lane & 3);
  a[0] = ldbits(p); a[1] = ldbits(p + 8 * LDS); a[2] = ldbits(p + 4); a[3] = ldbits(p + 8 * LDS + 4);
}
// acc[nt] (16 x 8 each, NT column tiles) += A(16 x DH, staged rows As) . T^T, T a staged tile whose rows are the output
// columns (mma_rows_x_tileT with the A operand from shared memory)
template <int DH, int PASSES, int NT>
__device__ __forceinline__ void mma_srows_x_tileT(float (&acc)[NT][4], const float* As, const float* Ts, int lane) {
  constexpr int LDS = Pitch<float, DH>::LDS;
  const int g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int k = 0; k < DH / 8; ++k) {
    uint32_t a[4];
    lds_a_frag<DH>(a, As, k, lane);
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
      const float* p = Ts + (nt * 8 + g) * LDS + k * 8 + t;
      mma_x<PASSES>(acc[nt], a, ldbits(p), ldbits(p + 4));
    }
  }
}
// acc[dt] += P(16 x 8 NT, accumulator-layout fragments) . T, T a staged tile whose rows are the contraction index
// (mma_p_x_tile over NT k-steps)
template <int DH, int PASSES, int NT>
__device__ __forceinline__ void mma_pn_x_tile(float (&acc)[DH / 8][4], const uint32_t (&p)[NT][4], const float* Ts, int lane) {
  constexpr int LDS = Pitch<float, DH>::LDS;
  const int g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int kt = 0; kt < NT; ++kt)
#pragma unroll
    for (int dt = 0; dt < DH / 8; ++dt) {
      const float* q = Ts + (kt * 8 + 2 * t) * LDS + dt * 8 + g;
      mma_x<PASSES>(acc[dt], p[kt], ldbits(q), ldbits(q + LDS));
    }
}

// forward: grid (ceil(N/128), heads, B); Q[128 rows], K[2][64 rows], V[2][64 rows]
template <int DH, int PASSES>
__global__ void __launch_bounds__(256, 1)
attn_fwd_wide_kernel(const float* __restrict__ qkv, float* __restrict__ out, float* __restrict__ lse, int N, int heads, float scale,
                     int cond, int round_out) {
  constexpr int LDS = Pitch<float, DH>::LDS;
  constexpr int KB = 64, NT = KB / 8;
  constexpr int TILE = KB * LDS;
  extern __shared__ __align__(16) uint8_t sm_raw[];
  float* Qs = reinterpret_cast<float*>(sm_raw);
  float* Ks = Qs + kWideRows * LDS;
  float* Vs = Ks + 2 * TILE;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3;
  const int h = blockIdx.y, b = blockIdx.z;
  const int inner = heads * DH;
  const long long ld = 3ll * inner;
  const float* qbase = qkv + (long long)b * N * ld + h * DH;
  const float* kbase = qbase + inner;
  const float* vbase = qbase + 2 * inner;
  const int qb = blockIdx.x * kWideRows;
  const int q0 = qb + warp * 16;
  const float* Qw = Qs + warp * 16 * LDS;
  const float c = scale * kLog2e;

  float o[DH / 8][4];
#pragma unroll
  for (int i = 0; i < DH / 8; ++i) { o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f; }
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;

  // the mask and tile skipping of attn_fwd_kernel (cond >= 0 always here)
  const int lim0 = max(q0 + g, cond - 1), lim1 = max(q0 + g + 8, cond - 1);
  const int ntiles = min((N + KB - 1) / KB, max(min(N - 1, qb + kWideRows - 1), cond - 1) / KB + 1);
  load_tile<DH, kWideRows, 256>(Qs, qbase, ld, qb, N, tid);
  load_tile<DH, KB, 256>(Ks, kbase, ld, 0, N, tid);
  load_tile<DH, KB, 256>(Vs, vbase, ld, 0, N, tid);
  cpa_commit();
  for (int j = 0; j < ntiles; ++j) {
    const int buf = j & 1;
    cpa_wait<0>();
    __syncthreads();
    if (j + 1 < ntiles) {
      load_tile<DH, KB, 256>(Ks + (buf ^ 1) * TILE, kbase, ld, (j + 1) * KB, N, tid);
      load_tile<DH, KB, 256>(Vs + (buf ^ 1) * TILE, vbase, ld, (j + 1) * KB, N, tid);
      cpa_commit();
    }
    float s[NT][4];
#pragma unroll
    for (int i = 0; i < NT; ++i) { s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f; }
    mma_srows_x_tileT<DH, PASSES, NT>(s, Qw, Ks + buf * TILE, lane);
    if ((j + 1) * KB > N || j * KB + KB - 1 > min(lim0, lim1)) {
#pragma unroll
      for (int nt = 0; nt < NT; ++nt) {
        const int key = j * KB + nt * 8 + 2 * t;
        if (key >= N || key > lim0) s[nt][0] = -INFINITY;
        if (key + 1 >= N || key + 1 > lim0) s[nt][1] = -INFINITY;
        if (key >= N || key > lim1) s[nt][2] = -INFINITY;
        if (key + 1 >= N || key + 1 > lim1) s[nt][3] = -INFINITY;
      }
    }
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
      mx0 = fmaxf(mx0, fmaxf(s[nt][0], s[nt][1]));
      mx1 = fmaxf(mx1, fmaxf(s[nt][2], s[nt][3]));
    }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    const float mn0 = fmaxf(m0, mx0), mn1 = fmaxf(m1, mx1);
    const float al0 = exp2f((m0 - mn0) * c), al1 = exp2f((m1 - mn1) * c);
    m0 = mn0; m1 = mn1;
    l0 *= al0; l1 *= al1;
#pragma unroll
    for (int i = 0; i < DH / 8; ++i) { o[i][0] *= al0; o[i][1] *= al0; o[i][2] *= al1; o[i][3] *= al1; }
    uint32_t pf[NT][4];
    const float mc0 = m0 * c, mc1 = m1 * c;
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
      const float p0 = exp2f(s[nt][0] * c - mc0), p1 = exp2f(s[nt][1] * c - mc0);
      const float p2 = exp2f(s[nt][2] * c - mc1), p3 = exp2f(s[nt][3] * c - mc1);
      l0 += p0 + p1; l1 += p2 + p3;
      acc_to_a<PASSES>(pf[nt], p0, p1, p2, p3);
    }
    mma_pn_x_tile<DH, PASSES, NT>(o, pf, Vs + buf * TILE, lane);
  }
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const float inv0 = 1.f / l0, inv1 = 1.f / l1;
  const int r0 = q0 + g, r1 = q0 + g + 8;
  const long long ob = (long long)b * N * inner + h * DH;
#pragma unroll
  for (int dt = 0; dt < DH / 8; ++dt) {
    if (r0 < N) store2<0>(out, ob + (long long)r0 * inner + dt * 8 + 2 * t, o[dt][0] * inv0, o[dt][1] * inv0, round_out);
    if (r1 < N) store2<0>(out, ob + (long long)r1 * inner + dt * 8 + 2 * t, o[dt][2] * inv1, o[dt][3] * inv1, round_out);
  }
  if (t == 0) {
    float* lb = lse + ((long long)b * heads + h) * N;
    if (r0 < N) lb[r0] = m0 * scale + logf(l0);
    if (r1 < N) lb[r1] = m1 * scale + logf(l1);
  }
}

// backward, key side: grid (ceil(N/128), heads, B); K[128 rows], V[128 rows], Q[2][32 rows], dO[2][32 rows], lse[2][32],
// delta[2][32].  Transposed score tiles as in attn_bwd_dkv_kernel.
template <int DH, int PASSES>
__global__ void __launch_bounds__(256, 1)
attn_bwd_dkv_wide_kernel(const float* __restrict__ qkv, const float* __restrict__ dout, const float* __restrict__ lse,
                         const float* __restrict__ delta, float* __restrict__ dqkv, int N, int heads, float scale, int cond,
                         int round_out) {
  constexpr int LDS = Pitch<float, DH>::LDS;
  constexpr int KB = 32, NT = KB / 8;
  constexpr int TILE = KB * LDS;
  extern __shared__ __align__(16) uint8_t sm_raw[];
  float* Kr = reinterpret_cast<float*>(sm_raw);
  float* Vr = Kr + kWideRows * LDS;
  float* Qs = Vr + kWideRows * LDS;
  float* Ds = Qs + 2 * TILE;
  float* Ls = Ds + 2 * TILE;
  float* Es = Ls + 2 * KB;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3;
  const int h = blockIdx.y, b = blockIdx.z;
  const int inner = heads * DH;
  const long long ld = 3ll * inner;
  const float* qbase = qkv + (long long)b * N * ld + h * DH;
  const float* dobase = dout + (long long)b * N * inner + h * DH;
  const float* lb = lse + ((long long)b * heads + h) * N;
  const float* eb = delta + ((long long)b * heads + h) * N;
  const int kb = blockIdx.x * kWideRows;
  const int k0 = kb + warp * 16;
  const float* Kw = Kr + warp * 16 * LDS;
  const float* Vw = Vr + warp * 16 * LDS;
  const float c = scale * kLog2e;

  float dk[DH / 8][4], dv[DH / 8][4];
#pragma unroll
  for (int i = 0; i < DH / 8; ++i) { dk[i][0] = dk[i][1] = dk[i][2] = dk[i][3] = 0.f; dv[i][0] = dv[i][1] = dv[i][2] = dv[i][3] = 0.f; }

  auto stage = [&](int j, int buf) {
    load_tile<DH, KB, 256>(Qs + buf * TILE, qbase, ld, j * KB, N, tid);
    load_tile<DH, KB, 256>(Ds + buf * TILE, dobase, inner, j * KB, N, tid);
    if (tid < KB) {
      const int q = j * KB + tid;
      Ls[buf * KB + tid] = q < N ? lb[q] * kLog2e : INFINITY;   // +inf -> P = 0 for padded queries
      Es[buf * KB + tid] = q < N ? eb[q] : 0.f;
    }
  };
  const int ntiles = (N + KB - 1) / KB;
  // key k receives from query q iff k <= max(q, cond - 1): a CTA whose first key is at or past `cond` starts at its own
  // first key's query tile
  const int jbeg = kb >= cond ? kb / KB : 0;
  const int kr0 = k0 + g, kr1 = k0 + g + 8;
  load_tile<DH, kWideRows, 256>(Kr, qbase + inner, ld, kb, N, tid);
  load_tile<DH, kWideRows, 256>(Vr, qbase + 2 * inner, ld, kb, N, tid);
  stage(jbeg, 0);
  cpa_commit();
  for (int j = jbeg; j < ntiles; ++j) {
    const int buf = (j - jbeg) & 1;
    cpa_wait<0>();
    __syncthreads();
    if (j + 1 < ntiles) { stage(j + 1, buf ^ 1); cpa_commit(); }
    const float* Q = Qs + buf * TILE;
    const float* dO = Ds + buf * TILE;
    float s[NT][4];
#pragma unroll
    for (int i = 0; i < NT; ++i) { s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f; }
    mma_srows_x_tileT<DH, PASSES, NT>(s, Kw, Q, lane);       // S^T = K Q^T
    uint32_t pf[NT][4];
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
      const float la = Ls[buf * KB + nt * 8 + 2 * t], lbb = Ls[buf * KB + nt * 8 + 2 * t + 1];
      s[nt][0] = exp2f(s[nt][0] * c - la);  s[nt][1] = exp2f(s[nt][1] * c - lbb);
      s[nt][2] = exp2f(s[nt][2] * c - la);  s[nt][3] = exp2f(s[nt][3] * c - lbb);
      const int va = max(j * KB + nt * 8 + 2 * t, cond - 1), vb = max(j * KB + nt * 8 + 2 * t + 1, cond - 1);   // last key each query sees
      if (kr0 > va) s[nt][0] = 0.f;
      if (kr0 > vb) s[nt][1] = 0.f;
      if (kr1 > va) s[nt][2] = 0.f;
      if (kr1 > vb) s[nt][3] = 0.f;
      acc_to_a<PASSES>(pf[nt], s[nt][0], s[nt][1], s[nt][2], s[nt][3]);
    }
    mma_pn_x_tile<DH, PASSES, NT>(dv, pf, dO, lane);         // dV += P^T dO
    float dp[NT][4];
#pragma unroll
    for (int i = 0; i < NT; ++i) { dp[i][0] = dp[i][1] = dp[i][2] = dp[i][3] = 0.f; }
    mma_srows_x_tileT<DH, PASSES, NT>(dp, Vw, dO, lane);     // dP^T = V dO^T
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
      const float ea = Es[buf * KB + nt * 8 + 2 * t], ebb = Es[buf * KB + nt * 8 + 2 * t + 1];
      acc_to_a<PASSES>(pf[nt], s[nt][0] * (dp[nt][0] - ea), s[nt][1] * (dp[nt][1] - ebb), s[nt][2] * (dp[nt][2] - ea),
                       s[nt][3] * (dp[nt][3] - ebb));
    }
    mma_pn_x_tile<DH, PASSES, NT>(dk, pf, Q, lane);          // dK += dS^T Q
  }
  const long long dkb = (long long)b * N * ld + inner + h * DH;
  const long long dvb = dkb + inner;
#pragma unroll
  for (int dt = 0; dt < DH / 8; ++dt) {
    if (kr0 < N) {
      store2<0>(dqkv, dkb + (long long)kr0 * ld + dt * 8 + 2 * t, dk[dt][0] * scale, dk[dt][1] * scale, round_out);
      store2<0>(dqkv, dvb + (long long)kr0 * ld + dt * 8 + 2 * t, dv[dt][0], dv[dt][1], round_out);
    }
    if (kr1 < N) {
      store2<0>(dqkv, dkb + (long long)kr1 * ld + dt * 8 + 2 * t, dk[dt][2] * scale, dk[dt][3] * scale, round_out);
      store2<0>(dqkv, dvb + (long long)kr1 * ld + dt * 8 + 2 * t, dv[dt][2], dv[dt][3], round_out);
    }
  }
}

// backward, query side: grid (ceil(N/128), heads, B); Q[128 rows], dO[128 rows], K[2][32 rows], V[2][32 rows]
template <int DH, int PASSES>
__global__ void __launch_bounds__(256, 1)
attn_bwd_dq_wide_kernel(const float* __restrict__ qkv, const float* __restrict__ dout, const float* __restrict__ lse,
                        const float* __restrict__ delta, float* __restrict__ dqkv, int N, int heads, float scale, int cond,
                        int round_out) {
  constexpr int LDS = Pitch<float, DH>::LDS;
  constexpr int KB = 32, NT = KB / 8;
  constexpr int TILE = KB * LDS;
  extern __shared__ __align__(16) uint8_t sm_raw[];
  float* Qr = reinterpret_cast<float*>(sm_raw);
  float* Dr = Qr + kWideRows * LDS;
  float* Ks = Dr + kWideRows * LDS;
  float* Vs = Ks + 2 * TILE;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3;
  const int h = blockIdx.y, b = blockIdx.z;
  const int inner = heads * DH;
  const long long ld = 3ll * inner;
  const float* qbase = qkv + (long long)b * N * ld + h * DH;
  const float* kbase = qbase + inner;
  const float* vbase = qbase + 2 * inner;
  const float* dobase = dout + (long long)b * N * inner + h * DH;
  const int qb = blockIdx.x * kWideRows;
  const int q0 = qb + warp * 16;
  const float* Qw = Qr + warp * 16 * LDS;
  const float* Dw = Dr + warp * 16 * LDS;
  const float c = scale * kLog2e;
  const int r0 = q0 + g, r1 = q0 + g + 8;
  const float* lb = lse + ((long long)b * heads + h) * N;
  const float* eb = delta + ((long long)b * heads + h) * N;
  const float lse0 = r0 < N ? lb[r0] * kLog2e : INFINITY, lse1 = r1 < N ? lb[r1] * kLog2e : INFINITY;
  const float e0 = r0 < N ? eb[r0] : 0.f, e1 = r1 < N ? eb[r1] : 0.f;

  float dq[DH / 8][4];
#pragma unroll
  for (int i = 0; i < DH / 8; ++i) { dq[i][0] = dq[i][1] = dq[i][2] = dq[i][3] = 0.f; }

  const int lim0 = max(r0, cond - 1), lim1 = max(r1, cond - 1);
  const int ntiles = min((N + KB - 1) / KB, max(min(N - 1, qb + kWideRows - 1), cond - 1) / KB + 1);
  load_tile<DH, kWideRows, 256>(Qr, qbase, ld, qb, N, tid);
  load_tile<DH, kWideRows, 256>(Dr, dobase, inner, qb, N, tid);
  load_tile<DH, KB, 256>(Ks, kbase, ld, 0, N, tid);
  load_tile<DH, KB, 256>(Vs, vbase, ld, 0, N, tid);
  cpa_commit();
  for (int j = 0; j < ntiles; ++j) {
    const int buf = j & 1;
    cpa_wait<0>();
    __syncthreads();
    if (j + 1 < ntiles) {
      load_tile<DH, KB, 256>(Ks + (buf ^ 1) * TILE, kbase, ld, (j + 1) * KB, N, tid);
      load_tile<DH, KB, 256>(Vs + (buf ^ 1) * TILE, vbase, ld, (j + 1) * KB, N, tid);
      cpa_commit();
    }
    float s[NT][4], dp[NT][4];
#pragma unroll
    for (int i = 0; i < NT; ++i) { s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f; dp[i][0] = dp[i][1] = dp[i][2] = dp[i][3] = 0.f; }
    mma_srows_x_tileT<DH, PASSES, NT>(s, Qw, Ks + buf * TILE, lane);    // S = Q K^T
    mma_srows_x_tileT<DH, PASSES, NT>(dp, Dw, Vs + buf * TILE, lane);   // dP = dO V^T
    uint32_t pf[NT][4];
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
      const int key = j * KB + nt * 8 + 2 * t;
      const bool ka = key < N, kbv = key + 1 < N;
      const float p0 = (ka && key <= lim0) ? exp2f(s[nt][0] * c - lse0) : 0.f, p1 = (kbv && key + 1 <= lim0) ? exp2f(s[nt][1] * c - lse0) : 0.f;
      const float p2 = (ka && key <= lim1) ? exp2f(s[nt][2] * c - lse1) : 0.f, p3 = (kbv && key + 1 <= lim1) ? exp2f(s[nt][3] * c - lse1) : 0.f;
      acc_to_a<PASSES>(pf[nt], p0 * (dp[nt][0] - e0), p1 * (dp[nt][1] - e0), p2 * (dp[nt][2] - e1), p3 * (dp[nt][3] - e1));
    }
    mma_pn_x_tile<DH, PASSES, NT>(dq, pf, Ks + buf * TILE, lane);       // dQ += dS K
  }
  const long long dqb = (long long)b * N * ld + h * DH;
#pragma unroll
  for (int dt = 0; dt < DH / 8; ++dt) {
    if (r0 < N) store2<0>(dqkv, dqb + (long long)r0 * ld + dt * 8 + 2 * t, dq[dt][0] * scale, dq[dt][1] * scale, round_out);
    if (r1 < N) store2<0>(dqkv, dqb + (long long)r1 * ld + dt * 8 + 2 * t, dq[dt][2] * scale, dq[dt][3] * scale, round_out);
  }
}

template <int DH, int PASSES>
static int fwd_wide_launch(const float* qkv, float* out, float* lse, int B, int N, int heads, float scale, int cond, int round_out,
                           cudaStream_t s) {
  constexpr size_t smem = (kWideRows + 4 * 64) * Pitch<float, DH>::LDS * sizeof(float);
  auto kern = attn_fwd_wide_kernel<DH, PASSES>;
  B200_CONFIGURE_SMEM_ONCE(kern, smem);
  kern<<<dim3((N + kWideRows - 1) / kWideRows, heads, B), 256, smem, s>>>(qkv, out, lse, N, heads, scale, cond, round_out);
  B200_LAUNCH_OK("attn_fwd_wide_kernel");
  return 0;
}

template <int DH, int PASSES>
static int bwd_wide_launch(const float* qkv, const float* dout, const float* lse, const float* delta, float* dqkv, int B, int N,
                           int heads, float scale, int cond, int round_out, cudaStream_t s) {
  constexpr size_t rows = 2 * kWideRows + 4 * 32;
  constexpr size_t smem_kv = rows * Pitch<float, DH>::LDS * sizeof(float) + 4 * 32 * sizeof(float);
  constexpr size_t smem_q = rows * Pitch<float, DH>::LDS * sizeof(float);
  auto k1 = attn_bwd_dkv_wide_kernel<DH, PASSES>;
  auto k2 = attn_bwd_dq_wide_kernel<DH, PASSES>;
  B200_CONFIGURE_SMEM_ONCE(k1, smem_kv);
  B200_CONFIGURE_SMEM_ONCE(k2, smem_q);
  const dim3 grid((N + kWideRows - 1) / kWideRows, heads, B);
  k1<<<grid, 256, smem_kv, s>>>(qkv, dout, lse, delta, dqkv, N, heads, scale, cond, round_out);
  B200_LAUNCH_OK("attn_bwd_dkv_wide_kernel");
  k2<<<grid, 256, smem_q, s>>>(qkv, dout, lse, delta, dqkv, N, heads, scale, cond, round_out);
  B200_LAUNCH_OK("attn_bwd_dq_wide_kernel");
  return 0;
}

static int check_wide(const void* qkv, int B, int N, int heads, int dh, int cond_len) {
  B200_CHECK_ARG(B > 0 && N > 0 && heads > 0, "attention: empty problem");
  B200_CHECK_ARG(dh == 96 || dh == 128, "attention: wide-head core takes head size 96 or 128 (got %d)", dh);
  B200_CHECK_ARG(B <= 65535 && heads <= 65535, "attention: grid too large");
  B200_CHECK_ARG(cond_len >= 0 && cond_len <= N, "attention: cond_len %d outside [0, %d]", cond_len, N);
  B200_CHECK_ARG((reinterpret_cast<uintptr_t>(qkv) & 15) == 0, "attention: qkv must be 16-byte aligned");
  return 0;
}

int attention_wide_forward(const float* qkv, float* out, float* lse, int B, int N, int heads, int dh, float scale, int cond_len,
                           int exact, int round_out, cudaStream_t stream) {
  if (int rc = check_wide(qkv, B, N, heads, dh, cond_len)) return rc;
  if (exact) return dh == 128 ? fwd_wide_launch<128, 3>(qkv, out, lse, B, N, heads, scale, cond_len, 0, stream)
                              : fwd_wide_launch<96, 3>(qkv, out, lse, B, N, heads, scale, cond_len, 0, stream);
  return dh == 128 ? fwd_wide_launch<128, 1>(qkv, out, lse, B, N, heads, scale, cond_len, round_out, stream)
                   : fwd_wide_launch<96, 1>(qkv, out, lse, B, N, heads, scale, cond_len, round_out, stream);
}

int attention_wide_backward(const float* qkv, const float* out, const float* lse, const float* dout, float* dqkv, float* delta,
                            int B, int N, int heads, int dh, float scale, int cond_len, int exact, int round_out,
                            cudaStream_t stream) {
  if (int rc = check_wide(qkv, B, N, heads, dh, cond_len)) return rc;
  B200_CHECK_ARG((reinterpret_cast<uintptr_t>(dout) & 15) == 0, "attention: dout must be 16-byte aligned");
  if (int rc = attention_delta(out, 0, dout, 0, delta, B, N, heads, dh, stream)) return rc;
  if (exact) return dh == 128 ? bwd_wide_launch<128, 3>(qkv, dout, lse, delta, dqkv, B, N, heads, scale, cond_len, 0, stream)
                              : bwd_wide_launch<96, 3>(qkv, dout, lse, delta, dqkv, B, N, heads, scale, cond_len, 0, stream);
  return dh == 128 ? bwd_wide_launch<128, 1>(qkv, dout, lse, delta, dqkv, B, N, heads, scale, cond_len, round_out, stream)
                   : bwd_wide_launch<96, 1>(qkv, dout, lse, delta, dqkv, B, N, heads, scale, cond_len, round_out, stream);
}

// ---------------------------------------------------------------------------------------------
template <int DH, int PASSES, int OUT16>
static int fwd_launch(const void* qkv, void* out, float* lse, int B, int N, int heads, float scale, int cond, int round_out,
                      cudaStream_t s) {
  using T = float;
  constexpr size_t smem = 4 * 64 * Pitch<T, DH>::LDS * sizeof(T);
  auto kern = attn_fwd_kernel<DH, PASSES, OUT16>;
  B200_CONFIGURE_SMEM_ONCE(kern, smem);
  kern<<<dim3((N + 127) / 128, heads, B), 256, smem, s>>>(qkv, out, lse, N, heads, scale, cond, round_out);
  B200_LAUNCH_OK("attn_fwd_kernel");
  return 0;
}

template <int DH, int PASSES, int OUT16>
static int bwd_launch(const void* qkv, const void* dout, const float* lse, const float* delta, void* dqkv, const float* out_scale,
                      int B, int N, int heads, float scale, int cond, int round_out, cudaStream_t s) {
  using T = float;
  constexpr size_t smem_kv = 4 * 64 * Pitch<T, DH>::LDS * sizeof(T) + 256 * sizeof(float);
  constexpr size_t smem_q = 4 * 64 * Pitch<T, DH>::LDS * sizeof(T);
  auto k1 = attn_bwd_dkv_kernel<DH, PASSES, OUT16>;
  auto k2 = attn_bwd_dq_kernel<DH, PASSES, OUT16>;
  B200_CONFIGURE_SMEM_ONCE(k1, smem_kv);
  B200_CONFIGURE_SMEM_ONCE(k2, smem_q);
  const dim3 grid((N + 63) / 64, heads, B);
  k1<<<grid, 128, smem_kv, s>>>(qkv, dout, lse, delta, dqkv, out_scale, N, heads, scale, cond, round_out);
  B200_LAUNCH_OK("attn_bwd_dkv_kernel");
  k2<<<grid, 128, smem_q, s>>>(qkv, dout, lse, delta, dqkv, out_scale, N, heads, scale, cond, round_out);
  B200_LAUNCH_OK("attn_bwd_dq_kernel");
  return 0;
}

static int check_problem(const void* qkv, int B, int N, int heads, int dh, int cond_len) {
  B200_CHECK_ARG(B > 0 && N > 0 && heads > 0, "attention: empty problem");
  B200_CHECK_ARG(dh == 64 || dh == 32, "attention: dim_head must be 32 or 64 (got %d)", dh);
  B200_CHECK_ARG(B <= 65535 && heads <= 65535, "attention: grid too large");
  B200_CHECK_ARG(cond_len <= N, "attention: cond_len %d exceeds the sequence length %d", cond_len, N);
  B200_CHECK_ARG((reinterpret_cast<uintptr_t>(qkv) & 15) == 0, "attention: qkv must be 16-byte aligned");
  return 0;
}

int attention_exact_forward(const float* qkv, float* out, float* lse, int B, int N, int heads, int dh, float scale,
                            int cond_len, cudaStream_t stream) {
  if (int rc = check_problem(qkv, B, N, heads, dh, cond_len)) return rc;
  if (dh == 64) return fwd_launch<64, 3, 0>(qkv, out, lse, B, N, heads, scale, cond_len, 0, stream);
  return fwd_launch<32, 3, 0>(qkv, out, lse, B, N, heads, scale, cond_len, 0, stream);
}

int attention_exact_backward(const float* qkv, const float* out, const float* lse, const float* dout, float* dqkv, float* delta,
                             int B, int N, int heads, int dh, float scale, int cond_len, cudaStream_t stream) {
  if (int rc = check_problem(qkv, B, N, heads, dh, cond_len)) return rc;
  int rc = attention_delta(out, 0, dout, 0, delta, B, N, heads, dh, stream);
  if (rc) return rc;
  if (dh == 64) return bwd_launch<64, 3, 0>(qkv, dout, lse, delta, dqkv, nullptr, B, N, heads, scale, cond_len, 0, stream);
  return bwd_launch<32, 3, 0>(qkv, dout, lse, delta, dqkv, nullptr, B, N, heads, scale, cond_len, 0, stream);
}

int attention_forward_tc(const float* qkv, void* out, int out_half, float* lse, int B, int N, int heads, int dh, float scale,
                         int round_out, int cond_len, cudaStream_t stream) {
  if (int rc = check_problem(qkv, B, N, heads, dh, cond_len)) return rc;
  if (dh == 64) return out_half ? fwd_launch<64, 1, 1>(qkv, out, lse, B, N, heads, scale, cond_len, 0, stream)
                                : fwd_launch<64, 1, 0>(qkv, out, lse, B, N, heads, scale, cond_len, round_out, stream);
  return out_half ? fwd_launch<32, 1, 1>(qkv, out, lse, B, N, heads, scale, cond_len, 0, stream)
                  : fwd_launch<32, 1, 0>(qkv, out, lse, B, N, heads, scale, cond_len, round_out, stream);
}

int attention_backward_tc(const float* qkv, const float* dout, const float* lse, const float* delta, void* dqkv, int out_half,
                          const float* out_scale, int B, int N, int heads, int dh, float scale, int round_out, int cond_len,
                          cudaStream_t stream) {
  if (int rc = check_problem(qkv, B, N, heads, dh, cond_len)) return rc;
  B200_CHECK_ARG((reinterpret_cast<uintptr_t>(dout) & 15) == 0, "attention: dout must be 16-byte aligned");
  if (dh == 64) return out_half ? bwd_launch<64, 1, 1>(qkv, dout, lse, delta, dqkv, out_scale, B, N, heads, scale, cond_len, 0, stream)
                                : bwd_launch<64, 1, 0>(qkv, dout, lse, delta, dqkv, nullptr, B, N, heads, scale, cond_len, round_out, stream);
  return out_half ? bwd_launch<32, 1, 1>(qkv, dout, lse, delta, dqkv, out_scale, B, N, heads, scale, cond_len, 0, stream)
                  : bwd_launch<32, 1, 0>(qkv, dout, lse, delta, dqkv, nullptr, B, N, heads, scale, cond_len, round_out, stream);
}

}  // namespace b200

using namespace b200;

extern "C" int b200vq_attention_exact_fwd(const float* qkv, float* out, float* lse, int B, int N, int heads, int dh, float scale,
                                          void* streamv) {
  return attention_exact_forward(qkv, out, lse, B, N, heads, dh, scale, -1, static_cast<cudaStream_t>(streamv));
}

extern "C" int b200vq_attention_exact_bwd(const float* qkv, const float* out, const float* lse, const float* dout, float* dqkv,
                                          float* delta, int B, int N, int heads, int dh, float scale, void* streamv) {
  return attention_exact_backward(qkv, out, lse, dout, dqkv, delta, B, N, heads, dh, scale, -1, static_cast<cudaStream_t>(streamv));
}
