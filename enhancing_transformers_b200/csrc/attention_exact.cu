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
#include <type_traits>

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
// row pitch (floats) of a staged tile: 16 bytes of padding per row
template <int DH> struct Pitch { static constexpr int LDS = DH + 4; };
__device__ __forceinline__ void cpa16(void* dst, const void* src, bool valid) {
  const int sz = valid ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(dst)), "l"(src), "r"(sz) : "memory");
}
__device__ __forceinline__ void cpa_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cpa_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// stage a [ROWS x DH] tile (row stride ld floats in global) into smem with row pitch Pitch::LDS;
// rows >= nvalid are zero-filled
template <int DH, int ROWS, int THREADS>
__device__ __forceinline__ void load_tile(float* s, const float* g, long long ld, int row0, int nvalid, int tid) {
  constexpr int V = DH / 4;   // 16-byte chunks per row
  constexpr int LDS = Pitch<DH>::LDS;
#pragma unroll
  for (int i = tid; i < ROWS * V; i += THREADS) {
    const int r = i / V, c = (i % V) * 4;
    const bool ok = row0 + r < nvalid;
    cpa16(s + r * LDS + c, g + (long long)(ok ? row0 + r : 0) * ld + c, ok);
  }
}

// A-operand fragments of a 16 x DH row block read straight from global memory (row stride ld)
template <int DH>
__device__ __forceinline__ void load_a_frags(uint32_t (&f)[DH / 8][4], const float* base, long long ld, int row_lo, int nvalid,
                                             int lane) {
  const int g = lane >> 2, t = lane & 3;
  const int r0 = row_lo + g, r1 = row_lo + g + 8;
  const float* p0 = base + (long long)(r0 < nvalid ? r0 : 0) * ld;
  const float* p1 = base + (long long)(r1 < nvalid ? r1 : 0) * ld;
  const bool ok0 = r0 < nvalid, ok1 = r1 < nvalid;
#pragma unroll
  for (int k = 0; k < DH / 8; ++k) {
    f[k][0] = ok0 ? ldbits(p0 + k * 8 + t) : 0u;
    f[k][1] = ok1 ? ldbits(p1 + k * 8 + t) : 0u;
    f[k][2] = ok0 ? ldbits(p0 + k * 8 + t + 4) : 0u;
    f[k][3] = ok1 ? ldbits(p1 + k * 8 + t + 4) : 0u;
  }
}

// A warp's resident operand: the 16 rows x DH (of Q, K, V or dO) that every product of the kernel multiplies from the
// left.  load() fetches the CTA's WARPS x 16 rows from row0 on, frag() gives the A fragment of k-step k.
// DH <= 64: fragments in registers (DH/2 per operand), read once from global memory.
template <int DH> struct RegRows {
  static constexpr bool kStaged = false;
  static constexpr int kSmemRows = 0;   // shared-memory rows per warp
  uint32_t f[DH / 8][4];
  template <int WARPS>
  __device__ __forceinline__ void load(float*, const float* g, long long ld, int row0, int nvalid, int tid) {
    load_a_frags<DH>(f, g, ld, row0 + (tid >> 5) * 16, nvalid, tid & 31);
  }
  __device__ __forceinline__ void frag(uint32_t (&a)[4], int k, int) const {
    a[0] = f[k][0]; a[1] = f[k][1]; a[2] = f[k][2]; a[3] = f[k][3];
  }
};
// DH > 64: the fragments would no longer fit beside the accumulators, so the CTA stages its rows in shared memory
// (cp.async, in the first commit group) and each k-step reads its fragment there, the way the streamed tiles' B
// fragments are read.
template <int DH> struct SmemRows {
  static constexpr bool kStaged = true;
  static constexpr int kSmemRows = 16;
  const float* rows;   // the warp's 16 rows
  template <int WARPS>
  __device__ __forceinline__ void load(float* s, const float* g, long long ld, int row0, int nvalid, int tid) {
    load_tile<DH, WARPS * 16, WARPS * 32>(s, g, ld, row0, nvalid, tid);
    rows = s + (tid >> 5) * 16 * Pitch<DH>::LDS;
  }
  __device__ __forceinline__ void frag(uint32_t (&a)[4], int k, int lane) const {
    constexpr int LDS = Pitch<DH>::LDS;
    const float* p = rows + (lane >> 2) * LDS + k * 8 + (lane & 3);
    a[0] = ldbits(p); a[1] = ldbits(p + 8 * LDS); a[2] = ldbits(p + 4); a[3] = ldbits(p + 8 * LDS + 4);
  }
};

// Everything that depends on the head size alone: where the resident operand lives and the CTA shape.
//   DH <= 64: forward 8 warps streaming 64-key tiles; backward 4 warps x 16 rows streaming 64-row tiles.
//   DH >  64: 8 warps x 16 rows everywhere, one CTA per SM; backward 32-row tiles, which keep the key side's score, dP
//             and dS tiles at 16 registers each beside the 2 x DH/2 registers of dK and dV.
// Shared memory at DH 128: 384 padded rows of 528 bytes = 198 KB per CTA.
template <int DH> struct AttnShape {
  using Rows = std::conditional_t<(DH > 64), SmemRows<DH>, RegRows<DH>>;
  static constexpr int kFwdWarps = 8, kFwdTile = 64;
  static constexpr int kBwdWarps = DH > 64 ? 8 : 4, kBwdTile = DH > 64 ? 32 : 64;
  static constexpr int kMinBlocks = DH > 64 ? 1 : 0;   // __launch_bounds__ minimum CTAs per SM, 0 = none
  // DH > 64 serves stage 2 only (check_problem rejects cond < 0 there), so its kernels compile the mask in
  // unconditionally rather than testing cond at run time
  static constexpr bool kMaskedOnly = DH > 64;
  // staged resident rows, then the double-buffered streamed tiles (and, key side, LSE and delta of each buffer)
  static constexpr size_t kFwdSmem = (kFwdWarps * Rows::kSmemRows + 4 * kFwdTile) * Pitch<DH>::LDS * sizeof(float);
  static constexpr size_t kDqSmem = (2 * kBwdWarps * Rows::kSmemRows + 4 * kBwdTile) * Pitch<DH>::LDS * sizeof(float);
  static constexpr size_t kDkvSmem = kDqSmem + 4 * kBwdTile * sizeof(float);
};

// acc[nt] (16 x 8 each, nt over NT column tiles) += A(16 x DH, the resident rows) . T^T where T is a smem tile
// [NT*8][DH+4] whose rows are the output columns ("K-like" read: b = T[n0+g][k0+t])
template <int DH, int PASSES, int NT, class Rows>
__device__ __forceinline__ void mma_rows_x_tileT(float (&acc)[NT][4], const Rows& a, const float* Ts, int lane) {
  constexpr int LDS = Pitch<DH>::LDS;
  const int g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int k = 0; k < DH / 8; ++k) {
    uint32_t af[4];
    a.frag(af, k, lane);
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
      const float* p = Ts + (nt * 8 + g) * LDS + k * 8 + t;
      mma_x<PASSES>(acc[nt], af, ldbits(p), ldbits(p + 4));
    }
  }
}
// acc[dt] (16 x 8 each, dt over DH/8 column tiles) += P(16 x NT*8, given as accumulator-layout
// fragments, full fp32) . T where T is a smem tile [NT*8][DH+4] whose rows are the
// contraction index ("V-like" read).  Accumulator columns (2t, 2t+1) of each 8-wide tile serve
// as k-slots (t, t+4), so the tile rows are read in the matching order 2t, 2t+1.
template <int DH, int PASSES, int NT>
__device__ __forceinline__ void mma_p_x_tile(float (&acc)[DH / 8][4], const uint32_t (&p)[NT][4], const float* Ts, int lane) {
  constexpr int LDS = Pitch<DH>::LDS;
  const int g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int kt = 0; kt < NT; ++kt)
#pragma unroll
    for (int dt = 0; dt < DH / 8; ++dt) {
      const float* q = Ts + (kt * 8 + 2 * t) * LDS + dt * 8 + g;
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

// ---------------------------------------------------------------------------------------------
// forward: grid (ceil(N/128), heads, B), 256 threads = 8 warps x 16 query rows; resident Q, streamed 64-key tiles
// ---------------------------------------------------------------------------------------------
template <int DH, int PASSES, int OUT16>
__global__ void __launch_bounds__(AttnShape<DH>::kFwdWarps * 32, AttnShape<DH>::kMinBlocks)
attn_fwd_kernel(const float* __restrict__ qkv, void* __restrict__ out, float* __restrict__ lse, int N, int heads, float scale,
                int cond, int round_out) {
  using Shape = AttnShape<DH>;
  constexpr int WARPS = Shape::kFwdWarps, ROWS = WARPS * 16, KB = Shape::kFwdTile;
  constexpr int LDS = Pitch<DH>::LDS;
  constexpr int TILE = KB * LDS;
  extern __shared__ __align__(16) uint8_t sm_raw[];   // [Q rows], K[2][TILE], V[2][TILE]
  float* Qs = reinterpret_cast<float*>(sm_raw);
  float* Ks = Qs + WARPS * Shape::Rows::kSmemRows * LDS;
  float* Vs = Ks + 2 * TILE;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3;
  const int h = blockIdx.y, b = blockIdx.z;
  const int inner = heads * DH;
  const long long ld = 3ll * inner;
  const float* qbase = qkv + (long long)b * N * ld + h * DH;
  const float* kbase = qbase + inner;
  const float* vbase = qbase + 2 * inner;
  const int q0 = blockIdx.x * ROWS + warp * 16;
  const float c = scale * kLog2e;

  // register fragments are fetched first, so their global loads overlap the set-up below; staged rows are issued with
  // the first K and V tiles
  typename Shape::Rows qr;
  if constexpr (!Shape::Rows::kStaged) qr.template load<WARPS>(Qs, qbase, ld, blockIdx.x * ROWS, N, tid);

  float o[DH / 8][4];
#pragma unroll
  for (int i = 0; i < DH / 8; ++i) { o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f; }
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;

  // cond >= 0: stage-2 mask (reference stage2/layers.py:43-48,83-85): query q sees key k iff k <= max(q, cond - 1)
  // (causal, with the first `cond` condition tokens fully visible to each other).  Key 0 is visible to every row, so the
  // running maximum is finite after the first tile and fully masked tiles contribute exp2(-inf) = 0.
  const bool masked = Shape::kMaskedOnly || cond >= 0;
  const int lim0 = masked ? max(q0 + g, cond - 1) : N, lim1 = masked ? max(q0 + g + 8, cond - 1) : N;
  int ntiles = (N + KB - 1) / KB;
  if (masked) ntiles = min(ntiles, max(min(N - 1, (int)blockIdx.x * ROWS + ROWS - 1), cond - 1) / KB + 1);   // tiles past the CTA's last visible key
  if constexpr (Shape::Rows::kStaged) qr.template load<WARPS>(Qs, qbase, ld, blockIdx.x * ROWS, N, tid);
  load_tile<DH, KB, WARPS * 32>(Ks, kbase, ld, 0, N, tid);
  load_tile<DH, KB, WARPS * 32>(Vs, vbase, ld, 0, N, tid);
  cpa_commit();
  for (int j = 0; j < ntiles; ++j) {
    const int buf = j & 1;
    cpa_wait<0>();
    __syncthreads();
    if (j + 1 < ntiles) {
      load_tile<DH, KB, WARPS * 32>(Ks + (buf ^ 1) * TILE, kbase, ld, (j + 1) * KB, N, tid);
      load_tile<DH, KB, WARPS * 32>(Vs + (buf ^ 1) * TILE, vbase, ld, (j + 1) * KB, N, tid);
      cpa_commit();
    }
    float s[KB / 8][4];
#pragma unroll
    for (int i = 0; i < KB / 8; ++i) { s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f; }
    mma_rows_x_tileT<DH, PASSES, KB / 8>(s, qr, Ks + buf * TILE, lane);
    // Keys past N, and under the mask keys past a row's limit, score -inf.  The one-pass and two-pass forms give the same
    // values; each is the one its head sizes compile best with (the two-pass form costs the 3xTF32 forward at DH 128
    // about 2 %, the one-pass form adds registers at DH 32).
    if constexpr (Shape::kMaskedOnly) {
      if ((j + 1) * KB > N || j * KB + KB - 1 > min(lim0, lim1)) {
#pragma unroll
        for (int nt = 0; nt < KB / 8; ++nt) {
          const int key = j * KB + nt * 8 + 2 * t;
          if (key >= N || key > lim0) s[nt][0] = -INFINITY;
          if (key + 1 >= N || key + 1 > lim0) s[nt][1] = -INFINITY;
          if (key >= N || key > lim1) s[nt][2] = -INFINITY;
          if (key + 1 >= N || key + 1 > lim1) s[nt][3] = -INFINITY;
        }
      }
    } else {
      if ((j + 1) * KB > N) {
#pragma unroll
        for (int nt = 0; nt < KB / 8; ++nt) {
          const int key = j * KB + nt * 8 + 2 * t;
          if (key >= N) { s[nt][0] = -INFINITY; s[nt][2] = -INFINITY; }
          if (key + 1 >= N) { s[nt][1] = -INFINITY; s[nt][3] = -INFINITY; }
        }
      }
      if (masked && j * KB + KB - 1 > min(lim0, lim1)) {
#pragma unroll
        for (int nt = 0; nt < KB / 8; ++nt) {
          const int key = j * KB + nt * 8 + 2 * t;
          if (key > lim0) s[nt][0] = -INFINITY;
          if (key + 1 > lim0) s[nt][1] = -INFINITY;
          if (key > lim1) s[nt][2] = -INFINITY;
          if (key + 1 > lim1) s[nt][3] = -INFINITY;
        }
      }
    }
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int nt = 0; nt < KB / 8; ++nt) {
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
    uint32_t pf[KB / 8][4];
    const float mc0 = m0 * c, mc1 = m1 * c;
#pragma unroll
    for (int nt = 0; nt < KB / 8; ++nt) {
      const float p0 = exp2f(s[nt][0] * c - mc0), p1 = exp2f(s[nt][1] * c - mc0);
      const float p2 = exp2f(s[nt][2] * c - mc1), p3 = exp2f(s[nt][3] * c - mc1);
      l0 += p0 + p1; l1 += p2 + p3;
      acc_to_a<PASSES>(pf[nt], p0, p1, p2, p3);
    }
    mma_p_x_tile<DH, PASSES, KB / 8>(o, pf, Vs + buf * TILE, lane);
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
// backward, key side: grid (ceil(N/ROWS), heads, B), WARPS x 16 keys per CTA; resident K and V, streamed KB-query tiles
// of Q, dO, LSE and delta.  Works on transposed score tiles S^T[key, query] so that P^T / dS^T come out of the tensor
// cores already in A-operand position for dV += P^T dO and dK += dS^T Q.
// ---------------------------------------------------------------------------------------------
template <int DH, int PASSES, int OUT16>
__global__ void __launch_bounds__(AttnShape<DH>::kBwdWarps * 32, AttnShape<DH>::kMinBlocks)
attn_bwd_dkv_kernel(const float* __restrict__ qkv, const float* __restrict__ dout, const float* __restrict__ lse,
                    const float* __restrict__ delta, void* __restrict__ dqkv, const float* __restrict__ out_scale, int N,
                    int heads, float scale, int cond, int round_out) {
  using Shape = AttnShape<DH>;
  constexpr int WARPS = Shape::kBwdWarps, ROWS = WARPS * 16, KB = Shape::kBwdTile, NT = KB / 8;
  constexpr int LDS = Pitch<DH>::LDS;
  constexpr int TILE = KB * LDS;
  extern __shared__ __align__(16) uint8_t sm_raw[];   // [K rows], [V rows], Q[2][TILE], dO[2][TILE], lse[2][KB], delta[2][KB]
  float* Kr = reinterpret_cast<float*>(sm_raw);
  float* Vr = Kr + WARPS * Shape::Rows::kSmemRows * LDS;
  float* Qs = Vr + WARPS * Shape::Rows::kSmemRows * LDS;
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
  const int k0 = blockIdx.x * ROWS + warp * 16;
  const float c = scale * kLog2e;

  typename Shape::Rows kr, vr;
  kr.template load<WARPS>(Kr, qbase + inner, ld, blockIdx.x * ROWS, N, tid);
  vr.template load<WARPS>(Vr, qbase + 2 * inner, ld, blockIdx.x * ROWS, N, tid);
  float dk[DH / 8][4], dv[DH / 8][4];
#pragma unroll
  for (int i = 0; i < DH / 8; ++i) { dk[i][0] = dk[i][1] = dk[i][2] = dk[i][3] = 0.f; dv[i][0] = dv[i][1] = dv[i][2] = dv[i][3] = 0.f; }

  auto stage = [&](int j, int buf) {
    load_tile<DH, KB, WARPS * 32>(Qs + buf * TILE, qbase, ld, j * KB, N, tid);
    load_tile<DH, KB, WARPS * 32>(Ds + buf * TILE, dobase, inner, j * KB, N, tid);
    if (tid < KB) {
      const int q = j * KB + tid;
      Ls[buf * KB + tid] = q < N ? lb[q] * kLog2e : INFINITY;   // +inf -> P = 0 for padded queries
      Es[buf * KB + tid] = q < N ? eb[q] : 0.f;
    }
    cpa_commit();
  };
  const int ntiles = (N + KB - 1) / KB;
  // stage-2 mask: key k receives from query q iff k <= max(q, cond - 1).  A CTA whose first key is at or past `cond`
  // starts at the query tile of its own first key.
  const bool masked = Shape::kMaskedOnly || cond >= 0;
  const int jbeg = (masked && (int)blockIdx.x * ROWS >= cond) ? (int)blockIdx.x * (ROWS / KB) : 0;
  const int kr0 = k0 + g, kr1 = k0 + g + 8;
  stage(jbeg, 0);
  for (int j = jbeg; j < ntiles; ++j) {
    const int buf = (j - jbeg) & 1;
    cpa_wait<0>();
    __syncthreads();
    if (j + 1 < ntiles) stage(j + 1, buf ^ 1);
    const float* Q = Qs + buf * TILE;
    const float* dO = Ds + buf * TILE;
    float s[NT][4];
#pragma unroll
    for (int i = 0; i < NT; ++i) { s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f; }
    mma_rows_x_tileT<DH, PASSES, NT>(s, kr, Q, lane);                // S^T = K Q^T
    uint32_t pf[NT][4];
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
      const float la = Ls[buf * KB + nt * 8 + 2 * t], lbb = Ls[buf * KB + nt * 8 + 2 * t + 1];
      s[nt][0] = exp2f(s[nt][0] * c - la);  s[nt][1] = exp2f(s[nt][1] * c - lbb);
      s[nt][2] = exp2f(s[nt][2] * c - la);  s[nt][3] = exp2f(s[nt][3] * c - lbb);
      if (masked) {
        const int va = max(j * KB + nt * 8 + 2 * t, cond - 1), vb = max(j * KB + nt * 8 + 2 * t + 1, cond - 1);   // last key each query sees
        if (kr0 > va) s[nt][0] = 0.f;
        if (kr0 > vb) s[nt][1] = 0.f;
        if (kr1 > va) s[nt][2] = 0.f;
        if (kr1 > vb) s[nt][3] = 0.f;
      }
      acc_to_a<PASSES>(pf[nt], s[nt][0], s[nt][1], s[nt][2], s[nt][3]);
    }
    mma_p_x_tile<DH, PASSES, NT>(dv, pf, dO, lane);                  // dV += P^T dO
    float dp[NT][4];
#pragma unroll
    for (int i = 0; i < NT; ++i) { dp[i][0] = dp[i][1] = dp[i][2] = dp[i][3] = 0.f; }
    mma_rows_x_tileT<DH, PASSES, NT>(dp, vr, dO, lane);              // dP^T = V dO^T
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
      const float ea = Es[buf * KB + nt * 8 + 2 * t], ebb = Es[buf * KB + nt * 8 + 2 * t + 1];
      acc_to_a<PASSES>(pf[nt], s[nt][0] * (dp[nt][0] - ea), s[nt][1] * (dp[nt][1] - ebb), s[nt][2] * (dp[nt][2] - ea),
                       s[nt][3] * (dp[nt][3] - ebb));
    }
    mma_p_x_tile<DH, PASSES, NT>(dk, pf, Q, lane);                   // dK += dS^T Q
  }
  const int r0 = k0 + g, r1 = k0 + g + 8;
  const long long dkb = (long long)b * N * ld + inner + h * DH;
  const long long dvb = dkb + inner;
  // fp16 output: the gradient scale it travels with.  DH > 64 stores fp32 only, so vm folds to 1 there.
  const float vm = (OUT16 || DH <= 64) && out_scale ? __ldg(out_scale) : 1.f;
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
// backward, query side: grid (ceil(N/ROWS), heads, B), WARPS x 16 queries per CTA; resident Q and dO, streamed KB-key
// tiles of K and V
// ---------------------------------------------------------------------------------------------
template <int DH, int PASSES, int OUT16>
__global__ void __launch_bounds__(AttnShape<DH>::kBwdWarps * 32, AttnShape<DH>::kMinBlocks)
attn_bwd_dq_kernel(const float* __restrict__ qkv, const float* __restrict__ dout, const float* __restrict__ lse,
                   const float* __restrict__ delta, void* __restrict__ dqkv, const float* __restrict__ out_scale, int N,
                   int heads, float scale, int cond, int round_out) {
  using Shape = AttnShape<DH>;
  constexpr int WARPS = Shape::kBwdWarps, ROWS = WARPS * 16, KB = Shape::kBwdTile, NT = KB / 8;
  constexpr int LDS = Pitch<DH>::LDS;
  constexpr int TILE = KB * LDS;
  extern __shared__ __align__(16) uint8_t sm_raw[];   // [Q rows], [dO rows], K[2][TILE], V[2][TILE]
  float* Qr = reinterpret_cast<float*>(sm_raw);
  float* Dr = Qr + WARPS * Shape::Rows::kSmemRows * LDS;
  float* Ks = Dr + WARPS * Shape::Rows::kSmemRows * LDS;
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
  const int q0 = blockIdx.x * ROWS + warp * 16;
  const float c = scale * kLog2e;
  const int r0 = q0 + g, r1 = q0 + g + 8;
  const float* lb = lse + ((long long)b * heads + h) * N;
  const float* eb = delta + ((long long)b * heads + h) * N;
  const float lse0 = r0 < N ? lb[r0] * kLog2e : INFINITY, lse1 = r1 < N ? lb[r1] * kLog2e : INFINITY;
  const float e0 = r0 < N ? eb[r0] : 0.f, e1 = r1 < N ? eb[r1] : 0.f;

  typename Shape::Rows qr, dr;
  qr.template load<WARPS>(Qr, qbase, ld, blockIdx.x * ROWS, N, tid);
  dr.template load<WARPS>(Dr, dobase, inner, blockIdx.x * ROWS, N, tid);
  float dq[DH / 8][4];
#pragma unroll
  for (int i = 0; i < DH / 8; ++i) { dq[i][0] = dq[i][1] = dq[i][2] = dq[i][3] = 0.f; }

  const bool masked = Shape::kMaskedOnly || cond >= 0;
  const int lim0 = masked ? max(r0, cond - 1) : N, lim1 = masked ? max(r1, cond - 1) : N;
  int ntiles = (N + KB - 1) / KB;
  if (masked) ntiles = min(ntiles, max(min(N - 1, (int)blockIdx.x * ROWS + ROWS - 1), cond - 1) / KB + 1);
  load_tile<DH, KB, WARPS * 32>(Ks, kbase, ld, 0, N, tid);
  load_tile<DH, KB, WARPS * 32>(Vs, vbase, ld, 0, N, tid);
  cpa_commit();
  for (int j = 0; j < ntiles; ++j) {
    const int buf = j & 1;
    cpa_wait<0>();
    __syncthreads();
    if (j + 1 < ntiles) {
      load_tile<DH, KB, WARPS * 32>(Ks + (buf ^ 1) * TILE, kbase, ld, (j + 1) * KB, N, tid);
      load_tile<DH, KB, WARPS * 32>(Vs + (buf ^ 1) * TILE, vbase, ld, (j + 1) * KB, N, tid);
      cpa_commit();
    }
    float s[NT][4], dp[NT][4];
#pragma unroll
    for (int i = 0; i < NT; ++i) { s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f; dp[i][0] = dp[i][1] = dp[i][2] = dp[i][3] = 0.f; }
    mma_rows_x_tileT<DH, PASSES, NT>(s, qr, Ks + buf * TILE, lane);     // S = Q K^T
    mma_rows_x_tileT<DH, PASSES, NT>(dp, dr, Vs + buf * TILE, lane);    // dP = dO V^T
    uint32_t pf[NT][4];
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
      const int key = j * KB + nt * 8 + 2 * t;
      const bool ka = key < N, kb = key + 1 < N;
      const float p0 = (ka && key <= lim0) ? exp2f(s[nt][0] * c - lse0) : 0.f, p1 = (kb && key + 1 <= lim0) ? exp2f(s[nt][1] * c - lse0) : 0.f;
      const float p2 = (ka && key <= lim1) ? exp2f(s[nt][2] * c - lse1) : 0.f, p3 = (kb && key + 1 <= lim1) ? exp2f(s[nt][3] * c - lse1) : 0.f;
      acc_to_a<PASSES>(pf[nt], p0 * (dp[nt][0] - e0), p1 * (dp[nt][1] - e0), p2 * (dp[nt][2] - e1), p3 * (dp[nt][3] - e1));
    }
    mma_p_x_tile<DH, PASSES, NT>(dq, pf, Ks + buf * TILE, lane);        // dQ += dS K
  }
  const long long dqb = (long long)b * N * ld + h * DH;
  const float qm = scale * ((OUT16 || DH <= 64) && out_scale ? __ldg(out_scale) : 1.f);
#pragma unroll
  for (int dt = 0; dt < DH / 8; ++dt) {
    if (r0 < N) store2<OUT16>(dqkv, dqb + (long long)r0 * ld + dt * 8 + 2 * t, dq[dt][0] * qm, dq[dt][1] * qm, round_out);
    if (r1 < N) store2<OUT16>(dqkv, dqb + (long long)r1 * ld + dt * 8 + 2 * t, dq[dt][2] * qm, dq[dt][3] * qm, round_out);
  }
}

// ---------------------------------------------------------------------------------------------
template <int DH, int PASSES, int OUT16>
static int fwd_launch(const float* qkv, void* out, float* lse, int B, int N, int heads, float scale, int cond, int round_out,
                      cudaStream_t s) {
  using Shape = AttnShape<DH>;
  constexpr int rows = Shape::kFwdWarps * 16;
  auto kern = attn_fwd_kernel<DH, PASSES, OUT16>;
  B200_CONFIGURE_SMEM_ONCE(kern, Shape::kFwdSmem);
  kern<<<dim3((N + rows - 1) / rows, heads, B), Shape::kFwdWarps * 32, Shape::kFwdSmem, s>>>(qkv, out, lse, N, heads, scale, cond,
                                                                                            round_out);
  B200_LAUNCH_OK("attn_fwd_kernel");
  return 0;
}

template <int DH, int PASSES, int OUT16>
static int bwd_launch(const float* qkv, const float* dout, const float* lse, const float* delta, void* dqkv, const float* out_scale,
                      int B, int N, int heads, float scale, int cond, int round_out, cudaStream_t s) {
  using Shape = AttnShape<DH>;
  constexpr int rows = Shape::kBwdWarps * 16;
  auto k1 = attn_bwd_dkv_kernel<DH, PASSES, OUT16>;
  auto k2 = attn_bwd_dq_kernel<DH, PASSES, OUT16>;
  B200_CONFIGURE_SMEM_ONCE(k1, Shape::kDkvSmem);
  B200_CONFIGURE_SMEM_ONCE(k2, Shape::kDqSmem);
  const dim3 grid((N + rows - 1) / rows, heads, B);
  k1<<<grid, Shape::kBwdWarps * 32, Shape::kDkvSmem, s>>>(qkv, dout, lse, delta, dqkv, out_scale, N, heads, scale, cond, round_out);
  B200_LAUNCH_OK("attn_bwd_dkv_kernel");
  k2<<<grid, Shape::kBwdWarps * 32, Shape::kDqSmem, s>>>(qkv, dout, lse, delta, dqkv, out_scale, N, heads, scale, cond, round_out);
  B200_LAUNCH_OK("attn_bwd_dq_kernel");
  return 0;
}

template <int DH_, int PASSES_, int OUT16_> struct Form { static constexpr int DH = DH_, PASSES = PASSES_, OUT16 = OUT16_; };
// f(Form<DH, PASSES, OUT16>{}) for the one instantiated form: at head sizes 32 and 64 tf32 with fp32 or fp16 output and
// 3xTF32; at 96 and 128 tf32 and 3xTF32.  The arguments have passed check_problem.
template <class F>
static int with_form(int dh, int passes, int out_half, F&& f) {
  if (out_half) return dh == 64 ? f(Form<64, 1, 1>{}) : f(Form<32, 1, 1>{});
  if (passes == 3) {
    switch (dh) {
      case 32: return f(Form<32, 3, 0>{});
      case 64: return f(Form<64, 3, 0>{});
      case 96: return f(Form<96, 3, 0>{});
      default: return f(Form<128, 3, 0>{});
    }
  }
  switch (dh) {
    case 32: return f(Form<32, 1, 0>{});
    case 64: return f(Form<64, 1, 0>{});
    case 96: return f(Form<96, 1, 0>{});
    default: return f(Form<128, 1, 0>{});
  }
}

static int check_problem(const float* qkv, int B, int N, int heads, int dh, int passes, int out_half, int cond_len) {
  B200_CHECK_ARG(B > 0 && N > 0 && heads > 0, "attention: empty problem");
  B200_CHECK_ARG(dh == 32 || dh == 64 || ((dh == 96 || dh == 128) && cond_len >= 0 && !out_half),
                 "attention: head size must be 32 or 64, or 96 or 128 with the stage-2 mask and fp32 output (got %d)", dh);
  B200_CHECK_ARG(passes == 1 || (passes == 3 && !out_half), "attention: %d passes (1, or 3 with fp32 output)", passes);
  B200_CHECK_ARG(B <= 65535 && heads <= 65535, "attention: grid too large");
  B200_CHECK_ARG(cond_len <= N, "attention: cond_len %d exceeds the sequence length %d", cond_len, N);
  B200_CHECK_ARG((reinterpret_cast<uintptr_t>(qkv) & 15) == 0, "attention: qkv must be 16-byte aligned");
  return 0;
}

int attention_forward(int dh, int passes, int out_half, int cond_len, int round_out, const float* qkv, void* out, float* lse, int B,
                      int N, int heads, float scale, cudaStream_t stream) {
  if (int rc = check_problem(qkv, B, N, heads, dh, passes, out_half, cond_len)) return rc;
  return with_form(dh, passes, out_half, [&](auto form) {
    using F = decltype(form);
    return fwd_launch<F::DH, F::PASSES, F::OUT16>(qkv, out, lse, B, N, heads, scale, cond_len, F::PASSES == 1 ? round_out : 0,
                                                  stream);
  });
}

int attention_backward(int dh, int passes, int dqkv_half, int cond_len, int round_out, const float* qkv, const void* o, int o_half,
                       const float* lse, const float* dout, float* delta, void* dqkv, const float* out_scale, int B, int N,
                       int heads, float scale, cudaStream_t stream) {
  if (int rc = check_problem(qkv, B, N, heads, dh, passes, dqkv_half, cond_len)) return rc;
  B200_CHECK_ARG((reinterpret_cast<uintptr_t>(dout) & 15) == 0, "attention: dout must be 16-byte aligned");
  if (int rc = attention_delta(o, o_half, dout, 0, delta, B, N, heads, dh, stream)) return rc;
  return with_form(dh, passes, dqkv_half, [&](auto form) {
    using F = decltype(form);
    return bwd_launch<F::DH, F::PASSES, F::OUT16>(qkv, dout, lse, delta, dqkv, F::OUT16 ? out_scale : nullptr, B, N, heads, scale,
                                                  cond_len, F::PASSES == 1 ? round_out : 0, stream);
  });
}

}  // namespace b200

using namespace b200;

extern "C" int b200vq_attention_exact_fwd(const float* qkv, float* out, float* lse, int B, int N, int heads, int dh, float scale,
                                          void* streamv) {
  B200_CHECK_ARG(B > 0 && N > 0 && heads > 0, "attention: empty problem");
  B200_CHECK_ARG(dh == 64 || dh == 32, "attention: dim_head must be 32 or 64 (got %d)", dh);
  return attention_forward(dh, 3, 0, -1, 0, qkv, out, lse, B, N, heads, scale, static_cast<cudaStream_t>(streamv));
}

extern "C" int b200vq_attention_exact_bwd(const float* qkv, const float* out, const float* lse, const float* dout, float* dqkv,
                                          float* delta, int B, int N, int heads, int dh, float scale, void* streamv) {
  B200_CHECK_ARG(B > 0 && N > 0 && heads > 0, "attention: empty problem");
  B200_CHECK_ARG(dh == 64 || dh == 32, "attention: dim_head must be 32 or 64 (got %d)", dh);
  return attention_backward(dh, 3, 0, -1, 0, qkv, out, 0, lse, dout, delta, dqkv, nullptr, B, N, heads, scale,
                            static_cast<cudaStream_t>(streamv));
}
