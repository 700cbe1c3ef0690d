// Fused vector-quantiser kernels (reference enhancing/modules/stage1/quantizers.py:38-92).
//
//   vq_prep : normalise the codebook once per call (quantizers.py:76), emit it transposed
//             [D][K] so the lookup streams it with coalesced 16-byte loads, plus |e_n|^2.
//   vq_fwd  : per 128-token tile: normalise z (:75), distance d = (|z|^2 + |e|^2) - 2 z.e in
//             the reference's association (:78-80) in exact fp32 FMA arithmetic, argmin with
//             lowest-index tie-break (:82), gather + normalise the winner (:85-86), loss partial
//             sums (:89-90), straight-through value z + (q - z) (:60-61); the residual mode's
//             depth loop (:42-57) runs inside the kernel.  The [tokens, n_embed] distance
//             matrix the reference materialises never exists.
//   vq_loss : deterministic reduction of the per-CTA partial sums into the scalar loss.
//   EMA codebook (EMAVectorQuantizer): vq_fwd with kStats != 0 also gathers, per code k, the count n_k and the sum s_k of
//             the vectors the lookup compared (a per-CTA shared-memory table flushed once per depth, or per-entry rows
//             summed by scatter_det.cu in a fixed order); vq_ema_* apply the update to the codebook on the device.
//   vq_bwd  : closed-form gradients (see oracle/vitvq_oracle.py:vq_backward_np).  The codebook gradient is scattered with
//             float atomics (vq_bwd_kernel) or, on request, stored per entry and summed in a fixed order
//             (vq_bwd_contrib_kernel + scatter_det.cu): bit-reproducible.
#include "../../include/b200vq.h"
#include "common.cuh"
#include "scatter_det.cuh"

namespace b200 {

constexpr int kVqD = 32;          // embed_dim of every shipped config (configs/*.yaml quantizer.embed_dim); wider: *_wide_kernel
constexpr int kVqTileM = 128;     // tokens per CTA
constexpr int kVqTileN = 128;     // codes per smem chunk
constexpr int kVqThreads = 256;
constexpr int kVqMaxDepth = 8;
constexpr float kNormEps = 1e-12f;

// ---------------------------------------------------------------------------------------------
__global__ void vq_prep_kernel(const float* __restrict__ E, float* __restrict__ EnT, float* __restrict__ ee, int K, int use_norm) {
  // 8 lanes per code row, one float4 each
  const int gid = blockIdx.x * blockDim.x + threadIdx.x;
  const int code = gid >> 3, part = gid & 7;
  float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
  if (code < K) v = *reinterpret_cast<const float4*>(E + (size_t)code * kVqD + part * 4);
  float s = v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
  s += __shfl_xor_sync(0xffffffffu, s, 1);
  s += __shfl_xor_sync(0xffffffffu, s, 2);
  s += __shfl_xor_sync(0xffffffffu, s, 4);
  const float nrm = use_norm ? fmaxf(sqrtf(s), kNormEps) : 1.f;   // use_norm=False: norm is the identity (quantizers.py:24)
  if (use_norm) { v.x /= nrm; v.y /= nrm; v.z /= nrm; v.w /= nrm; }   // true division, as F.normalize does
  float s2 = v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
  s2 += __shfl_xor_sync(0xffffffffu, s2, 1);
  s2 += __shfl_xor_sync(0xffffffffu, s2, 2);
  s2 += __shfl_xor_sync(0xffffffffu, s2, 4);
  if (code < K) {
    EnT[(size_t)(part * 4 + 0) * K + code] = v.x;
    EnT[(size_t)(part * 4 + 1) * K + code] = v.y;
    EnT[(size_t)(part * 4 + 2) * K + code] = v.z;
    EnT[(size_t)(part * 4 + 3) * K + code] = v.w;
    if (part == 0) ee[code] = s2;
  }
}

__device__ __forceinline__ float group8_sum(float s) {
  s += __shfl_xor_sync(0xffffffffu, s, 1);
  s += __shfl_xor_sync(0xffffffffu, s, 2);
  s += __shfl_xor_sync(0xffffffffu, s, 4);
  return s;
}
__device__ __forceinline__ float dot4(const float4& a, const float4& b) { return a.x * b.x + a.y * b.y + a.z * b.z + a.w * b.w; }
// F.normalize: x / max(|x|, eps).  True division, as ATen does.  use_norm == 0: identity (nrm = 1).
__device__ __forceinline__ float4 normalize8(const float4& v, float& nrm, int use_norm = 1) {
  if (!use_norm) { nrm = 1.f; return v; }
  nrm = fmaxf(sqrtf(group8_sum(dot4(v, v))), kNormEps);
  return make_float4(v.x / nrm, v.y / nrm, v.z / nrm, v.w / nrm);
}
// two independent fp32 FMAs: d.x += a * b.x, d.y += a * b.y, each rounded like a scalar fmaf, so the distances (and
// therefore the argmin) are bit-identical to the scalar loop
__device__ __forceinline__ void ffma2(float2& d, float a, const float2 b) {
  d.x = fmaf(a, b.x, d.x);
  d.y = fmaf(a, b.y, d.y);
}

__device__ __forceinline__ void cp_async16(void* dst, const void* src, bool valid) {
  const uint32_t d = smem_u32(dst);
  const int sz = valid ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(d), "l"(src), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// EMA statistics of one CTA and one depth step.  A CTA looks up 128 tokens per depth, so it meets at most 128 distinct
// codes: a 128-slot open-addressing table keyed by code never overflows.  Counts are integers (order-independent); the
// float sums of kVqStatsAtomic are shared-memory atomics here and one global atomic per (live slot, column) at the flush.
constexpr int kVqStatsOff = 0, kVqStatsAtomic = 1, kVqStatsDeterministic = 2;
constexpr int kVqStatSlots = 128;
struct VqStatTable {
  int keys[kVqStatSlots];
  int cnt[kVqStatSlots];
  float acc[kVqStatSlots][kVqD];
};
__device__ __forceinline__ void vq_stat_clear(VqStatTable& st, int tid) {
  for (int i = tid; i < kVqStatSlots; i += kVqThreads) { st.keys[i] = -1; st.cnt[i] = 0; }
#pragma unroll 1
  for (int i = tid; i < kVqStatSlots * kVqD; i += kVqThreads) (&st.acc[0][0])[i] = 0.f;
}
// every lane of the warp calls this (the slot travels by shuffle); dead tokens (live == false) add nothing
template <int kStats>
__device__ __forceinline__ void vq_stat_add(VqStatTable& st, int code, int part, bool live, const float4& x) {
  int slot = -1;
  if (part == 0 && live) {
    unsigned h = ((unsigned)code * 2654435761u) >> 25;
#pragma unroll 1
    for (int probe = 0; probe < kVqStatSlots; ++probe) {
      const int old = atomicCAS(&st.keys[h], -1, code);
      if (old == -1 || old == code) { slot = (int)h; break; }
      h = (h + 1) & (kVqStatSlots - 1);
    }
    atomicAdd(&st.cnt[slot], 1);
  }
  slot = __shfl_sync(0xffffffffu, slot, (threadIdx.x & 31) & ~7);
  if (kStats == kVqStatsAtomic && slot >= 0) {
    float* dst = &st.acc[slot][part * 4];
    atomicAdd(dst + 0, x.x); atomicAdd(dst + 1, x.y); atomicAdd(dst + 2, x.z); atomicAdd(dst + 3, x.w);
  }
}

// ---------------------------------------------------------------------------------------------
// z [M,32] fp32; EnT [32][K]; ee [K]; E [K,32] (un-normalised codebook, gathered for the winner)
// out [M,32]; idx [M,depth] int64; loss_part [depth][gridDim.x]
// kStats != 0 (EMA statistics): counts [K] int (accumulated); kVqStatsAtomic: sums [K,32] (accumulated);
// kVqStatsDeterministic: contrib [M*depth, 32] receives the compared vector of entry m*depth + t
template <int kStats>
__global__ void __launch_bounds__(kVqThreads, 2)
vq_fwd_kernel(const float* __restrict__ z, const float* __restrict__ EnT, const float* __restrict__ ee,
              const float* __restrict__ E, float* __restrict__ out, long long* __restrict__ idx_out,
              float* __restrict__ loss_part, int M, int K, int depth, int use_norm, int* __restrict__ counts,
              float* __restrict__ sums, float* __restrict__ contrib) {
  extern __shared__ __align__(16) uint8_t vq_smem[];
  float (*zT)[kVqTileM] = reinterpret_cast<float (*)[kVqTileM]>(vq_smem);                       // normalised residual, transposed
  float (*eT)[kVqD][kVqTileN] = reinterpret_cast<float (*)[kVqD][kVqTileN]>(vq_smem + sizeof(float) * kVqD * kVqTileM);  // chunk ring
  float (*ee_s)[kVqTileN] = reinterpret_cast<float (*)[kVqTileN]>(vq_smem + sizeof(float) * (kVqD * kVqTileM + 2 * kVqD * kVqTileN));
  float* zz_s = reinterpret_cast<float*>(ee_s) + 2 * kVqTileN;
  int* best_s = reinterpret_cast<int*>(zz_s + kVqTileM);
  float* red_s = reinterpret_cast<float*>(best_s + kVqTileM);
  // residual / accumulated-code state of the depth loop, parked in shared memory while the distance loop runs: it is only
  // touched in phases A and C, and keeping its 32 registers live across phase B spilled the 8x8 accumulator tile
  float4* park = reinterpret_cast<float4*>(red_s + 8);          // [8][256]: rreg[ps] at ps*256 + tid, acc[ps] at (4+ps)*256 + tid
  VqStatTable* st = reinterpret_cast<VqStatTable*>(park + 8 * kVqThreads);   // kStats != 0 only

  const int tid = threadIdx.x;
  const int m0 = blockIdx.x * kVqTileM;
  // phase A/C mapping: 8 lanes per token, 4 passes of 32 tokens
  const int part = tid & 7;
  // phase B mapping: 16 x 16 threads, 8 tokens x 8 codes each
  const int tx = tid & 15, ty = tid >> 4;

  // residual and accumulated code per (token, 4-float part); z itself is re-read at the end
#pragma unroll
  for (int ps = 0; ps < 4; ++ps) {
    const int tok = m0 + ps * 32 + (tid >> 3);
    park[ps * kVqThreads + tid] = tok < M ? *reinterpret_cast<const float4*>(z + (size_t)tok * kVqD + part * 4) : make_float4(1.f, 0.f, 0.f, 0.f);
    park[(4 + ps) * kVqThreads + tid] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  const int nchunks = (K + kVqTileN - 1) / kVqTileN;
  if constexpr (kStats != kVqStatsOff) vq_stat_clear(*st, tid);   // first used in phase C, after phase B's barriers

  for (int t = 0; t < depth; ++t) {
    // ---- phase A: normalise the residual, stage it transposed -------------------------------
#pragma unroll
    for (int ps = 0; ps < 4; ++ps) {
      float nrm;
      const float4 rn = normalize8(park[ps * kVqThreads + tid], nrm, use_norm);
      const int lt = ps * 32 + (tid >> 3);
      zT[part * 4 + 0][lt] = rn.x;
      zT[part * 4 + 1][lt] = rn.y;
      zT[part * 4 + 2][lt] = rn.z;
      zT[part * 4 + 3][lt] = rn.w;
      const float s = group8_sum(dot4(rn, rn));
      if (part == 0) zz_s[lt] = s;
    }
    // ---- phase B: distances + running argmin over the codebook ------------------------------
    auto load_chunk = [&](int c, int buf) {
      const int c0 = c * kVqTileN;
      // 32 rows x 128 floats = 1024 float4; 256 threads x 4
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int f = tid + i * kVqThreads;
        const int row = f >> 5, col4 = (f & 31) * 4;
        const bool ok = c0 + col4 < K;   // K % 4 == 0 enforced by the host
        cp_async16(&eT[buf][row][col4], EnT + (size_t)row * K + (ok ? c0 + col4 : 0), ok);
      }
      if (tid < kVqTileN / 4) {
        const bool ok = c0 + tid * 4 < K;
        cp_async16(&ee_s[buf][tid * 4], ee + (ok ? c0 + tid * 4 : 0), ok);
      }
      cp_async_commit();
    };
    float bestd[8];
    int besti[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) { bestd[i] = INFINITY; besti[i] = 0x7fffffff; }
    load_chunk(0, 0);
    for (int c = 0; c < nchunks; ++c) {
      const int buf = c & 1;
      if (c + 1 < nchunks) { load_chunk(c + 1, buf ^ 1); cp_async_wait<1>(); } else { cp_async_wait<0>(); }
      __syncthreads();   // chunk c (and, for c == 0, zT/zz_s) visible
      float2 dacc[8][4];     // 8 tokens x 8 codes, code pairs packed for FFMA2
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) dacc[i][j] = make_float2(0.f, 0.f);
#pragma unroll 8
      for (int k = 0; k < kVqD; ++k) {
        const float4 za = *reinterpret_cast<const float4*>(&zT[k][ty * 4]);
        const float4 zb = *reinterpret_cast<const float4*>(&zT[k][64 + ty * 4]);
        const float4 ea = *reinterpret_cast<const float4*>(&eT[buf][k][tx * 4]);
        const float4 eb = *reinterpret_cast<const float4*>(&eT[buf][k][64 + tx * 4]);
        const float zv[8] = {za.x, za.y, za.z, za.w, zb.x, zb.y, zb.z, zb.w};
        const float2 ev[4] = {make_float2(ea.x, ea.y), make_float2(ea.z, ea.w), make_float2(eb.x, eb.y), make_float2(eb.z, eb.w)};
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) ffma2(dacc[i][j], zv[i], ev[j]);   // same k-order and rounding as sequential fmaf
      }
      const int c0 = c * kVqTileN;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float zz = zz_s[(i < 4 ? 0 : 64) + ty * 4 + (i & 3)];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int lc = (j < 4 ? 0 : 64) + tx * 4 + (j & 3);
          const int code = c0 + lc;
          const float dot = (j & 1) ? dacc[i][j >> 1].y : dacc[i][j >> 1].x;
          const float d = fmaf(-2.f, dot, zz + ee_s[buf][lc]);   // (|z|^2+|e|^2) - 2 z.e
          if (code < K && d < bestd[i]) { bestd[i] = d; besti[i] = code; }   // codes ascend: first min kept
        }
      }
      __syncthreads();   // everyone done with buf before it is refilled
    }
    // reduce (d, idx) lexicographically over the 16 tx lanes that share a token
#pragma unroll
    for (int i = 0; i < 8; ++i) {
#pragma unroll
      for (int o = 1; o < 16; o <<= 1) {
        const float od = __shfl_xor_sync(0xffffffffu, bestd[i], o);
        const int oi = __shfl_xor_sync(0xffffffffu, besti[i], o);
        if (od < bestd[i] || (od == bestd[i] && oi < besti[i])) { bestd[i] = od; besti[i] = oi; }
      }
      if (tx == 0) best_s[(i < 4 ? 0 : 64) + ty * 4 + (i & 3)] = besti[i];
    }
    __syncthreads();
    // ---- phase C: gather, normalise, loss, residual update ----------------------------------
    float lsum = 0.f;
#pragma unroll
    for (int ps = 0; ps < 4; ++ps) {
      const int lt = ps * 32 + (tid >> 3);
      const int tok = m0 + lt;
      int code = best_s[lt];
      if (code >= K) code = 0;   // only for rows of NaNs: torch.argmin would also return some index
      const float4 e = *reinterpret_cast<const float4*>(E + (size_t)code * kVqD + part * 4);
      float nrm, nrm_r;
      const float4 q = normalize8(e, nrm, use_norm);
      float4 rr = park[ps * kVqThreads + tid], ac = park[(4 + ps) * kVqThreads + tid];
      const float4 rn = normalize8(rr, nrm_r, use_norm);   // same arithmetic as phase A: identical value
      const float dx = q.x - rn.x, dy = q.y - rn.y, dz = q.z - rn.z, dw = q.w - rn.w;
      if (tok < M) {
        lsum += dx * dx + dy * dy + dz * dz + dw * dw;
        if (part == 0) idx_out[(size_t)tok * depth + t] = code;
      }
      rr.x -= q.x; rr.y -= q.y; rr.z -= q.z; rr.w -= q.w;
      ac.x += q.x; ac.y += q.y; ac.z += q.z; ac.w += q.w;
      park[ps * kVqThreads + tid] = rr;
      park[(4 + ps) * kVqThreads + tid] = ac;
    }
    lsum = warp_sum(lsum);
    if ((tid & 31) == 0) red_s[tid >> 5] = lsum;
    __syncthreads();
    if constexpr (kStats != kVqStatsOff) {
      // EMA statistics of this depth.  zT still holds the vectors the lookup compared (phase C recomputed the same values)
      // and best_s the codes: reading them here, behind the barrier, keeps phase C's registers as they are.
#pragma unroll 1
      for (int ps = 0; ps < 4; ++ps) {
        const int lt = ps * 32 + (tid >> 3);
        const int tok = m0 + lt;
        int code = best_s[lt];
        if (code >= K) code = 0;   // as phase C
        const float4 x = make_float4(zT[part * 4 + 0][lt], zT[part * 4 + 1][lt], zT[part * 4 + 2][lt], zT[part * 4 + 3][lt]);
        vq_stat_add<kStats>(*st, code, part, tok < M, x);
        if (kStats == kVqStatsDeterministic && tok < M)
          *reinterpret_cast<float4*>(contrib + ((size_t)tok * depth + t) * kVqD + part * 4) = x;
      }
      __syncthreads();
      // flush the table, then clear it for the next depth (whose statistics follow phase B's barriers)
#pragma unroll 1
      for (int i = tid; i < kVqStatSlots * kVqD; i += kVqThreads) {
        const int slot = i / kVqD, col = i % kVqD;
        const int key = st->keys[slot];
        if (key >= 0) {
          if (kStats == kVqStatsAtomic) atomicAdd(sums + (size_t)key * kVqD + col, st->acc[slot][col]);
          if (col == 0) atomicAdd(counts + key, st->cnt[slot]);
        }
      }
      __syncthreads();
      vq_stat_clear(*st, tid);
    }
    if (tid == 0) {
      float s = 0.f;
      for (int w = 0; w < kVqThreads / 32; ++w) s += red_s[w];
      loss_part[(size_t)t * gridDim.x + blockIdx.x] = s;
    }
    // (the next depth's phase A rewrites zT only after the __syncthreads above; best_s/red_s are
    //  rewritten only after later barriers)
  }
  // straight-through value: z + (z_q - z)
#pragma unroll
  for (int ps = 0; ps < 4; ++ps) {
    const int tok = m0 + ps * 32 + (tid >> 3);
    if (tok < M) {
      const float4 zr = *reinterpret_cast<const float4*>(z + (size_t)tok * kVqD + part * 4);
      const float4 ac = park[(4 + ps) * kVqThreads + tid];
      float4 o;
      o.x = zr.x + (ac.x - zr.x);
      o.y = zr.y + (ac.y - zr.y);
      o.z = zr.z + (ac.z - zr.z);
      o.w = zr.w + (ac.w - zr.w);
      *reinterpret_cast<float4*>(out + (size_t)tok * kVqD + part * 4) = o;
    }
  }
}

// loss = mean_t( beta * m_t + m_t ),  m_t = sum_t / (M * D)      (quantizers.py:56-57,89-90)
// kEma: loss = mean_t( beta * m_t ) -- the EMA codebook has no codebook term
template <bool kEma>
__global__ void vq_loss_kernel(const float* __restrict__ loss_part, int nparts, int depth, float inv_count, float beta,
                               float* __restrict__ loss_out) {
  __shared__ float red[32];
  float total = 0.f;
  for (int t = 0; t < depth; ++t) {
    float s = 0.f;
    for (int i = threadIdx.x; i < nparts; i += blockDim.x) s += loss_part[(size_t)t * nparts + i];
    s = warp_sum(s);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
      float a = 0.f;
      for (int w = 0; w < (int)(blockDim.x >> 5); ++w) a += red[w];
      const float m = a * inv_count;
      if constexpr (kEma) total += beta * m;
      else total += beta * m + m;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) *loss_out = depth > 1 ? total / (float)depth : total;
}

// J_n(x)^T v = (v - xh (xh . v)) / max(|x|, eps), 8 lanes per vector (identity when use_norm == 0)
__device__ __forceinline__ float4 norm_jt8(const float4& xh, float nrm, const float4& v, int use_norm) {
  if (!use_norm) return v;
  const float p = group8_sum(dot4(xh, v));
  return make_float4((v.x - xh.x * p) / nrm, (v.y - xh.y * p) / nrm, (v.z - xh.z * p) / nrm, (v.w - xh.w * p) / nrm);
}

// Codebook-gradient scatter.  The reference's nn.Embedding backward is an atomic scatter-add into [K, D]; at
// initialisation an encoder hits only a few dozen codes per 4096 tokens, i.e. thousands of atomics land on the same
// few rows.  Each CTA therefore accumulates into a shared-memory table keyed by code (open addressing, 256 slots x
// 32 floats, shared-memory atomics) and flushes each live slot to global memory once: the global atomic count drops
// from tokens x 32 to CTAs x live codes x 32, whatever the code distribution.  A full table falls back to
// direct global atomics (uniform random codes: correct, just not better than before).
constexpr int kVqBwdSlots = 256;
constexpr int kVqBwdThreads = 256;
struct VqBwdTable {
  int keys[kVqBwdSlots];
  float acc[kVqBwdSlots][kVqD];
};
__device__ __forceinline__ void vq_scatter(VqBwdTable& tb, float* __restrict__ gE, long long code, int part, const float4& v) {
  // lane `part == 0` of the 8-lane group finds / claims the slot, the group shares it
  int slot = -1;
  if (part == 0) {
    unsigned h = ((unsigned)code * 2654435761u) >> 24;
#pragma unroll 1
    for (int probe = 0; probe < 8; ++probe) {
      const int old = atomicCAS(&tb.keys[h], -1, (int)code);
      if (old == -1 || old == (int)code) { slot = (int)h; break; }
      h = (h + 1) & (kVqBwdSlots - 1);
    }
  }
  slot = __shfl_sync(0xffffffffu, slot, (threadIdx.x & 31) & ~7);
  float* dst = slot >= 0 ? &tb.acc[slot][part * 4] : gE + (size_t)code * kVqD + part * 4;
  atomicAdd(dst + 0, v.x); atomicAdd(dst + 1, v.y); atomicAdd(dst + 2, v.z); atomicAdd(dst + 3, v.w);
}

// The per-token closed-form gradients of the backward, shared by the atomic and the deterministic kernel so both run the
// same arithmetic: returns g_z's 4-float `part` of token tk and hands every codebook contribution to
// emit(t, code, value) -- the plain quantiser once (t = 0), the residual one per depth step, deepest first.  A dead
// token (past M, kept so that 8-lane groups stay whole) emits zeros.
template <class Emit>
__device__ __forceinline__ float4 vq_bwd_token(const float* __restrict__ z, const float* __restrict__ E,
                                               const long long* __restrict__ idx, const float* __restrict__ g_out,
                                               float g_loss, int tk, bool live, int part, int M, int depth, int residual,
                                               float beta, int use_norm, Emit&& emit) {
  const float c = 2.f / ((float)M * (float)kVqD);
  const float4 zv = *reinterpret_cast<const float4*>(z + (size_t)tk * kVqD + part * 4);
  float4 go = g_out ? *reinterpret_cast<const float4*>(g_out + (size_t)tk * kVqD + part * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
  if (!residual) {
    const long long code = idx[tk];
    const float4 e = *reinterpret_cast<const float4*>(E + (size_t)code * kVqD + part * 4);
    float nz, ne;
    const float4 zn = normalize8(zv, nz, use_norm);
    const float4 qn = normalize8(e, ne, use_norm);
    const float4 dzq = make_float4(zn.x - qn.x, zn.y - qn.y, zn.z - qn.z, zn.w - qn.w);
    const float4 jz = norm_jt8(zn, nz, dzq, use_norm);
    const float sz = g_loss * beta * c;
    go.x += sz * jz.x; go.y += sz * jz.y; go.z += sz * jz.z; go.w += sz * jz.w;
    const float4 dqz = make_float4(-dzq.x, -dzq.y, -dzq.z, -dzq.w);
    const float4 je = norm_jt8(qn, ne, dqz, use_norm);
    const float se = live ? g_loss * c : 0.f;
    emit(0, code, make_float4(se * je.x, se * je.y, se * je.z, se * je.w));
  } else {
    const float gl = g_loss / (float)depth;
    float4 r = zv;
    float4 gq[kVqMaxDepth], gr[kVqMaxDepth], qh[kVqMaxDepth];
    float qn_norm[kVqMaxDepth];
#pragma unroll
    for (int t = 0; t < kVqMaxDepth; ++t) {
      if (t < depth) {
        const long long code = idx[(size_t)tk * depth + t];
        const float4 e = *reinterpret_cast<const float4*>(E + (size_t)code * kVqD + part * 4);
        float nr, ne;
        const float4 rn = normalize8(r, nr, use_norm);
        const float4 qn = normalize8(e, ne, use_norm);
        qh[t] = qn; qn_norm[t] = ne;
        const float s1 = gl * c;
        gq[t] = make_float4(s1 * (qn.x - rn.x), s1 * (qn.y - rn.y), s1 * (qn.z - rn.z), s1 * (qn.w - rn.w));
        const float4 d = make_float4(rn.x - qn.x, rn.y - qn.y, rn.z - qn.z, rn.w - qn.w);
        const float4 j = norm_jt8(rn, nr, d, use_norm);
        const float s2 = gl * beta * c;
        gr[t] = make_float4(s2 * j.x, s2 * j.y, s2 * j.z, s2 * j.w);
        r.x -= qn.x; r.y -= qn.y; r.z -= qn.z; r.w -= qn.w;
      }
    }
    float4 suffix = make_float4(0.f, 0.f, 0.f, 0.f);   // sum_{t > s} gr[t]
#pragma unroll
    for (int s = kVqMaxDepth - 1; s >= 0; --s) {
      if (s < depth) {
        const float4 tot = make_float4(gq[s].x - suffix.x, gq[s].y - suffix.y, gq[s].z - suffix.z, gq[s].w - suffix.w);
        float4 je = norm_jt8(qh[s], qn_norm[s], tot, use_norm);
        if (!live) je = make_float4(0.f, 0.f, 0.f, 0.f);
        const long long code = idx[(size_t)tk * depth + s];
        emit(s, code, je);
        suffix.x += gr[s].x; suffix.y += gr[s].y; suffix.z += gr[s].z; suffix.w += gr[s].w;
      }
    }
  }
  return go;
}

// gz [M,32] (written), gE [K,32] (atomically accumulated; caller zero-fills)
__global__ void __launch_bounds__(kVqBwdThreads)
vq_bwd_kernel(const float* __restrict__ z, const float* __restrict__ E, const long long* __restrict__ idx,
              const float* __restrict__ g_out, const float* __restrict__ g_loss_ptr, float* __restrict__ gz,
              float* __restrict__ gE, int M, int K, int depth, int residual, float beta, int use_norm) {
  __shared__ VqBwdTable tb;
  for (int i = threadIdx.x; i < kVqBwdSlots; i += kVqBwdThreads) tb.keys[i] = -1;
  for (int i = threadIdx.x; i < kVqBwdSlots * kVqD; i += kVqBwdThreads) (&tb.acc[0][0])[i] = 0.f;
  __syncthreads();
  const int part = threadIdx.x & 7;
  const float g_loss = g_loss_ptr ? *g_loss_ptr : 0.f;
  // 32 tokens per CTA pass; M % 4 == 0 (host) keeps every 8-lane group and every warp uniform
  for (int tok0 = blockIdx.x * (kVqBwdThreads / 8); tok0 < M; tok0 += gridDim.x * (kVqBwdThreads / 8)) {
    const int tok = tok0 + (threadIdx.x >> 3);
    const bool live = tok < M;
    const int tk = live ? tok : 0;
    const float4 go = vq_bwd_token(z, E, idx, g_out, g_loss, tk, live, part, M, depth, residual, beta, use_norm,
                                   [&](int, long long code, const float4& v) { vq_scatter(tb, gE, code, part, v); });
    if (live) *reinterpret_cast<float4*>(gz + (size_t)tok * kVqD + part * 4) = go;
  }
  __syncthreads();
  // flush: one global atomic per (live slot, column)
  for (int i = threadIdx.x; i < kVqBwdSlots * kVqD; i += kVqBwdThreads) {
    const int slot = i / kVqD;
    const int key = tb.keys[slot];
    if (key >= 0) {
      const float v = tb.acc[slot][i % kVqD];
      if (v != 0.f) atomicAdd(gE + (size_t)key * kVqD + (i % kVqD), v);
    }
  }
}

// Deterministic backward, first half: the same per-token work as vq_bwd_kernel, one pass of 32 tokens per CTA.  Instead of
// scattering, entry m * depth + t (m for the plain quantiser: the layout of idx) stores its codebook contribution in
// contrib [entries, 32]; scatter_rows_det then sums them into gE in a fixed order.
__global__ void __launch_bounds__(kVqBwdThreads)
vq_bwd_contrib_kernel(const float* __restrict__ z, const float* __restrict__ E, const long long* __restrict__ idx,
                      const float* __restrict__ g_out, const float* __restrict__ g_loss_ptr, float* __restrict__ gz,
                      float* __restrict__ contrib, int M, int depth, int residual, float beta, int use_norm) {
  const int part = threadIdx.x & 7;
  const float g_loss = g_loss_ptr ? *g_loss_ptr : 0.f;
  const int tok = blockIdx.x * (kVqBwdThreads / 8) + (threadIdx.x >> 3);
  const bool live = tok < M;
  const int tk = live ? tok : 0;
  const float4 go = vq_bwd_token(z, E, idx, g_out, g_loss, tk, live, part, M, depth, residual, beta, use_norm,
                                 [&](int t, long long, const float4& v) {
                                   const size_t entry = residual ? (size_t)tk * depth + t : (size_t)tk;
                                   if (live) *reinterpret_cast<float4*>(contrib + entry * kVqD + part * 4) = v;
                                 });
  if (live) *reinterpret_cast<float4*>(gz + (size_t)tok * kVqD + part * 4) = go;
}

// decode_codes support (vitvqgan.py:81-86): out[m] = sum_t normalize(E[code[m,t]])
__global__ void vq_embed_kernel(const float* __restrict__ E, const long long* __restrict__ codes, float* __restrict__ out,
                                int M, int K, int depth, int use_norm) {
  const int gid = blockIdx.x * blockDim.x + threadIdx.x;
  const int tok = gid >> 3, part = gid & 7;
  if (tok >= M) return;
  float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int t = 0; t < depth; ++t) {
    long long code = codes[(size_t)tok * depth + t];
    if (code < 0 || code >= K) code = 0;
    const float4 e = *reinterpret_cast<const float4*>(E + (size_t)code * kVqD + part * 4);
    float n;
    const float4 q = normalize8(e, n, use_norm);
    a.x += q.x; a.y += q.y; a.z += q.z; a.w += q.w;
  }
  *reinterpret_cast<float4*>(out + (size_t)tok * kVqD + part * 4) = a;
}

// ---------------------------------------------------------------------------------------------
constexpr size_t kVqSmemBytes =
    sizeof(float) * (kVqD * kVqTileM + 2 * kVqD * kVqTileN + 2 * kVqTileN + kVqTileM + kVqTileM + kVqThreads / 32) +
    sizeof(float4) * 8 * kVqThreads;

// =============================================================================================
// Wide codes: D = 32 * S for S in [2, 8] (D = 64 .. 256; RQ-VAE quantises 256-wide features).  The entry points pick these
// kernels for D > 32 through one host path (vq_lookup), and the EMA update kernels below serve every width.  The D = 32
// kernels above stay separate: the two families normalise in different summation orders (each vq_embed must equal its
// own lookup bit for bit), and running the D = 32 lookup on this kernel's phase B and statistics pass measured slower
// (DESIGN.md §7.6).  Same arithmetic contract: distances fmaf(-2, dot, |z|^2 + |e|^2) with dot summed by fmaf in
// ascending k, lowest index among equal distances, straight-through z + (acc - z), normalisation by true division by
// max(|x|, 1e-12).
//   - A row's squared norm is one thread's fmaf chain in column order (vq_row_sq): the lookup's phase A, its gather,
//     vq_prep and vq_embed all normalise a row with the same bits, so vq_embed equals the lookup's accumulated code.
//   - The lookup keeps the whole normalised tile zT [D][128] in shared memory and streams E^T through a two-stage ring
//     in 32-row k-slices; the 8 x 8 accumulator tile stays in registers across a chunk's S slices, so every dot still
//     sums k in order.  Phases A and C run one thread per token, so the transposed stores to zT are conflict-free.
//   - The raw residual of the depth loop lives in a global workspace [M, D] (L2-resident at the shapes this serves) and
//     the accumulated code in `out` itself, which the last depth overwrites with the straight-through value.
//   - EMA statistics: the same 128-slot table keyed by code, filled one 32-column slice of the sums at a time.
//   - Backward: one warp per token, lanes over columns; the per-token routine recomputes the depth recursion column by
//     column in a few passes instead of holding depth x D values per lane, and is shared by the atomic and the
//     deterministic kernel, so their gz agree bit for bit.
constexpr int kVqSlice = 32;
constexpr int kVqMaxD = 256;
__host__ __device__ constexpr bool vq_width_ok(int D) { return D >= kVqSlice && D <= kVqMaxD && D % kVqSlice == 0; }

__device__ __forceinline__ float vq_row_sq(const float* __restrict__ row, int D) {
  float s = 0.f;
  for (int c = 0; c < D; c += 4) {
    const float4 v = *reinterpret_cast<const float4*>(row + c);
    s = fmaf(v.x, v.x, s); s = fmaf(v.y, v.y, s); s = fmaf(v.z, v.z, s); s = fmaf(v.w, v.w, s);
  }
  return s;
}
__device__ __forceinline__ float vq_row_norm(const float* __restrict__ row, int D, int use_norm) {
  return use_norm ? fmaxf(sqrtf(vq_row_sq(row, D)), kNormEps) : 1.f;   // x / 1 == x: use_norm == 0 divides by 1
}
__device__ __forceinline__ float4 div4(const float4& v, float n) { return make_float4(v.x / n, v.y / n, v.z / n, v.w / n); }

// one thread per code: EnT [D][K] (coalesced across the warp's codes), ee [K]
__global__ void vq_prep_wide_kernel(const float* __restrict__ E, float* __restrict__ EnT, float* __restrict__ ee, int K, int D,
                                    int use_norm) {
  const int code = blockIdx.x * blockDim.x + threadIdx.x;
  if (code >= K) return;
  const float* row = E + (size_t)code * D;
  const float nrm = vq_row_norm(row, D, use_norm);
  float s2 = 0.f;
  for (int c = 0; c < D; c += 4) {
    const float4 v = div4(*reinterpret_cast<const float4*>(row + c), nrm);
    EnT[(size_t)(c + 0) * K + code] = v.x;
    EnT[(size_t)(c + 1) * K + code] = v.y;
    EnT[(size_t)(c + 2) * K + code] = v.z;
    EnT[(size_t)(c + 3) * K + code] = v.w;
    s2 = fmaf(v.x, v.x, s2); s2 = fmaf(v.y, v.y, s2); s2 = fmaf(v.z, v.z, s2); s2 = fmaf(v.w, v.w, s2);
  }
  ee[code] = s2;
}

struct VqWideStatTable {
  int keys[kVqStatSlots];
  int cnt[kVqStatSlots];
  int slot[kVqTileM];                    // the slot of each of the CTA's tokens (-1: dead token)
  float acc[kVqStatSlots][kVqSlice];     // one 32-column slice of the sums
};

__host__ __device__ constexpr size_t vq_wide_smem_bytes(int D, bool stats) {
  return sizeof(float) * ((size_t)D * kVqTileM + 2 * kVqSlice * kVqTileN + 2 * kVqTileN + kVqTileM + kVqTileM + kVqThreads / 32) +
         sizeof(int) * 8 * kVqThreads + (stats ? sizeof(VqWideStatTable) : 0);
}

// z [M,D]; EnT [D][K]; ee [K]; E [K,D]; out [M,D] (holds the accumulated code between depths); rws [M,D] raw residual
// (depth > 1 only); idx [M,depth]; loss_part [depth][gridDim.x]; statistics as vq_fwd_kernel with D-wide rows
template <int kStats>
__global__ void __launch_bounds__(kVqThreads, 2)
vq_fwd_wide_kernel(const float* __restrict__ z, const float* __restrict__ EnT, const float* __restrict__ ee,
                   const float* __restrict__ E, float* __restrict__ out, float* __restrict__ rws, long long* __restrict__ idx_out,
                   float* __restrict__ loss_part, int M, int K, int D, int depth, int use_norm, int* __restrict__ counts,
                   float* __restrict__ sums, float* __restrict__ contrib) {
  extern __shared__ __align__(16) uint8_t vq_smem[];
  float (*zT)[kVqTileM] = reinterpret_cast<float (*)[kVqTileM]>(vq_smem);
  float (*eT)[kVqSlice][kVqTileN] = reinterpret_cast<float (*)[kVqSlice][kVqTileN]>(vq_smem + sizeof(float) * D * kVqTileM);
  float (*ee_s)[kVqTileN] = reinterpret_cast<float (*)[kVqTileN]>(eT + 2);
  float* zz_s = reinterpret_cast<float*>(ee_s + 2);
  int* best_s = reinterpret_cast<int*>(zz_s + kVqTileM);
  float* red_s = reinterpret_cast<float*>(best_s + kVqTileM);
  // each thread's 8 running argmin indices, [i][tid]: only stored when a distance improves and read once per depth, so
  // the 8 registers they would take stay with the accumulator tile (128 per thread for two CTAs per SM, no spills)
  int (*besti)[kVqThreads] = reinterpret_cast<int (*)[kVqThreads]>(red_s + kVqThreads / 32);
  VqWideStatTable* st = reinterpret_cast<VqWideStatTable*>(besti + 8);   // kStats != 0 only

  const int tid = threadIdx.x;
  const int m0 = blockIdx.x * kVqTileM;
  const int lt = tid, tok = m0 + tid;                 // phases A and C: one thread per token (threads < 128)
  const bool row_thread = tid < kVqTileM, live = row_thread && tok < M;
  const int tx = tid & 15, ty = tid >> 4;             // phase B: 16 x 16 threads, 8 tokens x 8 codes each
  const int S = D / kVqSlice;
  const int nchunks = (K + kVqTileN - 1) / kVqTileN;
  const int nsteps = nchunks * S;
  if constexpr (kStats != kVqStatsOff) {
    for (int i = tid; i < kVqStatSlots; i += kVqThreads) { st->keys[i] = -1; st->cnt[i] = 0; }
#pragma unroll 1
    for (int i = tid; i < kVqStatSlots * kVqSlice; i += kVqThreads) (&st->acc[0][0])[i] = 0.f;
  }

  for (int t = 0; t < depth; ++t) {
    const float* src = (t == 0 ? z : rws) + (size_t)tok * D;    // the raw residual entering depth t
    // ---- phase A: normalise the residual, stage it transposed -------------------------------
    if (row_thread) {
      float s2 = 0.f;
      if (live) {
        const float nrm = vq_row_norm(src, D, use_norm);
        for (int c = 0; c < D; c += 4) {
          const float4 v = div4(*reinterpret_cast<const float4*>(src + c), nrm);
          zT[c + 0][lt] = v.x; zT[c + 1][lt] = v.y; zT[c + 2][lt] = v.z; zT[c + 3][lt] = v.w;
          s2 = fmaf(v.x, v.x, s2); s2 = fmaf(v.y, v.y, s2); s2 = fmaf(v.z, v.z, s2); s2 = fmaf(v.w, v.w, s2);
        }
      } else {
        for (int c = 0; c < D; ++c) zT[c][lt] = 0.f;
      }
      zz_s[lt] = s2;
    }
    // ---- phase B: distances + running argmin, E^T streamed in 32-row k-slices -----------------
    auto load_slice = [&](int step, int buf) {
      const int c = step / S, s = step - c * S;
      const int c0 = c * kVqTileN;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int f = tid + i * kVqThreads;
        const int row = f >> 5, col4 = (f & 31) * 4;
        const bool ok = c0 + col4 < K;   // K % 4 == 0 enforced by the host
        cp_async16(&eT[buf][row][col4], EnT + (size_t)(s * kVqSlice + row) * K + (ok ? c0 + col4 : 0), ok);
      }
      if (s == 0 && tid < kVqTileN / 4) {
        const bool ok = c0 + tid * 4 < K;
        cp_async16(&ee_s[c & 1][tid * 4], ee + (ok ? c0 + tid * 4 : 0), ok);
      }
      cp_async_commit();
    };
    float bestd[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) { bestd[i] = INFINITY; besti[i][tid] = 0x7fffffff; }
    float2 dacc[8][4];     // 8 tokens x 8 codes, kept across the chunk's slices
    load_slice(0, 0);
    for (int step = 0; step < nsteps; ++step) {
      const int buf = step & 1;
      const int c = step / S, s = step - c * S;
      if (step + 1 < nsteps) { load_slice(step + 1, buf ^ 1); cp_async_wait<1>(); } else { cp_async_wait<0>(); }
      __syncthreads();   // slice `step` (and, for step 0, zT / zz_s) visible
      if (s == 0) {
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) dacc[i][j] = make_float2(0.f, 0.f);
      }
      const float (*zs)[kVqTileM] = zT + s * kVqSlice;
#pragma unroll 8
      for (int k = 0; k < kVqSlice; ++k) {
        const float4 za = *reinterpret_cast<const float4*>(&zs[k][ty * 4]);
        const float4 zb = *reinterpret_cast<const float4*>(&zs[k][64 + ty * 4]);
        const float4 ea = *reinterpret_cast<const float4*>(&eT[buf][k][tx * 4]);
        const float4 eb = *reinterpret_cast<const float4*>(&eT[buf][k][64 + tx * 4]);
        const float zv[8] = {za.x, za.y, za.z, za.w, zb.x, zb.y, zb.z, zb.w};
        const float2 ev[4] = {make_float2(ea.x, ea.y), make_float2(ea.z, ea.w), make_float2(eb.x, eb.y), make_float2(eb.z, eb.w)};
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) ffma2(dacc[i][j], zv[i], ev[j]);
      }
      if (s == S - 1) {
        const int c0 = c * kVqTileN;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float zz = zz_s[(i < 4 ? 0 : 64) + ty * 4 + (i & 3)];
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const int lc = (j < 4 ? 0 : 64) + tx * 4 + (j & 3);
            const int code = c0 + lc;
            const float dot = (j & 1) ? dacc[i][j >> 1].y : dacc[i][j >> 1].x;
            const float d = fmaf(-2.f, dot, zz + ee_s[c & 1][lc]);
            if (code < K && d < bestd[i]) { bestd[i] = d; besti[i][tid] = code; }
          }
        }
      }
      __syncthreads();   // everyone done with buf before it is refilled
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      int bi = besti[i][tid];
#pragma unroll
      for (int o = 1; o < 16; o <<= 1) {
        const float od = __shfl_xor_sync(0xffffffffu, bestd[i], o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (od < bestd[i] || (od == bestd[i] && oi < bi)) { bestd[i] = od; bi = oi; }
      }
      if (tx == 0) best_s[(i < 4 ? 0 : 64) + ty * 4 + (i & 3)] = bi;
    }
    __syncthreads();
    // ---- phase C: gather, normalise, loss, residual and accumulated code ------------------------
    float lsum = 0.f;
    if (live) {
      int code = best_s[lt];
      if (code >= K) code = 0;   // only for rows of NaNs: torch.argmin would also return some index
      const float* er = E + (size_t)code * D;
      const float ne = vq_row_norm(er, D, use_norm);
      float* orow = out + (size_t)tok * D;
      const float* zrow = z + (size_t)tok * D;
      float* rrow = rws + (size_t)tok * D;
      for (int c = 0; c < D; c += 4) {
        const float4 q = div4(*reinterpret_cast<const float4*>(er + c), ne);
        const float dx = q.x - zT[c + 0][lt], dy = q.y - zT[c + 1][lt], dz = q.z - zT[c + 2][lt], dw = q.w - zT[c + 3][lt];
        lsum = fmaf(dx, dx, lsum); lsum = fmaf(dy, dy, lsum); lsum = fmaf(dz, dz, lsum); lsum = fmaf(dw, dw, lsum);
        if (t + 1 < depth) {
          float4 r = *reinterpret_cast<const float4*>(src + c);
          r.x -= q.x; r.y -= q.y; r.z -= q.z; r.w -= q.w;
          *reinterpret_cast<float4*>(rrow + c) = r;
        }
        float4 a = t == 0 ? make_float4(0.f, 0.f, 0.f, 0.f) : *reinterpret_cast<const float4*>(orow + c);
        a.x += q.x; a.y += q.y; a.z += q.z; a.w += q.w;
        if (t + 1 == depth) {
          const float4 zr = *reinterpret_cast<const float4*>(zrow + c);
          a = make_float4(zr.x + (a.x - zr.x), zr.y + (a.y - zr.y), zr.z + (a.z - zr.z), zr.w + (a.w - zr.w));
        }
        *reinterpret_cast<float4*>(orow + c) = a;
      }
      idx_out[(size_t)tok * depth + t] = code;
    }
    lsum = warp_sum(lsum);
    if ((tid & 31) == 0) red_s[tid >> 5] = lsum;
    __syncthreads();
    if constexpr (kStats != kVqStatsOff) {
      // zT still holds the vectors the lookup compared, best_s the codes
      if (row_thread) {
        int slot = -1;
        if (live) {
          int code = best_s[lt];
          if (code >= K) code = 0;   // as phase C
          unsigned h = ((unsigned)code * 2654435761u) >> 25;
#pragma unroll 1
          for (int probe = 0; probe < kVqStatSlots; ++probe) {
            const int old = atomicCAS(&st->keys[h], -1, code);
            if (old == -1 || old == code) { slot = (int)h; break; }
            h = (h + 1) & (kVqStatSlots - 1);
          }
          atomicAdd(&st->cnt[slot], 1);
          if (kStats == kVqStatsDeterministic) {
            float* crow = contrib + ((size_t)tok * depth + t) * D;
            for (int c = 0; c < D; c += 4)
              *reinterpret_cast<float4*>(crow + c) = make_float4(zT[c][lt], zT[c + 1][lt], zT[c + 2][lt], zT[c + 3][lt]);
          }
        }
        st->slot[lt] = slot;
      }
      __syncthreads();
      if constexpr (kStats == kVqStatsAtomic) {
#pragma unroll 1
        for (int s = 0; s < S; ++s) {
          if (row_thread && st->slot[lt] >= 0) {
            float* acc = st->acc[st->slot[lt]];
#pragma unroll 4
            for (int j = 0; j < kVqSlice; ++j) {
              const int col = (j + tid) & (kVqSlice - 1);    // lanes start on different banks
              atomicAdd(acc + col, zT[s * kVqSlice + col][lt]);
            }
          }
          __syncthreads();
#pragma unroll 1
          for (int i = tid; i < kVqStatSlots * kVqSlice; i += kVqThreads) {
            const int slot = i / kVqSlice, col = i % kVqSlice;
            const int key = st->keys[slot];
            if (key >= 0) {
              atomicAdd(sums + (size_t)key * D + s * kVqSlice + col, st->acc[slot][col]);
              st->acc[slot][col] = 0.f;
            }
          }
          __syncthreads();
        }
      }
      // counts, then an empty table for the next depth (whose statistics follow phase B's barriers)
      for (int i = tid; i < kVqStatSlots; i += kVqThreads) {
        const int key = st->keys[i];
        if (key >= 0) atomicAdd(counts + key, st->cnt[i]);
        st->keys[i] = -1;
        st->cnt[i] = 0;
      }
    }
    if (tid == 0) {
      float s = 0.f;
      for (int w = 0; w < kVqThreads / 32; ++w) s += red_s[w];
      loss_part[(size_t)t * gridDim.x + blockIdx.x] = s;
    }
  }
}

// Per-token closed-form gradients at width D, one warp per token (lane l owns columns l, l + 32, ...): writes gz's row
// and hands every codebook contribution to claim(t, code) -> handle (once per depth step, warp-uniform) and
// emit(handle, code, column, value).  The residual recursion r_{t+1} = r_t - q_t is recomputed column by column in each
// pass (norms, then J^T dot products), so a lane holds O(depth) scalars instead of depth x D floats.
template <class Claim, class Emit>
__device__ __forceinline__ void vq_bwd_token_wide(const float* __restrict__ z, const float* __restrict__ E,
                                                  const long long* __restrict__ idx, const float* __restrict__ g_out,
                                                  float* __restrict__ gz, float g_loss, int tk, int lane, int M, int D,
                                                  int depth, int residual, float beta, int use_norm, Claim&& claim, Emit&& emit) {
  const float cc = 2.f / ((float)M * (float)D);
  const float* zr = z + (size_t)tk * D;
  auto nrm_of = [&](float s) { return use_norm ? fmaxf(sqrtf(warp_sum(s)), kNormEps) : 1.f; };
  for (int c = lane; c < D; c += 32) gz[(size_t)tk * D + c] = g_out ? g_out[(size_t)tk * D + c] : 0.f;
  if (!residual) {
    const long long code = idx[tk];
    const float* er = E + (size_t)code * D;
    float sz = 0.f, se = 0.f;
    for (int c = lane; c < D; c += 32) { sz = fmaf(zr[c], zr[c], sz); se = fmaf(er[c], er[c], se); }
    const float nz = nrm_of(sz), ne = nrm_of(se);
    float pz = 0.f, pe = 0.f;
    for (int c = lane; c < D; c += 32) {
      const float zn = zr[c] / nz, qn = er[c] / ne, d = zn - qn;
      pz = fmaf(zn, d, pz);
      pe = fmaf(qn, -d, pe);
    }
    pz = warp_sum(pz);
    pe = warp_sum(pe);
    const float sz_ = g_loss * beta * cc, se_ = g_loss * cc;
    const int h = claim(0, code);
    for (int c = lane; c < D; c += 32) {
      const float zn = zr[c] / nz, qn = er[c] / ne, d = zn - qn;
      const float jz = use_norm ? fmaf(-zn, pz, d) / nz : d;
      const float je = use_norm ? fmaf(-qn, pe, -d) / ne : -d;
      gz[(size_t)tk * D + c] = fmaf(sz_, jz, gz[(size_t)tk * D + c]);
      emit(h, code, c, se_ * je);
    }
    return;
  }
  const float gl = g_loss / (float)depth;
  const float s1 = gl * cc, s2 = gl * beta * cc;
  int cd[kVqMaxDepth];                     // codes index K < 2^31 rows: an int, and E + cd * D recomputed, keep registers free
  float ne[kVqMaxDepth], nr[kVqMaxDepth], pr[kVqMaxDepth], pq[kVqMaxDepth];
  auto er = [&](int t, int c) { return E[(size_t)cd[t] * D + c]; };
#pragma unroll
  for (int t = 0; t < kVqMaxDepth; ++t) {
    cd[t] = t < depth ? (int)idx[(size_t)tk * depth + t] : 0;
    float se = 0.f;
    if (t < depth)
      for (int c = lane; c < D; c += 32) se = fmaf(er(t, c), er(t, c), se);
    ne[t] = t < depth ? nrm_of(se) : 1.f;
    pr[t] = 0.f; pq[t] = 0.f;
  }
  // |r_t|
  {
    float sr[kVqMaxDepth];
#pragma unroll
    for (int t = 0; t < kVqMaxDepth; ++t) sr[t] = 0.f;
    for (int c = lane; c < D; c += 32) {
      float r = zr[c];
#pragma unroll
      for (int t = 0; t < kVqMaxDepth; ++t)
        if (t < depth) { sr[t] = fmaf(r, r, sr[t]); r -= er(t, c) / ne[t]; }
    }
#pragma unroll
    for (int t = 0; t < kVqMaxDepth; ++t) nr[t] = t < depth ? nrm_of(sr[t]) : 1.f;
  }
  // rn_t . (rn_t - qn_t)
  for (int c = lane; c < D; c += 32) {
    float r = zr[c];
#pragma unroll
    for (int t = 0; t < kVqMaxDepth; ++t)
      if (t < depth) {
        const float rn = r / nr[t], qn = er(t, c) / ne[t];
        pr[t] = fmaf(rn, rn - qn, pr[t]);
        r -= qn;
      }
  }
#pragma unroll
  for (int t = 0; t < kVqMaxDepth; ++t) pr[t] = warp_sum(pr[t]);
  // column c of tot_s = gq_s - sum_{t > s} gr_t for every depth s, handed to f(s, qn_s, tot_s)
  auto column = [&](int c, auto&& f) {
    float qn[kVqMaxDepth], gq[kVqMaxDepth], gr[kVqMaxDepth];
    float r = zr[c];
#pragma unroll
    for (int t = 0; t < kVqMaxDepth; ++t)
      if (t < depth) {
        const float rn = r / nr[t];
        qn[t] = er(t, c) / ne[t];
        gq[t] = s1 * (qn[t] - rn);
        const float d = rn - qn[t];
        gr[t] = s2 * (use_norm ? fmaf(-rn, pr[t], d) / nr[t] : d);
        r -= qn[t];
      }
    float suffix = 0.f;
#pragma unroll
    for (int s = kVqMaxDepth - 1; s >= 0; --s)
      if (s < depth) {
        f(s, qn[s], gq[s] - suffix);
        suffix += gr[s];
      }
  };
  for (int c = lane; c < D; c += 32) column(c, [&](int s, float qn, float tot) { pq[s] = fmaf(qn, tot, pq[s]); });
  int h[kVqMaxDepth];
#pragma unroll
  for (int t = 0; t < kVqMaxDepth; ++t) {
    pq[t] = warp_sum(pq[t]);
    h[t] = t < depth ? claim(t, cd[t]) : -1;
  }
  for (int c = lane; c < D; c += 32)
    column(c, [&](int s, float qn, float tot) { emit(h[s], cd[s], c, use_norm ? fmaf(-qn, pq[s], tot) / ne[s] : tot); });
}

// The atomic backward's table: slots x D floats (64 KB whatever D) keyed by code, probed by lane 0 of a token's warp.
__host__ __device__ constexpr int vq_wide_bwd_slots(int D) { return 16384 / D; }
__host__ __device__ constexpr size_t vq_wide_bwd_smem_bytes(int D) {
  return (size_t)vq_wide_bwd_slots(D) * (sizeof(int) + sizeof(float) * D);
}
constexpr size_t kVqWideBwdSmemMax = vq_wide_bwd_smem_bytes(2 * kVqSlice);   // the narrowest wide code has the most keys

// gz [M,D] (written), gE [K,D] (atomically accumulated; caller zero-fills)
__global__ void __launch_bounds__(kVqBwdThreads)
vq_bwd_wide_kernel(const float* __restrict__ z, const float* __restrict__ E, const long long* __restrict__ idx,
                   const float* __restrict__ g_out, const float* __restrict__ g_loss_ptr, float* __restrict__ gz,
                   float* __restrict__ gE, int M, int D, int depth, int residual, float beta, int use_norm) {
  extern __shared__ __align__(16) uint8_t vq_smem[];
  const int slots = vq_wide_bwd_slots(D);
  float* acc = reinterpret_cast<float*>(vq_smem);
  int* keys = reinterpret_cast<int*>(acc + (size_t)slots * D);
  for (int i = threadIdx.x; i < slots; i += kVqBwdThreads) keys[i] = -1;
  for (int i = threadIdx.x; i < slots * D; i += kVqBwdThreads) acc[i] = 0.f;
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const float g_loss = g_loss_ptr ? *g_loss_ptr : 0.f;
  auto claim = [&](int, long long code) {
    int slot = -1;
    if (lane == 0) {
      unsigned hh = (((unsigned)code * 2654435761u) >> 16) % (unsigned)slots;
#pragma unroll 1
      for (int probe = 0; probe < 8; ++probe) {
        const int old = atomicCAS(&keys[hh], -1, (int)code);
        if (old == -1 || old == (int)code) { slot = (int)hh; break; }
        hh = hh + 1 == (unsigned)slots ? 0 : hh + 1;
      }
    }
    return __shfl_sync(0xffffffffu, slot, 0);
  };
  auto emit = [&](int slot, long long code, int c, float v) {
    atomicAdd(slot >= 0 ? &acc[(size_t)slot * D + c] : gE + (size_t)code * D + c, v);
  };
  for (int tk = blockIdx.x * (kVqBwdThreads / 32) + warp; tk < M; tk += gridDim.x * (kVqBwdThreads / 32))
    vq_bwd_token_wide(z, E, idx, g_out, gz, g_loss, tk, lane, M, D, depth, residual, beta, use_norm, claim, emit);
  __syncthreads();
  for (int i = threadIdx.x; i < slots * D; i += kVqBwdThreads) {
    const int key = keys[i / D];
    if (key >= 0 && acc[i] != 0.f) atomicAdd(gE + (size_t)key * D + i % D, acc[i]);
  }
}

// deterministic backward, first half: entry m * depth + t (m for the plain quantiser) stores its row in contrib [entries, D]
__global__ void __launch_bounds__(kVqBwdThreads)
vq_bwd_contrib_wide_kernel(const float* __restrict__ z, const float* __restrict__ E, const long long* __restrict__ idx,
                           const float* __restrict__ g_out, const float* __restrict__ g_loss_ptr, float* __restrict__ gz,
                           float* __restrict__ contrib, int M, int D, int depth, int residual, float beta, int use_norm) {
  const int lane = threadIdx.x & 31;
  const int tk = blockIdx.x * (kVqBwdThreads / 32) + (threadIdx.x >> 5);
  if (tk >= M) return;    // whole warp
  const float g_loss = g_loss_ptr ? *g_loss_ptr : 0.f;
  vq_bwd_token_wide(z, E, idx, g_out, gz, g_loss, tk, lane, M, D, depth, residual, beta, use_norm,
                    [&](int t, long long) { return residual ? tk * depth + t : tk; },
                    [&](int entry, long long, int c, float v) { contrib[(size_t)entry * D + c] = v; });
}

// decode_codes at width D, one thread per token: the lookup's normalisation and accumulation order, so the result is
// bit-identical to the accumulated code of vq_fwd_wide_kernel
__global__ void vq_embed_wide_kernel(const float* __restrict__ E, const long long* __restrict__ codes, float* __restrict__ out, int M,
                                     int K, int D, int depth, int use_norm) {
  const int tok = blockIdx.x * blockDim.x + threadIdx.x;
  if (tok >= M) return;
  float* orow = out + (size_t)tok * D;
  for (int t = 0; t < depth; ++t) {
    long long code = codes[(size_t)tok * depth + t];
    if (code < 0 || code >= K) code = 0;
    const float* er = E + (size_t)code * D;
    const float ne = vq_row_norm(er, D, use_norm);
    for (int c = 0; c < D; c += 4) {
      const float4 q = div4(*reinterpret_cast<const float4*>(er + c), ne);
      float4 a = t == 0 ? make_float4(0.f, 0.f, 0.f, 0.f) : *reinterpret_cast<const float4*>(orow + c);
      a.x += q.x; a.y += q.y; a.z += q.z; a.w += q.w;
      *reinterpret_cast<float4*>(orow + c) = a;
    }
  }
}

}  // namespace b200

using namespace b200;

static size_t align256(size_t b) { return (b + 255) & ~size_t(255); }

// The lookup's workspace, byte offsets: [EnT D x K | ee K | loss parts depth x blocks], then for D > 32 at depth > 1 the
// raw residual [M, D] of the depth loop (rws == 0: none)
struct VqFwdLayout {
  size_t ee, part, rws, bytes;
};
static VqFwdLayout vq_fwd_layout(int M, int K, int D, int depth) {
  const size_t nblk = (M + kVqTileM - 1) / kVqTileM;
  VqFwdLayout l;
  l.ee = (size_t)D * K * sizeof(float);
  l.part = l.ee + (size_t)K * sizeof(float);
  l.bytes = l.part + (size_t)depth * nblk * sizeof(float);
  l.rws = 0;
  if (D > kVqD && depth > 1) {
    l.rws = align256(l.bytes);
    l.bytes = l.rws + (size_t)M * D * sizeof(float);
  }
  return l;
}

extern "C" size_t b200vq_vq_workspace_bytes(int M, int K, int depth) { return vq_fwd_layout(M, K, kVqD, depth).bytes; }

extern "C" size_t b200vq_vq_fwd_workspace_bytes(int M, int K, int D, int depth) {
  return vq_width_ok(D) ? vq_fwd_layout(M, K, D, depth).bytes : 0;
}

// The shape checks of the quantiser's entry points, in this order: width, sizes, depth.  `who` prefixes the messages.
static int vq_check_shapes(const char* who, int M, int K, int D, int depth) {
  B200_CHECK_ARG(vq_width_ok(D), "%s: embed_dim must be a multiple of 32 in [32, 256] (got %d)", who, D);
  B200_CHECK_ARG(M > 0 && K > 0 && K % 4 == 0 && M % 4 == 0, "%s: need M %% 4 == 0 and n_embed %% 4 == 0 (M=%d K=%d)", who, M, K);
  B200_CHECK_ARG(depth >= 1 && depth <= kVqMaxDepth, "%s: num_quantizers must be in [1,%d] (got %d)", who, kVqMaxDepth, depth);
  return 0;
}

template <int kStats>
static int vq_launch_lookup(const float* z, const float* EnT, const float* ee, const float* E, float* out, float* rws, long long* idx,
                            float* part, int M, int K, int D, int depth, int use_norm, int* icounts, float* sums, float* contrib,
                            cudaStream_t stream) {
  constexpr bool stats = kStats != kVqStatsOff;
  const int nblk = (M + kVqTileM - 1) / kVqTileM;
  if (D == kVqD) {
    constexpr size_t smem = kVqSmemBytes + (stats ? sizeof(VqStatTable) : 0);
    B200_CONFIGURE_SMEM_ONCE(vq_fwd_kernel<kStats>, smem);
    vq_fwd_kernel<kStats><<<nblk, kVqThreads, smem, stream>>>(z, EnT, ee, E, out, idx, part, M, K, depth, use_norm, icounts, sums,
                                                              contrib);
    B200_LAUNCH_OK("vq_fwd_kernel");
  } else {
    B200_CONFIGURE_SMEM_ONCE(vq_fwd_wide_kernel<kStats>, vq_wide_smem_bytes(kVqMaxD, stats));
    vq_fwd_wide_kernel<kStats><<<nblk, kVqThreads, vq_wide_smem_bytes(D, stats), stream>>>(z, EnT, ee, E, out, rws, idx, part, M, K,
                                                                                           D, depth, use_norm, icounts, sums,
                                                                                           contrib);
    B200_LAUNCH_OK("vq_fwd_wide_kernel");
  }
  return 0;
}

// vq_prep + the lookup at any width and in any statistics mode, in the vq_fwd_layout workspace; *part receives the loss
// partial sums
static int vq_lookup(const float* z, const float* E, float* out, long long* idx, int M, int K, int D, int depth, int use_norm,
                     int stats, int* icounts, float* sums, float* contrib, void* workspace, float** part, cudaStream_t stream) {
  const VqFwdLayout l = vq_fwd_layout(M, K, D, depth);
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  float* EnT = reinterpret_cast<float*>(ws);
  float* ee = reinterpret_cast<float*>(ws + l.ee);
  float* rws = l.rws ? reinterpret_cast<float*>(ws + l.rws) : nullptr;
  *part = reinterpret_cast<float*>(ws + l.part);
  if (D == kVqD) {
    vq_prep_kernel<<<(K * 8 + 255) / 256, 256, 0, stream>>>(E, EnT, ee, K, use_norm);
    B200_LAUNCH_OK("vq_prep_kernel");
  } else {
    vq_prep_wide_kernel<<<(K + 255) / 256, 256, 0, stream>>>(E, EnT, ee, K, D, use_norm);
    B200_LAUNCH_OK("vq_prep_wide_kernel");
  }
  if (stats == kVqStatsOff)
    return vq_launch_lookup<kVqStatsOff>(z, EnT, ee, E, out, rws, idx, *part, M, K, D, depth, use_norm, icounts, sums, contrib,
                                         stream);
  if (stats == kVqStatsAtomic)
    return vq_launch_lookup<kVqStatsAtomic>(z, EnT, ee, E, out, rws, idx, *part, M, K, D, depth, use_norm, icounts, sums, contrib,
                                            stream);
  return vq_launch_lookup<kVqStatsDeterministic>(z, EnT, ee, E, out, rws, idx, *part, M, K, D, depth, use_norm, icounts, sums, contrib,
                                                 stream);
}

extern "C" int b200vq_vq_fwd(const float* z, const float* E, float* out, long long* idx, float* loss, int M, int K, int D, int depth,
                             float beta, int use_norm, void* workspace, size_t ws_bytes, void* streamv) {
  const cudaStream_t stream = static_cast<cudaStream_t>(streamv);
  if (const int rc = vq_check_shapes("vq", M, K, D, depth)) return rc;
  B200_CHECK_ARG(ws_bytes >= b200vq_vq_fwd_workspace_bytes(M, K, D, depth), "vq: workspace too small");
  float* part;
  if (const int rc = vq_lookup(z, E, out, idx, M, K, D, depth, use_norm, kVqStatsOff, nullptr, nullptr, nullptr, workspace, &part,
                               stream))
    return rc;
  const int nblk = (M + kVqTileM - 1) / kVqTileM;
  vq_loss_kernel<false><<<1, 256, 0, stream>>>(part, nblk, depth, 1.f / ((float)M * (float)D), beta, loss);
  B200_LAUNCH_OK("vq_loss_kernel");
  return 0;
}

extern "C" int b200vq_vq_bwd(const float* z, const float* E, const long long* idx, const float* g_out, const float* g_loss, float* gz,
                             float* gE, int M, int K, int D, int depth, int residual, float beta, int use_norm, void* streamv) {
  const cudaStream_t stream = static_cast<cudaStream_t>(streamv);
  if (const int rc = vq_check_shapes("vq", M, K, D, depth)) return rc;
  B200_CUDA_OK(cudaMemsetAsync(gE, 0, (size_t)K * D * sizeof(float), stream));
  const int cap = num_sms() * 2;          // few, long-lived CTAs: each aggregates ~M / cap tokens in its table
  if (D == kVqD) {
    int blocks = (M + 31) / 32;
    if (blocks > cap) blocks = cap;
    vq_bwd_kernel<<<blocks, kVqBwdThreads, 0, stream>>>(z, E, idx, g_out, g_loss, gz, gE, M, K, depth, residual, beta, use_norm);
    B200_LAUNCH_OK("vq_bwd_kernel");
    return 0;
  }
  int blocks = (M + kVqBwdThreads / 32 - 1) / (kVqBwdThreads / 32);
  if (blocks > cap) blocks = cap;
  B200_CONFIGURE_SMEM_ONCE(vq_bwd_wide_kernel, kVqWideBwdSmemMax);
  vq_bwd_wide_kernel<<<blocks, kVqBwdThreads, vq_wide_bwd_smem_bytes(D), stream>>>(z, E, idx, g_out, g_loss, gz, gE, M, D, depth,
                                                                                  residual, beta, use_norm);
  B200_LAUNCH_OK("vq_bwd_wide_kernel");
  return 0;
}

// contributions [M * depth, D], then the scatter's own scratch
extern "C" size_t b200vq_vq_bwd_deterministic_workspace_bytes(int M, int K, int D, int depth) {
  if (M <= 0 || K <= 0 || depth < 1 || depth > kVqMaxDepth || !vq_width_ok(D)) return 0;
  const long long n = (long long)M * depth;
  const size_t contrib = ((size_t)n * D * sizeof(float) + 255) & ~size_t(255);
  return contrib + scatter_det_workspace_bytes(n, K, D, kScatterRunVq);
}

extern "C" int b200vq_vq_bwd_deterministic(const float* z, const float* E, const long long* idx, const float* g_out,
                                           const float* g_loss, float* gz, float* gE, int M, int K, int D, int depth, int residual,
                                           float beta, int use_norm, void* workspace, size_t ws_bytes, void* streamv) {
  const cudaStream_t stream = static_cast<cudaStream_t>(streamv);
  if (const int rc = vq_check_shapes("vq", M, K, D, depth)) return rc;
  B200_CHECK_ARG(z && E && idx && gz && gE && workspace, "vq_bwd_deterministic: null pointer argument");
  B200_CHECK_ARG(ws_bytes >= b200vq_vq_bwd_deterministic_workspace_bytes(M, K, D, depth), "vq_bwd_deterministic: workspace too small");
  const long long n = residual ? (long long)M * depth : M;   // entries: the plain quantiser reads idx[m]
  float* contrib = static_cast<float*>(workspace);
  const size_t contrib_bytes = ((size_t)M * depth * D * sizeof(float) + 255) & ~size_t(255);
  if (D == kVqD) {
    vq_bwd_contrib_kernel<<<(M + 31) / 32, kVqBwdThreads, 0, stream>>>(z, E, idx, g_out, g_loss, gz, contrib, M, depth, residual,
                                                                        beta, use_norm);
    B200_LAUNCH_OK("vq_bwd_contrib_kernel");
  } else {
    vq_bwd_contrib_wide_kernel<<<(M + kVqBwdThreads / 32 - 1) / (kVqBwdThreads / 32), kVqBwdThreads, 0, stream>>>(
        z, E, idx, g_out, g_loss, gz, contrib, M, D, depth, residual, beta, use_norm);
    B200_LAUNCH_OK("vq_bwd_contrib_wide_kernel");
  }
  return scatter_rows_det<kScatterRunVq>(idx, n, K, contrib, n, 0, 0, D, gE, static_cast<uint8_t*>(workspace) + contrib_bytes,
                                         ws_bytes - contrib_bytes, stream);
}

extern "C" int b200vq_vq_embed(const float* E, const long long* codes, float* out, int M, int K, int D, int depth, int use_norm,
                               void* streamv) {
  const cudaStream_t stream = static_cast<cudaStream_t>(streamv);
  if (const int rc = vq_check_shapes("vq_embed", M, K, D, depth)) return rc;
  if (D == kVqD) {
    vq_embed_kernel<<<(M * 8 + 255) / 256, 256, 0, stream>>>(E, codes, out, M, K, depth, use_norm);
    B200_LAUNCH_OK("vq_embed_kernel");
  } else {
    vq_embed_wide_kernel<<<(M + 127) / 128, 128, 0, stream>>>(E, codes, out, M, K, D, depth, use_norm);
    B200_LAUNCH_OK("vq_embed_wide_kernel");
  }
  return 0;
}

// ---------------------------------------------------------------------------------------------
// EMA codebook (van den Oord et al. 2017, appendix A.1, in the form of Taming Transformers' EMAVectorQuantizer)
namespace b200 {

__global__ void vq_counts_to_float_kernel(const int* __restrict__ icounts, float* __restrict__ counts, int K) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < K) counts[k] = (float)icounts[k];    // exact: a count never exceeds M * depth < 2^24 (checked by the host)
}

// cluster_size <- decay * cluster_size + (1 - decay) * n;  embed_avg <- decay * embed_avg + (1 - decay) * s  (any width D)
__global__ void vq_ema_accumulate_wide_kernel(const float* __restrict__ counts, const float* __restrict__ sums,
                                              float* __restrict__ cluster_size, float* __restrict__ embed_avg, int K, int D, float decay,
                                              float one_minus_decay) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= K * D) return;
  embed_avg[i] = decay * embed_avg[i] + one_minus_decay * sums[i];
  if (i % D == 0) cluster_size[i / D] = decay * cluster_size[i / D] + one_minus_decay * counts[i / D];
}

// weight_k = embed_avg_k / ((cluster_size_k + eps) / (N + K eps) * N),  N = sum_k cluster_size_k.  Every CTA sums N itself
// in the same fixed order (strided per thread, then the warps' partials in order), so N has the same bits in every CTA
// and on every run, and no grid-wide barrier or scratch is needed.
constexpr int kVqEmaRowsPerCta = 64;
__global__ void __launch_bounds__(256)
vq_ema_weight_wide_kernel(const float* __restrict__ cluster_size, const float* __restrict__ embed_avg, float* __restrict__ weight, int K,
                          int D, float eps, float k_eps) {
  __shared__ float red[8];
  float s = 0.f;
  for (int k = threadIdx.x; k < K; k += 256) s += cluster_size[k];
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  float N = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) N += red[w];
  const float denom = N + k_eps;
  const int r0 = blockIdx.x * kVqEmaRowsPerCta;
  for (int i = threadIdx.x; i < kVqEmaRowsPerCta * D; i += 256) {
    const int k = r0 + i / D;
    if (k >= K) break;
    const float smoothed = (cluster_size[k] + eps) / denom * N;
    weight[(size_t)k * D + i % D] = embed_avg[(size_t)k * D + i % D] / smoothed;
  }
}

}  // namespace b200

// after the lookup: the EMA loss, the deterministic sums and the float counts
static int vq_ema_finish(const long long* idx, float* loss, float* counts, float* sums, const int* icounts, const float* contrib,
                         const float* part, int M, int K, int D, int depth, float beta, int deterministic, void* workspace,
                         size_t ws_bytes, cudaStream_t stream) {
  const long long n = (long long)M * depth;
  const int nblk = (M + kVqTileM - 1) / kVqTileM;
  vq_loss_kernel<true><<<1, 256, 0, stream>>>(part, nblk, depth, 1.f / ((float)M * (float)D), beta, loss);
  B200_LAUNCH_OK("vq_loss_kernel");
  if (!counts) return 0;
  if (deterministic) {
    uint8_t* scratch = const_cast<uint8_t*>(reinterpret_cast<const uint8_t*>(contrib)) + align256((size_t)n * D * sizeof(float));
    const size_t used = (size_t)(scratch - static_cast<uint8_t*>(workspace));
    const int rc = scatter_rows_det<kScatterRunVq>(idx, n, K, contrib, n, 0, 0, D, sums, scratch, ws_bytes - used, stream);
    if (rc != 0) return rc;
  }
  vq_counts_to_float_kernel<<<(K + 255) / 256, 256, 0, stream>>>(icounts, counts, K);
  B200_LAUNCH_OK("vq_counts_to_float_kernel");
  return 0;
}

// [b200vq_vq_fwd's workspace], [int counts K], deterministic: [contributions M*depth x D | scatter scratch]
extern "C" size_t b200vq_vq_fwd_ema_workspace_bytes(int M, int K, int D, int depth, int deterministic) {
  if (M <= 0 || K <= 0 || depth < 1 || depth > kVqMaxDepth || !vq_width_ok(D)) return 0;
  size_t b = align256(b200vq_vq_fwd_workspace_bytes(M, K, D, depth)) + align256((size_t)K * sizeof(int));
  if (deterministic) {
    const long long n = (long long)M * depth;
    b += align256((size_t)n * D * sizeof(float)) + scatter_det_workspace_bytes(n, K, D, kScatterRunVq);
  }
  return b;
}

extern "C" int b200vq_vq_fwd_ema(const float* z, const float* E, float* out, long long* idx, float* loss, float* counts, float* sums,
                                 int M, int K, int D, int depth, float beta, int use_norm, int deterministic, void* workspace,
                                 size_t ws_bytes, void* streamv) {
  const cudaStream_t stream = static_cast<cudaStream_t>(streamv);
  if (const int rc = vq_check_shapes("vq_fwd_ema", M, K, D, depth)) return rc;
  B200_CHECK_ARG(z && E && out && idx && loss && workspace, "vq_fwd_ema: null pointer argument");
  B200_CHECK_ARG((counts == nullptr) == (sums == nullptr), "vq_fwd_ema: counts and sums must both be given or both be NULL");
  B200_CHECK_ARG((long long)M * depth < (1ll << 24), "vq_fwd_ema: M * depth must be below 2^24 (fp32 counts stay exact)");
  B200_CHECK_ARG(ws_bytes >= b200vq_vq_fwd_ema_workspace_bytes(M, K, D, depth, deterministic), "vq_fwd_ema: workspace too small");
  uint8_t* ws = static_cast<uint8_t*>(workspace) + align256(b200vq_vq_fwd_workspace_bytes(M, K, D, depth));
  int* icounts = reinterpret_cast<int*>(ws);
  float* contrib = reinterpret_cast<float*>(ws + align256((size_t)K * sizeof(int)));
  const bool stats = counts != nullptr;
  if (stats) {
    B200_CUDA_OK(cudaMemsetAsync(icounts, 0, (size_t)K * sizeof(int), stream));
    if (!deterministic) B200_CUDA_OK(cudaMemsetAsync(sums, 0, (size_t)K * D * sizeof(float), stream));
  }
  const int mode = !stats ? kVqStatsOff : deterministic ? kVqStatsDeterministic : kVqStatsAtomic;
  float* part;
  if (const int rc = vq_lookup(z, E, out, idx, M, K, D, depth, use_norm, mode, icounts, sums, contrib, workspace, &part, stream))
    return rc;
  return vq_ema_finish(idx, loss, counts, sums, icounts, contrib, part, M, K, D, depth, beta, deterministic, workspace, ws_bytes,
                       stream);
}

extern "C" int b200vq_vq_ema_update(const float* counts, const float* sums, float* cluster_size, float* embed_avg, float* weight,
                                    int K, int D, float decay, float eps, void* streamv) {
  const cudaStream_t stream = static_cast<cudaStream_t>(streamv);
  B200_CHECK_ARG(vq_width_ok(D), "vq_ema_update: embed_dim must be a multiple of 32 in [32, 256] (got %d)", D);
  B200_CHECK_ARG(K > 0, "vq_ema_update: n_embed must be positive (got %d)", K);
  B200_CHECK_ARG(counts && sums && cluster_size && embed_avg && weight, "vq_ema_update: null pointer argument");
  B200_CHECK_ARG(decay >= 0.f && decay <= 1.f, "vq_ema_update: decay must be in [0, 1] (got %g)", (double)decay);
  B200_CHECK_ARG(eps >= 0.f, "vq_ema_update: eps must be non-negative (got %g)", (double)eps);
  vq_ema_accumulate_wide_kernel<<<(K * D + 255) / 256, 256, 0, stream>>>(counts, sums, cluster_size, embed_avg, K, D, decay,
                                                                         (float)(1.0 - (double)decay));
  B200_LAUNCH_OK("vq_ema_accumulate_wide_kernel");
  vq_ema_weight_wide_kernel<<<(K + kVqEmaRowsPerCta - 1) / kVqEmaRowsPerCta, 256, 0, stream>>>(cluster_size, embed_avg, weight, K, D,
                                                                                             eps, (float)((double)K * (double)eps));
  B200_LAUNCH_OK("vq_ema_weight_wide_kernel");
  return 0;
}
