// Stage-2 RQTransformer (reference enhancing/modules/stage2/layers.py:306-547): what its residual-code prior needs beyond
// the GPT kernels of stage2.cu.
//   short_attention  the depth transformer's causal attention over B' sequences of D <= 16 tokens (layers.py:76-89 with
//                    ctx_len = D, cond_len = 0).  One warp per (sequence, head), grid-stride: no grid dimension grows
//                    with B'.  Plain fp32 FMA -- 4 D hs FLOP per query against 16 hs bytes per token is far below the
//                    tensor-core break-even -- so every data path gets fp32-grade results.
//   rq_embed         cat(Wc[conds] + pos_c, cumsum_C(Wi[codes[..., D-1]]) + pos_i): the spatial input   (layers.py:375-384)
//   rq_depth_input   v[s, 0] = h[s], v[s, d] = cumsum_C(Wi[codes[s, d-1]]) + pos_d[d-1]: the depth input (layers.py:388-391)
//   code_sum_embed   sum_j Wi[codes[b, j]] + pos[row]: the sampling steps' inputs                        (layers.py:501-502,534-535)
// The channel prefix sums are scanned in fp64 and rounded once, which is what torch's CPU cumsum over fp32 does, so the
// embedding rows equal the reference's bit for bit.  Their backward is linear: the raw gradient rows are summed by id
// (float atomics, or scatter_det.cu's fixed-order sum on request) and one reverse channel scan over the [V, C] table
// follows; no per-entry scan is materialised.
#include "../../include/b200vq.h"
#include "common.cuh"
#include "scatter_det.cuh"

namespace b200 {

constexpr int kShortMaxD = 16;

static inline int rq_grid(long long work_items, int per_block) {
  long long blocks = (work_items + per_block - 1) / per_block;
  const long long cap = (long long)num_sms() * 16;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return (int)blocks;
}

// ------------------------------------------------------------------------------------------------ short attention
// Per warp: its sequence's rows of one head staged in shared memory (rows padded by 4 floats so that the pair-parallel
// dot products below fall on different banks), then
//   S[i][j] = scale q_i.k_j         one lane per (i, j) pair, j <= max(i, cond - 1)
//   P = softmax(S) per row          one lane per row
//   out rows                        one lane per (row, float4 column), reading P and the staged rows
// Every element of qkv (and dout) is read once with 16-byte loads; every output element is written once.
__host__ __device__ constexpr int short_ld(int hs) { return hs + 4; }
// per-warp shared floats: `mats` staged [D, hs + 4] matrices and two [D, D + 1] score tiles, rounded to whole float4s
__host__ __device__ constexpr size_t short_warp_floats(int D, int hs, int mats) {
  return ((size_t)mats * D * short_ld(hs) + 2 * (size_t)D * (D + 1) + 3) & ~(size_t)3;
}

__device__ __forceinline__ bool short_visible(int q, int k, int cond) { return k <= (q > cond - 1 ? q : cond - 1); }

template <int HS>
__device__ __forceinline__ void short_stage(const float* __restrict__ base, long long ld, float* s, int D, int lane) {
  constexpr int G = HS / 4;
  for (int e = lane; e < D * G; e += 32) {
    const int r = e / G, c = e - r * G;
    *reinterpret_cast<float4*>(s + r * short_ld(HS) + 4 * c) = *reinterpret_cast<const float4*>(base + r * ld + 4 * c);
  }
}

template <int HS>
__device__ __forceinline__ float short_dot(const float* a, const float* b) {
  float acc = 0.f;
#pragma unroll
  for (int c = 0; c < HS / 4; ++c) {
    const float4 x = *reinterpret_cast<const float4*>(a + 4 * c), y = *reinterpret_cast<const float4*>(b + 4 * c);
    acc = fmaf(x.x, y.x, acc); acc = fmaf(x.y, y.y, acc); acc = fmaf(x.z, y.z, acc); acc = fmaf(x.w, y.w, acc);
  }
  return acc;
}

__device__ __forceinline__ void f4_fma(float4& acc, float p, const float4 v) {
  acc.x = fmaf(p, v.x, acc.x); acc.y = fmaf(p, v.y, acc.y); acc.z = fmaf(p, v.z, acc.z); acc.w = fmaf(p, v.w, acc.w);
}

// row-wise softmax of S (in place, masked entries set to 0); one lane per row
__device__ __forceinline__ void short_softmax_rows(float* S, int D, int cond, int lane) {
  if (lane < D) {
    float* row = S + lane * (D + 1);
    float m = -INFINITY;
    for (int j = 0; j < D; ++j) if (short_visible(lane, j, cond)) m = fmaxf(m, row[j]);
    float l = 0.f;
    for (int j = 0; j < D; ++j) {
      const float e = short_visible(lane, j, cond) ? expf(row[j] - m) : 0.f;
      row[j] = e;
      l += e;
    }
    const float inv = 1.f / l;
    for (int j = 0; j < D; ++j) row[j] *= inv;
  }
}

template <int HS>
__global__ void __launch_bounds__(256, 4)
short_attention_fwd_kernel(const float* __restrict__ qkv, float* __restrict__ out, long long nseq, int D, int heads, int cond,
                           float scale) {
  extern __shared__ __align__(16) float smem_f[];
  constexpr int G = HS / 4;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, wpb = blockDim.x >> 5;
  const int C = heads * HS, ld = short_ld(HS);
  float* Q = smem_f + (size_t)warp * short_warp_floats(D, HS, 3);
  float* K = Q + D * ld;
  float* V = K + D * ld;
  float* S = V + D * ld;
  const int tasks = (int)nseq * heads;                    // < 2^31, checked by the host
  for (int task = blockIdx.x * wpb + warp; task < tasks; task += gridDim.x * wpb) {
    const long long seq = task / heads;
    const int h = task - (int)seq * heads;
    const float* base = qkv + seq * D * 3LL * C + h * HS;
    short_stage<HS>(base, 3LL * C, Q, D, lane);
    short_stage<HS>(base + C, 3LL * C, K, D, lane);
    short_stage<HS>(base + 2 * C, 3LL * C, V, D, lane);
    __syncwarp();
    for (int e = lane; e < D * D; e += 32) {
      const int i = e / D, j = e - i * D;
      if (short_visible(i, j, cond)) S[i * (D + 1) + j] = short_dot<HS>(Q + i * ld, K + j * ld) * scale;
    }
    __syncwarp();
    short_softmax_rows(S, D, cond, lane);
    __syncwarp();
    float* obase = out + seq * D * (long long)C + h * HS;
    for (int e = lane; e < D * G; e += 32) {
      const int r = e / G, c = e - r * G;
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int j = 0; j < D; ++j)
        if (short_visible(r, j, cond)) f4_fma(acc, S[r * (D + 1) + j], *reinterpret_cast<const float4*>(V + j * ld + 4 * c));
      *reinterpret_cast<float4*>(obase + r * (long long)C + 4 * c) = acc;
    }
    __syncwarp();                                         // the next task overwrites the staged rows
  }
}

// Backward with the scores recomputed in-kernel: P, dP = dO V^T, delta_i = rowsum(P o dP), dS = P o (dP - delta);
// dq_i = scale sum_j dS_ij k_j, dk_j = scale sum_i dS_ij q_i, dv_j = sum_i P_ij dO_i.  The warp writes the whole dqkv row
// block of its (sequence, head): no atomics, the same bits on every run.
template <int HS>
__global__ void __launch_bounds__(256, 4)
short_attention_bwd_kernel(const float* __restrict__ qkv, const float* __restrict__ dout, float* __restrict__ dqkv, long long nseq,
                           int D, int heads, int cond, float scale) {
  extern __shared__ __align__(16) float smem_f[];
  constexpr int G = HS / 4;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, wpb = blockDim.x >> 5;
  const int C = heads * HS, ld = short_ld(HS);
  float* Q = smem_f + (size_t)warp * short_warp_floats(D, HS, 4);
  float* K = Q + D * ld;
  float* V = K + D * ld;
  float* dO = V + D * ld;
  float* S = dO + D * ld;
  float* dP = S + D * (D + 1);
  const int tasks = (int)nseq * heads;                    // < 2^31, checked by the host
  for (int task = blockIdx.x * wpb + warp; task < tasks; task += gridDim.x * wpb) {
    const long long seq = task / heads;
    const int h = task - (int)seq * heads;
    const float* base = qkv + seq * D * 3LL * C + h * HS;
    short_stage<HS>(base, 3LL * C, Q, D, lane);
    short_stage<HS>(base + C, 3LL * C, K, D, lane);
    short_stage<HS>(base + 2 * C, 3LL * C, V, D, lane);
    short_stage<HS>(dout + seq * D * (long long)C + h * HS, C, dO, D, lane);
    __syncwarp();
    for (int e = lane; e < D * D; e += 32) {
      const int i = e / D, j = e - i * D;
      if (short_visible(i, j, cond)) {
        S[i * (D + 1) + j] = short_dot<HS>(Q + i * ld, K + j * ld) * scale;
        dP[i * (D + 1) + j] = short_dot<HS>(dO + i * ld, V + j * ld);
      }
    }
    __syncwarp();
    short_softmax_rows(S, D, cond, lane);
    if (lane < D) {                                       // the lane that normalised row `lane` turns dP into scale * dS
      const float* p = S + lane * (D + 1);
      float* dp = dP + lane * (D + 1);
      float delta = 0.f;
      for (int j = 0; j < D; ++j) if (short_visible(lane, j, cond)) delta = fmaf(p[j], dp[j], delta);
      for (int j = 0; j < D; ++j) dp[j] = short_visible(lane, j, cond) ? p[j] * (dp[j] - delta) * scale : 0.f;
    }
    __syncwarp();
    float* gbase = dqkv + seq * D * 3LL * C + h * HS;
    for (int e = lane; e < D * G; e += 32) {
      const int r = e / G, c = e - r * G;
      float4 dq = make_float4(0.f, 0.f, 0.f, 0.f), dk = dq, dv = dq;
      for (int j = 0; j < D; ++j) {
        f4_fma(dq, dP[r * (D + 1) + j], *reinterpret_cast<const float4*>(K + j * ld + 4 * c));      // masked entries are 0
        f4_fma(dk, dP[j * (D + 1) + r], *reinterpret_cast<const float4*>(Q + j * ld + 4 * c));
        f4_fma(dv, S[j * (D + 1) + r], *reinterpret_cast<const float4*>(dO + j * ld + 4 * c));
      }
      float* g = gbase + r * 3LL * C + 4 * c;
      *reinterpret_cast<float4*>(g) = dq;
      *reinterpret_cast<float4*>(g + C) = dk;
      *reinterpret_cast<float4*>(g + 2 * C) = dv;
    }
    __syncwarp();
  }
}

// ------------------------------------------------------------------------------------------------ embeddings
// dst[c] = round(sum_{c' <= c} src[c'] in fp64) + pos[c]: one warp per row, 128 columns per step (a float4 per lane), the
// lane's 4 values scanned serially, the lane totals by a shuffle scan, the carry between steps in fp64.
__device__ __forceinline__ void scan_row_add(const float* __restrict__ src, const float* __restrict__ pos, float* __restrict__ dst,
                                             int C, int lane) {
  double carry = 0.0;
  for (int c0 = 0; c0 < C; c0 += 128) {
    const int c = c0 + 4 * lane;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (c < C) v = __ldg(reinterpret_cast<const float4*>(src + c));
    const double a = v.x, b = a + v.y, d = b + v.z, e = d + v.w;
    double pre = e;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const double t = __shfl_up_sync(0xffffffffu, pre, o);
      if (lane >= o) pre += t;
    }
    const double excl = carry + (pre - e);
    if (c < C) {
      const float4 p = __ldg(reinterpret_cast<const float4*>(pos + c));
      *reinterpret_cast<float4*>(dst + c) = make_float4((float)(excl + a) + p.x, (float)(excl + b) + p.y, (float)(excl + d) + p.z,
                                                        (float)(excl + e) + p.w);
    }
    carry += __shfl_sync(0xffffffffu, pre, 31);
  }
}

__device__ __forceinline__ long long clamp_id(long long id, int V) { return id < 0 ? 0 : (id >= V ? V - 1 : id); }

// x[b, t] = t < Tc ? Wc[conds[b, t]] + pos_c[t] : scan(Wi[codes[b, t - Tc, D - 1]]) + pos_i[t - Tc]
__global__ void __launch_bounds__(256, 4)
rq_embed_fwd_kernel(const long long* __restrict__ conds, const long long* __restrict__ codes, const float* __restrict__ Wc,
                    const float* __restrict__ pos_c, const float* __restrict__ Wi, const float* __restrict__ pos_i, float* __restrict__ x,
                    int B, int Tc, int T, int D, int C, int Vc, int Vi) {
  const int lane = threadIdx.x & 31;
  const int Tt = Tc + T;
  const int rows = B * Tt;                                // < 2^31, checked by the host
  for (int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < rows; r += (gridDim.x * blockDim.x) >> 5) {
    const int b = r / Tt, t = r - b * Tt;
    float* dst = x + (long long)r * C;
    if (t < Tc) {
      const float* w = Wc + clamp_id(conds[(long long)b * Tc + t], Vc) * C;
      const float* p = pos_c + (long long)t * C;
      for (int c = 4 * lane; c < C; c += 128) {
        const float4 e = __ldg(reinterpret_cast<const float4*>(w + c)), q = __ldg(reinterpret_cast<const float4*>(p + c));
        *reinterpret_cast<float4*>(dst + c) = make_float4(e.x + q.x, e.y + q.y, e.z + q.z, e.w + q.w);
      }
    } else {
      const long long id = clamp_id(codes[((long long)b * T + (t - Tc)) * D + (D - 1)], Vi);
      scan_row_add(Wi + id * C, pos_i + (long long)(t - Tc) * C, dst, C, lane);
    }
  }
}

// v[s, 0] = h[s]; v[s, d] = scan(Wi[codes[s, d - 1]]) + pos_d[d - 1]   (s over B*T sequences of D rows)
__global__ void __launch_bounds__(256, 4)
rq_depth_input_fwd_kernel(const float* __restrict__ h, const long long* __restrict__ codes, const float* __restrict__ Wi,
                          const float* __restrict__ pos_d, float* __restrict__ v, long long nseq, int D, int C, int Vi) {
  const int lane = threadIdx.x & 31;
  const int rows = (int)nseq * D;                         // < 2^31, checked by the host
  for (int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < rows; r += (gridDim.x * blockDim.x) >> 5) {
    const long long s = r / D;
    const int d = r - (int)s * D;
    float* dst = v + (long long)r * C;
    if (d == 0) {
      for (int c = 4 * lane; c < C; c += 128) *reinterpret_cast<float4*>(dst + c) = *reinterpret_cast<const float4*>(h + s * C + c);
    } else {
      const long long id = clamp_id(codes[s * D + d - 1], Vi);
      scan_row_add(Wi + id * C, pos_d + (long long)(d - 1) * C, dst, C, lane);
    }
  }
}

// In place over a [V, C] table: t[v, c] = sum_{c' >= c} t[v, c'] (fp64, rounded once) -- the adjoint of the channel prefix sum.
__global__ void __launch_bounds__(256, 4)
reverse_scan_rows_kernel(float* __restrict__ t, int V, int C) {
  const int lane = threadIdx.x & 31;
  for (long long r = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < V; r += ((long long)gridDim.x * blockDim.x) >> 5) {
    float* row = t + r * C;
    double carry = 0.0;
    const int last = ((C - 1) / 128) * 128;
    for (int c0 = last; c0 >= 0; c0 -= 128) {
      const int c = c0 + 4 * lane;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (c < C) v = *reinterpret_cast<const float4*>(row + c);
      const double w = v.w, z = w + v.z, y = z + v.y, x = y + v.x;
      double suf = x;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const double u = __shfl_down_sync(0xffffffffu, suf, o);
        if (lane + o < 32) suf += u;
      }
      const double excl = carry + (suf - x);
      if (c < C) *reinterpret_cast<float4*>(row + c) = make_float4((float)(excl + x), (float)(excl + y), (float)(excl + z), (float)(excl + w));
      carry += __shfl_sync(0xffffffffu, suf, 0);
    }
  }
}

// Entry e of a strided id list: ids[(e / Tn) * stride + (e % Tn) * step + off]
struct IdMap { int Tn; long long stride; int step, off; };
__device__ __forceinline__ long long id_at(const long long* __restrict__ ids, IdMap m, long long e) {
  const long long s = e / m.Tn;
  return ids[s * m.stride + (e - s * m.Tn) * m.step + m.off];
}

// Scatter of the raw embedding gradient rows with float atomics (nn.Embedding dense backward).  Entry e's id is id_at(e);
// its gradient row is rows + ((e / Tn) * Tr + off + e % Tn) * C.
__global__ void __launch_bounds__(256, 4)
scatter_rows_atomic_kernel(const long long* __restrict__ ids, long long N, IdMap im, const float* __restrict__ rows, int Tr, int off,
                           int C, float* __restrict__ out, int V) {
  const int C4 = C / 4;
  const long long total = N * C4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long e = i / C4;
    const int c = (int)(i - e * C4);
    const long long s = e / im.Tn;
    const int k = (int)(e - s * im.Tn);
    const long long id = clamp_id(id_at(ids, im, e), V);
    const float4 g = *reinterpret_cast<const float4*>(rows + (s * Tr + off + k) * C + 4 * c);
    float* o = out + id * C + 4 * c;
    atomicAdd(o, g.x); atomicAdd(o + 1, g.y); atomicAdd(o + 2, g.z); atomicAdd(o + 3, g.w);
  }
}

// ids of the same entries, compacted into a dense list (the deterministic scatter takes one id per entry)
__global__ void __launch_bounds__(256, 4)
compact_ids_kernel(const long long* __restrict__ ids, long long N, IdMap im, long long* __restrict__ out) {
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < N; e += (long long)gridDim.x * blockDim.x)
    out[e] = id_at(ids, im, e);
}

// out[w] = sum_m X[m * ld + w] for w < 4 * W4, in an order fixed by the shape: a block owns 8 float4 columns and 32 row
// lanes; lane y sums rows y, y + 32, ... in order; the 32 lane partials are added in lane order.
__global__ void __launch_bounds__(256, 4)
colsum_fixed_kernel(const float* __restrict__ X, long long ld, long long M, int W4, float* __restrict__ out) {
  __shared__ float4 part[32][8];
  const int tx = threadIdx.x & 7, ty = threadIdx.x >> 3;
  const long long w = (long long)blockIdx.x * 8 + tx;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  if (w < W4)
    for (long long m = ty; m < M; m += 32) {
      const float4 v = *reinterpret_cast<const float4*>(X + m * ld + 4 * w);
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
  part[ty][tx] = acc;
  __syncthreads();
  if (ty == 0 && w < W4) {
    float4 s = part[0][tx];
    for (int y = 1; y < 32; ++y) { const float4 p = part[y][tx]; s.x += p.x; s.y += p.y; s.z += p.z; s.w += p.w; }
    reinterpret_cast<float4*>(out)[w] = s;
  }
}

// out[b] = sum_{j < n} Wi[codes[b * ld + j]] (in order, fp32) + pos
__global__ void __launch_bounds__(256, 4)
code_sum_embed_kernel(const long long* __restrict__ codes, long long ld, int n, const float* __restrict__ Wi, const float* __restrict__ pos,
                      float* __restrict__ out, int B, int C, int V) {
  const int C4 = C / 4;
  const long long total = (long long)B * C4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long b = i / C4;
    const int c = (int)(i - b * C4);
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int j = 0; j < n; ++j) {
      const float4 e = __ldg(reinterpret_cast<const float4*>(Wi + clamp_id(codes[b * ld + j], V) * C) + c);
      if (j == 0) acc = e;
      else { acc.x += e.x; acc.y += e.y; acc.z += e.z; acc.w += e.w; }
    }
    const float4 p = __ldg(reinterpret_cast<const float4*>(pos) + c);
    reinterpret_cast<float4*>(out)[i] = make_float4(acc.x + p.x, acc.y + p.y, acc.z + p.z, acc.w + p.w);
  }
}

}  // namespace b200

// ------------------------------------------------------------------------------------------------ host side
using namespace b200;

static int short_check(const void* a, const void* b, const void* c, long long nseq, int D, int heads, int hs, int cond,
                       const char* what) {
  B200_CHECK_ARG(a && b && c, "%s: null pointer argument", what);
  B200_CHECK_ARG(nseq > 0 && heads > 0, "%s: bad shape (sequences=%lld heads=%d)", what, nseq, heads);
  B200_CHECK_ARG(D >= 1 && D <= kShortMaxD, "%s: sequence length must be 1..%d (got %d)", what, kShortMaxD, D);
  B200_CHECK_ARG(hs == 32 || hs == 64 || hs == 96 || hs == 128, "%s: head size must be 32, 64, 96 or 128 (got %d)", what, hs);
  B200_CHECK_ARG(heads * hs <= 2048, "%s: heads * head size must be <= 2048 (got %d)", what, heads * hs);
  B200_CHECK_ARG(cond >= 0, "%s: cond_len must be >= 0 (got %d)", what, cond);
  B200_CHECK_ARG(nseq * heads < (1LL << 31), "%s: too many (sequence, head) pairs", what);
  return 0;
}

// The short-attention kernels are persistent (grid-stride over (sequence, head) tasks), so b200vq_set_sm_limit caps their
// grid like the GEMM's: at most sm_limit() CTAs.  One warp owns each task whatever the grid, so results do not change.
static int short_grid(long long tasks, int wpb) {
  int grid = rq_grid(tasks, wpb);
  const int cap = sm_limit();
  if (cap > 0 && grid > cap) grid = cap;
  return grid;
}

static int short_warps(size_t warp_bytes) {
  int w = (int)((48 * 1024) / warp_bytes);
  return w < 1 ? 1 : (w > 8 ? 8 : w);
}

// Head sizes 96 / 128: a warp's staged rows take up to 27 KB (forward) / 36 KB (backward) at D = 16, so the CTA's rows are
// sized against a larger opt-in budget, which still lets two CTAs share an SM.
constexpr size_t kShortWideSmem = 110 * 1024;
static int short_warps_wide(size_t warp_bytes) {
  const int w = (int)(kShortWideSmem / warp_bytes);
  return w > 8 ? 8 : w;                                   // >= 3: warp_bytes <= 36 KB for D <= 16
}

template <int HS>
static int short_fwd_wide(const float* qkv, float* out, long long nseq, int D, int heads, int cond, float scale, cudaStream_t stream) {
  const size_t wb = short_warp_floats(D, HS, 3) * sizeof(float);
  const int wpb = short_warps_wide(wb);
  auto kern = short_attention_fwd_kernel<HS>;
  B200_CONFIGURE_SMEM_ONCE(kern, kShortWideSmem);
  kern<<<short_grid(nseq * heads, wpb), wpb * 32, wpb * wb, stream>>>(qkv, out, nseq, D, heads, cond, scale);
  B200_LAUNCH_OK("short_attention_fwd_kernel");
  return 0;
}

template <int HS>
static int short_bwd_wide(const float* qkv, const float* dout, float* dqkv, long long nseq, int D, int heads, int cond, float scale,
                          cudaStream_t stream) {
  const size_t wb = short_warp_floats(D, HS, 4) * sizeof(float);
  const int wpb = short_warps_wide(wb);
  auto kern = short_attention_bwd_kernel<HS>;
  B200_CONFIGURE_SMEM_ONCE(kern, kShortWideSmem);
  kern<<<short_grid(nseq * heads, wpb), wpb * 32, wpb * wb, stream>>>(qkv, dout, dqkv, nseq, D, heads, cond, scale);
  B200_LAUNCH_OK("short_attention_bwd_kernel");
  return 0;
}

extern "C" int b200vq_short_attention_fwd(const float* qkv, float* out, long long nseq, int D, int heads, int hs, int cond,
                                          float scale, void* streamv) {
  const cudaStream_t stream = static_cast<cudaStream_t>(streamv);
  if (int rc = short_check(qkv, out, out, nseq, D, heads, hs, cond, "short_attention_fwd")) return rc;
  if (hs == 128) return short_fwd_wide<128>(qkv, out, nseq, D, heads, cond, scale, stream);
  if (hs == 96) return short_fwd_wide<96>(qkv, out, nseq, D, heads, cond, scale, stream);
  const size_t wb = short_warp_floats(D, hs, 3) * sizeof(float);
  const int wpb = short_warps(wb);
  const int grid = short_grid(nseq * heads, wpb);
  if (hs == 64) short_attention_fwd_kernel<64><<<grid, wpb * 32, wpb * wb, stream>>>(qkv, out, nseq, D, heads, cond, scale);
  else          short_attention_fwd_kernel<32><<<grid, wpb * 32, wpb * wb, stream>>>(qkv, out, nseq, D, heads, cond, scale);
  B200_LAUNCH_OK("short_attention_fwd_kernel");
  return 0;
}

extern "C" int b200vq_short_attention_bwd(const float* qkv, const float* dout, float* dqkv, long long nseq, int D, int heads, int hs,
                                          int cond, float scale, void* streamv) {
  const cudaStream_t stream = static_cast<cudaStream_t>(streamv);
  if (int rc = short_check(qkv, dout, dqkv, nseq, D, heads, hs, cond, "short_attention_bwd")) return rc;
  if (hs == 128) return short_bwd_wide<128>(qkv, dout, dqkv, nseq, D, heads, cond, scale, stream);
  if (hs == 96) return short_bwd_wide<96>(qkv, dout, dqkv, nseq, D, heads, cond, scale, stream);
  const size_t wb = short_warp_floats(D, hs, 4) * sizeof(float);
  const int wpb = short_warps(wb);
  const int grid = short_grid(nseq * heads, wpb);
  if (hs == 64) short_attention_bwd_kernel<64><<<grid, wpb * 32, wpb * wb, stream>>>(qkv, dout, dqkv, nseq, D, heads, cond, scale);
  else          short_attention_bwd_kernel<32><<<grid, wpb * 32, wpb * wb, stream>>>(qkv, dout, dqkv, nseq, D, heads, cond, scale);
  B200_LAUNCH_OK("short_attention_bwd_kernel");
  return 0;
}

static int embed_shape_ok(int B, int Tc, int T, int D, int C, int Vc, int Vi, const char* what) {
  B200_CHECK_ARG(B > 0 && Tc >= 0 && T > 0 && C > 0 && C % 4 == 0, "%s: bad shape B=%d Tc=%d T=%d C=%d", what, B, Tc, T, C);
  B200_CHECK_ARG(D >= 1 && D <= kShortMaxD, "%s: depth must be 1..%d (got %d)", what, kShortMaxD, D);
  B200_CHECK_ARG(Vi > 0 && (Tc == 0 || Vc > 0), "%s: vocabulary sizes must be positive (Vc=%d Vi=%d)", what, Vc, Vi);
  B200_CHECK_ARG((long long)B * (Tc + T) * D <= (1LL << 30), "%s: too many tokens", what);
  return 0;
}

static int colsum_fixed(const float* X, long long ld, long long M, long long W, float* out, cudaStream_t stream) {
  const long long W4 = W / 4;
  colsum_fixed_kernel<<<(unsigned)((W4 + 7) / 8), 256, 0, stream>>>(X, ld, M, (int)W4, out);
  B200_LAUNCH_OK("colsum_fixed_kernel");
  return 0;
}

static int reverse_scan_rows(float* t, int V, int C, cudaStream_t stream) {
  reverse_scan_rows_kernel<<<rq_grid(V, 8), 256, 0, stream>>>(t, V, C);
  B200_LAUNCH_OK("reverse_scan_rows_kernel");
  return 0;
}

extern "C" int b200vq_rq_embed_fwd(const long long* conds, const long long* codes, const float* Wc, const float* pos_c,
                                   const float* Wi, const float* pos_i, float* x, int B, int Tc, int T, int D, int C, int Vc, int Vi,
                                   void* streamv) {
  const cudaStream_t stream = static_cast<cudaStream_t>(streamv);
  if (int rc = embed_shape_ok(B, Tc, T, D, C, Vc, Vi, "rq_embed_fwd")) return rc;
  B200_CHECK_ARG(codes && Wi && pos_i && x && (Tc == 0 || (conds && Wc && pos_c)), "rq_embed_fwd: null pointer argument");
  rq_embed_fwd_kernel<<<rq_grid((long long)B * (Tc + T), 8), 256, 0, stream>>>(conds, codes, Wc, pos_c, Wi, pos_i, x, B, Tc, T, D, C,
                                                                              Vc, Vi);
  B200_LAUNCH_OK("rq_embed_fwd_kernel");
  return 0;
}

// gWc / gWi zero-filled, then the cond rows and the code rows scattered with atomics; gpos = column sums over the batch;
// gWi reverse-scanned
extern "C" int b200vq_rq_embed_bwd(const long long* conds, const long long* codes, const float* g, float* gWc, float* gpos_c,
                                   float* gWi, float* gpos_i, int B, int Tc, int T, int D, int C, int Vc, int Vi,
                                   void* streamv) {
  const cudaStream_t stream = static_cast<cudaStream_t>(streamv);
  if (int rc = embed_shape_ok(B, Tc, T, D, C, Vc, Vi, "rq_embed_bwd")) return rc;
  B200_CHECK_ARG(codes && g && gWi && gpos_i && (Tc == 0 || (conds && gWc && gpos_c)), "rq_embed_bwd: null pointer argument");
  const int Tt = Tc + T;
  if (Tc > 0) {
    B200_CUDA_OK(cudaMemsetAsync(gWc, 0, (size_t)Vc * C * sizeof(float), stream));
    scatter_rows_atomic_kernel<<<rq_grid((long long)B * Tc * (C / 4), 256), 256, 0, stream>>>(conds, (long long)B * Tc, IdMap{Tc, Tc, 1, 0}, g,
                                                                                             Tt, 0, C, gWc, Vc);
    B200_LAUNCH_OK("scatter_rows_atomic_kernel");
    if (int rc = colsum_fixed(g, (long long)Tt * C, B, (long long)Tc * C, gpos_c, stream)) return rc;
  } else if (gWc && Vc > 0) {                             // no cond rows: the cond table's gradient is zero
    B200_CUDA_OK(cudaMemsetAsync(gWc, 0, (size_t)Vc * C * sizeof(float), stream));
  }
  B200_CUDA_OK(cudaMemsetAsync(gWi, 0, (size_t)Vi * C * sizeof(float), stream));
  scatter_rows_atomic_kernel<<<rq_grid((long long)B * T * (C / 4), 256), 256, 0, stream>>>(codes, (long long)B * T, IdMap{T, (long long)T * D, D, D - 1},
                                                                                          g, Tt, Tc, C, gWi, Vi);
  B200_LAUNCH_OK("scatter_rows_atomic_kernel");
  if (int rc = colsum_fixed(g + (long long)Tc * C, (long long)Tt * C, B, (long long)T * C, gpos_i, stream)) return rc;
  return reverse_scan_rows(gWi, Vi, C, stream);
}

static size_t align256(size_t n) { return (n + 255) & ~(size_t)255; }

extern "C" size_t b200vq_rq_embed_bwd_deterministic_workspace_bytes(int B, int Tc, int T, int D, int C, int Vc, int Vi) {
  if (B <= 0 || Tc < 0 || T <= 0 || C <= 0 || D < 1 || Vi <= 0) return 0;
  const size_t wc = (Tc > 0 && Vc > 0) ? scatter_det_workspace_bytes((long long)B * Tc, Vc, C, kScatterRunToken) : 0;
  const size_t wi = scatter_det_workspace_bytes((long long)B * T, Vi, C, kScatterRunToken);
  return align256((size_t)B * T * sizeof(long long)) + (wc > wi ? wc : wi);
}

extern "C" int b200vq_rq_embed_bwd_deterministic(const long long* conds, const long long* codes, const float* g, float* gWc,
                                                 float* gpos_c, float* gWi, float* gpos_i, int B, int Tc, int T, int D, int C, int Vc,
                                                 int Vi, void* workspace, size_t ws_bytes, void* streamv) {
  const cudaStream_t stream = static_cast<cudaStream_t>(streamv);
  if (int rc = embed_shape_ok(B, Tc, T, D, C, Vc, Vi, "rq_embed_bwd_deterministic")) return rc;
  B200_CHECK_ARG(codes && g && gWi && gpos_i && workspace && (Tc == 0 || (conds && gWc && gpos_c)),
                 "rq_embed_bwd_deterministic: null pointer argument");
  B200_CHECK_ARG((long long)B * (Tc + T) <= (1LL << 30), "rq_embed_bwd_deterministic: too many tokens");
  B200_CHECK_ARG(ws_bytes >= b200vq_rq_embed_bwd_deterministic_workspace_bytes(B, Tc, T, D, C, Vc, Vi),
                 "rq_embed_bwd_deterministic: workspace too small");
  const long long Tt = Tc + T;
  long long* ids = static_cast<long long*>(workspace);
  const size_t id_bytes = align256((size_t)B * T * sizeof(long long));
  void* sws = static_cast<char*>(workspace) + id_bytes;
  const size_t sws_bytes = ws_bytes - id_bytes;
  if (Tc > 0) {
    if (int rc = scatter_rows_det<kScatterRunToken>(conds, (long long)B * Tc, Vc, g, Tc, Tt, 0, C, gWc, sws, sws_bytes, stream)) return rc;
    if (int rc = colsum_fixed(g, Tt * C, B, (long long)Tc * C, gpos_c, stream)) return rc;
  } else if (gWc && Vc > 0) {
    B200_CUDA_OK(cudaMemsetAsync(gWc, 0, (size_t)Vc * C * sizeof(float), stream));
  }
  compact_ids_kernel<<<rq_grid((long long)B * T, 256), 256, 0, stream>>>(codes, (long long)B * T, IdMap{T, (long long)T * D, D, D - 1}, ids);
  B200_LAUNCH_OK("compact_ids_kernel");
  if (int rc = scatter_rows_det<kScatterRunToken>(ids, (long long)B * T, Vi, g, T, Tt, Tc, C, gWi, sws, sws_bytes, stream)) return rc;
  if (int rc = colsum_fixed(g + (long long)Tc * C, Tt * C, B, (long long)T * C, gpos_i, stream)) return rc;
  return reverse_scan_rows(gWi, Vi, C, stream);
}

static int depth_shape_ok(long long nseq, int D, int C, int Vi, const char* what) {
  B200_CHECK_ARG(nseq > 0 && C > 0 && C % 4 == 0 && Vi > 0, "%s: bad shape (sequences=%lld C=%d V=%d)", what, nseq, C, Vi);
  B200_CHECK_ARG(D >= 1 && D <= kShortMaxD, "%s: depth must be 1..%d (got %d)", what, kShortMaxD, D);
  B200_CHECK_ARG(nseq * D <= (1LL << 30), "%s: too many tokens", what);
  return 0;
}

extern "C" int b200vq_rq_depth_input_fwd(const float* h, const long long* codes, const float* Wi, const float* pos_d, float* v,
                                         long long nseq, int D, int C, int Vi, void* streamv) {
  const cudaStream_t stream = static_cast<cudaStream_t>(streamv);
  if (int rc = depth_shape_ok(nseq, D, C, Vi, "rq_depth_input_fwd")) return rc;
  B200_CHECK_ARG(h && codes && Wi && v && (D == 1 || pos_d), "rq_depth_input_fwd: null pointer argument");
  rq_depth_input_fwd_kernel<<<rq_grid(nseq * D, 8), 256, 0, stream>>>(h, codes, Wi, pos_d, v, nseq, D, C, Vi);
  B200_LAUNCH_OK("rq_depth_input_fwd_kernel");
  return 0;
}

// gh = the row-0 gradients; gpos_d = column sums of rows d >= 1 over the sequences; gWi from rows d >= 1
static int depth_common_bwd(const float* g, float* gh, float* gpos_d, long long nseq, int D, int C, cudaStream_t stream) {
  B200_CUDA_OK(cudaMemcpy2DAsync(gh, (size_t)C * sizeof(float), g, (size_t)D * C * sizeof(float), (size_t)C * sizeof(float), (size_t)nseq,
                                 cudaMemcpyDeviceToDevice, stream));
  if (D > 1) return colsum_fixed(g + C, (long long)D * C, nseq, (long long)(D - 1) * C, gpos_d, stream);
  return 0;
}

extern "C" int b200vq_rq_depth_input_bwd(const long long* codes, const float* g, float* gh, float* gWi, float* gpos_d, long long nseq,
                                         int D, int C, int Vi, void* streamv) {
  const cudaStream_t stream = static_cast<cudaStream_t>(streamv);
  if (int rc = depth_shape_ok(nseq, D, C, Vi, "rq_depth_input_bwd")) return rc;
  B200_CHECK_ARG(codes && g && gh && gWi && (D == 1 || gpos_d), "rq_depth_input_bwd: null pointer argument");
  B200_CUDA_OK(cudaMemsetAsync(gWi, 0, (size_t)Vi * C * sizeof(float), stream));
  if (D > 1) {
    const long long N = nseq * (D - 1);
    scatter_rows_atomic_kernel<<<rq_grid(N * (C / 4), 256), 256, 0, stream>>>(codes, N, IdMap{D - 1, D, 1, 0}, g, D, 1, C, gWi, Vi);
    B200_LAUNCH_OK("scatter_rows_atomic_kernel");
  }
  if (int rc = depth_common_bwd(g, gh, gpos_d, nseq, D, C, stream)) return rc;
  return reverse_scan_rows(gWi, Vi, C, stream);
}

extern "C" size_t b200vq_rq_depth_input_bwd_deterministic_workspace_bytes(long long nseq, int D, int C, int Vi) {
  if (nseq <= 0 || D < 2 || C <= 0 || Vi <= 0) return 0;
  const long long N = nseq * (D - 1);
  return align256((size_t)N * sizeof(long long)) + scatter_det_workspace_bytes(N, Vi, C, kScatterRunToken);
}

extern "C" int b200vq_rq_depth_input_bwd_deterministic(const long long* codes, const float* g, float* gh, float* gWi, float* gpos_d,
                                                       long long nseq, int D, int C, int Vi, void* workspace, size_t ws_bytes,
                                                       void* streamv) {
  const cudaStream_t stream = static_cast<cudaStream_t>(streamv);
  if (int rc = depth_shape_ok(nseq, D, C, Vi, "rq_depth_input_bwd_deterministic")) return rc;
  B200_CHECK_ARG(codes && g && gh && gWi && (D == 1 || (gpos_d && workspace)), "rq_depth_input_bwd_deterministic: null pointer argument");
  B200_CHECK_ARG(nseq * D <= (1LL << 30), "rq_depth_input_bwd_deterministic: too many tokens");
  B200_CHECK_ARG(ws_bytes >= b200vq_rq_depth_input_bwd_deterministic_workspace_bytes(nseq, D, C, Vi),
                 "rq_depth_input_bwd_deterministic: workspace too small");
  if (D > 1) {
    const long long N = nseq * (D - 1);
    long long* ids = static_cast<long long*>(workspace);
    const size_t id_bytes = align256((size_t)N * sizeof(long long));
    compact_ids_kernel<<<rq_grid(N, 256), 256, 0, stream>>>(codes, N, IdMap{D - 1, D, 1, 0}, ids);
    B200_LAUNCH_OK("compact_ids_kernel");
    if (int rc = scatter_rows_det<kScatterRunToken>(ids, N, Vi, g, D - 1, D, 1, C, gWi, static_cast<char*>(workspace) + id_bytes,
                                                    ws_bytes - id_bytes, stream))
      return rc;
  } else {
    B200_CUDA_OK(cudaMemsetAsync(gWi, 0, (size_t)Vi * C * sizeof(float), stream));
  }
  if (int rc = depth_common_bwd(g, gh, gpos_d, nseq, D, C, stream)) return rc;
  return reverse_scan_rows(gWi, Vi, C, stream);
}

extern "C" int b200vq_code_sum_embed(const long long* codes, long long ld, int n, const float* Wi, const float* pos, float* out,
                                     int B, int C, int Vi, void* streamv) {
  const cudaStream_t stream = static_cast<cudaStream_t>(streamv);
  B200_CHECK_ARG(codes && Wi && pos && out, "code_sum_embed: null pointer argument");
  B200_CHECK_ARG(B > 0 && C > 0 && C % 4 == 0 && Vi > 0 && n >= 1 && ld >= n, "code_sum_embed: bad shape (B=%d n=%d ld=%lld C=%d)", B, n,
                 ld, C);
  code_sum_embed_kernel<<<rq_grid((long long)B * (C / 4), 256), 256, 0, stream>>>(codes, ld, n, Wi, pos, out, B, C, Vi);
  B200_LAUNCH_OK("code_sum_embed_kernel");
  return 0;
}
