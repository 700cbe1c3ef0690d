// Deterministic "sum rows by id": out[v] = sum over the entries e with id(e) == v of row(e), in ascending entry order.
// The opt-in bit-reproducible backward of the codebook (vq.cu) and of the stage-2 token embeddings (stage2.cu) reduce
// through it instead of float atomics.  Two stages, no atomics of any kind, launch geometry from the shape alone:
//
//   1. stable LSD radix sort of the entry indices by id, on the ceil(log2 V) bits of the id, in passes of at most 8 bits.
//      One warp owns a tile of kSortTile entries.  Per pass: every tile counts its digits (sort_hist_kernel), one CTA
//      scans the digit-major [digit][tile] count table (sort_scan_kernel), and every tile scatters its entries to
//      offset[digit][tile] + their rank among the tile's equal digits (sort_scatter_kernel).  The rank comes from
//      __match_any_sync over each 32-entry step, taken in entry order, so the sort is stable; since every (id, entry)
//      pair is distinct, any stable sort yields this one permutation.
//   2. fixed-order segmented row sum.  The sorted array is cut into runs of R positions.  One group of lanes per run
//      walks it in order, one lane per column, and sums each id's piece sequentially (seg_run_kernel).  A piece that is
//      the whole segment is stored straight to out; a piece of a segment that crosses a run boundary is stored as that
//      run's head or tail partial.  seg_join_kernel then adds each crossing segment's partials in run order and
//      zero-fills the ids no entry names.
//
// The summation order therefore depends on the ids and the shape only: not on the SM count, the SM limit or timing.
#include "common.cuh"
#include "scatter_det.cuh"

namespace b200 {

constexpr int kSortItems = 16;                   // entries per lane per tile
constexpr int kSortTile = 32 * kSortItems;       // one warp per tile
constexpr int kSortWarps = 4;                    // tiles per CTA
constexpr int kDigitBits = 8;                    // at most 256 buckets per pass
constexpr int kScanThreads = 1024;
constexpr int kSegThreads = 256;
constexpr int kSegBatch = 8;                     // positions loaded ahead of the sequential adds

static inline size_t align256(size_t b) { return (b + 255) & ~size_t(255); }

// id of position i: in the first pass straight from the caller's int64 ids (clamped into [0, V), as the gathers that
// produced the rows clamp them), afterwards from the previous pass's sorted keys
__device__ __forceinline__ int sort_key(const long long* __restrict__ ids, const int* __restrict__ keys, int i, int V) {
  if (keys) return keys[i];
  const long long id = ids[i];
  return id < 0 ? 0 : (id >= V ? V - 1 : (int)id);
}

__global__ void __launch_bounds__(32 * kSortWarps)
sort_hist_kernel(const long long* __restrict__ ids, const int* __restrict__ keys, int N, int V, int shift, int nd, int ntiles,
                 int* __restrict__ hist) {
  __shared__ int cnt[kSortWarps][1 << kDigitBits];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tile = blockIdx.x * kSortWarps + warp;
  if (tile >= ntiles) return;                    // whole warp
  for (int d = lane; d < nd; d += 32) cnt[warp][d] = 0;
  __syncwarp();
#pragma unroll 4
  for (int it = 0; it < kSortItems; ++it) {
    const int i = tile * kSortTile + it * 32 + lane;
    const int d = i < N ? (sort_key(ids, keys, i, V) >> shift) & (nd - 1) : -1;
    const unsigned peers = __match_any_sync(0xffffffffu, d);
    if (d >= 0 && lane == __ffs(peers) - 1) cnt[warp][d] += __popc(peers);   // one leader per digit: no race
    __syncwarp();
  }
  for (int d = lane; d < nd; d += 32) hist[(size_t)d * ntiles + tile] = cnt[warp][d];
}

// exclusive prefix sum of a[0, n) in place, one CTA, in chunks of 4 * kScanThreads
__global__ void __launch_bounds__(kScanThreads)
sort_scan_kernel(int* __restrict__ a, int n) {
  __shared__ int wsum[kScanThreads / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int carry = 0;
  for (int base = 0; base < n; base += 4 * kScanThreads) {
    const int i = base + threadIdx.x * 4;
    int v[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) v[k] = i + k < n ? a[i + k] : 0;
    const int s = v[0] + v[1] + v[2] + v[3];
    int x = s;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, x, o);
      if (lane >= o) x += y;
    }
    if (lane == 31) wsum[warp] = x;
    __syncthreads();
    if (warp == 0) {
      int w = wsum[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, w, o);
        if (lane >= o) w += y;
      }
      wsum[lane] = w;
    }
    __syncthreads();
    int run = carry + (warp ? wsum[warp - 1] : 0) + x - s;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (i + k < n) a[i + k] = run;
      run += v[k];
    }
    carry += wsum[kScanThreads / 32 - 1];
    __syncthreads();                             // wsum is rewritten by the next chunk
  }
}

__global__ void __launch_bounds__(32 * kSortWarps)
sort_scatter_kernel(const long long* __restrict__ ids, const int* __restrict__ keys, const int* __restrict__ vals, int N, int V,
                    int shift, int nd, int ntiles, const int* __restrict__ offs, int* __restrict__ keys_out, int* __restrict__ vals_out) {
  __shared__ int cnt[kSortWarps][1 << kDigitBits];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tile = blockIdx.x * kSortWarps + warp;
  if (tile >= ntiles) return;
  for (int d = lane; d < nd; d += 32) cnt[warp][d] = offs[(size_t)d * ntiles + tile];
  __syncwarp();
  const unsigned lt = (1u << lane) - 1u;
#pragma unroll 4
  for (int it = 0; it < kSortItems; ++it) {
    const int i = tile * kSortTile + it * 32 + lane;
    int k = 0, d = -1;
    if (i < N) {
      k = sort_key(ids, keys, i, V);
      d = (k >> shift) & (nd - 1);
    }
    const unsigned peers = __match_any_sync(0xffffffffu, d);
    const int base = d >= 0 ? cnt[warp][d] : 0;
    if (d >= 0) {
      const int pos = base + __popc(peers & lt);   // lanes below me with my digit come first: stable
      keys_out[pos] = k;
      vals_out[pos] = vals ? vals[i] : i;
    }
    __syncwarp();                                  // every peer has read `base`
    if (d >= 0 && lane == __ffs(peers) - 1) cnt[warp][d] = base + __popc(peers);
    __syncwarp();
  }
}

// seg_begin[v] / seg_end[v]: the positions of id v in the sorted keys (both 0 when v does not occur)
__global__ void __launch_bounds__(256)
seg_bounds_kernel(const int* __restrict__ skeys, int N, int* __restrict__ seg_begin, int* __restrict__ seg_end) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  const int k = skeys[i];
  if (i == 0 || skeys[i - 1] != k) seg_begin[k] = i;
  if (i == N - 1 || skeys[i + 1] != k) seg_end[k] = i + 1;
}

// entry e -> its row: rows + ((e / Tn) * T + off + e % Tn) * C  (a [B, T, C] tensor whose rows off .. off + Tn - 1 of
// every batch entry are the entries, in order; a plain [N, C] matrix is Tn = N, T = 0, off = 0)
// (row indices fit in an int: scatter_rows_det checks the map against N before launching)
struct RowMap {
  const float* rows;
  int Tn, T, off;
};
__device__ __forceinline__ const float* row_of(const RowMap& rm, int e, int C) {
  const int b = e / rm.Tn;
  return rm.rows + (long long)(b * rm.T + rm.off + (e - b * rm.Tn)) * C;
}

// lanes per run group: one per column up to kSegThreads, a power of two so groups tile the CTA
static inline int seg_lanes(int C) {
  int t = 1;
  while (t < C && t < kSegThreads) t <<= 1;
  return t;
}

template <int R>
__global__ void __launch_bounds__(kSegThreads)
seg_run_kernel(const int* __restrict__ skeys, const int* __restrict__ svals, int N, RowMap rm, int C, int lanes, int nruns,
               float* __restrict__ out, float* __restrict__ p_head, float* __restrict__ p_tail) {
  const int run = blockIdx.x * (kSegThreads / lanes) + threadIdx.x / lanes;
  if (run >= nruns) return;
  const int sub = threadIdx.x % lanes;
  const int i0 = run * R, i1 = min(N, i0 + R);
  const int kprev = i0 > 0 ? skeys[i0 - 1] : -1;
  const int knext = i1 < N ? skeys[i1] : -1;
  for (int c = sub; c < C; c += lanes) {
    float acc = 0.f;
    int piece = i0;                                // first position of the current id's piece
    for (int b = i0; b < i1; b += kSegBatch) {
      int kk[kSegBatch + 1];
      float vv[kSegBatch];
#pragma unroll
      for (int j = 0; j < kSegBatch; ++j) {
        const bool ok = b + j < i1;
        kk[j] = ok ? skeys[b + j] : -2;
        vv[j] = ok ? row_of(rm, svals[b + j], C)[c] : 0.f;
      }
      kk[kSegBatch] = b + kSegBatch < i1 ? skeys[b + kSegBatch] : -2;   // the run's end closes its last piece
#pragma unroll
      for (int j = 0; j < kSegBatch; ++j) {
        if (b + j >= i1) break;
        acc += vv[j];
        if (kk[j + 1] != kk[j]) {
          const int k = kk[j];
          const bool from_before = piece == i0 && kprev == k;   // the segment began in an earlier run
          const bool goes_on = b + j + 1 == i1 && knext == k;   // ... or continues into a later one
          if (from_before)  p_head[(size_t)run * C + c] = acc;
          else if (goes_on) p_tail[(size_t)run * C + c] = acc;
          else              out[(size_t)k * C + c] = acc;
          acc = 0.f;
          piece = b + j + 1;
        }
      }
    }
  }
}

// segments that cross a run boundary: tail partial of their first run + head partials of the following runs, in run
// order; ids without entries: zero rows
__global__ void __launch_bounds__(kSegThreads)
seg_join_kernel(const int* __restrict__ seg_begin, const int* __restrict__ seg_end, const float* __restrict__ p_head,
                const float* __restrict__ p_tail, float* __restrict__ out, int V, int C, int lanes, int R) {
  const int v = blockIdx.x * (kSegThreads / lanes) + threadIdx.x / lanes;
  if (v >= V) return;
  const int sub = threadIdx.x % lanes;
  const int s = seg_begin[v], e = seg_end[v];
  if (s == e) {
    for (int c = sub; c < C; c += lanes) out[(size_t)v * C + c] = 0.f;
    return;
  }
  const int r0 = s / R, r1 = (e - 1) / R;
  if (r0 == r1) return;                            // stored whole by seg_run_kernel
  for (int c = sub; c < C; c += lanes) {
    float acc = p_tail[(size_t)r0 * C + c];
#pragma unroll 8
    for (int r = r0 + 1; r <= r1; ++r) acc += p_head[(size_t)r * C + c];
    out[(size_t)v * C + c] = acc;
  }
}

// ---------------------------------------------------------------------------------------------
struct ScatterLayout {
  int ntiles, nruns;
  size_t keys0, vals0, keys1, vals1, hist, seg_begin, seg_end, p_head, p_tail, total;
};
static ScatterLayout scatter_layout(long long N, int V, int C, int R) {
  ScatterLayout L{};
  L.ntiles = (int)((N + kSortTile - 1) / kSortTile);
  L.nruns = (int)((N + R - 1) / R);
  size_t o = 0;
  auto take = [&](size_t bytes) { const size_t at = o; o += align256(bytes); return at; };
  L.keys0 = take((size_t)N * 4);
  L.vals0 = take((size_t)N * 4);
  L.keys1 = take((size_t)N * 4);
  L.vals1 = take((size_t)N * 4);
  L.hist = take((size_t)(1 << kDigitBits) * L.ntiles * 4);
  L.seg_begin = take((size_t)V * 4);
  L.seg_end = take((size_t)V * 4);
  L.p_head = take((size_t)L.nruns * C * 4);
  L.p_tail = take((size_t)L.nruns * C * 4);
  L.total = o;
  return L;
}

size_t scatter_det_workspace_bytes(long long N, int V, int C, int R) { return N > 0 ? scatter_layout(N, V, C, R).total : 0; }

template <int R>
int scatter_rows_det(const long long* ids, long long N, int V, const float* rows, long long Tn, long long T, long long off, int C,
                     float* out, void* workspace, size_t ws_bytes, cudaStream_t stream) {
  B200_CHECK_ARG(N >= 0 && N <= (1LL << 30) && V > 0 && C > 0, "scatter_det: bad shape N=%lld V=%d C=%d", N, V, C);
  if (N == 0) {                                    // no entries: every row of out is zero
    B200_CUDA_OK(cudaMemsetAsync(out, 0, (size_t)V * C * sizeof(float), stream));
    return 0;
  }
  B200_CHECK_ARG(Tn > 0 && T >= 0 && off >= 0 && T <= (1LL << 30) && off <= (1LL << 30) && (N / Tn) * T + off + Tn <= 0x7fffffffLL,
                 "scatter_det: row map out of range (Tn=%lld T=%lld off=%lld)", Tn, T, off);
  const ScatterLayout L = scatter_layout(N, V, C, R);
  B200_CHECK_ARG(ws_bytes >= L.total, "scatter_det: workspace too small");
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  int* kbuf[2] = {reinterpret_cast<int*>(ws + L.keys0), reinterpret_cast<int*>(ws + L.keys1)};
  int* vbuf[2] = {reinterpret_cast<int*>(ws + L.vals0), reinterpret_cast<int*>(ws + L.vals1)};
  int* hist = reinterpret_cast<int*>(ws + L.hist);
  int* seg_begin = reinterpret_cast<int*>(ws + L.seg_begin);
  int* seg_end = reinterpret_cast<int*>(ws + L.seg_end);
  float* p_head = reinterpret_cast<float*>(ws + L.p_head);
  float* p_tail = reinterpret_cast<float*>(ws + L.p_tail);
  const int n = (int)N;

  int bits = 0;
  while ((1LL << bits) < V) ++bits;
  const int npass = bits == 0 ? 1 : (bits + kDigitBits - 1) / kDigitBits;
  const int width = (bits + npass - 1) / npass;
  const int sort_blocks = (L.ntiles + kSortWarps - 1) / kSortWarps;
  const int* keys = nullptr;                       // first pass: read (and clamp) the caller's ids
  const int* vals = nullptr;                       // first pass: the entry index itself
  for (int p = 0; p < npass; ++p) {
    const int shift = p * width;
    const int w = min(width, bits - shift);
    const int nd = 1 << (w > 0 ? w : 0);
    sort_hist_kernel<<<sort_blocks, 32 * kSortWarps, 0, stream>>>(ids, keys, n, V, shift, nd, L.ntiles, hist);
    B200_LAUNCH_OK("sort_hist_kernel");
    sort_scan_kernel<<<1, kScanThreads, 0, stream>>>(hist, nd * L.ntiles);
    B200_LAUNCH_OK("sort_scan_kernel");
    sort_scatter_kernel<<<sort_blocks, 32 * kSortWarps, 0, stream>>>(ids, keys, vals, n, V, shift, nd, L.ntiles, hist, kbuf[p & 1],
                                                                      vbuf[p & 1]);
    B200_LAUNCH_OK("sort_scatter_kernel");
    keys = kbuf[p & 1];
    vals = vbuf[p & 1];
  }

  B200_CUDA_OK(cudaMemsetAsync(seg_begin, 0, L.seg_end + (size_t)V * 4 - L.seg_begin, stream));
  seg_bounds_kernel<<<(n + 255) / 256, 256, 0, stream>>>(keys, n, seg_begin, seg_end);
  B200_LAUNCH_OK("seg_bounds_kernel");
  const int lanes = seg_lanes(C);
  const int groups = kSegThreads / lanes;
  const RowMap rm{rows, (int)Tn, (int)T, (int)off};
  seg_run_kernel<R><<<(L.nruns + groups - 1) / groups, kSegThreads, 0, stream>>>(keys, vals, n, rm, C, lanes, L.nruns, out, p_head, p_tail);
  B200_LAUNCH_OK("seg_run_kernel");
  seg_join_kernel<<<(V + groups - 1) / groups, kSegThreads, 0, stream>>>(seg_begin, seg_end, p_head, p_tail, out, V, C, lanes, R);
  B200_LAUNCH_OK("seg_join_kernel");
  return 0;
}

// the run lengths of the two callers: the codebook (32-float rows, up to M * depth entries on a few dozen ids) and the
// token embeddings (C-float rows, B * T entries)
template int scatter_rows_det<kScatterRunVq>(const long long*, long long, int, const float*, long long, long long, long long, int, float*,
                                             void*, size_t, cudaStream_t);
template int scatter_rows_det<kScatterRunToken>(const long long*, long long, int, const float*, long long, long long, long long, int,
                                                float*, void*, size_t, cudaStream_t);

}  // namespace b200
