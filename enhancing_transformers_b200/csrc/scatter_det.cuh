// Deterministic "sum rows by id" (scatter_det.cu): out[v] = sum of row(e) over the entries e with ids[e] == v, summed in
// ascending entry order within fixed runs of R sorted positions and the runs in order.  No atomics; the summation order
// and the launch geometry depend on the ids and the shape only.  Used by the opt-in bit-reproducible backward of the
// codebook (vq.cu) and of the stage-2 token embeddings (stage2.cu).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

namespace b200 {

constexpr int kScatterRunVq = 128;      // D-float codebook rows: up to M * depth entries, often on a few dozen ids
constexpr int kScatterRunToken = 32;    // C-float embedding rows: B * T entries

size_t scatter_det_workspace_bytes(long long N, int V, int C, int R);
// ids int64 [N] (clamped into [0, V)); entry e's row: rows + ((e / Tn) * T + off + e % Tn) * C; out [V, C] (every row
// written).  Validates its arguments before any CUDA call.
template <int R>
int scatter_rows_det(const long long* ids, long long N, int V, const float* rows, long long Tn, long long T, long long off, int C,
                     float* out, void* workspace, size_t ws_bytes, cudaStream_t stream);

}  // namespace b200
