// Persistent tensor-core GEMM for sm_90a: TMA -> 128B-swizzled smem ring (mbarrier full / empty pairs) ->
// mma.sync on eight consumer warps (fp32 accumulators in registers) -> fused epilogue stored straight from
// registers.  Replaces every cuBLAS/cuDNN call the reference issues for nn.Linear / Conv2d(k=s) /
// ConvTranspose2d(k=s) on the hot path (reference enhancing/modules/stage1/layers.py:99-101,118-132,168-171,
// 202-205) and their dgrad / wgrad.
//
//   C[M,N] = epilogue( alpha * sum_k A[m,k] * B[n,k] )              (per split z)
//
// Operand kinds (template KIND):
//   0  fp32 storage, mma.sync m16n8k8 .tf32 (the tensor core keeps 10 mantissa bits: operands are rounded to
//      nearest where they are produced).  With passes == 3 the contraction runs three times over
//      (A_lo, B), (A, B_lo), (A, B) -- the error-compensated "3xTF32" product (lo = x - trunc_tf32(x),
//      written by split_tf32_lo): fp32-grade results for the parity mode, at a third of the rate.
//   1  fp16 storage, wgmma m64n256k16 .f16 straight from the swizzled tiles (either major: wgmma transposes fp16
//      operands itself), fp32 accumulate: the same 11-bit significand as tf32 at twice
//      the tensor rate and half the operand bytes; gradients travel scaled by a power of two (alpha
//      undoes it), so fp16's narrower exponent range is never the limit.
// Output: fp32 (optionally tf32-rounded) or, with OUT16, fp16 (saturating).
//
// Operand storage ("major"):
//   a_major = 0 : A is [M, K]        row-major, K contiguous   (K-major)
//   a_major = 1 : A is [K_total, M]  row-major, M contiguous   (MN-major; wgrad reads dY^T)
//   b_major = 0 : B is [N, K]        row-major                 (nn.Linear weight)
//   b_major = 1 : B is [K_total, N]  row-major                 (dgrad reads W, wgrad reads X)
// Split-K: split z contracts rows/cols [z*K, (z+1)*K) and writes C + z*c_split_stride.
//
// Why the tf32 kinds use mma.sync: Hopper's wgmma reads tf32 operands from shared memory in K-major form only, and the
// dgrad / wgrad products of the tf32 and parity data paths read MN-major operands.  Their mma.sync fragments are gathered
// by the consumer warps themselves (scalar loads from the swizzled tiles), behind the same TMA ring and epilogue.
//
// Warp roles (288 threads): warps 0..7 consume, warp 8 is the TMA producer.  fp16: warpgroup w (warps 4w..4w+3) owns
// rows 64w .. 64w+63 of the 128 x 256 tile (warp 4w+i: rows 64w+16i .. +15); tf32: warp w owns rows 32*(w%4) .. +31
// and half of the BN columns.
#include "../../include/b200vq.h"
#include "common.cuh"

#include <mutex>
#include <type_traits>
#include <unordered_map>

namespace b200 {

struct GemmParams {
  int M, N, K;                 // output rows / cols, contraction length per split
  int num_m_blocks;            // ceil(M / 128)
  int num_n_blocks;            // ceil(N / BN)
  int num_splits;
  int k_blocks;                // ceil(K / BK)
  void* C;                     // fp32 or (OUT16) fp16
  long long ldc, c_split_stride;
  const float* alpha_ptr;      // device scalar multiplied into the accumulators (null = 1): undoes gradient scaling
  int passes;                  // 1, or 3 for the 3xTF32 split-operand product (KIND 0 only)
  const float* bias;           // [N] or null
  const float* res;            // residual row (row % res_row_mod) added in the epilogue, or null
  long long ldres;
  int res_row_mod;
  const void* in;              // in_mode 1: fp32 residual [M, ldin]; in_mode 2: tanh' input, output dtype [M, ldin]
  long long ldin;
  int in_mode;                 // 0 none, 1: + in (residual), 2: * (1 - in^2) (tanh backward)
  int act;                     // 0 none, 1 tanh
  int round_out;               // 1: round the stored value to tf32 (it only feeds another GEMM)
  float* colsum_part;          // null, or [ceil(M/16)][N]: column sums of every 16-row group of the stored C
};

constexpr int kBM = 128;
constexpr int kBNHalf = 256;      // tile width of the fp16 kind (ops.GEMM_TILE mirrors it for the split-K model)
constexpr int kConsumerWarps = 8;
constexpr int kGemmThreads = 32 * (kConsumerWarps + 1);

// per operand kind: a k-block is one 128-byte swizzle row of the operand's element type
template <int KIND> struct Elem;
template <> struct Elem<0> { static constexpr int BYTES = 4, BK = 32, ATOM = 32, MMA_K = 8; };
template <> struct Elem<1> { static constexpr int BYTES = 2, BK = 64, ATOM = 64, MMA_K = 16; };

template <int BN>
struct GemmCfg {
  static constexpr int A_BYTES = kBM * 128;       // 128 rows (or k-rows x atoms) of 128 bytes, either kind
  static constexpr int B_BYTES = BN * 128;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int MAX_SMEM = 232448;         // 227 KB opt-in limit
  static constexpr int RING_BUDGET = MAX_SMEM - 1024 - 256;
  static constexpr int STAGES = (RING_BUDGET / STAGE_BYTES) > 8 ? 8 : (RING_BUDGET / STAGE_BYTES);
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
};

// Byte offset of element (mn, k) of a stage tile, as TMA wrote it with SWIZZLE_128B (the tile base is 1024-aligned, so
// the swizzle phase is the 128-byte row index mod 8).
//   K-major : [mn][128 B of k]
//   MN-major: [mn / ATOM][BK k-rows][128 B of mn]
template <int KIND, int MAJ>
__device__ __forceinline__ uint32_t tile_off(int mn, int k) {
  using El = Elem<KIND>;
  if constexpr (MAJ == 0) {
    const uint32_t b = (uint32_t)k * El::BYTES;
    return (uint32_t)mn * 128u + ((((b >> 4) ^ (uint32_t)mn) & 7u) << 4) + (b & 15u);
  } else {
    const uint32_t b = (uint32_t)(mn % El::ATOM) * El::BYTES;
    return (uint32_t)(mn / El::ATOM) * (El::BK * 128u) + (uint32_t)k * 128u + ((((b >> 4) ^ (uint32_t)k) & 7u) << 4) + (b & 15u);
  }
}

__device__ __forceinline__ float2 pair_to_float2(float2 v) { return v; }
__device__ __forceinline__ float2 pair_to_float2(uint32_t v) { return __half22float2(*reinterpret_cast<const __half2*>(&v)); }

// P3: the 3xTF32 product (KIND 0, passes == 3), with per-k-block promotion of the partial sums
template <int KIND, int BN, int AMAJ, int BMAJ, int OUT16, int P3>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
               const __grid_constant__ CUtensorMap tmA2, const __grid_constant__ CUtensorMap tmB2, const GemmParams p) {
  using Cfg = GemmCfg<BN>;
  using El = Elem<KIND>;
  constexpr int kBK = El::BK;
  constexpr int STAGES = Cfg::STAGES;
  constexpr int WN = BN / 2;          // columns per consumer warp
  constexpr int NT = WN / 8;          // n8 tiles per consumer warp
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_align1024(smem_raw);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * Cfg::STAGE_BYTES);   // [STAGES]
  uint64_t* empty_bar = full_bar + STAGES;                                               // [STAGES]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);                  // the producer's expect_tx arrival
      mbar_init(&empty_bar[s], kConsumerWarps);    // one arrival per consumer warp
    }
    fence_barrier_init();
  }
  __syncthreads();

  const int tiles_per_split = p.num_m_blocks * p.num_n_blocks;
  const int total_tiles = tiles_per_split * p.num_splits;
  const int kb_total = p.k_blocks * p.passes;

  if (warp == kConsumerWarps) {
    // ---------------------------------------------------------------- TMA producer (one lane)
    if (lane == 0) {
      tma_prefetch_desc(&tmA);
      tma_prefetch_desc(&tmB);
      int stage = 0;
      uint32_t phase = 0;
      for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
        const int z = t / tiles_per_split;
        const int r = t - z * tiles_per_split;
        const int mb = r / p.num_n_blocks, nb = r - mb * p.num_n_blocks;
        const int m0 = mb * kBM, n0 = nb * BN;
        const int kbase = z * p.K;
        for (int pass = 0; pass < p.passes; ++pass) {
          // 3xTF32: (A_lo, B) then (A, B_lo) then (A, B) -- small terms first; a single pass uses (A, B)
          const CUtensorMap* mapA = (p.passes == 3 && pass == 0) ? &tmA2 : &tmA;
          const CUtensorMap* mapB = (p.passes == 3 && pass == 1) ? &tmB2 : &tmB;
          for (int kb = 0; kb < p.k_blocks; ++kb) {
            mbar_wait(&empty_bar[stage], phase ^ 1);
            uint8_t* sa = smem + stage * Cfg::STAGE_BYTES;
            uint8_t* sb = sa + Cfg::A_BYTES;
            const int k0 = kbase + kb * kBK;
            mbar_arrive_expect_tx(&full_bar[stage], Cfg::STAGE_BYTES);
            if constexpr (AMAJ == 0) tma_load_2d(sa, mapA, &full_bar[stage], k0, m0);
            else                     tma_load_3d(sa, mapA, &full_bar[stage], 0, k0, m0 / El::ATOM);
            if constexpr (BMAJ == 0) tma_load_2d(sb, mapB, &full_bar[stage], k0, n0);
            else                     tma_load_3d(sb, mapB, &full_bar[stage], 0, k0, n0 / El::ATOM);
            if (++stage == STAGES) { stage = 0; phase ^= 1; }
          }
        }
      }
    }
    return;
  }

  // ------------------------------------------------------------------ consumers: main loop + epilogue
  const int wm = warp & 3, wn = warp >> 2;
  const int g = lane >> 2, tq = lane & 3;
  const float alpha = p.alpha_ptr ? __ldg(p.alpha_ptr) : 1.f;
  const uint32_t smem_base = smem_u32(smem);
  // accumulator shape per warp: MT m16 tiles x NTW n8 tiles, each in the mma.sync / wgmma fragment layout
  // (c0, c1: row g, columns 2tq, 2tq+1; c2, c3: row g + 8)
  constexpr bool WG = KIND == 1;
  constexpr int MT = WG ? 1 : 2;
  constexpr int NTW = WG ? BN / 8 : NT;
  int stage = 0;
  uint32_t phase = 0;
  for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
    const int z = t / tiles_per_split;
    const int r = t - z * tiles_per_split;
    const int mb = r / p.num_n_blocks, nb = r - mb * p.num_n_blocks;
    float acc[MT][NTW][4];
#pragma unroll
    for (int i = 0; i < MT; ++i)
#pragma unroll
      for (int j = 0; j < NTW; ++j) acc[i][j][0] = acc[i][j][1] = acc[i][j][2] = acc[i][j][3] = 0.f;
    // 3xTF32: the tensor core's internal fp32 accumulation truncates, which over a long contraction costs the product
    // its fp32 grade.  Each k-block is therefore summed into a zeroed partial and promoted into acc with a rounded FADD.
    constexpr bool promote = P3 != 0;
    float part[MT][NTW][4];
#pragma unroll
    for (int i = 0; i < MT; ++i)
#pragma unroll
      for (int j = 0; j < NTW; ++j) part[i][j][0] = part[i][j][1] = part[i][j][2] = part[i][j][3] = 0.f;

    float (&d)[BN / 2] = *reinterpret_cast<float(*)[BN / 2]>(&acc[0][0][0]);   // the wgmma accumulator (fp16 kind)
    int held = -1;                                                            // fp16: the stage of the MMAs in flight
    if constexpr (WG) wgmma_fence_regs(d);
    for (int kb = 0; kb < kb_total; ++kb) {
      mbar_wait(&full_bar[stage], phase);
      const uint8_t* sa = smem + stage * Cfg::STAGE_BYTES;
      const uint8_t* sb = sa + Cfg::A_BYTES;
      if constexpr (KIND == 0) {
#pragma unroll
        for (int ks = 0; ks < kBK / El::MMA_K; ++ks) {
          const int k0 = ks * El::MMA_K;
          uint32_t af[2][4], bf[NT][2];
#pragma unroll
          for (int mt = 0; mt < 2; ++mt) {
            const int m = wm * 32 + mt * 16 + g;
            af[mt][0] = *reinterpret_cast<const uint32_t*>(sa + tile_off<0, AMAJ>(m, k0 + tq));
            af[mt][1] = *reinterpret_cast<const uint32_t*>(sa + tile_off<0, AMAJ>(m + 8, k0 + tq));
            af[mt][2] = *reinterpret_cast<const uint32_t*>(sa + tile_off<0, AMAJ>(m, k0 + tq + 4));
            af[mt][3] = *reinterpret_cast<const uint32_t*>(sa + tile_off<0, AMAJ>(m + 8, k0 + tq + 4));
          }
#pragma unroll
          for (int nt = 0; nt < NT; ++nt) {
            const int n = wn * WN + nt * 8 + g;
            bf[nt][0] = *reinterpret_cast<const uint32_t*>(sb + tile_off<0, BMAJ>(n, k0 + tq));
            bf[nt][1] = *reinterpret_cast<const uint32_t*>(sb + tile_off<0, BMAJ>(n, k0 + tq + 4));
          }
          if constexpr (promote) {
#pragma unroll
            for (int mt = 0; mt < 2; ++mt)
#pragma unroll
              for (int nt = 0; nt < NT; ++nt) mma_tf32(part[mt][nt], af[mt], bf[nt][0], bf[nt][1]);
          } else {
#pragma unroll
            for (int mt = 0; mt < 2; ++mt)
#pragma unroll
              for (int nt = 0; nt < NT; ++nt) mma_tf32(acc[mt][nt], af[mt], bf[nt][0], bf[nt][1]);
          }
        }
      } else {
        // one warpgroup-wide MMA per 16-deep k step: A = this warpgroup's 64 rows, B = the whole 256-column tile.
        // (256 rather than 128 columns halves the shared-memory B reads per FLOP and the A loads from L2 per FLOP.)
        // K-major: 8-row groups 1024 B apart (SBO), a k step is 32 B along the row.  MN-major: 64-element atoms
        // kBK*128 B apart (LBO), 8-k-row groups 1024 B apart (SBO), a k step is 16 k-rows = 2048 B.
        const int wg = warp >> 2;
        const uint32_t sa_u = smem_base + stage * Cfg::STAGE_BYTES, sb_u = sa_u + Cfg::A_BYTES;
        const uint32_t a0 = sa_u + wg * (AMAJ ? kBK * 128 : 64 * 128);
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < kBK / El::MMA_K; ++ks) {
          const uint64_t ad = wgmma_desc_sw128(a0 + ks * (AMAJ ? 2048 : 32), kBK * 128, 1024);
          const uint64_t bd = wgmma_desc_sw128(sb_u + ks * (BMAJ ? 2048 : 32), kBK * 128, 1024);
          static_assert(BN == kBNHalf, "the fp16 kind runs on 256-column tiles");
          wgmma_m64n256k16_f16<AMAJ, BMAJ>(d, ad, bd);
        }
        wgmma_commit();
        // one k-block stays in flight, so the tensor pipe is not drained between k-blocks: this wait retires the
        // previous k-block, whose stage the producer may now refill.  MMAs into one accumulator complete in order, so
        // every element still sums its k16 products in k order.
        wgmma_wait<1>();
        if (held >= 0) {
          __syncwarp();
          if (lane == 0) mbar_arrive(&empty_bar[held]);
        }
        held = stage;
      }
      if constexpr (KIND == 0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[stage]);
      }
      if (++stage == STAGES) { stage = 0; phase ^= 1; }
      if constexpr (promote) {
#pragma unroll
        for (int i = 0; i < MT; ++i)
#pragma unroll
          for (int j = 0; j < NTW; ++j)
#pragma unroll
            for (int e = 0; e < 4; ++e) { acc[i][j][e] += part[i][j][e]; part[i][j][e] = 0.f; }
      }
    }

    if constexpr (WG) {
      // ---------------------------------------------------------------- epilogue (rows g, g + 8 of each m16 tile)
      // As far as the compiler knows the output may alias an epilogue input, so it keeps every load below the stores
      // that precede it in the source: loading each n8 tile's inputs right before its stores would cost every warp one
      // memory round trip per n8 tile.  The bias pairs and epilogue-input pairs are therefore loaded ahead of the stores,
      // the first tile's before the last k-block's MMAs are waited for.  The lookahead grows only as fast as the stored
      // tiles free their accumulator registers, up to kAheadMax tiles: ptxas caps the kernel at 168 registers (9 warps at
      // one CTA per SM put 3 warps on one SM sub-partition's 16 K registers), and the fp16 kind's accumulators take 128.
      // The loads are predicated rather than branched over: branches around them cost the allocator spills.  Every element
      // goes through the same operations in the same order as when loaded in place, and is only ever loaded by the thread
      // that stores it, before it stores it, so an output written in place over its epilogue input stays correct.
      //
      // One input slot per element pair ("ex"): the in_mode 1 / 2 input (output dtype), or else the residual-table row.
      // With both (in_mode 2 and a table, fp32 output only) the table row is loaded where it is added.
      using OutT = std::conditional_t<OUT16 != 0, __half, float>;
      using ExPair = std::conditional_t<OUT16 != 0, uint32_t, float2>;   // an fp16 pair travels as its bits
      constexpr int kTileRegs = 2 + MT * 2 * (OUT16 ? 1 : 2);          // one n8 tile's bias and input pairs
      constexpr int kAheadMax = 8;
      const int col0 = nb * BN + 2 * tq;                                // this thread's first column; n8 tile nt adds 8 nt
      const bool has_bias = p.bias != nullptr, ex_is_in = p.in_mode != 0, has_ex = ex_is_in || p.res != nullptr;
      bool row_ok[MT][2];
      OutT* c_row[MT][2];
      const ExPair* ex_row[MT][2];
  #pragma unroll
      for (int mt = 0; mt < MT; ++mt)
  #pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = mb * kBM + warp * 16 + g + h * 8;
          row_ok[mt][h] = row < p.M;
          c_row[mt][h] = static_cast<OutT*>(p.C) + (long long)z * p.c_split_stride + (long long)row * p.ldc + col0;
          ex_row[mt][h] = ex_is_in ? reinterpret_cast<const ExPair*>(static_cast<const OutT*>(p.in) + (long long)row * p.ldin + col0)
                                   : reinterpret_cast<const ExPair*>(p.res + (long long)(row % (p.res_row_mod > 0 ? p.res_row_mod : 1)) * p.ldres + col0);
        }
      float2 bias_v[NTW];
      ExPair ex_v[NTW][MT][2];
      // N is even, so col < N implies col + 1 < N
      auto fetch = [&](int nt) {
        const bool col_ok = col0 + nt * 8 < p.N;
        bias_v[nt] = has_bias && col_ok ? reinterpret_cast<const float2*>(p.bias + col0)[nt * 4] : make_float2(0.f, 0.f);
  #pragma unroll
        for (int mt = 0; mt < MT; ++mt)
  #pragma unroll
          for (int h = 0; h < 2; ++h) ex_v[nt][mt][h] = has_ex && row_ok[mt][h] && col_ok ? ex_row[mt][h][nt * 4] : ExPair{};
      };
      // tiles [0, fetched(nt)) are loaded before tile nt is stored: as many tiles ahead as the accumulator registers of
      // the tiles already stored can hold, at least one and at most kAheadMax.
      auto fetched = [](int nt) {
        int ahead = 4 * MT * nt / kTileRegs;
        ahead = ahead < 1 ? 1 : ahead > kAheadMax ? kAheadMax : ahead;
        return nt + ahead < NTW ? nt + ahead : NTW;
      };
  #pragma unroll
      for (int nt = 0; nt < fetched(0); ++nt) fetch(nt);

      wgmma_wait<0>();
      wgmma_fence_regs(d);
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[held]);

  #pragma unroll
      for (int nt = 0; nt < NTW; ++nt) {
  #pragma unroll
        for (int f = nt == 0 ? fetched(0) : fetched(nt - 1); f < fetched(nt); ++f) fetch(f);
        const int col = col0 + nt * 8;
        const bool col_ok = col < p.N;
        const float2 bias2 = bias_v[nt];
  #pragma unroll
        for (int mt = 0; mt < MT; ++mt) {
          const int row16 = mb * kBM + (WG ? warp * 16 : wm * 32 + mt * 16);
          float cs0 = 0.f, cs1 = 0.f;
  #pragma unroll
          for (int h = 0; h < 2; ++h) {    // row half: g, g + 8
            float o0 = acc[mt][nt][h * 2] * alpha + bias2.x;
            float o1 = acc[mt][nt][h * 2 + 1] * alpha + bias2.y;
            if (!row_ok[mt][h] || !col_ok) continue;
            if (p.act == 1) { o0 = fast_tanh(o0); o1 = fast_tanh(o1); }
            const float2 a = pair_to_float2(ex_v[nt][mt][h]);
            if constexpr (!OUT16) {          // fp16 output takes no fp32 residual (gemm_launch)
              if (p.in_mode == 1) { o0 += a.x; o1 += a.y; }
            }
            if (p.in_mode == 2) { o0 *= 1.f - a.x * a.x; o1 *= 1.f - a.y * a.y; }
            if constexpr (!OUT16) {
              if (p.res) {
                const int row = row16 + g + h * 8;
                const float2 rr = ex_is_in ? *reinterpret_cast<const float2*>(p.res + (long long)(row % p.res_row_mod) * p.ldres + col) : a;
                o0 += rr.x; o1 += rr.y;
              }
            }
            if constexpr (OUT16) {
              const uint32_t pk = pack_half2_sat(o0, o1);
              reinterpret_cast<uint32_t*>(c_row[mt][h])[nt * 4] = pk;
              const float2 st = __half22float2(*reinterpret_cast<const __half2*>(&pk));
              cs0 += st.x; cs1 += st.y;
            } else {
              if (p.round_out) { o0 = round_tf32(o0); o1 = round_tf32(o1); }
              reinterpret_cast<float2*>(c_row[mt][h])[nt * 4] = make_float2(o0, o1);
              cs0 += o0; cs1 += o1;
            }
          }
          if (p.colsum_part) {
            // bias gradient for free: the m16 tile's rows are one 16-row group of the partial-sum table
  #pragma unroll
            for (int off = 4; off < 32; off <<= 1) {
              cs0 += __shfl_xor_sync(0xffffffffu, cs0, off);
              cs1 += __shfl_xor_sync(0xffffffffu, cs1, off);
            }
            if (g == 0 && col_ok && row16 < p.M)
              *reinterpret_cast<float2*>(p.colsum_part + (size_t)(row16 >> 4) * p.N + col) = make_float2(cs0, cs1);
          }
        }
      }
    } else {
      // tf32 kinds: each element pair's inputs are loaded where they are used.  The same loads run ahead of the
      // stores, as above, changed results from launch to launch once a CTA ran several tiles with column sums
      // (test_gemm_epilogue_input_refill_is_race_free): whole n8 tiles of a warp came out wrong, which points at the
      // mma.sync main loop's shared-memory fragment loads and the stage release under a different schedule, not at
      // the epilogue.  Not resolved; these kinds keep the schedule they were validated with.
      // ---------------------------------------------------------------- epilogue (rows g, g + 8 of each m16 tile)
      const long long zoff = (long long)z * p.c_split_stride;
  #pragma unroll
      for (int nt = 0; nt < NTW; ++nt) {
        const int col = nb * BN + (WG ? 0 : wn * WN) + nt * 8 + 2 * tq;
        const bool col_ok = col < p.N;     // N is even, so col + 1 < N as well
        float2 bias2 = make_float2(0.f, 0.f);
        if (p.bias && col_ok) bias2 = *reinterpret_cast<const float2*>(p.bias + col);
  #pragma unroll
        for (int mt = 0; mt < MT; ++mt) {
          const int row16 = mb * kBM + (WG ? warp * 16 : wm * 32 + mt * 16);
          float cs0 = 0.f, cs1 = 0.f;
  #pragma unroll
          for (int h = 0; h < 2; ++h) {    // row half: g, g + 8
            const int row = row16 + g + h * 8;
            float o0 = acc[mt][nt][h * 2] * alpha + bias2.x;
            float o1 = acc[mt][nt][h * 2 + 1] * alpha + bias2.y;
            if (row >= p.M || !col_ok) continue;
            if (p.act == 1) { o0 = fast_tanh(o0); o1 = fast_tanh(o1); }
            if (p.in_mode == 1) {
              const float2 a = *reinterpret_cast<const float2*>(static_cast<const float*>(p.in) + (long long)row * p.ldin + col);
              o0 += a.x; o1 += a.y;
            } else if (p.in_mode == 2) {
              float2 a;
              if constexpr (OUT16) a = __half22float2(*reinterpret_cast<const __half2*>(static_cast<const __half*>(p.in) + (long long)row * p.ldin + col));
              else                 a = *reinterpret_cast<const float2*>(static_cast<const float*>(p.in) + (long long)row * p.ldin + col);
              o0 *= 1.f - a.x * a.x; o1 *= 1.f - a.y * a.y;
            }
            if (p.res) {
              const float2 rr = *reinterpret_cast<const float2*>(p.res + (long long)(row % p.res_row_mod) * p.ldres + col);
              o0 += rr.x; o1 += rr.y;
            }
            if constexpr (OUT16) {
              const uint32_t pk = pack_half2_sat(o0, o1);
              *reinterpret_cast<uint32_t*>(static_cast<__half*>(p.C) + zoff + (long long)row * p.ldc + col) = pk;
              const float2 st = __half22float2(*reinterpret_cast<const __half2*>(&pk));
              cs0 += st.x; cs1 += st.y;
            } else {
              if (p.round_out) { o0 = round_tf32(o0); o1 = round_tf32(o1); }
              *reinterpret_cast<float2*>(static_cast<float*>(p.C) + zoff + (long long)row * p.ldc + col) = make_float2(o0, o1);
              cs0 += o0; cs1 += o1;
            }
          }
          if (p.colsum_part) {
            // bias gradient for free: the m16 tile's rows are one 16-row group of the partial-sum table
  #pragma unroll
            for (int off = 4; off < 32; off <<= 1) {
              cs0 += __shfl_xor_sync(0xffffffffu, cs0, off);
              cs1 += __shfl_xor_sync(0xffffffffu, cs1, off);
            }
            if (g == 0 && col_ok && row16 < p.M)
              *reinterpret_cast<float2*>(p.colsum_part + (size_t)(row16 >> 4) * p.N + col) = make_float2(cs0, cs1);
          }
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// host side: tensor maps (cuTensorMapEncodeTiled through the runtime's driver entry point, so
// the library has no link-time dependency on libcuda) and launch
// ---------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

struct TmapKey {
  const void* ptr; int rank, swz, esz; unsigned long long dims[5], strides[4]; unsigned box[5];
  bool operator==(const TmapKey& o) const {
    if (ptr != o.ptr || rank != o.rank || swz != o.swz || esz != o.esz) return false;
    for (int i = 0; i < rank; ++i) if (dims[i] != o.dims[i] || box[i] != o.box[i]) return false;
    for (int i = 0; i + 1 < rank; ++i) if (strides[i] != o.strides[i]) return false;
    return true;
  }
};
struct TmapKeyHash {
  size_t operator()(const TmapKey& k) const {
    size_t h = std::hash<const void*>()(k.ptr);
    auto mix = [&h](size_t v) { h ^= v + 0x9e3779b97f4a7c15ull + (h << 6) + (h >> 2); };
    mix((size_t)k.rank * 16 + k.swz * 4 + k.esz);
    for (int i = 0; i < k.rank; ++i) { mix((size_t)k.dims[i]); mix((size_t)k.box[i]); }
    for (int i = 0; i + 1 < k.rank; ++i) mix((size_t)k.strides[i]);
    return h;
  }
};

int make_tensor_map(CUtensorMap* out, const void* ptr, int elem_bytes, int rank, const unsigned long long* dims,
                    const unsigned long long* strides_bytes, const unsigned* box, int swizzle) {
  // The encoded map depends only on (address, geometry): it is valid on whichever device owns the address, so one
  // process-wide cache serves every device.
  static std::unordered_map<TmapKey, CUtensorMap, TmapKeyHash> cache;
  static std::mutex mu;
  TmapKey key{};
  key.ptr = ptr; key.rank = rank; key.swz = swizzle; key.esz = elem_bytes;
  for (int i = 0; i < rank; ++i) { key.dims[i] = dims[i]; key.box[i] = box[i]; }
  for (int i = 0; i + 1 < rank; ++i) key.strides[i] = strides_bytes[i];
  {
    std::lock_guard<std::mutex> g(mu);
    auto it = cache.find(key);
    if (it != cache.end()) { *out = it->second; return 0; }
  }
  EncodeTiledFn enc = get_encode_fn();
  if (!enc) return set_error(-4, "cuTensorMapEncodeTiled entry point not available");
  cuuint64_t d[5], st[4];
  cuuint32_t bx[5], es[5];
  for (int i = 0; i < rank; ++i) { d[i] = dims[i]; bx[i] = box[i]; es[i] = 1; }
  for (int i = 0; i + 1 < rank; ++i) st[i] = strides_bytes[i];
  static const CUtensorMapSwizzle kSwz[3] = {CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_SWIZZLE_NONE};
  CUresult r = enc(out, elem_bytes == 2 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, (cuuint32_t)rank,
                   const_cast<void*>(ptr), d, st, bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE, kSwz[swizzle < 0 || swizzle > 2 ? 2 : swizzle],
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return set_error(-4, "cuTensorMapEncodeTiled failed (%d) ptr=%p esz=%d rank=%d dims0=%llu box0=%u", (int)r, ptr, elem_bytes, rank,
                     dims[0], box[0]);
  std::lock_guard<std::mutex> g(mu);
  if (cache.size() > 8192) cache.clear();
  cache.emplace(key, *out);
  return 0;
}

// esz 4 (tf32 operands) or 2 (f16 operands); a k-block / an MN atom is 128 bytes = 128/esz elements
// major 0: matrix [rows = MN extent, cols = K extent], box {128/esz k, box_mn rows}
// major 1: matrix [rows = K extent, cols = MN extent], viewed as {atom, rows, cols/atom}, box {atom, 128/esz k-rows, box_mn/atom}
static int make_operand_tmap(CUtensorMap* out, const void* ptr, int esz, long long ld, int rows, int cols, int major, int box_mn) {
  const unsigned atom = 128u / esz;
  if (major == 0) {
    const unsigned long long dims[2] = {(unsigned long long)cols, (unsigned long long)rows};
    const unsigned long long strides[1] = {(unsigned long long)ld * esz};
    const unsigned box[2] = {atom, (unsigned)box_mn};
    return make_tensor_map(out, ptr, esz, 2, dims, strides, box, 0);
  }
  const unsigned long long dims[3] = {atom, (unsigned long long)rows, (unsigned long long)(cols / atom)};
  const unsigned long long strides[2] = {(unsigned long long)ld * esz, 128};
  const unsigned box[3] = {atom, atom, (unsigned)(box_mn / atom)};
  return make_tensor_map(out, ptr, esz, 3, dims, strides, box, 0);
}

struct GemmMaps { CUtensorMap a, b, a2, b2; };

template <int KIND, int BN, int AMAJ, int BMAJ, int OUT16, int P3 = 0>
static int launch_gemm(const GemmMaps& tm, const GemmParams& p, cudaStream_t stream) {
  using Cfg = GemmCfg<BN>;
  auto kern = gemm_tc_kernel<KIND, BN, AMAJ, BMAJ, OUT16, P3>;
  B200_CONFIGURE_SMEM_ONCE(kern, Cfg::SMEM_BYTES);
  const int total = p.num_m_blocks * p.num_n_blocks * p.num_splits;
  // persistent kernel: launch exactly as many CTAs as can be co-resident, so that none waits for a second wave behind
  // CTAs that never exit early
  static PerDevice occ;
  const int dev = current_device();
  if (dev < 0 || dev >= kMaxDevices) return set_error(-2, "no current CUDA device");
  if (!occ.done[dev]) {
    int n = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kern, kGemmThreads, Cfg::SMEM_BYTES) != cudaSuccess || n <= 0) n = 1;
    occ.value[dev] = n * num_sms();
    occ.done[dev] = true;
  }
  int ctas = occ.value[dev] < total ? occ.value[dev] : total;
  const int cap = sm_limit();          // optional cap (B200VQ_SM_LIMIT / b200vq_set_sm_limit): leave SMs to a concurrent NCCL kernel
  if (cap > 0 && ctas > cap) ctas = cap;
  kern<<<ctas, kGemmThreads, Cfg::SMEM_BYTES, stream>>>(tm.a, tm.b, tm.a2, tm.b2, p);
  B200_LAUNCH_OK("gemm_tc_kernel");
  return 0;
}

template <int KIND, int BN, int P3 = 0>
static int dispatch_major(int am, int bm, int out16, const GemmMaps& tm, const GemmParams& p, cudaStream_t s) {
  if constexpr (KIND == 0) {
    if (am == 0 && bm == 0) return launch_gemm<0, BN, 0, 0, 0, P3>(tm, p, s);
    if (am == 0 && bm == 1) return launch_gemm<0, BN, 0, 1, 0, P3>(tm, p, s);
    if (am == 1 && bm == 1) return launch_gemm<0, BN, 1, 1, 0, P3>(tm, p, s);
    if (am == 1 && bm == 0) return launch_gemm<0, BN, 1, 0, 0, P3>(tm, p, s);
  } else {
    // the combinations the fp16 data path uses: forward x W^T and dgrad g W with fp32 or fp16 output; wgrad (fp32)
    if (am == 0 && bm == 0) return out16 ? launch_gemm<1, BN, 0, 0, 1>(tm, p, s) : launch_gemm<1, BN, 0, 0, 0>(tm, p, s);
    if (am == 0 && bm == 1) return out16 ? launch_gemm<1, BN, 0, 1, 1>(tm, p, s) : launch_gemm<1, BN, 0, 1, 0>(tm, p, s);
    if (am == 1 && bm == 1 && !out16) return launch_gemm<1, BN, 1, 1, 0>(tm, p, s);
  }
  return set_error(-1, "gemm: operand major (%d,%d) with out16=%d is not built for kind %d", am, bm, out16, KIND);
}

// kind 0: A/B fp32 (tf32 tensor cores; A_lo/B_lo non-null selects the 3-pass error-compensated product)
// kind 1: A/B fp16
// cta_group is accepted for ABI stability and ignored (one CTA per tile on sm_90a).  The fp16 kind always runs on
// 128 x 256 tiles (4 ring stages).  tf32: bn <= 64 selects 64-column tiles, anything else 128; the 3xTF32 product
// always runs on 64-column tiles: its promoted partial sums double the accumulator registers.
static int gemm_launch(int kind, const void* A, long long lda, int a_major, const void* B, long long ldb, int b_major, void* C,
                       long long ldc, int out16, int M, int N, int K, int splits, long long c_split_stride, const float* bias,
                       const float* res, long long ldres, int res_row_mod, const void* aux, long long ldaux, float* colsum_part,
                       int act, int round_out, const float* alpha_ptr, const float* A_lo, const float* B_lo, int cta_group, int bn,
                       cudaStream_t stream) {
  (void)cta_group;
  const int esz = kind == 0 ? 4 : 2;          // operand element bytes
  const int osz = out16 ? 2 : 4;              // output element bytes
  const int atom = 128 / esz;
  B200_CHECK_ARG(!colsum_part || splits == 1, "gemm: colsum_part cannot be combined with split-K");
  B200_CHECK_ARG(M > 0 && N > 0 && K > 0 && splits > 0, "gemm: empty problem M=%d N=%d K=%d splits=%d", M, N, K, splits);
  B200_CHECK_ARG((long long)N * osz % 16 == 0 && ldc * osz % 16 == 0, "gemm: N and ldc must give 16-byte rows (N=%d ldc=%lld)", N, ldc);
  B200_CHECK_ARG(lda * esz % 16 == 0 && ldb * esz % 16 == 0, "gemm: lda/ldb must give 16-byte strides (TMA)");
  B200_CHECK_ARG((reinterpret_cast<uintptr_t>(A) & 15) == 0 && (reinterpret_cast<uintptr_t>(B) & 15) == 0 &&
                     (reinterpret_cast<uintptr_t>(C) & 15) == 0, "gemm: operands must be 16-byte aligned");
  B200_CHECK_ARG(!(a_major == 1 && M % atom), "gemm: MN-major A needs M %% %d == 0 (M=%d)", atom, M);
  B200_CHECK_ARG(!(b_major == 1 && N % atom), "gemm: MN-major B needs N %% %d == 0 (N=%d)", atom, N);
  B200_CHECK_ARG(splits == 1 || K % atom == 0, "gemm: split-K needs K %% %d == 0", atom);
  B200_CHECK_ARG(!res || ldres % 4 == 0, "gemm: ldres %% 4");
  B200_CHECK_ARG(!aux || ldaux * (out16 ? 2 : 4) % 16 == 0, "gemm: ldaux must give 16-byte rows");
  B200_CHECK_ARG(!out16 || (!res && splits == 1 && !round_out), "gemm: fp16 output takes no residual / split-K / tf32 rounding");
  B200_CHECK_ARG(!(A_lo || B_lo) || (kind == 0 && A_lo && B_lo), "gemm: the 3xTF32 product needs both A_lo and B_lo (fp32 operands)");
  B200_CHECK_ARG(splits == 1 || c_split_stride % 4 == 0, "gemm: c_split_stride %% 4");
  B200_CHECK_ARG(!(aux && res && res_row_mod == 0), "gemm: residual and tanh' inputs cannot be combined");
  if (bn <= 0) bn = N > 64 ? 128 : 64;
  B200_CHECK_ARG(bn == 64 || bn == 128 || bn == 192 || bn == 256, "gemm: unsupported BN %d", bn);
  bn = kind == 1 ? kBNHalf : (bn <= 64 || A_lo) ? 64 : 128;

  GemmParams p;
  p.M = M; p.N = N; p.K = K;
  p.num_m_blocks = (M + kBM - 1) / kBM;
  p.num_n_blocks = (N + bn - 1) / bn;
  p.num_splits = splits;
  p.k_blocks = (K + atom - 1) / atom;
  p.C = C; p.ldc = ldc; p.c_split_stride = c_split_stride;
  p.alpha_ptr = alpha_ptr;
  p.passes = A_lo ? 3 : 1;
  p.bias = bias; p.act = act; p.round_out = round_out; p.colsum_part = colsum_part;
  p.res = (res && res_row_mod > 0) ? res : nullptr; p.ldres = ldres; p.res_row_mod = res_row_mod;
  p.in_mode = aux ? 2 : ((res && res_row_mod == 0) ? 1 : 0);
  p.in = aux ? aux : static_cast<const void*>(res);
  p.ldin = aux ? ldaux : ldres;
  B200_CHECK_ARG(!p.in_mode || (reinterpret_cast<uintptr_t>(p.in) & 15) == 0, "gemm: epilogue input must be 16-byte aligned");

  GemmMaps tm;
  const int ktot = K * splits;
  int rc;
  auto opmap = [&](CUtensorMap* out, const void* ptr, long long ld, int mn, int major, int box_mn) {
    return major == 0 ? make_operand_tmap(out, ptr, esz, ld, mn, ktot, 0, box_mn) : make_operand_tmap(out, ptr, esz, ld, ktot, mn, 1, box_mn);
  };
  if ((rc = opmap(&tm.a, A, lda, M, a_major, kBM))) return rc;
  if ((rc = opmap(&tm.b, B, ldb, N, b_major, bn))) return rc;
  tm.a2 = tm.a; tm.b2 = tm.b;
  if (A_lo) {
    if ((rc = opmap(&tm.a2, A_lo, lda, M, a_major, kBM))) return rc;
    if ((rc = opmap(&tm.b2, B_lo, ldb, N, b_major, bn))) return rc;
  }
  if (A_lo) return dispatch_major<0, 64, 1>(a_major, b_major, 0, tm, p, stream);
  if (kind == 1) return dispatch_major<1, kBNHalf>(a_major, b_major, out16, tm, p, stream);
  return bn == 64 ? dispatch_major<0, 64>(a_major, b_major, 0, tm, p, stream) : dispatch_major<0, 128>(a_major, b_major, 0, tm, p, stream);
}

}  // namespace b200

using namespace b200;

extern "C" int b200vq_gemm_tf32(const float* A, long long lda, int a_major, const float* B, long long ldb, int b_major, float* C,
                                long long ldc, int M, int N, int K, int splits, long long c_split_stride, const float* bias,
                                const float* res, long long ldres, int res_row_mod, const float* aux, long long ldaux,
                                float* colsum_part, int act, int round_out, int cta_group, int bn, void* streamv) {
  const cudaStream_t stream = static_cast<cudaStream_t>(streamv);
  return gemm_launch(0, A, lda, a_major, B, ldb, b_major, C, ldc, 0, M, N, K, splits, c_split_stride, bias, res, ldres, res_row_mod,
                     aux, ldaux, colsum_part, act, round_out, nullptr, nullptr, nullptr, cta_group, bn, stream);
}

extern "C" int b200vq_gemm_3xtf32(const float* A, const float* A_lo, long long lda, int a_major, const float* B, const float* B_lo,
                                  long long ldb, int b_major, float* C, long long ldc, int M, int N, int K, int splits,
                                  long long c_split_stride, const float* bias, const float* res, long long ldres, int res_row_mod,
                                  const float* aux, long long ldaux, float* colsum_part, int act, int cta_group, int bn, void* streamv) {
  const cudaStream_t stream = static_cast<cudaStream_t>(streamv);
  B200_CHECK_ARG(A_lo && B_lo, "gemm_3xtf32: A_lo and B_lo are required");
  return gemm_launch(0, A, lda, a_major, B, ldb, b_major, C, ldc, 0, M, N, K, splits, c_split_stride, bias, res, ldres, res_row_mod,
                     aux, ldaux, colsum_part, act, 0, nullptr, A_lo, B_lo, cta_group, bn, stream);
}

extern "C" int b200vq_gemm_f16(const void* A, long long lda, int a_major, const void* B, long long ldb, int b_major, void* C,
                               long long ldc, int out_half, int M, int N, int K, int splits, long long c_split_stride,
                               const float* bias, const float* res, long long ldres, int res_row_mod, const void* aux,
                               long long ldaux, float* colsum_part, int act, int round_out, const float* alpha_ptr, int cta_group,
                               int bn, void* streamv) {
  const cudaStream_t stream = static_cast<cudaStream_t>(streamv);
  return gemm_launch(1, A, lda, a_major, B, ldb, b_major, C, ldc, out_half, M, N, K, splits, c_split_stride, bias, res, ldres,
                     res_row_mod, aux, ldaux, colsum_part, act, round_out, alpha_ptr, nullptr, nullptr, cta_group, bn, stream);
}
