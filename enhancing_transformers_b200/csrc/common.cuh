// Shared device helpers: inline-PTX wrappers for mbarrier / TMA / mma.sync / wgmma (sm_90a).
// Hand-written after the PTX ISA.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#if defined(__CUDA_ARCH__) && !defined(__CUDA_ARCH_FEAT_SM90_ALL)
#error "b200vq kernels must be compiled with -gencode arch=compute_90a,code=sm_90a"
#endif

namespace b200 {

// ------------------------------------------------------------------------------------------
// error plumbing shared by all translation units (defined in api.cu)
// ------------------------------------------------------------------------------------------
int set_error(int code, const char* fmt, ...);
#define B200_CHECK_ARG(cond, ...)                                  \
  do {                                                             \
    if (!(cond)) return ::b200::set_error(-1, __VA_ARGS__);        \
  } while (0)
#define B200_CUDA_OK(expr)                                                                     \
  do {                                                                                         \
    cudaError_t e__ = (expr);                                                                  \
    if (e__ != cudaSuccess)                                                                    \
      return ::b200::set_error(-2, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__),    \
                               __FILE__, __LINE__);                                            \
  } while (0)
void count_launch();
#define B200_LAUNCH_OK(name)                                                                   \
  do {                                                                                         \
    ::b200::count_launch();                                                                    \
    cudaError_t e__ = cudaGetLastError();                                                      \
    if (e__ != cudaSuccess)                                                                    \
      return ::b200::set_error(-3, "launch of %s failed: %s", name, cudaGetErrorString(e__));  \
  } while (0)

int num_sms();            // SM count of the *current* device (cached per device)
int current_device();     // cudaGetDevice, or -1
int sm_limit();           // 0 = none; otherwise persistent kernels launch at most this many CTAs (leaves SMs to NCCL)
// Per-kernel, per-device one-time setup (cudaFuncSetAttribute is a per-device property: a process that drives
// several GPUs -- DataParallel, a multi-device script -- must set it once on each of them).
constexpr int kMaxDevices = 64;
struct PerDevice { bool done[kMaxDevices] = {}; int value[kMaxDevices] = {}; };
#define B200_CONFIGURE_SMEM_ONCE(kern, bytes)                                                                \
  do {                                                                                                       \
    static ::b200::PerDevice once__;                                                                         \
    const int dev__ = ::b200::current_device();                                                              \
    if (dev__ < 0 || dev__ >= ::b200::kMaxDevices) return ::b200::set_error(-2, "no current CUDA device");   \
    if (!once__.done[dev__]) {                                                                               \
      B200_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(bytes)));   \
      once__.done[dev__] = true;                                                                             \
    }                                                                                                        \
  } while (0)
// generic tiled tensor map (rank <= 5), cached.  elem_bytes: 4 = fp32, 2 = fp16;
// swizzle: 0 = SWIZZLE_128B, 1 = SWIZZLE_64B, 2 = none
int make_tensor_map(CUtensorMap* out, const void* ptr, int elem_bytes, int rank, const unsigned long long* dims,
                    const unsigned long long* strides_bytes, const unsigned* box, int swizzle);

#ifdef __CUDACC__
// ------------------------------------------------------------------------------------------
// small utilities
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
// 1024-byte alignment of the dynamic shared-memory base (SWIZZLE_128B atoms) as pointer arithmetic on the __shared__
// symbol: a round trip through uintptr_t loses the address space and every later access becomes a generic LD / ST.
__device__ __forceinline__ uint8_t* smem_align1024(uint8_t* raw) { return raw + ((1024u - (smem_u32(raw) & 1023u)) & 1023u); }
// round-to-nearest (ties away from zero, like cvt.rna.tf32.f32) fp32 -> tf32 (10-bit mantissa),
// result kept in an fp32 container with the low 13 bits cleared.  Integer ops on the ALU pipe
// instead of cvt.rna.tf32, which issues on the XU pipe shared with ex2.  A NaN keeps its sign and gets
// the quiet bit instead of the rounding carry: the carry would run out of the mantissa (0x7FFFFFFF, the
// NaN every fp32 operation on the GPU makes, would become -0.0), and the quiet bit survives the tensor
// core's truncation.  Finite values and +-inf round as before.
__device__ __forceinline__ float round_tf32(float x) {
  const uint32_t u = __float_as_uint(x);
  const bool nan = (u & 0x7FFFFFFFu) > 0x7F800000u;
  return __uint_as_float((nan ? (u | 0x00400000u) : (u + 0x1000u)) & 0xFFFFE000u);
}
// tanh(x) = 1 - 2 / (exp(2x) + 1) with one ex2.approx and one rcp.approx (absolute error ~1e-7, far below the
// tf32 rounding applied to the result).  libdevice's tanhf costs ~40 instructions per element of the MLP-1 epilogue.
__device__ __forceinline__ float fast_tanh(float x) {
  float e, r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(x * 2.8853900817779268f));   // exp(2x) = 2^(2x log2 e)
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(e + 1.0f));
  return fmaf(-2.0f, r, 1.0f);                                                    // e = inf -> r = 0 -> 1; e = 0 -> -1
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ------------------------------------------------------------------------------------------
// mbarrier
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
// Spin on a phase parity.  A deadlocked pipeline would otherwise hang the GPU until the watchdog kills the box, so
// after 2^28 failed probes (each try_wait suspends the thread for a hardware-defined slice: seconds in total) the kernel
// traps instead.  The loop body is the probe, one add and one compare: a spinning producer warp shares its scheduler's
// issue slots with the consumer warps.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  const uint32_t addr = smem_u32(bar);
  uint32_t done = 0;
  for (uint32_t it = 0;; ++it) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(addr), "r"(parity)
        : "memory");
    if (done) break;
    if (it == (1u << 28)) __trap();
  }
}

// ------------------------------------------------------------------------------------------
// TMA (cp.async.bulk.tensor), tile mode, completion on an mbarrier
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
// ------------------------------------------------------------------------------------------
// warp-level tensor-core MMA (fp32 accumulate)
// ------------------------------------------------------------------------------------------
// c[16x8] += a[16x8] . b[8x8], tf32 operands given as fp32 bit patterns (the tensor core ignores the low 13 bits)
__device__ __forceinline__ void mma_tf32(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// ------------------------------------------------------------------------------------------
// wgmma (sm_90a): warpgroup MMA on shared-memory descriptors, fp16 operands, fp32 accumulators in registers
// ------------------------------------------------------------------------------------------
// SWIZZLE_128B shared-memory matrix descriptor: start address, leading / stride byte offsets (16-byte units), layout 1
__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  return (uint64_t)((saddr & 0x3FFFFu) >> 4) | ((uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16) |
         ((uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32) | (1ull << 62);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accesses of the accumulator registers across the asynchronous MMA
template <int N>
__device__ __forceinline__ void wgmma_fence_regs(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// D[64 x 256] += A[64 x 16] . B[16 x 256]; TA / TB = 1: the operand is MN-major in shared memory (transposed)
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n256k16_f16(float (&d)[128], uint64_t adesc, uint64_t bdesc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, "
      "%128, %129, p, 1, 1, %130, %131;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(adesc), "l"(bdesc), "n"(TA), "n"(TB)
      : "memory");
}
// D[64 x 64] (+)= A[64 x 16] . B[16 x 64], A K-major in shared memory; accumulate = 0 overwrites D with the product
template <int TB>
__device__ __forceinline__ void wgmma_m64n64k16_ss(float (&d)[32], uint64_t adesc, uint64_t bdesc, int accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "%32, %33, p, 1, 1, 0, %35;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(adesc), "l"(bdesc), "r"(accumulate), "n"(TB)
      : "memory");
}
// D[64 x 64] += A[64 x 16] . B[16 x 64], A from registers: per warp the m16n8k16 A fragment of its 16 rows, which is the
// accumulator layout of two adjacent n8 column tiles packed to fp16 pairs
template <int TB>
__device__ __forceinline__ void wgmma_m64n64k16_rs(float (&d)[32], const uint32_t (&a)[4], uint64_t bdesc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "{%32, %33, %34, %35}, %36, p, 1, 1, %37;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "n"(TB)
      : "memory");
}
// two fp32 -> packed fp16x2 (round to nearest), saturating at +-65504 instead of overflowing to inf
__device__ __forceinline__ uint32_t pack_half2_sat(float a, float b) {
  uint32_t r;      // one F2FP.SATFINITE: a -> low half, b -> high half
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));
  return r;
}
#endif  // __CUDACC__

}  // namespace b200
