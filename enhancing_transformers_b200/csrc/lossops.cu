// The two native ops of the reference's loss stage (SURVEY.md section 8f-2), rebuilt for sm_90a behind the C ABI:
//   bias_act   -- reference enhancing/losses/op/fused_bias_act_kernel.cu (StyleGAN2 fused bias + leaky-ReLU + gain, and
//                 its first/second derivative forms), called by losses/op/fused_act.py:62-91;
//   upfirdn2d  -- reference enhancing/losses/op/upfirdn2d_kernel.cu (zero-insert upsample -> FIR -> decimate),
//                 called by losses/op/upfirdn2d.py:89-146 (Blur, losses/layers.py:140-160).
// Both are HBM-bound streams: float4 grid-stride loops sized to the SM count; the FIR reads each input pixel from L1/L2
// for its <= 16 taps (4 x 4 blur kernels in every shipped discriminator).  The JIT-compiled extensions of the
// reference (torch.utils.cpp_extension.load at import time) are not needed once loss_ops.py is installed.
#include "../../include/b200vq.h"
#include "common.cuh"

namespace b200 {

// out = act'(x [+ b[c]], ref) * scale
//   grad 0: y = lrelu(x + b)            (ref unused)
//   grad 1: y = x * (ref > 0 ? 1 : a)   (first derivative applied to an incoming gradient x; ref = forward output)
//   grad 2: y = 0                       (second derivative of a piecewise-linear function)
// act 1 = linear, 3 = leaky ReLU (the numbering of the reference kernel, fused_bias_act_kernel.cu:43-64)
__global__ void __launch_bounds__(256)
bias_act_kernel(const float* __restrict__ x, const float* __restrict__ b, const float* __restrict__ ref, float* __restrict__ out,
                long long n, int step_b, int size_b, int act, int grad, float alpha, float scale) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float v = x[i];
    if (b) v += __ldg(b + (i / step_b) % size_b);
    const float r = ref ? ref[i] : 0.f;
    float y;
    if (grad == 2) y = 0.f;
    else if (act == 3) y = ((grad == 0 ? v : r) > 0.f) ? v : v * alpha;
    else y = v;
    out[i] = y * scale;
  }
}

// out[p, oy, ox] = sum_{ky,kx} U[p, oy*down_y + ky, ox*down_x + kx] * K[kh-1-ky, kw-1-kx]
// U = the input plane zero-inserted by (up_y, up_x) and padded / cropped by (pad_y0, pad_x0)   (upfirdn2d.py:168-206)
__global__ void __launch_bounds__(256)
upfirdn2d_kernel(const float* __restrict__ in, const float* __restrict__ kern, float* __restrict__ out, long long planes, int in_h,
                 int in_w, int out_h, int out_w, int kh, int kw, int up_x, int up_y, int down_x, int down_y, int pad_x0, int pad_y0) {
  extern __shared__ float ks[];                    // flipped kernel
  for (int i = threadIdx.x; i < kh * kw; i += blockDim.x) ks[i] = kern[(kh - 1 - i / kw) * kw + (kw - 1 - i % kw)];
  __syncthreads();
  const long long total = planes * out_h * out_w;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int ox = (int)(i % out_w);
    const long long t = i / out_w;
    const int oy = (int)(t % out_h);
    const long long pl = t / out_h;
    const float* src = in + pl * in_h * in_w;
    const int uy0 = oy * down_y - pad_y0, ux0 = ox * down_x - pad_x0;     // top-left tap in upsampled coordinates
    float acc = 0.f;
    for (int ky = 0; ky < kh; ++ky) {
      const int uy = uy0 + ky;
      if (uy < 0 || uy % up_y) continue;
      const int iy = uy / up_y;
      if (iy >= in_h) continue;
      for (int kx = 0; kx < kw; ++kx) {
        const int ux = ux0 + kx;
        if (ux < 0 || ux % up_x) continue;
        const int ix = ux / up_x;
        if (ix >= in_w) continue;
        acc = fmaf(src[iy * in_w + ix], ks[ky * kw + kx], acc);
      }
    }
    out[i] = acc;
  }
}

static inline int lo_grid(long long work, int threads) {
  long long blocks = (work + threads - 1) / threads;
  const long long cap = (long long)num_sms() * 8;
  if (blocks > cap) blocks = cap;
  return (int)(blocks < 1 ? 1 : blocks);
}

}  // namespace b200

using namespace b200;

extern "C" int b200vq_bias_act(const float* x, const float* b, const float* ref, float* out, long long n, int step_b, int size_b,
                               int act, int grad, float alpha, float scale, void* streamv) {
  const cudaStream_t stream = static_cast<cudaStream_t>(streamv);
  B200_CHECK_ARG(n > 0, "bias_act: empty input");
  B200_CHECK_ARG(act == 1 || act == 3, "bias_act: act must be 1 (linear) or 3 (leaky ReLU), got %d", act);
  B200_CHECK_ARG(grad >= 0 && grad <= 2, "bias_act: grad must be 0, 1 or 2");
  B200_CHECK_ARG(!b || (step_b > 0 && size_b > 0), "bias_act: bad bias geometry");
  B200_CHECK_ARG(grad == 0 || ref, "bias_act: derivative forms need the forward output as ref");
  bias_act_kernel<<<lo_grid(n, 256), 256, 0, stream>>>(x, b, ref, out, n, step_b > 0 ? step_b : 1, size_b > 0 ? size_b : 1, act, grad,
                                                       alpha, scale);
  B200_LAUNCH_OK("bias_act_kernel");
  return 0;
}

extern "C" int b200vq_upfirdn2d(const float* in, const float* kern, float* out, long long planes, int in_h, int in_w, int kh, int kw,
                                int up_x, int up_y, int down_x, int down_y, int pad_x0, int pad_x1, int pad_y0, int pad_y1,
                                void* streamv) {
  const cudaStream_t stream = static_cast<cudaStream_t>(streamv);
  B200_CHECK_ARG(planes > 0 && in_h > 0 && in_w > 0 && kh > 0 && kw > 0 && kh * kw <= 1024, "upfirdn2d: bad sizes");
  B200_CHECK_ARG(up_x > 0 && up_y > 0 && down_x > 0 && down_y > 0, "upfirdn2d: up/down factors must be positive");
  const int out_h = (in_h * up_y + pad_y0 + pad_y1 - kh + down_y) / down_y;
  const int out_w = (in_w * up_x + pad_x0 + pad_x1 - kw + down_x) / down_x;
  B200_CHECK_ARG(out_h > 0 && out_w > 0, "upfirdn2d: empty output (%d x %d)", out_h, out_w);
  upfirdn2d_kernel<<<lo_grid(planes * out_h * out_w, 256), 256, kh * kw * sizeof(float), stream>>>(
      in, kern, out, planes, in_h, in_w, out_h, out_w, kh, kw, up_x, up_y, down_x, down_y, pad_x0, pad_y0);
  B200_LAUNCH_OK("upfirdn2d_kernel");
  return 0;
}
