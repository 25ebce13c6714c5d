// dorefa.cu -- DoReFa weight quantizer (SURVEY §8f #2): tanh squash + abs-max normalise fused into the fake-quant op.
//
// Replaces the ATen op chain in front of STE.apply in
//   sparsebit/quantization/quantizers/dorefa.py:15-20 (_forward), :22-26 (update_observer):
//       t = x.tanh();  x_normed = t / t.detach().abs().max();  y = STE(x_normed, scale, zero_point)
// which the reference runs as tanh (8 B/elem) + abs (8) + max (4) + div (8) + fake-quant (8) = 36 B/elem in five
// launches, and autograd walks back through div and tanh with three more passes.  Here:
//   sb200_dorefa_absmax   m = max |tanh(x)|                                   4 B/elem   (NaN propagates like torch.max)
//   sb200_dorefa_fwd      y = QDQ(tanh(x) / m)  (or tanh(x) / m alone for the observer)   8 B/elem
//   sb200_dorefa_bwd      gx = ((gy * [qmin <= round(xn / s) + zp <= qmax]) / m) * (1 - t^2)   12 B/elem
// Same IEEE op sequence as the eager chain: libdevice tanhf (what ATen's CUDA tanh calls), a true division by m
// (`tensor / 0-dim tensor` is a real division in ATen, not a reciprocal multiply: dorefa_norm of common.cuh gives that
// IEEE quotient), then quant_tensor.py:181-184.
// Plain chunked grid-stride kernels like adaround.cu, with 64-bit element indices throughout: besides weights they serve
// whole activations, whose max |tanh| the integer-grid layers take on DoReFa inputs, and those pass 2^31 elements
// (tests/test_gpu_far_end_conv.py runs all three past it, and dorefa_absmax past 2^32).
#include "common.cuh"

namespace sb200 {
namespace {

constexpr int kThreads = 256;

__global__ void __launch_bounds__(kThreads) dorefa_absmax_kernel(const float* __restrict__ x, long long n, uint32_t* __restrict__ state) {
  __shared__ uint32_t s_red[kThreads / 32];
  uint32_t best = 0u;  // bit pattern of a non-negative float: unsigned order == value order, NaN (0x7fc00000) above +inf
  const long long t0 = (long long)blockIdx.x * blockDim.x + threadIdx.x, nt = (long long)gridDim.x * blockDim.x;
  const bool vec = (reinterpret_cast<uintptr_t>(x) & 15u) == 0;
  const long long nv = vec ? (n >> 2) : 0;
  auto one = [&](float v) {
    const float t = fabsf(tanhf(v));
    const uint32_t b = (t != t) ? 0x7FC00000u : __float_as_uint(t);
    best = b > best ? b : best;
  };
  for (long long i = t0; i < nv; i += nt) {
    const float4 v = __ldg(reinterpret_cast<const float4*>(x) + i);
    one(v.x); one(v.y); one(v.z); one(v.w);
  }
  for (long long i = (nv << 2) + t0; i < n; i += nt) one(__ldg(x + i));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const uint32_t other = __shfl_xor_sync(0xffffffffu, best, o);
    best = other > best ? other : best;
  }
  if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = best;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < kThreads / 32; ++w) best = s_red[w] > best ? s_red[w] : best;
    atomicMax(state, best);
  }
}

// OP 0: out = tanh(x) / m            (what the observer sees, dorefa.py:22-26)
// OP 1: out = QDQ(tanh(x) / m)       (dorefa.py:15-20)
// OP 2: out = d loss / d x given gy  (autograd of the same chain; scale / zero_point are buffers there: no gs / gzp)
template <int OP>
__device__ __forceinline__ float one_elem(float x, float gy, const QP& p, float m, double rm) {
  float t;
  const float xn = dorefa_norm(x, rm, t);
  if (OP == 0) return xn;
  if (OP == 1) return qdq1<0>(xn, p, 0);
  const float vq = __fadd_rn(round_q<0>(div_exact(xn, p), 0), p.zp);
  const float g = (vq >= p.qmin && vq <= p.qmax) ? gy : 0.f;  // NaN compares false: no gradient, like the reference mask
  return __fmul_rn(__fdiv_rn(g, m), __fsub_rn(1.f, __fmul_rn(t, t)));
}

// One CTA walks chunks of (row = outer*C index, 1024 consecutive elements of that row): channel parameters once per chunk.
template <int OP, bool VEC>
__global__ void __launch_bounds__(kThreads) dorefa_kernel(const float* __restrict__ x, const float* __restrict__ gy,
                                                          const float* __restrict__ absmax, const float* __restrict__ scale,
                                                          const float* __restrict__ zp, float* __restrict__ out, long long rows,
                                                          long long C, long long inner, float qmin, float qmax) {
  constexpr int kChunk = kThreads * 4;
  const long long chunks_per_row = (inner + kChunk - 1) / kChunk;
  const long long total = rows * chunks_per_row;
  const float m = __ldg(absmax);
  const double rm = dorefa_rcp(m);
  for (long long tix = blockIdx.x; tix < total; tix += gridDim.x) {
    const long long row = tix / chunks_per_row;
    const long long k0 = (tix - row * chunks_per_row) * kChunk;
    QP p;
    p.qmin = qmin;
    p.qmax = qmax;
    if (OP != 0) p.set(__ldg(scale + row % C), __ldg(zp + row % C));
    const long long base = row * inner + k0;
    const long long left = inner - k0;
    if (VEC) {
      const long long k = (long long)threadIdx.x * 4;
      if (k < left) {  // inner % 4 == 0: whole float4 in range
        const float4 xv = *reinterpret_cast<const float4*>(x + base + k);
        float4 gv = make_float4(0.f, 0.f, 0.f, 0.f), o;
        if (OP == 2) gv = *reinterpret_cast<const float4*>(gy + base + k);
        o.x = one_elem<OP>(xv.x, gv.x, p, m, rm); o.y = one_elem<OP>(xv.y, gv.y, p, m, rm);
        o.z = one_elem<OP>(xv.z, gv.z, p, m, rm); o.w = one_elem<OP>(xv.w, gv.w, p, m, rm);
        *reinterpret_cast<float4*>(out + base + k) = o;
      }
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const long long k = threadIdx.x + (long long)j * kThreads;
        if (k < left) out[base + k] = one_elem<OP>(x[base + k], OP == 2 ? gy[base + k] : 0.f, p, m, rm);
      }
    }
  }
}

template <int OP>
int launch(const float* x, const float* gy, const float* absmax, const float* scale, const float* zp, float* out,
           long long outer, long long C, long long inner, int qmin, int qmax, cudaStream_t st) {
  const long long rows = outer * C;
  const long long chunks = rows * ((inner + kThreads * 4 - 1) / (kThreads * 4));
  const long long cap = (long long)sm_count() * 8;
  const unsigned grid = (unsigned)(chunks < cap ? chunks : cap);
  const bool vec = (inner % 4 == 0) && aligned16(x) && aligned16(out) && (OP != 2 || aligned16(gy));
  if (vec)
    dorefa_kernel<OP, true><<<grid, kThreads, 0, st>>>(x, gy, absmax, scale, zp, out, rows, C, inner, (float)qmin, (float)qmax);
  else
    dorefa_kernel<OP, false><<<grid, kThreads, 0, st>>>(x, gy, absmax, scale, zp, out, rows, C, inner, (float)qmin, (float)qmax);
  SB_LAUNCHED();
  return SB200_OK;
}

}  // namespace
}  // namespace sb200

using namespace sb200;

extern "C" {

int sb200_dorefa_absmax(const float* x, int64_t n, float* absmax, void* stream) {
  SB_REQUIRE(x && absmax, "sb200_dorefa_absmax: null pointer argument");
  SB_REQUIRE(n > 0, "sb200_dorefa_absmax: empty tensor");
  const long long want = (n / 4 + kThreads - 1) / kThreads + 1;
  const long long cap = (long long)sm_count() * 8;
  dorefa_absmax_kernel<<<(unsigned)(want < cap ? want : cap), kThreads, 0, (cudaStream_t)stream>>>(x, n, reinterpret_cast<uint32_t*>(absmax));
  SB_LAUNCHED();
  return SB200_OK;
}

int sb200_dorefa_fwd(const float* x, const float* absmax, const float* scale, const float* zero_point, float* out,
                     int64_t outer, int64_t channels, int64_t inner, int qmin, int qmax, int quantize, void* stream) {
  SB_REQUIRE(x && absmax && out, "sb200_dorefa_fwd: null pointer argument");
  SB_REQUIRE(outer > 0 && channels > 0 && inner > 0, "sb200_dorefa_fwd: empty tensor");
  SB_REQUIRE(quantize == 0 || quantize == 1, "sb200_dorefa_fwd: quantize must be 0 (normalise only) or 1");
  if (!quantize) return launch<0>(x, nullptr, absmax, nullptr, nullptr, out, outer, channels, inner, 0, 0, (cudaStream_t)stream);
  SB_REQUIRE(scale && zero_point, "sb200_dorefa_fwd: null qparams");
  SB_REQUIRE(qmin <= qmax, "sb200_dorefa_fwd: qmin > qmax");
  return launch<1>(x, nullptr, absmax, scale, zero_point, out, outer, channels, inner, qmin, qmax, (cudaStream_t)stream);
}

int sb200_dorefa_bwd(const float* x, const float* absmax, const float* scale, const float* zero_point, const float* grad_y,
                     float* grad_x, int64_t outer, int64_t channels, int64_t inner, int qmin, int qmax, void* stream) {
  SB_REQUIRE(x && absmax && scale && zero_point && grad_y && grad_x, "sb200_dorefa_bwd: null pointer argument");
  SB_REQUIRE(outer > 0 && channels > 0 && inner > 0, "sb200_dorefa_bwd: empty tensor");
  SB_REQUIRE(qmin <= qmax, "sb200_dorefa_bwd: qmin > qmax");
  return launch<2>(x, grad_y, absmax, scale, zero_point, grad_x, outer, channels, inner, qmin, qmax, (cudaStream_t)stream);
}

}  // extern "C"
