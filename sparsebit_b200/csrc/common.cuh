// common.cuh -- shared device/host helpers for the sm_90a kernels behind include/sparsebit_b200.h.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <atomic>

#include "../../include/sparsebit_b200.h"

namespace sb200 {

// ---------------------------------------------------------------- host-side error plumbing
void set_error(const char* fmt, ...);
int sm_count();
extern std::atomic<long long> g_launches;
extern int g_variant;

#define SB_REQUIRE(cond, ...)          \
  do {                                 \
    if (!(cond)) {                     \
      sb200::set_error(__VA_ARGS__);   \
      return SB200_E_INVALID;          \
    }                                  \
  } while (0)

#define SB_CUDA(call)                                                                    \
  do {                                                                                   \
    cudaError_t e__ = (call);                                                            \
    if (e__ != cudaSuccess) {                                                            \
      sb200::set_error("%s failed: %s (%s:%d)", #call, cudaGetErrorString(e__), __FILE__, \
                       __LINE__);                                                        \
      return SB200_E_CUDA;                                                               \
    }                                                                                    \
  } while (0)

// Call after every kernel launch: counts it and surfaces launch-configuration errors.
#define SB_LAUNCHED()                                                                     \
  do {                                                                                    \
    sb200::g_launches.fetch_add(1, std::memory_order_relaxed);                            \
    cudaError_t e__ = cudaPeekAtLastError();                                              \
    if (e__ != cudaSuccess) {                                                             \
      (void)cudaGetLastError();                                                           \
      sb200::set_error("kernel launch failed: %s (%s:%d)", cudaGetErrorString(e__), __FILE__, \
                       __LINE__);                                                         \
      return SB200_E_CUDA;                                                                \
    }                                                                                     \
  } while (0)

// Per-device one-time cudaFuncSetAttribute(MaxDynamicSharedMemorySize): the attribute is per device, so a process
// driving several GPUs must set it on each (a process-wide `static bool` would skip the second device).
template <typename KernelT>
static inline cudaError_t ensure_dyn_smem(KernelT kernel, int bytes, std::atomic<int>* done_per_device /*[64]*/) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  if (dev < 0 || dev >= 64) return cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (done_per_device[dev].load(std::memory_order_acquire) >= bytes) return cudaSuccess;
  e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e == cudaSuccess) done_per_device[dev].store(bytes, std::memory_order_release);
  return e;
}

static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// ---------------------------------------------------------------- order-preserving float key
// enc() maps fp32 to uint32 such that a < b  <=>  enc(a) < enc(b) (with -0 < +0, NaN at the ends).
__host__ __device__ __forceinline__ uint32_t enc_f32(float f) {
#ifdef __CUDA_ARCH__
  uint32_t b = __float_as_uint(f);
#else
  union { float f; uint32_t u; } c; c.f = f; uint32_t b = c.u;
#endif
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__host__ __device__ __forceinline__ float dec_f32(uint32_t k) {
  uint32_t b = (k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k;
#ifdef __CUDA_ARCH__
  return __uint_as_float(b);
#else
  union { float f; uint32_t u; } c; c.u = b; return c.f;
#endif
}
// Running min/max state: {enc(min), enc(max)} ; "empty" = {0xFFFFFFFF, 0}.  A NaN input poisons
// both slots with the canonical NaN marker below (torch.min / torch.max propagate NaN).
#define SB_MM_EMPTY_MIN 0xFFFFFFFFu
#define SB_MM_EMPTY_MAX 0x00000000u

#ifdef __CUDACC__
// ---------------------------------------------------------------- streaming 128-bit access
__device__ __forceinline__ float4 ld_stream4(const float4* p) { return __ldcs(p); }
__device__ __forceinline__ void st_stream4(float4* p, float4 v) { __stcs(p, v); }
__device__ __forceinline__ float ld_stream1(const float* p) { return __ldcs(p); }
__device__ __forceinline__ void st_stream1(float* p, float v) { __stcs(p, v); }

// ---------------------------------------------------------------- QDQ scalar math (oracle order)
// Follows sparsebit/quantization/quantizers/quant_tensor.py:181-184 exactly:
//   zp = round(zero_point); x_q = clamp(round(x / scale) + zp, qmin, qmax); x_dq = (x_q - zp) * scale
// with IEEE semantics for every step, no FMA contraction, NaN propagating through the clamp
// (torch.clamp semantics).
//
// Division.  The IEEE quotient RN32(x/s) is obtained as RN32(RN64(x * RN64(1/s))): the quotient of
// two binary32 numbers is at least 2^-49 (relative) away from every binary32 rounding midpoint
// (|X*2^24 - M*S| >= 1 for 24-bit X, S and a 25-bit odd M), while the double-precision product is
// within 2^-52 of it, so both round to the same float for every input including zero, subnormal,
// infinite and NaN operands.  This is 3 instructions per element (cvt, DMUL, cvt) with the
// reciprocal hoisted out of the loop, instead of the ~35-instruction div.rn.f32 expansion (MUFU +
// Newton + range check + slow-path call) per element.
__device__ __forceinline__ float fmin_nan(float a, float b) {
  float r;
  asm("min.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
}
__device__ __forceinline__ float fmax_nan(float a, float b) {
  float r;
  asm("max.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
}

struct QP {
  float s, zp, qmin, qmax;
  double rs;  // RN64(1 / s)
  float r;    // RN32(1 / s)
  bool fast;  // |s| in [2^-60, 2^60]: the fp32 fast path below is valid
  float gz_hi;  // STE backward only: largest vq that counts as "inside" for the zero-point gradient (qmax, or qmax - 1
                // under the reference's per-channel rule, fake_quant_tensor.cu:264)
  __device__ __forceinline__ void set(float scale, float zero_point_raw) {
    s = scale;
    zp = rintf(zero_point_raw);
    rs = __drcp_rn((double)scale);
    r = __double2float_rn(rs);
    const float a = fabsf(scale);
    fast = (a >= 0x1p-60f) && (a <= 0x1p60f);
  }
};

__device__ __forceinline__ float div_exact(float x, const QP& p) {
  return __double2float_rn(__dmul_rn((double)x, p.rs));
}

// ROUNDING: 0 half-to-even (torch.round / nearbyint); -1 = runtime `rounding` in {0, 1, 2}
// (1: floor(v + .5), 2: ceil(v - .5), torch_extensions/common.cuh:66-74).
// rint() without the XU pipe: adding 1.5 * 2^23 rounds to an integer with the FPU's own
// round-half-even; exact for |v| < 2^22, everything else (incl. NaN) takes the FRND path.  The
// only difference from rintf is the sign of a zero result, which cannot reach the output:
// (+-0 + zp) and (+-0 - q) are the same values either way.
__device__ __forceinline__ float rint_fast(float v) {
  float r = __fadd_rn(__fadd_rn(v, 12582912.f), -12582912.f);
  if (!(fabsf(v) < 4194304.f)) r = rintf(v);
  return r;
}

template <int ROUNDING>
__device__ __forceinline__ float round_q(float v, int rounding) {
  if (ROUNDING == 0) return rint_fast(v);
  if (rounding == 1) return floorf(__fadd_rn(v, 0.5f));
  if (rounding == 2) return ceilf(__fsub_rn(v, 0.5f));
  return rintf(v);
}

// round(x / s) for the forward pass, bit-identical to round_q(div_exact(x)) but on the FP32 pipe:
//   q1 = Markstein quotient (x*r, exact residual by FMA, one correction) -- within 1/2 ulp (+2^-47)
//        of x/s, like the IEEE quotient itself;
//   t1 = q1 rounded to an integer by the 1.5*2^23 trick;
//   the two can only round to different integers if a half-integer lies within 2 ulp of q1, i.e.
//   0.5 - |q1 - t1| <= |q1| * 2^-22.  Those elements (a ~1e-4 fraction for 8-bit data), huge or
//   non-finite quotients, and out-of-range scales take the exact fp64 route.
// Verified against rintf(x / s) on 4e9 random + adversarial (k + 0.5) * s +- few-ulp inputs.
// LAZY: p.rs is not populated (per-channel parameters come from a shared-memory table holding only
// s, 1/s, zp); the rare exact fallback computes the fp64 reciprocal on the spot.
template <int ROUNDING, bool LAZY = false>
__device__ __forceinline__ float quant_round(float x, const QP& p, int rounding) {
  if (ROUNDING == 0 && p.fast) {
    const float q0 = __fmul_rn(x, p.r);
    const float e = __fmaf_rn(-q0, p.s, x);
    const float q1 = __fmaf_rn(e, p.r, q0);
    const float t1 = __fadd_rn(__fadd_rn(q1, 12582912.f), -12582912.f);
    const float d = __fsub_rn(q1, t1);
    const float c = __fmaf_rn(fabsf(q1), -0x1p-22f, __fsub_rn(0.5f, fabsf(d)));
    if (c > 0.f) return t1;
  }
  if (LAZY) return round_q<ROUNDING>(__double2float_rn(__dmul_rn((double)x, __drcp_rn((double)p.s))), rounding);
  return round_q<ROUNDING>(div_exact(x, p), rounding);
}

template <int ROUNDING, bool LAZY = false>
__device__ __forceinline__ float qdq1(float x, const QP& p, int rounding) {
  float v = __fadd_rn(quant_round<ROUNDING, LAZY>(x, p, rounding), p.zp);
  v = fmax_nan(fmin_nan(v, p.qmax), p.qmin);
  return __fmul_rn(__fsub_rn(v, p.zp), p.s);
}

// DoReFa's normalised value tanh(x) / m (dorefa.py:16-17), m = max |tanh| over the tensor: libdevice tanhf (what
// ATen's CUDA tanh calls), then the IEEE quotient (`tensor / 0-dim tensor` is a true division in ATen).  The one
// sequence of the DoReFa kernels (dorefa.cu) and of the integer-grid kernels' DoReFa inputs (int8_grid.cuh); `t`
// receives tanh(x).
//
// The quotient is RN32(RN64(t * rm)), rm = dorefa_rcp(m) hoisted out of the loop, as div_exact above: a binary32
// quotient lies at least 2^-49 (relative) from every binary32 rounding midpoint, and rm is 1 / m within 2^-51 for every
// finite nonzero m (a normal double even for a subnormal float m), so the product rounds to RN32(t / m) for every t,
// zero, subnormal, infinite and NaN included.  rm comes from the approximate reciprocal and two Newton steps (error
// 2^-20 -> 2^-40 -> under 2^-51) rather than rcp.rn / div.rn, whose slow-path calls make the integer-grid kernels spill
// registers; the exact reciprocals of +-0 (+-inf) and +-inf (+-0) are set apart, and a NaN m gives a NaN rm.  So the
// quotient equals __fdiv_rn(t, m) for every float m, not only the 0, (0, 1] or NaN that a max |tanh| can be.
__device__ __forceinline__ double dorefa_rcp(float m) {
  const double md = (double)m;
  double r;
  asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(md));
  r = __fma_rn(r, __fma_rn(-md, r, 1.0), r);
  r = __fma_rn(r, __fma_rn(-md, r, 1.0), r);
  if (m == 0.f) r = copysign(__longlong_as_double(0x7ff0000000000000LL), md);
  if (isinf(m)) r = copysign(0.0, md);
  return r;
}
__device__ __forceinline__ float dorefa_norm(float x, double rm, float& t) {
  t = tanhf(x);
  return __double2float_rn(__dmul_rn((double)t, rm));
}

// ---------------------------------------------------------------- mbarrier + TMA bulk copy (sm_90+)
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE;\n\t"
      "bra WAIT_LOOP;\n\t"
      "DONE:\n\t}" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
// mbarrier wait with an optional back-off between polls (sb200_gptq4_set_wait_backoff; 0 = poll continuously)
__device__ __forceinline__ void mbar_wait_relaxed(uint64_t* bar, uint32_t parity, int backoff_ns) {
  for (;;) {
    uint32_t done;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    if (done) return;
    if (backoff_ns > 0) __nanosleep((unsigned)backoff_ns);
  }
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// 1-D TMA: global -> shared, completion signalled on an mbarrier (bytes % 16 == 0, both 16 B aligned)
__device__ __forceinline__ void tma_bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst_smem)),
               "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// ---------------------------------------------------------------- warp / block reductions
__device__ __forceinline__ float warp_min(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fminf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Per-thread running min/max.  min.NaN / max.NaN propagate NaN like torch.min / torch.max.
struct MinMaxAcc {
  float lo, hi;
  __device__ __forceinline__ void init() { lo = __int_as_float(0x7f800000); hi = __int_as_float(0xff800000); }
  __device__ __forceinline__ void add(float v) {
    lo = fmin_nan(lo, v);
    hi = fmax_nan(hi, v);
  }
  __device__ __forceinline__ void add4(const float4& v) { add(v.x); add(v.y); add(v.z); add(v.w); }
  __device__ __forceinline__ void warp_reduce() {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      lo = fmin_nan(lo, __shfl_xor_sync(0xffffffffu, lo, o));
      hi = fmax_nan(hi, __shfl_xor_sync(0xffffffffu, hi, o));
    }
  }
  // Publish into the {enc(min), enc(max)} state of one channel.  NaN -> both slots get the
  // extreme keys, which decode to NaN (see minmax_read).
  __device__ __forceinline__ void publish(uint32_t* st) const {
    if (lo != lo || hi != hi) {
      atomicMin(st, 0u);
      atomicMax(st + 1, 0xFFFFFFFFu);
    } else if (lo <= hi) {
      atomicMin(st, enc_f32(lo));
      atomicMax(st + 1, enc_f32(hi));
    }
  }
};

// Block-level reduce of a MinMaxAcc; result valid in warp 0.  `sm` needs 2*32 words.
__device__ __forceinline__ void block_reduce_minmax(MinMaxAcc& a, float* sm) {
  a.warp_reduce();
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  if (lane == 0) {
    sm[wid] = a.lo;
    sm[32 + wid] = a.hi;
  }
  __syncthreads();
  if (wid == 0) {
    a.lo = lane < nw ? sm[lane] : __int_as_float(0x7f800000);
    a.hi = lane < nw ? sm[32 + lane] : __int_as_float(0xff800000);
    a.warp_reduce();
  }
  __syncthreads();
}
// Fixed-order finish of per-tile fp64 partials:  out[row * nval + k] += sum_j partial[(row * tpr + j) * nval + k].
// One CTA per row; thread (s, k) = (tid / nval, tid % nval) sums the tiles j = s, s + S, s + 2S, ... (S = blockDim / nval
// slices, four independent accumulators so that four loads are in flight), the S slice sums are combined in slice order
// by thread k.  The association depends only on (tpr, blockDim), never on scheduling: run-to-run deterministic.
// (The one-thread-per-output loops this replaces took 100 - 290 us for a single per-tensor row: a serial chain of
// dependent-latency loads, longer than the streaming pass that produced the partials.)  Dynamic smem: S * nval doubles.
__global__ void strided_finish_kernel(const double* __restrict__ partial, long long tpr, int nval, double* __restrict__ out);
static inline int strided_finish_threads(long long tpr, int nval) {
  long long slices = (tpr + 3) / 4;  // at least ~4 tiles per slice
  if (slices < 1) slices = 1;
  long long t = slices * nval;
  if (t > 1024) t = (1024 / nval) * (long long)nval;
  if (t < nval) t = nval;
  return (int)((t + 31) / 32 * 32 > 1024 ? 1024 : (t + 31) / 32 * 32);
}
#endif  // __CUDACC__

}  // namespace sb200
