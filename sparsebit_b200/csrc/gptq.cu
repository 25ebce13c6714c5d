// gptq.cu -- C-ABI entry points of the GPTQ 2 / 3 / 4-bit dequant-matmul and its input gradient: the argument
// checks and the SIMT / decode / tensor-core dispatch.
//
// Boundary replaced: cuda_kernel.vecquant4matmul / vecgroupquant4matmul
// (large_language_models/llama/quantization/cuda/cuda_kernel.cpp:10-23,70,73) and their argument
// checks (cuda_kernel_4bit.cu:44-60).
#include <stdio.h>

#include "gptq_launch.cuh"
#include "gptq_unpack.cuh"

namespace sb200 {
static int g_gptq_impl = 0;

// fp16 <-> fp32 staging for the paths of sb200_gptq4_linear_f16 that run the fp32 kernels (small M)
__global__ void __launch_bounds__(256) f16_to_f32_kernel(const __half* __restrict__ src, float* __restrict__ dst, long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) dst[i] = __half2float(src[i]);
}
__global__ void __launch_bounds__(256) bias_rows_kernel(const float* __restrict__ bias, float* __restrict__ dst, long long rows, long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < rows * n; i += (long long)gridDim.x * blockDim.x) dst[i] = bias ? bias[i % n] : 0.f;
}
__global__ void __launch_bounds__(256) f32_to_f16_kernel(const float* __restrict__ src, __half* __restrict__ dst, long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) dst[i] = __float2half_rn(src[i]);
}
static inline unsigned ew_grid(long long n) {
  long long b = (n + 255) / 256, cap = (long long)sm_count() * 16;
  return (unsigned)(b < 1 ? 1 : (b > cap ? cap : b));
}

// The operand rules of every GPTQ entry point, checked before any CUDA call (cuda_kernel_{2,3,4}bit.cu argument
// checks): 2, 3 or 4 bits, non-null operands, 1 <= M, K, N < 2^31, at least the packed rows QuantLinear allocates for K,
// and a group size that is a multiple of 128 (2-bit: 64).  `fn` names the caller in the messages.  *group_size == 0
// means one group and is replaced by K.
static int check_gptq_args(const char* fn, int bits, const void* x, const int32_t* qweight, const void* out,
                           const float* scales, const float* zeros, int64_t m, int64_t k, int64_t n, int64_t qweight_rows,
                           int* group_size) {
  SB_REQUIRE(bits == 2 || bits == 3 || bits == 4, "%s: only support 2/3/4 bit now (got %d)", fn, bits);
  SB_REQUIRE(x && qweight && out && scales && zeros, "%s: null pointer argument", fn);
  SB_REQUIRE(m > 0 && k > 0 && n > 0, "%s: empty operand (M=%lld K=%lld N=%lld)", fn, (long long)m, (long long)k, (long long)n);
  SB_REQUIRE(m < (1LL << 31) && k < (1LL << 31) && n < (1LL << 31), "%s: dimension too large", fn);
  const long long need = gptq_packed_rows(bits, k);
  SB_REQUIRE(qweight_rows >= need, "%s: qweight has %lld rows, %d-bit K=%lld needs %lld", fn, (long long)qweight_rows, bits,
             (long long)k, need);
  const int min_group = bits == 2 ? 64 : 128;  // cuda_kernel_2bit.cu:58, cuda_kernel_3bit.cu:60, cuda_kernel_4bit.cu:60
  SB_REQUIRE(*group_size >= 0 && *group_size % min_group == 0,
             "only group_size divisible by %d is supported in %d-bit quantization (got %d)", min_group, bits, *group_size);
  if (*group_size == 0) *group_size = (int)k;
  return SB200_OK;
}
}  // namespace sb200

using namespace sb200;

extern "C" {

int sb200_gptq4_set_impl(int impl) {
  SB_REQUIRE(impl >= 0 && impl <= 4 && impl != 3, "sb200_gptq4_set_impl: impl must be 0, 1, 2 or 4 (got %d)", impl);
  g_gptq_impl = impl;
  return SB200_OK;
}

int sb200_gptq4_set_wait_backoff(int nanoseconds) {
  SB_REQUIRE(nanoseconds >= 0 && nanoseconds <= 100000, "sb200_gptq4_set_wait_backoff: 0..100000 ns (got %d)", nanoseconds);
  gptq4_tc_set_backoff(nanoseconds);
  return SB200_OK;
}

int sb200_gptq4_set_decode(int mode) {
  SB_REQUIRE(mode >= 0 && mode <= 255, "sb200_gptq4_set_decode: mode is a bit mask 0 .. 255 (got %d)", mode);
  gptq4_decode_set_mode(mode);
  return SB200_OK;
}

size_t sb200_gptq4_workspace_bytes(int64_t m, int64_t k, int64_t n, int group_size) {
  if (m <= 0 || k <= 0 || n <= 0) return 0;
  if (group_size <= 0) group_size = (int)k;
  return gptq4_tc_workspace(m, k, n, group_size);
}

// Arguments as check_gptq_args left them, impl in {0, 1, 2, 4}.
static int gptq4_dispatch(const float* x, const int32_t* qweight, float* out, const float* scales, const float* zeros,
                          int64_t m, int64_t k, int64_t n, int64_t qweight_rows, int group_size, int impl,
                          void* workspace, size_t workspace_bytes, void* stream, int flags = 0) {
  cudaStream_t st = (cudaStream_t)stream;
  // 1 = small-M path: warp-level HMMA streaming kernel (gptq_decode.cu) when N % 4 == 0, else the scalar kernel;
  // 4 = scalar SIMT kernel (gptq_simt.cu, any shape);  2 = wgmma, exact int4 operands + per-128-K-group fp32 rescale (gptq_tc.cu).
  int use = 1;
  if (impl != 1 && impl != 4) {
    const bool ok2 = gptq4_tc_supported(x, qweight, out, m, k, n, qweight_rows, group_size) && workspace &&
                     workspace_bytes >= gptq4_tc_workspace(m, k, n, group_size);
    if (impl == 2 && !ok2) {
      set_error("sb200_gptq4_matmul: tensor-core path forced but shape/workspace unsupported (M=%lld K=%lld N=%lld gs=%d ws=%zu)",
                (long long)m, (long long)k, (long long)n, group_size, workspace_bytes);
      return SB200_E_UNSUPPORTED;
    }
    if (ok2 && (impl == 2 || m >= 32)) use = 2;
  }
  if (use == 2)
    return gptq4_tc(x, qweight, out, scales, zeros, m, k, n, qweight_rows, group_size, workspace, workspace_bytes, st);
  if (impl != 4 && gptq4_decode_supported(qweight, n))
    return gptq4_decode(x, qweight, out, scales, zeros, m, k, n, qweight_rows, group_size, flags, st);
  return gptq_simt(4, x, qweight, out, scales, zeros, m, k, n, qweight_rows, group_size, st);
}

int sb200_gptq4_matmul(const float* x, const int32_t* qweight, float* out, const float* scales, const float* zeros,
                       int64_t m, int64_t k, int64_t n, int64_t qweight_rows, int group_size, void* workspace,
                       size_t workspace_bytes, void* stream) {
  if (const int rc = check_gptq_args("sb200_gptq4_matmul", 4, x, qweight, out, scales, zeros, m, k, n, qweight_rows, &group_size))
    return rc;
  return gptq4_dispatch(x, qweight, out, scales, zeros, m, k, n, qweight_rows, group_size, g_gptq_impl, workspace,
                        workspace_bytes, stream);
}

int sb200_gptq4_matmul_ex(const float* x, const int32_t* qweight, float* out, const float* scales, const float* zeros,
                          int64_t m, int64_t k, int64_t n, int64_t qweight_rows, int group_size,
                          const sb200_gptq4_options* options, void* workspace, size_t workspace_bytes, void* stream) {
  const int impl = options ? options->impl : 0, flags = options ? options->flags : 0;
  if (options) {
    SB_REQUIRE(impl >= 0 && impl <= 4 && impl != 3, "sb200_gptq4_matmul_ex: impl must be 0 (auto), 1 (small-M), 2 (tensor core), 4 (scalar) (got %d)", impl);
    SB_REQUIRE((flags & ~SB200_GPTQ4_STATIC_WEIGHTS) == 0, "sb200_gptq4_matmul_ex: unknown flags 0x%x", flags);
    SB_REQUIRE(options->chunk_k == 0, "sb200_gptq4_matmul_ex: chunk_k is reserved and must be zero (got %d)", options->chunk_k);
    for (int i = 0; i < 5; ++i) SB_REQUIRE(options->reserved[i] == 0, "sb200_gptq4_matmul_ex: reserved option fields must be zero");
  }
  if (const int rc = check_gptq_args("sb200_gptq4_matmul_ex", 4, x, qweight, out, scales, zeros, m, k, n, qweight_rows, &group_size))
    return rc;
  return gptq4_dispatch(x, qweight, out, scales, zeros, m, k, n, qweight_rows, group_size, impl, workspace,
                        workspace_bytes, stream, flags);
}

int sb200_gptq4_matmul_batch(const sb200_gptq4_problem* problems, int count, int64_t m, void* stream) {
  return sb200_gptq4_matmul_batch_ex(problems, count, m, 0, stream);
}

int sb200_gptq4_matmul_batch_ex(const sb200_gptq4_problem* problems, int count, int64_t m, int flags, void* stream) {
  SB_REQUIRE((flags & ~SB200_GPTQ4_STATIC_WEIGHTS) == 0, "sb200_gptq4_matmul_batch_ex: unknown flags 0x%x", flags);
  SB_REQUIRE(problems && count >= 1 && count <= kDecMaxProblems, "sb200_gptq4_matmul_batch: 1 .. %d problems (got %d)", kDecMaxProblems, count);
  SB_REQUIRE(m >= 1 && m <= 32, "sb200_gptq4_matmul_batch: decode-sized M only (1 .. 32, got %lld)", (long long)m);
  sb200_gptq4_problem p[kDecMaxProblems];
  for (int i = 0; i < count; ++i) {
    p[i] = problems[i];
    char fn[64];
    snprintf(fn, sizeof fn, "sb200_gptq4_matmul_batch: problem %d", i);
    if (const int rc = check_gptq_args(fn, 4, p[i].x, p[i].qweight, p[i].out, p[i].scales, p[i].zeros, m, p[i].k, p[i].n,
                                       p[i].qweight_rows, &p[i].group_size))
      return rc;
    SB_REQUIRE(gptq4_decode_supported(p[i].qweight, p[i].n), "%s needs N %% 4 == 0 and a 16-byte aligned qweight", fn);
  }
  return gptq4_decode_batch(p, count, m, flags, (cudaStream_t)stream);
}

constexpr int64_t kF16SingleLaunchMaxM = 32;
constexpr size_t kF16StateBytes = 65536;  // one int per 128-feature block: N <= 2 097 152

size_t sb200_gptq4_linear_f16_workspace_bytes(int64_t m, int64_t k, int64_t n, int group_size) {
  if (m <= 0 || k <= 0 || n <= 0) return 0;
  // fp32 staging of x and y for the small-M paths + the kernels' own workspace + the per-slice partial sums of the
  // single-launch decode path
  const size_t part = m <= kF16SingleLaunchMaxM ? gptq4_decode_f16_partial_bytes(m, k, n) + 256 : 0;
  return sb200_gptq4_workspace_bytes(m, k, n, group_size) + (size_t)m * (size_t)(k + n) * sizeof(float) + 2048 + part;
}

size_t sb200_gptq4_linear_f16_state_bytes(void) { return kF16StateBytes; }

int sb200_gptq4_linear_f16(const void* x_f16, const int32_t* qweight, void* out_f16, const float* bias, const float* scales,
                           const float* zeros, int64_t m, int64_t k, int64_t n, int64_t qweight_rows, int group_size,
                           void* workspace, size_t workspace_bytes, void* stream) {
  return sb200_gptq4_linear_f16_ex(x_f16, qweight, out_f16, bias, scales, zeros, m, k, n, qweight_rows, group_size, nullptr, 0,
                                   workspace, workspace_bytes, stream);
}

int sb200_gptq4_linear_f16_ex(const void* x_f16, const int32_t* qweight, void* out_f16, const float* bias, const float* scales,
                              const float* zeros, int64_t m, int64_t k, int64_t n, int64_t qweight_rows, int group_size,
                              void* state, int flags, void* workspace, size_t workspace_bytes, void* stream) {
  if (const int rc = check_gptq_args("sb200_gptq4_linear_f16", 4, x_f16, qweight, out_f16, scales, zeros, m, k, n, qweight_rows,
                                     &group_size))
    return rc;
  SB_REQUIRE((flags & ~SB200_GPTQ4_STATIC_WEIGHTS) == 0, "sb200_gptq4_linear_f16_ex: unknown flags 0x%x", flags);
  SB_REQUIRE(workspace && workspace_bytes >= sb200_gptq4_linear_f16_workspace_bytes(m, k, n, group_size), "sb200_gptq4_linear_f16: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  const __half* xh = reinterpret_cast<const __half*>(x_f16);
  __half* yh = reinterpret_cast<__half*>(out_f16);
  if (m >= 768 && gptq4_tc_supported(x_f16, qweight, nullptr, m, k, n, qweight_rows, group_size))  // fp16 in, fp16 out, no fp32 round trip of x or y
    return gptq4_tc(nullptr, qweight, nullptr, scales, zeros, m, k, n, qweight_rows, group_size, workspace, workspace_bytes, st, xh, yh, bias);
  if (state && m <= kF16SingleLaunchMaxM && gptq4_decode_supported(qweight, n) && n <= (int64_t)(kF16StateBytes / sizeof(int)) * 128) {
    // decode-sized M with a caller-provided (zero-initialised, self-resetting) arrival-counter state: ONE launch -- fp16
    // activations are read by the kernel's staging, the last K-slice CTA of every feature block writes bias + sum as fp16
    float* partial = reinterpret_cast<float*>(((reinterpret_cast<uintptr_t>(workspace) + 255) / 256) * 256);
    return gptq4_decode_f16(xh, qweight, yh, bias, scales, zeros, m, k, n, qweight_rows, group_size, partial,
                            reinterpret_cast<int*>(state), flags, st);
  }
  // small M: stage through fp32 inside the library (a few MB at most) and run the fp32 kernels
  unsigned char* ws = reinterpret_cast<unsigned char*>(((reinterpret_cast<uintptr_t>(workspace) + 255) / 256) * 256);
  float* x32 = reinterpret_cast<float*>(ws);
  float* y32 = x32 + (size_t)m * k;
  unsigned char* rest = reinterpret_cast<unsigned char*>(y32 + (size_t)m * n);
  const size_t rest_bytes = workspace_bytes - (size_t)(rest - reinterpret_cast<unsigned char*>(workspace));
  f16_to_f32_kernel<<<ew_grid(m * k), 256, 0, st>>>(xh, x32, m * k);
  SB_LAUNCHED();
  bias_rows_kernel<<<ew_grid(m * n), 256, 0, st>>>(bias, y32, m, n);
  SB_LAUNCHED();
  // the kernel immediately in front is bias_rows_kernel (writes y32 only): the weight tables cannot be its output
  const int rc = gptq4_dispatch(x32, qweight, y32, scales, zeros, m, k, n, qweight_rows, group_size, 0, rest, rest_bytes, stream,
                                SB200_GPTQ4_STATIC_WEIGHTS);
  if (rc) return rc;
  f32_to_f16_kernel<<<ew_grid(m * n), 256, 0, st>>>(y32, yh, m * n);
  SB_LAUNCHED();
  return SB200_OK;
}

int sb200_gptq_matmul(const float* x, const int32_t* qweight, float* out, const float* scales, const float* zeros,
                      int64_t m, int64_t k, int64_t n, int64_t qweight_rows, int bits, int group_size, void* workspace,
                      size_t workspace_bytes, void* stream) {
  if (const int rc = check_gptq_args("sb200_gptq_matmul", bits, x, qweight, out, scales, zeros, m, k, n, qweight_rows, &group_size))
    return rc;
  if (bits == 4)
    return gptq4_dispatch(x, qweight, out, scales, zeros, m, k, n, qweight_rows, group_size, g_gptq_impl, workspace,
                          workspace_bytes, stream);
  return gptq_simt(bits, x, qweight, out, scales, zeros, m, k, n, qweight_rows, group_size, (cudaStream_t)stream);
}

// Auto dispatch of the input gradient: the tensor-core kernel from this many rows of grad_out on (4-bit shapes it takes).
// Measured crossover (scripts/bench_gptq_dgrad.py, H100 80GB HBM3 at a 700 W power limit, LLaMA-7B g128 shapes): at
// M = 32 the SIMT kernel wins on 4096x4096 and 4096x11008 (84 vs 119 us, 223 vs 308 us), at M = 48 the two tie there
// (120 vs 120 us, 317 vs 314 us), from M = 64 on the tensor-core kernel wins on every shape (11008x4096: from M = 32).
constexpr int64_t kDgradTcMinM = 48;

size_t sb200_gptq_dgrad_workspace_bytes(int64_t m, int64_t k, int64_t n, int bits, int group_size) {
  if (m <= 0 || k <= 0 || n <= 0) return 0;
  if (group_size <= 0) group_size = (int)k;
  const size_t a = gptq_dgrad_simt_workspace(m, k, n, group_size);
  const size_t b = bits == 4 ? gptq_dgrad_tc_workspace(m, k, n, group_size) : 0;
  return a > b ? a : b;
}

int sb200_gptq_matmul_dgrad(const float* grad_out, const int32_t* qweight, float* grad_in, const float* scales,
                            const float* zeros, int64_t m, int64_t k, int64_t n, int64_t qweight_rows, int bits,
                            int group_size, int impl, void* workspace, size_t workspace_bytes, void* stream) {
  if (const int rc = check_gptq_args("sb200_gptq_matmul_dgrad", bits, grad_out, qweight, grad_in, scales, zeros, m, k, n,
                                     qweight_rows, &group_size))
    return rc;
  SB_REQUIRE(impl >= 0 && impl <= 2, "sb200_gptq_matmul_dgrad: impl must be 0 (auto), 1 (SIMT) or 2 (tensor core) (got %d)", impl);
  cudaStream_t st = (cudaStream_t)stream;
  const bool tc_ok = bits == 4 && gptq_dgrad_tc_supported(grad_out, k, n, group_size) && workspace &&
                     workspace_bytes >= gptq_dgrad_tc_workspace(m, k, n, group_size);
  if (impl == 2 && !tc_ok) {
    set_error("sb200_gptq_matmul_dgrad: tensor-core path forced but shape/workspace unsupported (bits=%d M=%lld K=%lld N=%lld gs=%d ws=%zu)",
              bits, (long long)m, (long long)k, (long long)n, group_size, workspace_bytes);
    return SB200_E_UNSUPPORTED;
  }
  if (impl == 2 || (impl == 0 && tc_ok && m >= kDgradTcMinM))
    return gptq4_dgrad_tc(grad_out, qweight, grad_in, scales, zeros, m, k, n, qweight_rows, group_size, workspace,
                          workspace_bytes, st);
  return gptq_dgrad_simt(bits, grad_out, qweight, grad_in, scales, zeros, m, k, n, qweight_rows, group_size, workspace,
                         workspace_bytes, st);
}

}  // extern "C"
