// gptq.cu -- C-ABI entry points of the GPTQ int4 dequant-matmul and the SIMT / tensor-core dispatch.
//
// Boundary replaced: cuda_kernel.vecquant4matmul / vecgroupquant4matmul
// (large_language_models/llama/quantization/cuda/cuda_kernel.cpp:10-23,70,73) and their argument
// checks (cuda_kernel_4bit.cu:44-60).
#include <cuda_fp16.h>

#include "common.cuh"

namespace sb200 {
int gptq4_simt(const float* x, const int32_t* qweight, float* out, const float* scales, const float* zeros,
               long long M, long long K, long long N, long long KW, int group_size, cudaStream_t st);
int gptq4_decode(const float* x, const int32_t* qweight, float* out, const float* scales, const float* zeros, long long M,
                 long long K, long long N, long long KW, int group_size, int flags, cudaStream_t st);
bool gptq4_tc_supported(const float* x, const int32_t* qweight, const float* out, long long M, long long K, long long N,
                        long long KW, int group_size);
size_t gptq4_tc_workspace(long long M, long long K, long long N, int group_size);
int gptq4_tc(const float* x, const int32_t* qweight, float* out, const float* scales, const float* zeros, long long M,
             long long K, long long N, long long KW, int group_size, void* workspace, size_t workspace_bytes,
             cudaStream_t st);
size_t gptq4_ts_workspace(long long M, long long K, long long N, int group_size);
int gptq4_ts(const float* x, const int32_t* qweight, float* out, const float* scales, const float* zeros, long long M,
             long long K, long long N, long long KW, int group_size, int chunk_kb, void* workspace, size_t workspace_bytes,
             cudaStream_t st, const __half* x_h = nullptr, __half* out_h = nullptr, const float* bias = nullptr);
size_t gptq4_decode_f16_partial_bytes(long long M, long long K, long long N);
int gptq4_decode_f16(const __half* x_h, const int32_t* qweight, __half* out_h, const float* bias, const float* scales,
                     const float* zeros, long long M, long long K, long long N, long long KW, int group_size, float* partial,
                     int* counters, int flags, cudaStream_t st);
bool gptq4_decode_supported(const int32_t* qweight, long long N);
void gptq4_tc_set_backoff(int ns);
void gptq4_decode_set_mode(int mode);
int gptq_lowbit(int bits, const float* x, const int32_t* qweight, float* out, const float* scales, const float* zeros,
                long long M, long long K, long long N, long long KW, int group_size, cudaStream_t st);
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
}  // namespace sb200

using namespace sb200;

extern "C" {

int sb200_gptq4_set_impl(int impl) {
  SB_REQUIRE(impl >= 0 && impl <= 4, "sb200_gptq4_set_impl: impl must be 0 .. 4 (got %d)", impl);
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
  const size_t a = gptq4_tc_workspace(m, k, n, group_size), b = gptq4_ts_workspace(m, k, n, group_size);
  return a > b ? a : b;
}

static int gptq4_dispatch(const float* x, const int32_t* qweight, float* out, const float* scales, const float* zeros,
                          int64_t m, int64_t k, int64_t n, int64_t qweight_rows, int group_size, int impl, int chunk_k,
                          void* workspace, size_t workspace_bytes, void* stream, int flags = 0) {
  SB_REQUIRE(x && qweight && out && scales && zeros, "sb200_gptq4_matmul: null pointer argument");
  SB_REQUIRE(m > 0 && k > 0 && n > 0, "sb200_gptq4_matmul: empty operand (M=%lld K=%lld N=%lld)", (long long)m,
             (long long)k, (long long)n);
  SB_REQUIRE(m < (1LL << 31) && k < (1LL << 31) && n < (1LL << 31), "sb200_gptq4_matmul: dimension too large");
  SB_REQUIRE(qweight_rows >= (k + 7) / 8,
             "sb200_gptq4_matmul: qweight has %lld rows, need ceil(K/8) = %lld", (long long)qweight_rows,
             (long long)((k + 7) / 8));
  SB_REQUIRE(impl >= 0 && impl <= 4, "sb200_gptq4_matmul: impl must be 0 (auto), 1 (small-M), 2 or 3 (tensor core), 4 (scalar) (got %d)", impl);
  SB_REQUIRE(chunk_k >= 0 && chunk_k % 64 == 0, "sb200_gptq4_matmul: chunk_k must be a multiple of 64 (got %d)", chunk_k);
  if (group_size != 0) {
    // cuda_kernel_4bit.cu:60
    SB_REQUIRE(group_size > 0 && group_size % 128 == 0,
               "only group_size divisible by 128 is supported in 4-bit quantization (got %d)", group_size);
  } else {
    group_size = (int)k;
  }
  cudaStream_t st = (cudaStream_t)stream;
  // 1 = small-M path: warp-level HMMA streaming kernel (gptq_decode.cu) when N % 4 == 0, else the scalar kernel;
  // 4 = scalar SIMT kernel (gptq_simt.cu, any shape);  2 = wgmma, exact int4 operands + per-128-K-group fp32 rescale (gptq_tc.cu);
  // 3 = wgmma, scaled fp16 weight planes as the register operand, whole-K accumulation (gptq_ts.cu).
  int use = 1;
  if (impl != 1 && impl != 4) {
    const bool shape_ok = gptq4_tc_supported(x, qweight, out, m, k, n, qweight_rows, group_size) && workspace;
    const bool ok2 = shape_ok && workspace_bytes >= gptq4_tc_workspace(m, k, n, group_size);
    const bool ok3 = shape_ok && workspace_bytes >= gptq4_ts_workspace(m, k, n, group_size);
    if (impl == 2 || impl == 3) {
      if (!(impl == 2 ? ok2 : ok3)) {
        set_error("sb200_gptq4_matmul: tensor-core path forced but shape/workspace unsupported (M=%lld K=%lld N=%lld gs=%d ws=%zu)",
                  (long long)m, (long long)k, (long long)n, group_size, workspace_bytes);
        return SB200_E_UNSUPPORTED;
      }
      use = impl;
    } else if (ok2 && m >= 32) {  // on the H100 the per-group kernel is faster than impl 3 at every M (DESIGN.md section 7)
      use = 2;
    }
  }
  if (use == 3)
    return gptq4_ts(x, qweight, out, scales, zeros, m, k, n, qweight_rows, group_size, chunk_k / 64, workspace,
                    workspace_bytes, st);
  if (use == 2)
    return gptq4_tc(x, qweight, out, scales, zeros, m, k, n, qweight_rows, group_size, workspace, workspace_bytes, st);
  if (impl != 4 && gptq4_decode_supported(qweight, n))
    return gptq4_decode(x, qweight, out, scales, zeros, m, k, n, qweight_rows, group_size, flags, st);
  return gptq4_simt(x, qweight, out, scales, zeros, m, k, n, qweight_rows, group_size, st);
}

int sb200_gptq4_matmul(const float* x, const int32_t* qweight, float* out, const float* scales, const float* zeros,
                       int64_t m, int64_t k, int64_t n, int64_t qweight_rows, int group_size, void* workspace,
                       size_t workspace_bytes, void* stream) {
  return gptq4_dispatch(x, qweight, out, scales, zeros, m, k, n, qweight_rows, group_size, g_gptq_impl, 0, workspace,
                        workspace_bytes, stream);
}

int sb200_gptq4_matmul_ex(const float* x, const int32_t* qweight, float* out, const float* scales, const float* zeros,
                          int64_t m, int64_t k, int64_t n, int64_t qweight_rows, int group_size,
                          const sb200_gptq4_options* options, void* workspace, size_t workspace_bytes, void* stream) {
  const int impl = options ? options->impl : 0, chunk_k = options ? options->chunk_k : 0, flags = options ? options->flags : 0;
  if (options) {
    SB_REQUIRE((flags & ~SB200_GPTQ4_STATIC_WEIGHTS) == 0, "sb200_gptq4_matmul_ex: unknown flags 0x%x", flags);
    for (int i = 0; i < 5; ++i) SB_REQUIRE(options->reserved[i] == 0, "sb200_gptq4_matmul_ex: reserved option fields must be zero");
  }
  return gptq4_dispatch(x, qweight, out, scales, zeros, m, k, n, qweight_rows, group_size, impl, chunk_k, workspace,
                        workspace_bytes, stream, flags);
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
  SB_REQUIRE(x_f16 && qweight && out_f16 && scales && zeros, "sb200_gptq4_linear_f16: null pointer argument");
  SB_REQUIRE((flags & ~SB200_GPTQ4_STATIC_WEIGHTS) == 0, "sb200_gptq4_linear_f16_ex: unknown flags 0x%x", flags);
  const int group_size_arg = group_size;  // 0 = one group: handed on unchanged (K itself need not be a multiple of 128)
  SB_REQUIRE(m > 0 && k > 0 && n > 0, "sb200_gptq4_linear_f16: empty operand (M=%lld K=%lld N=%lld)", (long long)m, (long long)k, (long long)n);
  SB_REQUIRE(m < (1LL << 31) && k < (1LL << 31) && n < (1LL << 31), "sb200_gptq4_linear_f16: dimension too large");
  SB_REQUIRE(qweight_rows >= (k + 7) / 8, "sb200_gptq4_linear_f16: qweight has %lld rows, need ceil(K/8) = %lld", (long long)qweight_rows, (long long)((k + 7) / 8));
  if (group_size != 0) {
    SB_REQUIRE(group_size > 0 && group_size % 128 == 0, "only group_size divisible by 128 is supported in 4-bit quantization (got %d)", group_size);
  } else {
    group_size = (int)k;
  }
  SB_REQUIRE(workspace && workspace_bytes >= sb200_gptq4_linear_f16_workspace_bytes(m, k, n, group_size), "sb200_gptq4_linear_f16: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  const __half* xh = reinterpret_cast<const __half*>(x_f16);
  __half* yh = reinterpret_cast<__half*>(out_f16);
  const bool ts_ok = m >= 768 && (k % 8 == 0) && (n % 4 == 0) && aligned16(x_f16) && aligned16(qweight) &&
                     gptq4_ts_workspace(m, k, n, group_size) > 0;
  if (ts_ok)  // fp16 in, fp16 out, no fp32 round trip of x or y
    return gptq4_ts(nullptr, qweight, nullptr, scales, zeros, m, k, n, qweight_rows, group_size, 0, workspace, workspace_bytes, st, xh, yh, bias);
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
  const int rc = gptq4_dispatch(x32, qweight, y32, scales, zeros, m, k, n, qweight_rows, group_size_arg, 0, 0, rest, rest_bytes, stream,
                                SB200_GPTQ4_STATIC_WEIGHTS);
  if (rc) return rc;
  f32_to_f16_kernel<<<ew_grid(m * n), 256, 0, st>>>(y32, yh, m * n);
  SB_LAUNCHED();
  return SB200_OK;
}

int sb200_gptq_matmul(const float* x, const int32_t* qweight, float* out, const float* scales, const float* zeros,
                      int64_t m, int64_t k, int64_t n, int64_t qweight_rows, int bits, int group_size, void* workspace,
                      size_t workspace_bytes, void* stream) {
  SB_REQUIRE(bits == 2 || bits == 3 || bits == 4, "sb200_gptq_matmul: only support 2/3/4 bit now (got %d)", bits);
  if (bits == 4)
    return sb200_gptq4_matmul(x, qweight, out, scales, zeros, m, k, n, qweight_rows, group_size, workspace,
                              workspace_bytes, stream);
  SB_REQUIRE(x && qweight && out && scales && zeros, "sb200_gptq_matmul: null pointer argument");
  SB_REQUIRE(m > 0 && k > 0 && n > 0, "sb200_gptq_matmul: empty operand (M=%lld K=%lld N=%lld)", (long long)m,
             (long long)k, (long long)n);
  SB_REQUIRE(m < (1LL << 31) && k < (1LL << 31) && n < (1LL << 31), "sb200_gptq_matmul: dimension too large");
  // rows QuantLinear allocates (utils/quant.py:172-184): ceil(K*bit / (32*p)) * p, p = 3 for 3-bit
  const int64_t need = bits == 2 ? (k + 15) / 16 : ((k * 3 + 95) / 96) * 3;
  SB_REQUIRE(qweight_rows >= need, "sb200_gptq_matmul: qweight has %lld rows, %d-bit K=%lld needs %lld",
             (long long)qweight_rows, bits, (long long)k, (long long)need);
  const int min_group = bits == 2 ? 64 : 128;  // cuda_kernel_2bit.cu:58, cuda_kernel_3bit.cu:60
  if (group_size != 0) {
    SB_REQUIRE(group_size > 0 && group_size % min_group == 0,
               "only group_size divisible by %d is supported in %d-bit quantization (got %d)", min_group, bits, group_size);
  } else {
    group_size = (int)k;
  }
  return gptq_lowbit(bits, x, qweight, out, scales, zeros, m, k, n, qweight_rows, group_size, (cudaStream_t)stream);
}

}  // extern "C"
