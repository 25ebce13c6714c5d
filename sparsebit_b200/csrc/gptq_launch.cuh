// gptq_launch.cuh -- the internal launchers behind the GPTQ entry points (gptq.cu).  Each one trusts its arguments:
// gptq.cu has checked them, and group_size is already the real group size (0 replaced by K).
#pragma once
#include <cuda_fp16.h>

#include "common.cuh"

namespace sb200 {

// gptq_simt.cu: 2 / 3 / 4-bit SIMT dequant-matmul, any shape
int gptq_simt(int bits, const float* x, const int32_t* qweight, float* out, const float* scales, const float* zeros,
              long long M, long long K, long long N, long long KW, int group_size, cudaStream_t st);

// gptq_decode.cu: 4-bit decode-sized M on warp-level HMMA (N % 4 == 0, 16-byte aligned qweight)
constexpr int kDecMaxProblems = 4;  // problems of one sb200_gptq4_matmul_batch launch
bool gptq4_decode_supported(const int32_t* qweight, long long N);
void gptq4_decode_set_mode(int mode);
int gptq4_decode(const float* x, const int32_t* qweight, float* out, const float* scales, const float* zeros, long long M,
                 long long K, long long N, long long KW, int group_size, int flags, cudaStream_t st);
int gptq4_decode_batch(const sb200_gptq4_problem* problems, int count, long long M, int flags, cudaStream_t st);
size_t gptq4_decode_f16_partial_bytes(long long M, long long K, long long N);
int gptq4_decode_f16(const __half* x_h, const int32_t* qweight, __half* out_h, const float* bias, const float* scales,
                     const float* zeros, long long M, long long K, long long N, long long KW, int group_size, float* partial,
                     int* counters, int flags, cudaStream_t st);

// gptq_tc.cu: 4-bit prefill on wgmma
bool gptq4_tc_supported(const void* x, const int32_t* qweight, const float* out, long long M, long long K, long long N,
                        long long KW, int group_size);
size_t gptq4_tc_workspace(long long M, long long K, long long N, int group_size);
int gptq4_tc(const float* x, const int32_t* qweight, float* out, const float* scales, const float* zeros, long long M,
             long long K, long long N, long long KW, int group_size, void* workspace, size_t workspace_bytes,
             cudaStream_t st, const __half* x_h = nullptr, __half* out_h = nullptr, const float* bias = nullptr);
void gptq4_tc_set_backoff(int ns);
int gptq4_tc_backoff();
int gptq_launch_split(const float* x, __half* a_hi, __half* a_lo, float* xsum, float* rowscale, int* need_lo, long long M,
                      int K, int G, cudaStream_t st);

// gptq_dgrad.cu: the input gradient, 2 / 3 / 4-bit SIMT and 4-bit wgmma
size_t gptq_dgrad_simt_workspace(long long M, long long K, long long N, int group_size);
size_t gptq_dgrad_tc_workspace(long long M, long long K, long long N, int group_size);
bool gptq_dgrad_tc_supported(const float* grad_out, long long K, long long N, int group_size);
int gptq_dgrad_simt(int bits, const float* go, const int32_t* qweight, float* grad_in, const float* scales, const float* zeros,
                    long long M, long long K, long long N, long long KW, int group_size, void* workspace,
                    size_t workspace_bytes, cudaStream_t st);
int gptq4_dgrad_tc(const float* go, const int32_t* qweight, float* grad_in, const float* scales, const float* zeros,
                   long long M, long long K, long long N, long long KW, int group_size, void* workspace, size_t workspace_bytes,
                   cudaStream_t st);

}  // namespace sb200
