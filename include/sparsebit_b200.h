/*
 * sparsebit_b200.h -- C-ABI of the H100-native (sm_90a) fake-quantization / observer / sparser /
 * GPTQ-int4 hot path.  This is the drop-in boundary: plain pointers and sizes, no torch types.
 *
 * Every entry point cites the reference interface it replaces (paths relative to the
 * megvii-research/Sparsebit tree, commit f473aef).  The reference exposes this path as two pybind
 * modules (`fake_quant`, `cuda_kernel`) plus chains of ATen ops inside its Python observers and
 * sparsers; INTEGRATION.md shows the ctypes / pybind stub a maintainer adds on the reference side.
 *
 * Conventions
 *   - All `const float*` / `float*` data arguments are DEVICE pointers (fp32, contiguous) unless the
 *     function name ends in `_host`, in which case the data arguments are HOST pointers (ideally
 *     pinned) and the call performs the H2D / D2H copies itself, pipelined over internal streams.
 *   - `stream` is a `cudaStream_t` passed as `void*` (NULL = legacy default stream).  Device
 *     entry points are asynchronous on that stream, never synchronise the host, keep no global
 *     state and are re-entrant (the reference kernels have the same contract:
 *     sparsebit/quantization/torch_extensions/fake_quant_tensor.cu:83,152,212,297).
 *   - Return value: 0 on success, a negative SB200_E_* code on error; `sb200_last_error()` returns
 *     a thread-local human readable message.  The reference reports the same conditions as
 *     C++ exceptions -> Python RuntimeError (torch_extensions/common.cuh:27-55,
 *     large_language_models/llama/quantization/cuda/cuda_kernel_4bit.cu:44-60); the Python host
 *     layer (`sparsebit_b200/`) turns non-zero codes back into RuntimeError.
 *   - `rounding`: 0 = half-to-even (the only value the reference ever passes,
 *     quantizers/quant_tensor.py:99,109,147,151), 1 = half-up, 2 = half-down
 *     (torch_extensions/common.cuh:21-23).
 *   - Numerics follow the reference's *CPU Python* path (quant_tensor.py:181-184), which is the
 *     parity oracle: zp = rint(zero_point) half-to-even, IEEE division x/scale, float clamp,
 *     (q - zp) * scale without FMA contraction.  Finite inputs agree bit-for-bit with both the
 *     reference CPU path and its CUDA kernels; NaN propagates like torch.clamp.
 */
#ifndef SPARSEBIT_B200_H_
#define SPARSEBIT_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif
#if defined(__GNUC__)
#pragma GCC visibility push(default) /* the library is built with -fvisibility=hidden */
#endif

#define SB200_OK 0
#define SB200_E_INVALID (-1)   /* bad argument (null pointer, empty tensor, bad size) */
#define SB200_E_CUDA (-2)      /* a CUDA runtime call failed */
#define SB200_E_UNSUPPORTED (-3)
#define SB200_E_WORKSPACE (-4) /* caller workspace too small */

/* ---- library ---------------------------------------------------------------------------- */
const char* sb200_last_error(void);
int sb200_version(void);
/* Number of SMs of the current device (grid sizing is derived from it). */
int sb200_sm_count(void);
/* Select an implementation variant for the streaming QDQ kernels: 0 = auto, 1 = 128-bit LDG/STG
 * register pipeline, 2 = TMA (cp.async.bulk) shared-memory ring.  For benchmarking only. */
int sb200_set_variant(int variant);

/* ---- (1) Quantizer.forward: quantize -> dequantize ---------------------------------------
 * Replaces fake_quant.quant_pertensor_forward   (torch_extensions/export.cc:4,
 *          fake_quant_tensor.cu:50-94)   and the CPU branch quant_tensor.py:181-184.
 * out[i] = (clamp(round(x[i]/scale[0]) + rint(zp[0]), qmin, qmax) - rint(zp[0])) * scale[0]
 * scale / zero_point: device pointers to 1 float each. */
int sb200_qdq_pertensor_fwd(const float* x, const float* scale, const float* zero_point,
                            float* out, int64_t n, int qmin, int qmax, int rounding, void* stream);

/* Replaces fake_quant.quant_perchannel_forward (export.cc:6, fake_quant_tensor.cu:170-224).
 * x is viewed as [outer, C, inner] (inner = prod(sizes[ch_axis+1:]), fake_quant_tensor.cu:203-208);
 * scale / zero_point hold C floats and are indexed by c = (i / inner) % C. */
int sb200_qdq_perchannel_fwd(const float* x, const float* scale, const float* zero_point,
                             float* out, int64_t outer, int64_t channels, int64_t inner, int qmin,
                             int qmax, int rounding, void* stream);

/* Fused QDQ + MinMax observer statistics of the INPUT x (new; the reference runs
 * Quantizer.forward and observers/minmax.py:14-25 as separate ATen passes).  `minmax_state` is a
 * running state of 2 uint32 {enc(min), enc(max)} created by sb200_minmax_init(.., 1, ..) and
 * decoded by sb200_minmax_read.  8 B/elem of HBM traffic, the kernel the 70 % roofline target is
 * quoted on. */
int sb200_qdq_stats_pertensor_fwd(const float* x, const float* scale, const float* zero_point,
                                  float* out, uint32_t* minmax_state, int64_t n, int qmin, int qmax,
                                  int rounding, void* stream);

/* Host-buffer (end-to-end) variants: x_host/out_host are host pointers; scale/zero_point are HOST
 * floats.  Copies are chunked and overlapped with the kernel on internal streams; the call
 * returns after the last D2H copy completed.  minmax_host receives {min, max} (may be NULL). */
int sb200_qdq_pertensor_fwd_host(const float* x_host, float scale, float zero_point,
                                 float* out_host, float* minmax_host, int64_t n, int qmin, int qmax,
                                 int rounding);
/* Asynchronous form: enqueues the copies / kernels and returns; host buffers (pinned for real overlap)
 * must stay valid and untouched until sb200_host_sync() returns.  Back-to-back calls keep the H2D and D2H
 * engines busy across calls instead of draining the pipeline once per tensor. */
int sb200_qdq_pertensor_fwd_host_async(const float* x_host, float scale, float zero_point,
                                       float* out_host, float* minmax_host, int64_t n, int qmin,
                                       int qmax, int rounding);
int sb200_host_sync(void);
int sb200_qdq_perchannel_fwd_host(const float* x_host, const float* scale_host,
                                  const float* zero_point_host, float* out_host, int64_t outer,
                                  int64_t channels, int64_t inner, int qmin, int qmax,
                                  int rounding);

/* ---- STE backward ------------------------------------------------------------------------
 * Replaces fake_quant.quant_pertensor_backward (export.cc:5, fake_quant_tensor.cu:97-167) and
 * quant_perchannel_backward (export.cc:7, fake_quant_tensor.cu:227-314).
 *   vq = round(x/s) + zp ;  gx = gy * [qmin <= vq <= qmax]
 *   gs  = sum gy * { round(x/s) - x/s  inside ; (qmin - zp) below ; (qmax - zp) above }
 *   gzp = sum -s * gy * [vq outside [qmin, qmax]]         per-tensor (fake_quant_tensor.cu:126)
 *   gzp = sum -s * gy * [vq outside [qmin, qmax)]         per-channel: the reference kernel counts vq == qmax
 *                                                         as clipped (fake_quant_tensor.cu:264); reproduced as is
 * gs / gzp may be NULL (the reference's enable_gs / enable_gzp = requires_grad flags).  They are
 * produced by a deterministic two-stage reduction (fp32 per thread, fp64 across CTAs) instead of
 * float atomics.  `workspace` must hold sb200_qdq_bwd_workspace_bytes(...) bytes. */
size_t sb200_qdq_bwd_workspace_bytes(int64_t outer, int64_t channels, int64_t inner);
int sb200_qdq_pertensor_bwd(const float* x, const float* scale, const float* zero_point,
                            const float* grad_y, float* grad_x, float* grad_scale, float* grad_zp,
                            int64_t n, int qmin, int qmax, int rounding, void* workspace,
                            size_t workspace_bytes, void* stream);
int sb200_qdq_perchannel_bwd(const float* x, const float* scale, const float* zero_point,
                             const float* grad_y, float* grad_x, float* grad_scale, float* grad_zp,
                             int64_t outer, int64_t channels, int64_t inner, int qmin, int qmax,
                             int rounding, void* workspace, size_t workspace_bytes, void* stream);

/* Same as sb200_qdq_perchannel_bwd with `flags`: SB200_BWD_GZP_CLOSED selects the closed interval
 * qmin <= vq <= qmax for the zero-point gradient, i.e. the rule of the reference's Python statement of the
 * backward (MySTE.backward, quantizers/quant_tensor.py:62-69) and of its per-tensor kernel. */
#define SB200_BWD_GZP_CLOSED 1
int sb200_qdq_perchannel_bwd_ex(const float* x, const float* scale, const float* zero_point,
                                const float* grad_y, float* grad_x, float* grad_scale, float* grad_zp,
                                int64_t outer, int64_t channels, int64_t inner, int qmin, int qmax,
                                int rounding, int flags, void* workspace, size_t workspace_bytes,
                                void* stream);

/* PACT (quantizers/pact.py:43-46) clamps the activation to the learnable [lower, alpha] in front of the fake-quant op and
 * lets autograd differentiate the clamp.  The clamp does not change the forward value (the QDQ grid derived from
 * [lower, alpha] clamps to the same points), so the native PACT quantizer skips that 8 B/elem pass and only needs the
 * clamp's backward:   grad_x = grad_y * [lo <= x <= hi],  grad_hi = sum grad_y * [x > hi],  grad_lo = sum grad_y * [x < lo]
 * (torch.clamp's convention).  lo / hi: device scalars.  grad_hi / grad_lo may be NULL.  Deterministic. */
size_t sb200_clamp_bwd_workspace_bytes(int64_t n);
int sb200_clamp_bwd(const float* x, const float* grad_y, const float* lo, const float* hi, float* grad_x,
                    float* grad_hi, float* grad_lo, int64_t n, void* workspace, size_t workspace_bytes,
                    void* stream);

/* ---- (2) Observer calibration reductions -------------------------------------------------
 * MinMax (observers/minmax.py:14-25 -- torch.cat + min/max).  Streaming: the state is updated
 * in place per batch, nothing is cached or concatenated.  State layout: uint32[2*C], entry 2c =
 * order-preserving encoding of the running min of channel c, 2c+1 = of the running max; a third
 * implicit NaN flag is encoded as enc(NaN).  C = 1 for per-tensor. */
int sb200_minmax_init(uint32_t* state, int64_t channels, void* stream);
int sb200_observe_minmax(const float* x, int64_t n, uint32_t* state, void* stream);
int sb200_observe_minmax_perchannel(const float* x, int64_t outer, int64_t channels, int64_t inner,
                                    uint32_t* state, void* stream);
/* Decode to floats: out_min[C], out_max[C] (device pointers). */
int sb200_minmax_read(const uint32_t* state, int64_t channels, float* out_min, float* out_max,
                      void* stream);

/* qparams of MANY MinMax observers in one launch: running state -> min, max, scale, zero_point
 * (observers/minmax.py:14-25 + Observer.calc_qparams_with_minmax, observers/base.py:63-79; the reference -- and a
 * per-quantizer port -- spends ~15 tiny ATen launches per quantizer here, which dominates a streaming calibration).
 *   symmetric: scale = max(max(-min(min,0), max(max,0)) * 2 / (qmax - qmin), 1e-6), zero_point = 0
 *   affine:    scale = max((max(max,0) - min(min,0)) / (qmax - qmin), 1e-6), zero_point = round(-min(min,0) / scale)
 * with IEEE fp32 operations in that order (bit-identical to the torch statement).  `device_table`: caller-owned scratch
 * of count * 64 bytes.  Outputs hold `channels` floats each. */
typedef struct sb200_minmax_qparams_desc {
  const uint32_t* state;
  float* out_min;
  float* out_max;
  float* out_scale;
  float* out_zero_point;
  int64_t channels;
  int qmin, qmax, symmetric;
} sb200_minmax_qparams_desc;
int sb200_minmax_qparams_multi(const sb200_minmax_qparams_desc* descs, int count, void* device_table,
                               size_t table_bytes, void* stream);

/* KL-histogram (observers/kl_histogram.py:47-50 -> torch.histc on CPU).  counts[bins] (int64) is
 * accumulated in place.  `range` = device {lo, hi}.  Bin rule = ATen's CPU histc
 * (HistogramKernel.cpp, linear interpolation): pos = (int64)(((x - lo) * bins) / (hi - lo)) in
 * fp32 with IEEE division, pos == bins folded into the last bin, x outside [lo, hi] and NaN
 * ignored. */
int sb200_observe_hist(const float* x, int64_t n, const float* range, int bins, int64_t* counts,
                       void* stream);

/* MSE observer sweep (observers/mse.py:46-61): for each row r (R rows of `row_len` contiguous
 * floats; R = 1 for per-tensor) and each of `ncand` candidate (scale, zp) pairs
 * cand_scale/cand_zp[r*ncand + i], accumulate sse[r*ncand + i] += sum_j (x - qdq_i(x))^2 in one
 * pass over x (the reference does ncand=80 full QDQ + loss passes).  sse is fp64, accumulated in
 * place (so several cached batches / several GPUs add up); workspace from
 * sb200_mse_workspace_bytes. */
size_t sb200_mse_workspace_bytes(int64_t rows, int64_t row_len, int ncand);
int sb200_observe_mse_sweep(const float* x, int64_t rows, int64_t row_len, const float* cand_scale,
                            const float* cand_zp, int ncand, int qmin, int qmax, double* sse,
                            void* workspace, size_t workspace_bytes, void* stream);

/* Exact order statistics by MSB-first radix select on an order-preserving 32-bit key
 * (replaces torch.kthvalue in observers/percentile.py:34-43 and torch.sort in
 * sparse/sparsers/l1norm.py:18-22).  Three passes over the data (11 + 11 + 10 key bits); each pass
 * is   sb200_select_hist (adds this shard's digit histogram for every live target)
 *      [optional: SUM all-reduce of `hist` across GPUs]
 *      sb200_select_scan (finds each target's bucket, narrows prefix and rank, clears hist).
 * `sel` is an opaque device state of SB200_SELECT_STATE_WORDS uint64 per target; `hist` holds
 * ntargets * 2048 int64.  key_mode 0: key = enc(x) (signed order); 1: key = enc(|x|).
 * Row-batched: `rows` independent rows of `row_len` floats, targets are per row
 * (ntargets_per_row of them), state index = row * ntargets_per_row + t. */
#define SB200_SELECT_STATE_WORDS 4
#define SB200_SELECT_BINS 2048
/* Reset `sel` (ntargets_total states) and `hist`; ranks (device, 0-based, may be NULL = 0). */
int sb200_select_init(uint64_t* sel, int64_t* hist, int64_t ntargets_total, const int64_t* ranks,
                      void* stream);
int sb200_select_hist(const float* x, int64_t rows, int64_t row_len, int ntargets_per_row,
                      const uint64_t* sel, int64_t* hist, int pass, int key_mode, void* stream);
/* Same, and in pass 0 also accumulates sign_counts[row*2+0] += #(x < 0),
 * sign_counts[row*2+1] += #(x >= 0) from the same read of x (percentile.py:27-28). */
int sb200_select_hist_counts(const float* x, int64_t rows, int64_t row_len, int ntargets_per_row,
                             const uint64_t* sel, int64_t* hist, int pass, int key_mode,
                             int64_t* sign_counts, void* stream);
int sb200_select_scan(uint64_t* sel, int64_t* hist, int64_t rows, int ntargets_per_row, int pass,
                      void* stream);
/* values[t] = float whose key is the selected one (valid after the pass-2 scan). */
int sb200_select_read(const uint64_t* sel, int64_t ntargets_total, int key_mode, float* values,
                      void* stream);

/* Percentile observer helpers (observers/percentile.py:27-43).
 * counts[row*2 + 0] += #(x < 0), counts[row*2 + 1] += #(x >= 0)  (int64, in place). */
int sb200_count_sign(const float* x, int64_t rows, int64_t row_len, int64_t* counts, void* stream);
/* Writes the two ranks of every row straight into its select states (2 targets per row):
 *   target 0 (min side): 0-based rank max(round(neg*alpha), 1) - 1
 *   target 1 (max side): 0-based rank total - max(round(pos*alpha), 0) - 1
 * with Python round() (half-to-even on the double product) -- percentile.py:36-42.
 * total[row] = number of elements of the row (NaN included), device int64. */
int sb200_percentile_ranks(const int64_t* counts, const int64_t* total, int64_t rows, double alpha,
                           uint64_t* sel, void* stream);

/* Row moments for the step-size initialisations of LSQ (lsq.py:32-51: mean |x|), LSQ+ (lsq_plus.py:21-55:
 * mean / unbiased std) and ACIQ-laplace (aciq.py:65-124: b = mean |x - mean x|).  x: [rows, row_len] contiguous.
 *   out[row*5 + 0..4] += { sum x, sum x^2, sum |x|, sum |x - c|, sum (x - c)^2 },  c = centre[row] (0 if NULL)
 * fp64 accumulation in a fixed order (deterministic); `out` is caller-zeroed and accumulates across batches.
 * workspace: sb200_moments_workspace_bytes(rows, row_len) bytes of device memory. */
size_t sb200_moments_workspace_bytes(int64_t rows, int64_t row_len);
int sb200_observe_moments(const float* x, int64_t rows, int64_t row_len, const double* centre, double* out,
                          void* workspace, size_t workspace_bytes, void* stream);

/* ---- (3) Sparser -------------------------------------------------------------------------
 * mask[i] = |w[i]| > thresh[0]   (sparse/sparsers/l1norm.py:23; strict, ties pruned; uint8 0/1 =
 * torch.bool storage).  thresh is a device float (from the radix select above with key_mode 1
 * and rank min(int(n*ratio), n-1), l1norm.py:19-21). */
int sb200_mask_gt(const float* w, const float* thresh, uint8_t* mask, int64_t n, void* stream);
/* Structured (filter) pruning, sparse/sparsers/l1norm.py:27-40: the per-filter L1 norms come from
 * sb200_observe_moments (column 2 = sum |x|, fp64), the rank-th smallest from the radix select above, and
 *   mask[r, :] = score[r] > thresh[0] ? 1.f : 0.f      (float mask shaped like the weight, as the reference builds). */
int sb200_mask_rows_gt(const float* score, const float* thresh, float* mask, int64_t rows, int64_t inner,
                       void* stream);
/* out = w * mask    (sparse/modules/conv.py:40, linear.py:31).  mask: uint8 (bool). */
int sb200_mask_apply(const float* w, const uint8_t* mask, float* out, int64_t n, void* stream);
/* out = w * mask_f32   (mask stored as float ones_like when ratio == 0, l1norm.py:15-16). */
int sb200_mask_apply_f32(const float* w, const float* mask, float* out, int64_t n, void* stream);
/* Fused  out = QDQ_perchannel(w * mask)  (mask-apply feeding the weight quantizer, one pass,
 * 9 B/elem instead of 4+1+4 + 4+4). */
int sb200_mask_apply_qdq_perchannel(const float* w, const uint8_t* mask, const float* scale,
                                    const float* zero_point, float* out, int64_t outer,
                                    int64_t channels, int64_t inner, int qmin, int qmax,
                                    int rounding, void* stream);

/* Multi-tensor form: the mask-apply + per-channel weight QDQ of EVERY QConv2d / QLinear of a model in one launch
 * (modules/conv.py:37-42, linear.py:30-35 run them once per layer per forward; ResNet-50: 54 launch-bound kernels).
 * Describe the tensors once -- sb200_qdq_multi_plan copies the table to `device_table`
 * (sb200_qdq_multi_table_bytes(count) bytes, caller-owned) and returns the number of (tensor, row) work items --
 * then every forward is one sb200_qdq_multi_run.  mask may be NULL per tensor; half-to-even rounding. */
typedef struct sb200_qdq_tensor_desc {
  const float* x;            /* device, [outer, channels, inner] contiguous */
  const uint8_t* mask;       /* device uint8 (torch.bool), same shape as x, or NULL */
  const float* scale;        /* device, `channels` floats */
  const float* zero_point;   /* device, `channels` floats */
  float* out;                /* device, same shape as x */
  int64_t outer, channels, inner;
  int qmin, qmax;
} sb200_qdq_tensor_desc;
size_t sb200_qdq_multi_table_bytes(int count);
int sb200_qdq_multi_plan(const sb200_qdq_tensor_desc* descs, int count, void* device_table,
                         size_t table_bytes, int64_t* total_rows, void* stream);
int sb200_qdq_multi_run(const void* device_table, int count, int64_t total_rows, void* stream);

/* ---- (3b) AdaRound weight quantizer (sparsebit/quantization/quantizers/adaround.py) -------
 * The one quantizer that bypasses STE.  [outer, channels, inner] geometry as above (per-tensor:
 * 1, 1, n); scale / zero_point hold `channels` floats; v has the shape of x.
 *   x_floor = floor(x / scale);  h(v) = clamp(sigmoid(v) * 1.2 - 0.1, 0, 1)
 *   soft = 1 (training, adaround.py:48-49):  x_q = x_floor + h(v)
 *   soft = 0 (eval,     adaround.py:50-51):  x_q = x_floor + (v >= 0)          -- exact
 *   out = (clamp(x_q + zero_point, qmin, qmax) - zero_point) * scale           (adaround.py:52-53)
 * zero_point is used as stored (not rounded), like the reference. */
int sb200_adaround_fwd(const float* x, const float* v, const float* scale, const float* zero_point,
                       float* out, int64_t outer, int64_t channels, int64_t inner, int qmin,
                       int qmax, int soft, void* stream);
/* grad_v = d out / d v * grad_y for soft = 1 (what autograd derives from adaround.py:40-54; x and
 * scale receive no gradient: floor() has none and scale is a buffer). */
int sb200_adaround_bwd(const float* x, const float* v, const float* scale, const float* zero_point,
                       const float* grad_y, float* grad_v, int64_t outer, int64_t channels,
                       int64_t inner, int qmin, int qmax, void* stream);
/* v = -log(1.2 / (x/scale - floor(x/scale) + 0.1) - 1), so that h(v) = frac(x/scale)
 * (init_variables, adaround.py:26-32). */
int sb200_adaround_init(const float* x, const float* scale, float* v, int64_t outer,
                        int64_t channels, int64_t inner, void* stream);

/* ---- (3c) DoReFa weight quantizer (sparsebit/quantization/quantizers/dorefa.py:15-26) ------
 * The reference squashes the weights with tanh, divides by the abs-max of the result and hands that to STE.apply:
 * five ATen passes (36 B/elem) in front of the fake-quant op, three more in autograd.  Here
 *   absmax:  *absmax = max(*absmax, max |tanh(x)|), updated through its bit pattern (zero-initialise the float;
 *            a NaN input leaves NaN, like torch.max)
 *   fwd:     quantize = 0: out = tanh(x) / *absmax                      (what update_observer caches, dorefa.py:22-26)
 *            quantize = 1: out = QDQ(tanh(x) / *absmax, scale, zero_point, qmin, qmax)      (dorefa.py:15-20)
 *   bwd:     grad_x = ((grad_y * [qmin <= round(xn / scale) + zp <= qmax]) / *absmax) * (1 - tanh(x)^2)
 * [outer, channels, inner] geometry as in (3b); scale / zero_point hold `channels` floats (buffers: no gradient). */
int sb200_dorefa_absmax(const float* x, int64_t n, float* absmax, void* stream);
int sb200_dorefa_fwd(const float* x, const float* absmax, const float* scale, const float* zero_point,
                     float* out, int64_t outer, int64_t channels, int64_t inner, int qmin, int qmax,
                     int quantize, void* stream);
int sb200_dorefa_bwd(const float* x, const float* absmax, const float* scale, const float* zero_point,
                     const float* grad_y, float* grad_x, int64_t outer, int64_t channels,
                     int64_t inner, int qmin, int qmax, void* stream);

/* ---- (4) GPTQ int4 group-wise dequant-matmul --------------------------------------------
 * Replaces cuda_kernel.vecquant4matmul / vecgroupquant4matmul
 * (large_language_models/llama/quantization/cuda/cuda_kernel.cpp:10-23,70,73;
 *  cuda_kernel_4bit.cu:36-180):
 *   out[m, n] += sum_k (scales[n*G + k/gs] * nib(qweight[k/8, n], k%8) - zeros[n*G + k/gs]) * x[m, k]
 * x: [M, K] fp32; qweight: int32 [ceil(K/8), N], 8 nibbles per word along K, LSB = lowest k
 * (utils/quant.py:220-225); out: [M, N] fp32, PRE-INITIALISED (bias) and accumulated in place;
 * scales / zeros (= zero*scale, utils/quant.py:188): fp32 [N, G], G = ceil(K / group_size).
 * group_size == 0 means one group (= K), like vecquant4matmul; otherwise it must be a multiple of
 * 128 (cuda_kernel_4bit.cu:60).  Large-M problems with TMA-compatible shapes run on wgmma
 * tensor cores (split-fp16 activations, exact int4 operands, fp32 register accumulation, per-group
 * scale/zero applied on the accumulator); everything else runs the HBM-bound SIMT path.
 * `workspace` from sb200_gptq4_workspace_bytes (may be 0 bytes / NULL for the SIMT path). */
size_t sb200_gptq4_workspace_bytes(int64_t m, int64_t k, int64_t n, int group_size);
int sb200_gptq4_matmul(const float* x, const int32_t* qweight, float* out, const float* scales,
                       const float* zeros, int64_t m, int64_t k, int64_t n, int64_t qweight_rows,
                       int group_size, void* workspace, size_t workspace_bytes, void* stream);
/* Per-call options instead of process-global switches.  impl: 0 = auto (M >= 32 -> 2, else 1),
 * 1 = small-M path (warp-level HMMA streaming kernel when N % 4 == 0, scalar kernel otherwise), 4 = scalar kernel,
 * 2 = wgmma with exact int4 operands and a per-128-K-group fp32 rescale of the register accumulator,
 * 3 = wgmma with the scaled weights as two fp16 planes in the register operand and whole-K accumulation, restarted
 * into a second fp32 register accumulator every chunk_k K (multiple of 64; 0 = default 512) to bound the tensor
 * core's truncating accumulation. */
/* flags: SB200_GPTQ4_STATIC_WEIGHTS -- the caller guarantees that qweight / scales / zeros are constants of the model,
 * i.e. NOT written by the kernel immediately in front of this call on the stream.  The decode kernel (M <= 32) is
 * launched programmatically dependent (it may begin while its predecessor drains); with this flag it requests the
 * weights before it waits for the predecessor, without it nothing is read before the wait (plain stream semantics). */
#define SB200_GPTQ4_STATIC_WEIGHTS 1
typedef struct sb200_gptq4_options {
  int impl;
  int chunk_k;
  int flags;
  int reserved[5]; /* must be zero */
} sb200_gptq4_options;
int sb200_gptq4_matmul_ex(const float* x, const int32_t* qweight, float* out, const float* scales,
                          const float* zeros, int64_t m, int64_t k, int64_t n, int64_t qweight_rows,
                          int group_size, const sb200_gptq4_options* options, void* workspace,
                          size_t workspace_bytes, void* stream);
/* Up to 4 independent decode-sized linears (1 <= M <= 32 tokens, the same M for all) in ONE launch -- q / k / v or
 * gate / up of a decoder layer.  A decode GEMV lives for a handful of DRAM latencies; launching them back to back leaves
 * HBM idle between kernels.  Same contract per problem as sb200_gptq4_matmul (out pre-initialised, accumulated in place);
 * requires N % 4 == 0 and a 16-byte aligned qweight. */
typedef struct sb200_gptq4_problem {
  const float* x;          /* [M, k] fp32 */
  const int32_t* qweight;  /* [qweight_rows, n] */
  float* out;              /* [M, n] fp32, accumulated in place */
  const float* scales;     /* [n, G] */
  const float* zeros;      /* [n, G] */
  int64_t k, n, qweight_rows;
  int group_size;          /* 0 = k */
} sb200_gptq4_problem;
int sb200_gptq4_matmul_batch(const sb200_gptq4_problem* problems, int count, int64_t m, void* stream);
/* The same with flags (SB200_GPTQ4_STATIC_WEIGHTS, see sb200_gptq4_options). */
int sb200_gptq4_matmul_batch_ex(const sb200_gptq4_problem* problems, int count, int64_t m, int flags, void* stream);

/* fp16 activations in, fp16 result out, WITHOUT the per-call casts of QuantLinear.forward (utils/quant.py:262-278 casts
 * x / scales / zeros / bias to fp32, materialises y = bias, and casts the result back):
 *   out_f16[m, n] = fp16( bias[n] + sum_k (scales * q - zeros) * x_f16[m, k] )          (overwrites out_f16)
 * bias may be NULL; scales / zeros are the fp32 [N, G] tables.  Prefill-sized M runs the weight-plane
 * wgmma kernel (impl 3) directly on the fp16 activations (their hi plane, no lo pass) and writes fp16 from the epilogue;
 * smaller M is staged through fp32 inside the library (cast, bias, kernel, cast) -- or runs as ONE launch through
 * sb200_gptq4_linear_f16_ex below.  Same accuracy as the fp32 entry point before the final rounding to fp16.  workspace: sb200_gptq4_linear_f16_workspace_bytes(...) bytes. */
size_t sb200_gptq4_linear_f16_workspace_bytes(int64_t m, int64_t k, int64_t n, int group_size);
/* Decode-sized M (<= 32) in ONE launch: the decode kernel reads the fp16 activations itself, every K-slice CTA stores its
 * fp32 partial sums into its own slot of the workspace and the last slice CTA of a 128-feature block to arrive adds the
 * slots in slice order, adds the bias and writes fp16 (deterministic; no cast / bias / cast launches around the kernel).
 * `state`: sb200_gptq4_linear_f16_state_bytes() bytes of device memory, ZERO-INITIALISED ONCE by the caller and then
 * left alone (the kernel returns its arrival counters to zero); one state + workspace pair serves one stream at a
 * time.  state == NULL (or M > 32) falls back to sb200_gptq4_linear_f16's staging.  flags: SB200_GPTQ4_STATIC_WEIGHTS. */
size_t sb200_gptq4_linear_f16_state_bytes(void);
int sb200_gptq4_linear_f16_ex(const void* x_f16, const int32_t* qweight, void* out_f16, const float* bias,
                              const float* scales, const float* zeros, int64_t m, int64_t k, int64_t n,
                              int64_t qweight_rows, int group_size, void* state, int flags, void* workspace,
                              size_t workspace_bytes, void* stream);
int sb200_gptq4_linear_f16(const void* x_f16, const int32_t* qweight, void* out_f16, const float* bias,
                           const float* scales, const float* zeros, int64_t m, int64_t k, int64_t n,
                           int64_t qweight_rows, int group_size, void* workspace, size_t workspace_bytes,
                           void* stream);
/* Any bit width of the reference's module: bits = 4 forwards to sb200_gptq4_matmul; bits = 3 / 2
 * replace vecquant3matmul / vecgroupquant3matmul / vecquant2matmul / vecgroupquant2matmul
 * (cuda_kernel.cpp:26-57,68-72; cuda_kernel_3bit.cu, cuda_kernel_2bit.cu).  Packed layouts of
 * QuantLinear.pack (utils/quant.py:210-258): 2-bit 16 values / word; 3-bit 32 values / 3 words with
 * values 10 and 21 straddling; qweight rows = ceil(K*bits / (32*p)) * p (p = 3 for 3-bit, else 1).
 * group_size: 0 = K, else a multiple of 64 (2-bit) / 128 (3-bit).  workspace is only used by bits = 4. */
int sb200_gptq_matmul(const float* x, const int32_t* qweight, float* out, const float* scales,
                      const float* zeros, int64_t m, int64_t k, int64_t n, int64_t qweight_rows,
                      int bits, int group_size, void* workspace, size_t workspace_bytes, void* stream);
/* Force a GPTQ implementation for sb200_gptq4_matmul (process-wide; tests / benchmarking only -- prefer the
 * per-call sb200_gptq4_matmul_ex): 0 = auto, 1 = small-M path, 2 / 3 = the two wgmma kernels, 4 = scalar kernel. */
int sb200_gptq4_set_impl(int impl);

/* Tuning knob of the wgmma kernels: nanoseconds their TMA producer sleeps between polls of a stage's mbarrier while it
 * waits for the consumers to free the stage.  0 (default) = poll continuously. */
int sb200_gptq4_set_wait_backoff(int nanoseconds);

/* Variant of the decode kernel (M <= 32; process-wide, tests / benchmarking only), a bit mask:
 *   bit 0  the CTA's packed-weight slab is fetched with cp.async.bulk (one copy per packed row, all in flight before
 *          the activations are touched; a multi-pass M reads the weights once) instead of per-lane LDG.128;
 *   bit 1  the kernel is launched with programmatic stream serialisation (it may begin while the previous kernel of
 *          the stream drains; griddepcontrol.wait before the first global read, or -- SB200_GPTQ4_STATIC_WEIGHTS --
 *          after the weights / scales / zeros have been requested);
 *   bit 3  treat every call as SB200_GPTQ4_STATIC_WEIGHTS (benchmarking the flag through entry points without one);
 *   bit 2  (register-staged variant) the 128-K blocks beyond the two a lane holds in registers are prefetched into L2
 *          at the start of the CTA, so the refills between the MMA groups do not pay a DRAM round trip;
 *   bits 4..7  resident CTAs per SM the K split aims at (0 = the default 5).
 * Default 6 (measured best at M = 1, profiles/r02_ab_decode.jsonl).  Results are identical in every mode up to the
 * order of the fp32 atomic adds across K slices. */
int sb200_gptq4_set_decode(int mode);

/* Number of kernels this library launched since load (bench.py's `gpu_launches`). */
int64_t sb200_launch_count(void);

#if defined(__GNUC__)
#pragma GCC visibility pop
#endif
#ifdef __cplusplus
}
#endif
#endif /* SPARSEBIT_B200_H_ */
