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
 * ignored.  An empty range (lo == hi) is widened to [lo - 1, hi + 1].  ATen widens it to the
 * data's own min and max first, so the two agree when every element of the data equals lo (for
 * range [0, 0] and data {0, 5} ATen counts both in [0, 5], this kernel drops 5).  The KL observer's
 * range [-absmax, absmax] is empty only when absmax == 0, i.e. for all-zero data. */
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
 * 2 = wgmma with exact int4 operands and a per-128-K-group fp32 rescale of the register accumulator.  Any other value
 * (3 included) is SB200_E_INVALID.  chunk_k is reserved and must be zero, like reserved[]. */
/* flags: SB200_GPTQ4_STATIC_WEIGHTS -- the caller guarantees that qweight / scales / zeros are constants of the model,
 * i.e. NOT written by the kernel immediately in front of this call on the stream.  The decode kernel (M <= 32) is
 * launched programmatically dependent (it may begin while its predecessor drains); with this flag it requests the
 * weights before it waits for the predecessor, without it nothing is read before the wait (plain stream semantics). */
#define SB200_GPTQ4_STATIC_WEIGHTS 1
typedef struct sb200_gptq4_options {
  int impl;
  int chunk_k; /* reserved, must be zero */
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
 * bias may be NULL; scales / zeros are the fp32 [N, G] tables.  Prefill-sized M (>= 768) runs the per-group
 * wgmma kernel (impl 2) directly on the fp16 activations (their hi plane, no lo pass) and writes fp16 from the epilogue;
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
/* Input gradient of the dequant-matmul above (the backward of QuantLinear with respect to its input), any bit width:
 *   grad_in[m, k] += sum_n grad_out[m, n] * (scales[n, k/gs] * q(k, n) - zeros[n, k/gs])
 * grad_out: [M, N] fp32; grad_in: [M, K] fp32, accumulated in place; qweight / scales / zeros / group_size / bits: the
 * tensors and values the forward takes, with the same argument checks (all before any CUDA call).  Results are
 * deterministic: two identical calls are bit-identical.
 * impl (per call): 0 = auto, 1 = SIMT kernel (any bits, any shape), 2 = wgmma kernel (bits = 4, N % 8 == 0, K % 4 == 0,
 * 16-byte aligned grad_out; the weights are repacked along N into the workspace for the call, the scaled weights enter
 * the MMA as two fp16 planes); forcing 2 on anything else returns SB200_E_UNSUPPORTED.  Auto takes the wgmma kernel for
 * the shapes it supports from a measured M on (gptq.cu).
 * workspace: sb200_gptq_dgrad_workspace_bytes(...) bytes (a pure function of its arguments). */
size_t sb200_gptq_dgrad_workspace_bytes(int64_t m, int64_t k, int64_t n, int bits, int group_size);
int sb200_gptq_matmul_dgrad(const float* grad_out, const int32_t* qweight, float* grad_in, const float* scales,
                            const float* zeros, int64_t m, int64_t k, int64_t n, int64_t qweight_rows, int bits,
                            int group_size, int impl, void* workspace, size_t workspace_bytes, void* stream);
/* ---- (5) Integer-grid inference of a calibrated QLinear (int8 wgmma, sm_90a) -----------------
 * New; the reference's QLinear (modules/linear.py) fake-quantises x and W and runs an fp32 matmul.  With
 * v = clamp(round(x / s) + Z, qmin, qmax) - Z and Z = rint(zero_point) the fake-quant product is
 *   y[m, n] = s_x * s_w[n] * sum_k v_x[m, k] * v_w[n, k] + bias[n]
 * whose sum is an integer, computed exactly here on the int8 tensor cores.
 *
 * Stored grid.  Integer ranges are stored as s8: g - 128 for unsigned ranges (qmin >= 0, at most [0, 255]), g itself
 * for signed ones (within [-128, 127]); the zero points on the stored grid are shifted by the same amount.  Rows are
 * Kp = round_up(K, 16) bytes long, the padding is zero.  K < 2^17 (|sum| <= K * 2^14 fits int32), else
 * SB200_E_UNSUPPORTED.  qmax - qmin > 255, or a range that fits neither form, is SB200_E_INVALID.
 *
 * sb200_int8_quantize_rows: x [rows, K] fp32 -> q [rows, Kp] s8 (16-byte aligned) holding the grid values
 * clamp(round(x / s) + Z, qmin, qmax) on the stored grid, bit-identical to the QDQ kernels (half-to-even);
 * row_sum[rows] int32 = sum of the stored row; nan_flag[rows] uint8 = 1 if the row holds a NaN (stored as 0).
 * +-inf clamp to qmin / qmax.  scale / zero_point: device, 1 float each (per_row = 0) or one per row (per_row = 1).
 *
 * sb200_int8_linear: out[M, N] fp32 (overwritten) for x [M, K] fp32 with per-tensor device scalars x_scale /
 * x_zero_point and the integer range [qmin_x, qmax_x]; the weights as sb200_int8_quantize_rows stored them:
 * w_q [N, Kp] s8 (16-byte aligned), w_rowsum [N] int32, w_scale [N] fp32, w_zero [N] int32 = rint(zero_point) on the
 * stored grid; bias [N] fp32 or NULL.  The zero points must lie in their integer ranges.  Epilogue: the zero points are
 * removed exactly in int64, I = sum a b - Z_w sum a - Z_x sum b + K Z_x Z_w, then y = fp32(fp64(I * s_x * s_w[n])) and
 * fp32 + bias[n]; a row of x holding a NaN gives a NaN row (a weight row holding a NaN is marked by w_scale[n] = NaN,
 * which gives a NaN column).  Deterministic, no state between calls (graph-capturable).
 * workspace: sb200_int8_linear_workspace_bytes(m, k) bytes (a pure function; too small -> SB200_E_WORKSPACE). */
int sb200_int8_quantize_rows(const float* x, const float* scale, const float* zero_point, int per_row, int qmin, int qmax,
                             int8_t* q, int32_t* row_sum, uint8_t* nan_flag, int64_t rows, int64_t k, void* stream);
size_t sb200_int8_linear_workspace_bytes(int64_t m, int64_t k);
int sb200_int8_linear(const float* x, const float* x_scale, const float* x_zero_point, int qmin_x, int qmax_x,
                      const int8_t* w_q, const int32_t* w_rowsum, const float* w_scale, const int32_t* w_zero,
                      const float* bias, float* out, int64_t m, int64_t k, int64_t n, void* workspace,
                      size_t workspace_bytes, void* stream);

/* ---- (5a) 2:4 structured sparsity on the integer grid (int8 sparse wgmma, sm_90a) ---------------
 * New; the reference's L1 sparser has only unstructured and per-filter masks, and its pruned layers run dense.
 *
 * sb200_sparse24_mask: mask [rows, cols] uint8 0 / 1 for w [rows, cols] fp32 (weight.reshape(C_out, -1)).  Each row is
 * walked in aligned groups of 4 from column 0; a group keeps the two elements of largest |w|: ties go to the lower
 * index, NaN ranks above every number (so it is kept), +-0 rank as 0; a tail group of r < 4 keeps min(2, r).
 *
 * Compressed weight format.  d[n, k] = w_q[n, k] - w_zero[n] (w_q / w_zero as sb200_int8_quantize_rows stores them) is
 * the centred weight grid, 0 exactly where the fake-quant weight is 0, for k < K; d = 0 for k >= K.  With K64 =
 * round_up(K, 64), group j of row n is d[n, 4j .. 4j + 3]; it keeps two indices i0 < i1: its nonzero positions, then its
 * lowest-index zero positions up to two (so an all-zero group, and every padding group, keeps (0, 1)).
 *   vals [N, K64 / 2] s8: vals[n, 2j] = d[n, 4j + i0], vals[n, 2j + 1] = d[n, 4j + i1].
 *   meta [ceil(N / 128), K64 / 64, 2, 128] uint32: word (b, s, h, t) is what thread t of consumer warpgroup h reads at
 *     k64 step s of 128-feature tile b: feature n = 128 b + 64 h + 16 (t >> 5) + ((t & 31) >> 2) + 8 (t & 1), groups
 *     j = 16 s + 8 ((t >> 1) & 1) + g for g = 0 .. 7 with i0 | i1 << 2 in bits [4 g, 4 g + 4).  Features n >= N hold
 *     0x44444444 (every group (0, 1)).  This is the sparse-metadata order of wgmma .sp .s8 m64nNk64, selector 0.
 *   dsum [N] int32 = sum_k d[n, k].
 *   bad [N] int32 = groups of row n with more than two nonzero d, or a d outside [-128, 127]; vals then do not hold
 *     row n and sb200_int8_sparse24_linear must not be given it.
 * A row whose w_scale is NaN is packed as d = 0 (its output column is NaN through w_scale).
 *
 * sb200_int8_sparse24_pack: the format above from w_q [N, Kp] s8, w_zero [N] int32, w_scale [N] fp32; vals 16-byte
 * aligned.  Once per weight, at conversion.
 *
 * sb200_int8_sparse24_linear: out [M, N] fp32 (overwritten) for x [M, K] fp32 with per-tensor device scalars x_scale /
 * x_zero_point and [qmin_x, qmax_x], the packed weight (vals, meta 16-byte aligned; dsum) with w_scale [N] and bias [N]
 * or NULL.  I = sum_k a d - Z_x dsum on the stored activation grid equals sb200_int8_linear's integer, and the epilogue
 * is the same: y = fp32(fp64(I) * (fp64(s_x) * fp64(w_scale[n]))) (+ bias[n] in fp32), NaN rows from x's NaN rows.
 * So out equals sb200_int8_linear on the dense weight bit for bit.  Argument rules, K < 2^17 and the workspace
 * (sb200_int8_linear_workspace_bytes(m, k), the same layout) are sb200_int8_linear's.  Deterministic, graph-capturable. */
int sb200_sparse24_mask(const float* w, uint8_t* mask, int64_t rows, int64_t cols, void* stream);
int sb200_int8_sparse24_pack(const int8_t* w_q, const int32_t* w_zero, const float* w_scale, int8_t* vals,
                             uint32_t* meta, int32_t* dsum, int32_t* bad, int64_t n, int64_t k, void* stream);
int sb200_int8_sparse24_linear(const float* x, const float* x_scale, const float* x_zero_point, int qmin_x, int qmax_x,
                               const int8_t* vals, const uint32_t* meta, const int32_t* dsum, const float* w_scale,
                               const float* bias, float* out, int64_t m, int64_t k, int64_t n, void* workspace,
                               size_t workspace_bytes, void* stream);

/* ---- (5b) Integer-grid inference of a calibrated QConv2d (int8 wgmma, sm_90a) ----------------
 * New; the reference's QConv2d (modules/conv.py) fake-quantises x and W (QDQ x 2) and runs F.conv2d.  Lowered, the
 * convolution is the integer linear above: M = n OH OW output pixels, K = c kh kw taps in the order (c, kh, kw) of
 * weight.reshape(c_out, -1), N = c_out.  The weights go through sb200_int8_quantize_rows as [c_out, K] rows.
 *
 * Geometry (host struct, passed by pointer): x is [n, c, h, w] fp32 contiguous; every size, stride and dilation > 0,
 * the four paddings >= 0 (asymmetric padding -- e.g. PyTorch's padding='same' for even kernels -- is allowed);
 *   OH = (h + pad_top + pad_bottom - dilation_h (kh - 1) - 1) / stride_h + 1, OW likewise.
 * Argument checks, all before any CUDA call: null pointers, a non-positive geometry, an empty output (OH or OW < 1)
 * and M >= 2^31 are SB200_E_INVALID, as are the range rules of the integer linear and a w_q / q not 16-byte aligned;
 * K >= 2^17 is SB200_E_UNSUPPORTED; a workspace that is too small is SB200_E_WORKSPACE.
 *
 * sb200_int8_im2col_quantize: the lowering alone.  q [M, Kp] s8 (16-byte aligned, Kp = round_up(K, 16)): element
 * (m, k) is the stored grid value (as in sb200_int8_quantize_rows) of x[img, c, oh sh - pad_top + kh dh,
 * ow sw - pad_left + kw dw] for m = (img OH + oh) OW + ow, k = (c kh_ + kh) kw_ + kw; a tap in the padding stores
 * rint(zero_point) - off (the grid point of the fake-quant input's zero padding); the K padding is zero.
 * row_sum[M] int32 = sum of the stored row; nan_flag[M] uint8 = 1 if the window holds a NaN.  scale / zero_point:
 * device, one float each.
 *
 * sb200_int8_conv2d: out [n, c_out, OH, OW] fp32 NCHW (overwritten) = the fake-quant conv2d of x with per-tensor
 * device scalars x_scale / x_zero_point and the integer range [qmin_x, qmax_x], and the weights as
 * sb200_int8_quantize_rows stored them (w_q [c_out, Kp], w_rowsum / w_scale / w_zero [c_out], bias [c_out] or NULL);
 * the epilogue, NaN rules and guarantees are those of sb200_int8_linear (groups = 1 only).
 * workspace: sb200_int8_conv2d_workspace_bytes(geom) bytes (a pure function; 0 for an invalid geometry). */
typedef struct sb200_conv2d_geom {
  int64_t n, c, h, w;                         /* input [n, c, h, w] */
  int64_t kh, kw;                             /* kernel */
  int64_t stride_h, stride_w;
  int64_t dilation_h, dilation_w;
  int64_t pad_top, pad_bottom, pad_left, pad_right;
} sb200_conv2d_geom;
int sb200_int8_im2col_quantize(const float* x, const sb200_conv2d_geom* geom, const float* scale,
                               const float* zero_point, int qmin, int qmax, int8_t* q, int32_t* row_sum,
                               uint8_t* nan_flag, void* stream);
size_t sb200_int8_conv2d_workspace_bytes(const sb200_conv2d_geom* geom);
int sb200_int8_conv2d(const float* x, const sb200_conv2d_geom* geom, const float* x_scale, const float* x_zero_point,
                      int qmin_x, int qmax_x, const int8_t* w_q, const int32_t* w_rowsum, const float* w_scale,
                      const int32_t* w_zero, const float* bias, float* out, int64_t c_out, void* workspace,
                      size_t workspace_bytes, void* stream);

/* sb200_int8_sparse24_conv2d: the conv2d above with a 2:4-sparse weight on the sparse int8 tensor cores.  The weight is
 * the (5a) operand that sb200_int8_sparse24_pack made from the stored rows of weight.reshape(c_out, -1) (K = c kh kw;
 * vals, meta 16-byte aligned, dsum, every `bad` entry 0) with w_scale [c_out] and bias [c_out] or NULL.  The input is
 * lowered by sb200_int8_im2col_quantize, whose K order (c, kh, kw) is the order the 2:4 groups follow, and a padding tap
 * stores rint(zero_point) - off, so I = sum_k a d - Z_x dsum is sb200_int8_conv2d's integer.  out [n, c_out, OH, OW] fp32
 * NCHW (overwritten) equals sb200_int8_conv2d on the dense stored weight bit for bit, NaNs included.  Argument checks
 * in sb200_int8_conv2d's order (vals and meta take w_q's alignment rule); the workspace is
 * sb200_int8_conv2d_workspace_bytes(geom), the same layout.  Deterministic, graph-capturable. */
int sb200_int8_sparse24_conv2d(const float* x, const sb200_conv2d_geom* geom, const float* x_scale,
                               const float* x_zero_point, int qmin_x, int qmax_x, const int8_t* vals,
                               const uint32_t* meta, const int32_t* dsum, const float* w_scale, const float* bias,
                               float* out, int64_t c_out, void* workspace, size_t workspace_bytes, void* stream);

/* ---- (5c) Integer-grid inference of a calibrated activation x activation matmul (int8 wgmma, sm_90a) ----
 * New; the reference's MatMul (modules/matmul.py) multiplies two fake-quantised activations (a QIdentity carrier in
 * front of each input) with an fp32 torch.matmul.  With both operands per-tensor the product is
 *   y[b, m, n] = s_a * s_b * sum_k v_a[b, m, k] * v_b[b, k, n],   v = clamp(round(x / s) + Z, qmin, qmax) - Z
 * over `batch` independent problems: a is [batch, m, k]; b is [batch, n, k] when b_k_major = 1 (the k^T of attention:
 * its rows go through the row quantizer as they lie) or [batch, k, n] when b_k_major = 0 (the column quantizer
 * transposes it).  All tensors fp32 contiguous, scales / zero points device scalars, the stored grid, range rules and
 * K < 2^17 as in (5).
 *
 * Argument checks, all before any CUDA call: null pointers, an empty operand, batch m or batch n >= 2^31 and the range
 * rules of the integer linear are SB200_E_INVALID, as is a q not 16-byte aligned; K >= 2^17 is SB200_E_UNSUPPORTED; a
 * workspace that is too small is SB200_E_WORKSPACE.
 *
 * sb200_int8_quantize_cols: the transposing quantizer alone.  x [batch, k, n] fp32 -> q [batch, n, Kp] s8 (16-byte
 * aligned, Kp = round_up(K, 16), padding zero): element (b, n, k) is the stored grid value (as in
 * sb200_int8_quantize_rows) of x[b, k, n]; col_sum[batch n] int32 = sum of the stored row of q; nan_flag[batch n] uint8
 * = 1 if the column holds a NaN (stored as 0).  +-inf clamp to qmin / qmax.  scale / zero_point: device, one float each.
 *
 * sb200_int8_matmul: out [batch, m, n] fp32 (overwritten).  Epilogue: the zero points are removed exactly in int64,
 * I = sum a b - Z_b sum_k a - Z_a sum_k b + K Z_a Z_b, then y = fp32(fp64(I) * (fp64(s_a) * fp64(s_b))).  A NaN in row
 * m of a[b] makes row m of out[b] NaN, a NaN in column n of b[b] makes column n of out[b] NaN (as the fake-quant matmul
 * does); no other batch entry is touched.  Exact against the fp64 product of the fake-quant operands when both scales
 * are powers of two, within 2^-21 * (|f_a| @ |f_b|) otherwise.  Deterministic, no state between calls
 * (graph-capturable).
 * workspace: sb200_int8_matmul_workspace_bytes(batch, m, k, n) bytes (a pure function; 0 for arguments the matmul
 * rejects). */
int sb200_int8_quantize_cols(const float* x, const float* scale, const float* zero_point, int qmin, int qmax,
                             int8_t* q, int32_t* col_sum, uint8_t* nan_flag, int64_t batch, int64_t k, int64_t n,
                             void* stream);
size_t sb200_int8_matmul_workspace_bytes(int64_t batch, int64_t m, int64_t k, int64_t n);
int sb200_int8_matmul(const float* a, const float* b, int b_k_major, const float* a_scale, const float* a_zero_point,
                      int qmin_a, int qmax_a, const float* b_scale, const float* b_zero_point, int qmin_b, int qmax_b,
                      float* out, int64_t batch, int64_t m, int64_t k, int64_t n, void* workspace,
                      size_t workspace_bytes, void* stream);

/* ---- (5d) Integer-grid inference of a calibrated grouped / depthwise QConv2d (direct int8 kernel, sm_90a) ----
 * New; the reference's QConv2d with groups > 1 fake-quantises x and W and runs a grouped F.conv2d.  With C_g = c /
 * groups input channels and C_out / groups output channels per group, g(n) = n / (c_out / groups):
 *   y[img, n, oh, ow] = fp32(fp64(I) * (fp64(s_x) * fp64(s_w[n])))  (+ bias[n] in fp32)
 *   I = sum over the C_g channels of group g(n) and the kh x kw taps of (v_x - Z_x)(v_w[n] - Z_w[n])
 * computed exactly in int32 / int64 by one kernel that quantizes its input tile (stored grid as in (5), padding taps
 * at the zero point) into shared memory; no workspace.  The epilogue is that of (5) operation for operation, so that a
 * group's output is bit-identical to sb200_int8_conv2d run on that group's channel slice and weight rows.
 *
 * x [n, c, h, w] fp32 contiguous, geometry as in (5b); out [n, c_out, OH, OW] fp32 NCHW (overwritten).  The weights
 * are sb200_int8_quantize_rows of weight.reshape(c_out, -1): w_q [c_out, round_up(K_g, 16)] s8 with K_g = C_g kh kw in
 * the order (c, kh, kw), w_rowsum / w_scale / w_zero [c_out]; bias [c_out] or NULL.  The zero points must lie in
 * their integer ranges.  A NaN in input channel c makes NaN every output of group g(c) whose window covers it, and no
 * other output; a weight row holding a NaN is marked by w_scale[n] = NaN and gives a NaN channel.  +-inf clamp.
 * Exact against the fp64 conv2d of the fake-quant operands when s_x and s_w are powers of two, within
 * 2^-21 (conv(|f_x|, |f_w|) + |bias|) elementwise otherwise.  Deterministic, no state between calls (graph-capturable).
 *
 * Argument checks, all before any CUDA call: null pointers, c_out <= 0 or >= 2^31, a non-positive geometry, an empty
 * output, n OH OW >= 2^31, groups < 2 (groups = 1 is sb200_int8_conv2d), c or c_out not divisible by groups and the
 * range rules of the integer linear are SB200_E_INVALID; K_g >= 2^17 (|sum a b| <= K_g 2^14 must fit int32) is
 * SB200_E_UNSUPPORTED. */
int sb200_int8_group_conv2d(const float* x, const sb200_conv2d_geom* geom, int64_t groups, const float* x_scale,
                            const float* x_zero_point, int qmin_x, int qmax_x, const int8_t* w_q, const int32_t* w_rowsum,
                            const float* w_scale, const int32_t* w_zero, const float* bias, float* out, int64_t c_out,
                            void* stream);

/* ---- (5f) Channels-last (NHWC) integer-grid convs ----------------------------------------------------------------
 * The entry points of (5b) and (5d) for an x stored NHWC: geom keeps its meaning (n, c, h, w) -- only the storage of x,
 * x[((img h + ih) w + iw) c + ch], and of out, out[((img OH + oh) OW + ow) c_out + n], changes.  Each takes the argument
 * list of its NCHW counterpart, makes the same checks in the same order with the same codes before any CUDA call, and
 * computes the same values: the lowered q / row_sum / nan_flag byte for byte, every output bit for bit, NaNs
 * included.  The weights are the same stored rows (K order (c, kh, kw)), so one stored weight serves both layouts.
 *
 * sb200_int8_im2col_quantize_nhwc: sb200_int8_im2col_quantize of an NHWC x.  A stride-1, unpadded 1 x 1 conv with
 * c >= 256 is the row quantizer over x as [n h w, c]; otherwise each window's channels are read with 16-byte loads when c % 4 = 0 and
 * x is 16-byte aligned.
 * sb200_int8_conv2d_nhwc, sb200_int8_sparse24_conv2d_nhwc: the lowering above, then the GEMM of sb200_int8_conv2d /
 * sb200_int8_sparse24_conv2d with its row-major [n OH OW, c_out] epilogue, which is out stored NHWC.  Workspace:
 * sb200_int8_conv2d_workspace_bytes(geom), as for NCHW.
 * sb200_int8_group_conv2d_nhwc: sb200_int8_group_conv2d, one direct kernel reading the channels of each tap with
 * vector loads; no workspace.  All deterministic and graph-capturable. */
int sb200_int8_im2col_quantize_nhwc(const float* x, const sb200_conv2d_geom* geom, const float* scale,
                                    const float* zero_point, int qmin, int qmax, int8_t* q, int32_t* row_sum,
                                    uint8_t* nan_flag, void* stream);
int sb200_int8_conv2d_nhwc(const float* x, const sb200_conv2d_geom* geom, const float* x_scale,
                           const float* x_zero_point, int qmin_x, int qmax_x, const int8_t* w_q, const int32_t* w_rowsum,
                           const float* w_scale, const int32_t* w_zero, const float* bias, float* out, int64_t c_out,
                           void* workspace, size_t workspace_bytes, void* stream);
int sb200_int8_sparse24_conv2d_nhwc(const float* x, const sb200_conv2d_geom* geom, const float* x_scale,
                                    const float* x_zero_point, int qmin_x, int qmax_x, const int8_t* vals,
                                    const uint32_t* meta, const int32_t* dsum, const float* w_scale, const float* bias,
                                    float* out, int64_t c_out, void* workspace, size_t workspace_bytes, void* stream);
int sb200_int8_group_conv2d_nhwc(const float* x, const sb200_conv2d_geom* geom, int64_t groups, const float* x_scale,
                                 const float* x_zero_point, int qmin_x, int qmax_x, const int8_t* w_q,
                                 const int32_t* w_rowsum, const float* w_scale, const int32_t* w_zero, const float* bias,
                                 float* out, int64_t c_out, void* stream);

/* ---- (5e) Integer-grid inference of a calibrated attention, fused (int8 wgmma, sm_90a) ----
 * New; the reference runs MatMul -> Softmax -> MatMul with a QIdentity carrier in front of every matmul input, so q,
 * k, the softmax output p and v are each fake-quantised per tensor.  Per batch entry, with q [tq, d], k [tk, d] and
 * v [tk, dv] fp32 contiguous:
 *   s = RN32(fp64(I_qk) * (fp64(s_q) * fp64(s_k)))  (then RN32(s * scale) when has_scale)
 *   I_qk = sum over d of (v_q - Z_q)(v_k - Z_k), exact: s is bit-identical to sb200_int8_matmul(q, k^T)
 *   p = softmax(s) along the keys, in fp32; g_p = its stored grid (the QDQ rule with p's qparams)
 *   out = RN32(fp64(I_pv) * (fp64(s_p) * fp64(s_v))),  I_pv = sum over the keys of (g_p - Z_p)(v_v - Z_v), exact
 * One kernel computes the scores, the softmax, p's grid and p @ v; the [tq, tk] scores never reach memory.  Only p is
 * inexact: |p - p64| <= 13 * 2^-24 * p64 + 2^-125, p64 the fp64 softmax of the same fp32 scores.
 * out [batch, tq, dv] fp32 (overwritten).  p_q: NULL, or [batch, tq, round_up(tk, 16)] s8 (16-byte aligned) that
 * receives the stored grid of p, the key padding 0.  scale: a host float, used when has_scale != 0.  Scales and zero
 * points: device, one float each; the stored grid and range rules as in (5).
 * NaN: a NaN in row i of q makes row i of out NaN; a NaN anywhere in k makes all of that entry's out NaN; a NaN in
 * column n of v makes column n of that entry's out NaN; +-inf clamp.  Deterministic, no state between calls
 * (graph-capturable).
 *
 * Argument checks, all before any CUDA call: null pointers, an empty dimension, batch tq or batch tk >= 2^31, the
 * range rules of the four operands, a non-finite scale with has_scale and a p_q not 16-byte aligned are
 * SB200_E_INVALID; d > 128, dv > 128 or tk >= 2^17 is SB200_E_UNSUPPORTED; a workspace that is too small is
 * SB200_E_WORKSPACE.
 * workspace: sb200_int8_attention_workspace_bytes(batch, tq, tk, d, dv) bytes, O(batch (tq + tk) d + batch dv tk)
 * (a pure function; 0 for arguments the attention rejects). */
size_t sb200_int8_attention_workspace_bytes(int64_t batch, int64_t tq, int64_t tk, int64_t d, int64_t dv);
int sb200_int8_attention(const float* q, const float* k, const float* v, const float* q_scale,
                         const float* q_zero_point, int qmin_q, int qmax_q, const float* k_scale,
                         const float* k_zero_point, int qmin_k, int qmax_k, const float* p_scale,
                         const float* p_zero_point, int qmin_p, int qmax_p, const float* v_scale,
                         const float* v_zero_point, int qmin_v, int qmax_v, int has_scale, float scale, float* out,
                         int8_t* p_q, int64_t batch, int64_t tq, int64_t tk, int64_t d, int64_t dv, void* workspace,
                         size_t workspace_bytes, void* stream);

/* ---- (5f) The fused attention of (5e) with an additive mask and a causal mode (int8 wgmma, sm_90a) ----
 * New; the reference's BERT (GLUE) adds a key-padding mask (1 - m) * -10000 to the scaled scores, its GPT-2 (wikitext)
 * keeps the scores of a causal band and adds an attention mask.  Per batch entry b, after s (and its scale) of (5e):
 *   causal: s[i, j] = -inf where j > i + (tk - tq)  (the band aligned bottom-right, as the GPT-2 example; this is not
 *           the top-left is_causal of PyTorch's scaled_dot_product_attention when tq != tk)
 *   mask:   s[i, j] = RN32(s[i, j] + mask[(b / mask_inner) mask_stride_outer + (b % mask_inner) mask_stride_inner
 *                                         + i mask_stride_row + j])          (fp32, column stride 1, 64-bit offsets)
 * then p, its grid and out as in (5e), with the same bound on p against the fp64 softmax of the masked fp32 scores.
 * A [B, 1, 1, tk] mask over [B, H] entries is mask_inner = H, mask_stride_outer = tk, mask_stride_inner = 0,
 * mask_stride_row = 0.  Under causal a block of 128 keys that no row of a 128-row tile sees is not read or computed;
 * its keys have p = 0 (p_q receives their grid).  A row that sees no key (causal with tq > tk, or an all -inf mask row)
 * is NaN.  NaN: as (5e), except that a NaN in k poisons only the rows whose band contains its key; a NaN in column n of
 * v still makes column n NaN (0 * NaN); a NaN or +inf mask value at a key of a skipped block is not read.
 * mask: NULL for none, then the four mask arguments are not read.  causal: 0 or 1.  mask == NULL with causal == 0
 * computes exactly sb200_int8_attention.
 *
 * Argument checks, all before any CUDA call: those of (5e); causal not 0 or 1, and with a mask a negative stride,
 * mask_inner <= 0 or not dividing batch, a mask not 4-byte aligned or a last offset >= 2^62 are SB200_E_INVALID.
 * workspace: sb200_int8_attention_masked_workspace_bytes(batch, tq, tk, d, dv, causal) bytes: that of (5e), and with
 * causal also batch dv ceil(tk / 128) int32 column sums of v (a pure function; 0 for arguments it rejects). */
size_t sb200_int8_attention_masked_workspace_bytes(int64_t batch, int64_t tq, int64_t tk, int64_t d, int64_t dv,
                                                   int causal);
int sb200_int8_attention_masked(const float* q, const float* k, const float* v, const float* q_scale,
                                const float* q_zero_point, int qmin_q, int qmax_q, const float* k_scale,
                                const float* k_zero_point, int qmin_k, int qmax_k, const float* p_scale,
                                const float* p_zero_point, int qmin_p, int qmax_p, const float* v_scale,
                                const float* v_zero_point, int qmin_v, int qmax_v, int has_scale, float scale,
                                const float* mask, int64_t mask_stride_outer, int64_t mask_stride_inner,
                                int64_t mask_inner, int64_t mask_stride_row, int causal, float* out, int8_t* p_q,
                                int64_t batch, int64_t tq, int64_t tk, int64_t d, int64_t dv, void* workspace,
                                size_t workspace_bytes, void* stream);

/* ---- (5h) The attention of (5e) / (5f) over an int8 key/value cache, for generation (sm_90a) ----
 * New; the reference's GPT-2 (wikitext) concatenates layer_past onto the new key and value at every step.  Here each
 * key and value is quantized once, when it is appended, into a cache that the caller allocates zeroed.  Per entry e of
 * `batch` (the flattened leading dimensions), capacity C, L keys stored, dp = round_up(d, 16), Cp = round_up(C, 16):
 *   k_q [batch, C, dp] s8     row j = the stored grid of key j as sb200_int8_quantize_rows writes it (padding 0)
 *   k_sum, k_nan [batch, C]   int32 / uint8: that row's sum and NaN flag
 *   v_t [batch, dv, Cp] s8    v^T, key-major, as sb200_int8_quantize_cols writes it
 *   v_sum, v_nan [batch, dv]  int32 / uint8: the column sums over the L stored keys; a sticky NaN flag
 * Every byte at a key position >= L stays 0.  k_q and v_t are 16-byte aligned.  The qparams and ranges of k and v must
 * be the same at every append and attention call of a cache.
 *
 * sb200_int8_kv_append writes k [batch, t, d] and v [batch, t, dv] (fp32 contiguous) at positions [length,
 * length + t) in one launch and updates v_sum / v_nan.  Checks, before any CUDA call: null pointers, an empty
 * dimension, a negative length, length + t > capacity, batch capacity >= 2^31, a k_q or v_t not 16-byte aligned and
 * the range rules are SB200_E_INVALID; capacity >= 2^17, d > 128 or dv > 128 is SB200_E_UNSUPPORTED.
 *
 * sb200_int8_attention_cached is sb200_int8_attention_masked (q [batch, tq, d], the four qparams, scale, mask, causal,
 * out, p_q) with k and v the first `length` keys of the cache.  tq > 16: q is quantized and the fused kernel of (5e)
 * runs over the cache; out and p_q are bit-identical to sb200_int8_attention_masked on the fp32 keys and values that
 * were appended.  tq <= 16 (decode): a split-key kernel pair plus a combine (at most four launches with q's
 * quantization): the scores are bit-identical to sb200_int8_matmul(q, k^T), every p is within the bound of (5e), out is
 * exactly the integer p @ v of the kernel's own p_q, and the NaN rules are those of (5f).  Only the fp64 summation
 * order of the softmax denominator differs from the fused kernel, so a p grid value can differ from it by one step
 * where RN32(1 / l) rounds differently.  Deterministic: the key split depends on the shape only.
 * Checks: those of (5f) with tk = length (length >= 1), then those of the append on the cache; a too small workspace
 * is SB200_E_WORKSPACE.
 * workspace: sb200_int8_attention_cached_workspace_bytes(batch, tq, capacity, length, d, dv, causal) bytes: q's grid,
 * and with tq <= 16 the fp32 scores [batch, tq, length] and per key split int32 partials (a pure function; 0 for
 * arguments it rejects). */
int sb200_int8_kv_append(const float* k, const float* v, const float* k_scale, const float* k_zero_point, int qmin_k,
                         int qmax_k, const float* v_scale, const float* v_zero_point, int qmin_v, int qmax_v,
                         int8_t* k_q, int32_t* k_sum, uint8_t* k_nan, int8_t* v_t, int32_t* v_sum, uint8_t* v_nan,
                         int64_t batch, int64_t capacity, int64_t length, int64_t t, int64_t d, int64_t dv,
                         void* stream);
size_t sb200_int8_attention_cached_workspace_bytes(int64_t batch, int64_t tq, int64_t capacity, int64_t length,
                                                   int64_t d, int64_t dv, int causal);
int sb200_int8_attention_cached(const float* q, const float* q_scale, const float* q_zero_point, int qmin_q, int qmax_q,
                                const float* k_scale, const float* k_zero_point, int qmin_k, int qmax_k,
                                const float* p_scale, const float* p_zero_point, int qmin_p, int qmax_p,
                                const float* v_scale, const float* v_zero_point, int qmin_v, int qmax_v, int has_scale,
                                float scale, const float* mask, int64_t mask_stride_outer, int64_t mask_stride_inner,
                                int64_t mask_inner, int64_t mask_stride_row, int causal, const int8_t* k_q,
                                const int32_t* k_sum, const uint8_t* k_nan, const int8_t* v_t, const int32_t* v_sum,
                                const uint8_t* v_nan, int64_t capacity, int64_t length, float* out, int8_t* p_q,
                                int64_t batch, int64_t tq, int64_t d, int64_t dv, void* workspace,
                                size_t workspace_bytes, void* stream);

/* ---- (5g) Integer-grid layers with a DoReFa input ------------------------------------------------------------------
 * Replaces the chain of sparsebit/quantization/quantizers/dorefa.py:15-20 (t = tanh(x); x_n = t / max |t|; QDQ(x_n))
 * feeding F.linear / F.conv2d when the layer's input quantizer is DoReFa: the lowering (or the grouped kernel) quantizes
 * x_n = tanh(x) / *x_absmax in registers, with the op sequence of sb200_dorefa_fwd (libdevice tanhf, a true division),
 * so that every output is bit-identical to the plain entry point run on sb200_dorefa_fwd(x, x_absmax, quantize = 0),
 * NaNs included.  x_absmax: device, one float, max |tanh(x)| over the layer's whole input as sb200_dorefa_absmax writes
 * it (the caller zeroes it and launches sb200_dorefa_absmax first, on the same stream).  A NaN in x makes *x_absmax
 * NaN and an all-zero x makes it 0 (0 / 0 = NaN): either way every output is NaN, as in the fake-quant op.  Padding
 * taps stay at the grid point of a real 0.
 *
 * Each takes its plain counterpart's arguments with x_absmax inserted after x_zero_point, makes the counterpart's checks
 * in the same order with the same codes, then rejects a null x_absmax (SB200_E_INVALID), all before any CUDA call.  The
 * workspace queries and layout are the counterpart's. */
int sb200_int8_linear_dorefa(const float* x, const float* x_scale, const float* x_zero_point, const float* x_absmax,
                             int qmin_x, int qmax_x, const int8_t* w_q, const int32_t* w_rowsum, const float* w_scale,
                             const int32_t* w_zero, const float* bias, float* out, int64_t m, int64_t k, int64_t n,
                             void* workspace, size_t workspace_bytes, void* stream);
int sb200_int8_conv2d_dorefa(const float* x, const sb200_conv2d_geom* geom, const float* x_scale,
                             const float* x_zero_point, const float* x_absmax, int qmin_x, int qmax_x, const int8_t* w_q,
                             const int32_t* w_rowsum, const float* w_scale, const int32_t* w_zero, const float* bias,
                             float* out, int64_t c_out, void* workspace, size_t workspace_bytes, void* stream);
int sb200_int8_conv2d_nhwc_dorefa(const float* x, const sb200_conv2d_geom* geom, const float* x_scale,
                                  const float* x_zero_point, const float* x_absmax, int qmin_x, int qmax_x,
                                  const int8_t* w_q, const int32_t* w_rowsum, const float* w_scale,
                                  const int32_t* w_zero, const float* bias, float* out, int64_t c_out, void* workspace,
                                  size_t workspace_bytes, void* stream);
int sb200_int8_group_conv2d_dorefa(const float* x, const sb200_conv2d_geom* geom, int64_t groups, const float* x_scale,
                                   const float* x_zero_point, const float* x_absmax, int qmin_x, int qmax_x,
                                   const int8_t* w_q, const int32_t* w_rowsum, const float* w_scale,
                                   const int32_t* w_zero, const float* bias, float* out, int64_t c_out, void* stream);
int sb200_int8_group_conv2d_nhwc_dorefa(const float* x, const sb200_conv2d_geom* geom, int64_t groups,
                                        const float* x_scale, const float* x_zero_point, const float* x_absmax,
                                        int qmin_x, int qmax_x, const int8_t* w_q, const int32_t* w_rowsum,
                                        const float* w_scale, const int32_t* w_zero, const float* bias, float* out,
                                        int64_t c_out, void* stream);

/* Force a GPTQ implementation for sb200_gptq4_matmul (process-wide; tests / benchmarking only -- prefer the
 * per-call sb200_gptq4_matmul_ex): 0 = auto, 1 = small-M path, 2 = wgmma kernel, 4 = scalar kernel; 3 is invalid. */
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
