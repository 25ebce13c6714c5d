// qdq.cu -- Quantizer.forward hot path for sm_90a: quantize->dequantize (per-tensor and
// per-channel), the fused QDQ + MinMax statistics kernel, per-tensor MinMax and the Sparser
// mask-apply, all instances of one streaming kernel skeleton.
//
// Replaces (reference, megvii-research/Sparsebit):
//   sparsebit/quantization/torch_extensions/fake_quant_tensor.cu:50-94   per-tensor forward
//   sparsebit/quantization/torch_extensions/fake_quant_tensor.cu:170-224 per-channel forward
//   sparsebit/quantization/quantizers/quant_tensor.py:181-184            CPU op chain (the oracle)
//   sparsebit/quantization/observers/minmax.py:14-25                     per-tensor min / max
//   sparsebit/sparse/modules/conv.py:40, linear.py:31                    weight * w_mask
//
// Design (HBM-bound, 8 B/elem): a persistent-sized grid (SM count x resident CTAs), every thread
// issues UNROLL independent 128-bit streaming loads (ld.global.cs.v4) before touching any of
// them, computes in registers and writes 128-bit streaming stores.  Per-channel work never does a
// per-element 64-bit div/mod (the reference does, fake_quant_tensor.cu:183): each thread divides
// once, then carries (channel, position-in-row) forward with precomputed per-step increments.
// Statistics are reduced with warp shuffles -> one shared-memory hop -> ONE atomic pair per CTA on
// an order-preserving integer key, so the result is exact and independent of scheduling order.
#include "common.cuh"

namespace sb200 {

enum { MODE_TENSOR = 0, MODE_CHANNEL = 1 };

constexpr int kThreads = 256;
constexpr int kUnroll = 4;
constexpr int kCtasPerSm = 4;  // 1024 threads/SM x 4 x 16 B in flight = 64 KB per SM

struct ChanGeom {
  long long inner;  // elements per channel row
  long long dpos;   // step % inner,            step = total_threads * VEC elements
  int channels;
  int dc;           // (step / inner) % channels
};

template <int VEC>
__device__ __forceinline__ void load_vec(const float* __restrict__ base, long long vi, float (&r)[VEC]) {
  if (VEC == 4) {
    float4 t = ld_stream4(reinterpret_cast<const float4*>(base) + vi);
    r[0] = t.x; r[1] = t.y; r[2] = t.z; r[3] = t.w;
  } else {
    r[0] = ld_stream1(base + vi);
  }
}
template <int VEC>
__device__ __forceinline__ void store_vec(float* __restrict__ base, long long vi, const float (&r)[VEC]) {
  if (VEC == 4) {
    st_stream4(reinterpret_cast<float4*>(base) + vi, make_float4(r[0], r[1], r[2], r[3]));
  } else {
    st_stream1(base + vi, r[0]);
  }
}
template <int VEC>
__device__ __forceinline__ void load_mask(const uint8_t* __restrict__ m, long long vi, float (&r)[VEC]) {
  if (VEC == 4) {
    uchar4 t = __ldcs(reinterpret_cast<const uchar4*>(m) + vi);
    r[0] = t.x ? 1.f : 0.f; r[1] = t.y ? 1.f : 0.f; r[2] = t.z ? 1.f : 0.f; r[3] = t.w ? 1.f : 0.f;
  } else {
    r[0] = __ldcs(m + vi) ? 1.f : 0.f;
  }
}

// One streaming kernel; everything that differs between the entry points is a template flag.
//   MODE    tensor | channel rows ([outer, C, inner])
//   DOQ     apply QDQ                STORE   write `out`
//   STATS   accumulate min/max of the (unmasked) input into mm[0..1]
//   MASK    multiply the input by a uint8 mask first (Sparser mask-apply)
template <int MODE, int VEC, bool DOQ, bool STORE, bool STATS, bool MASK, int ROUNDING>
__global__ void __launch_bounds__(kThreads, kCtasPerSm)
stream_kernel(const float* __restrict__ x, const uint8_t* __restrict__ mask, float* __restrict__ out,
              const float* __restrict__ scale, const float* __restrict__ zero_point, long long n,
              float qmin, float qmax, int rounding, ChanGeom g, uint32_t* __restrict__ mm, int use_tab) {
  // MODE_CHANNEL with use_tab: per-channel {scale, RN32(1/scale), rint(zp), in-range flag} staged once per
  // CTA in shared memory (one LDS.128 per vector instead of two global loads + an fp64 reciprocal).
  extern __shared__ __align__(16) float4 s_tab[];
  if (DOQ && MODE == MODE_CHANNEL && use_tab) {
    for (int ci = threadIdx.x; ci < g.channels; ci += blockDim.x) {
      QP t;
      t.set(__ldg(scale + ci), __ldg(zero_point + ci));
      s_tab[ci] = make_float4(t.s, t.r, t.zp, t.fast ? 1.f : 0.f);
    }
    __syncthreads();
  }
  const long long nvec = (VEC == 4) ? (n >> 2) : n;
  const long long T = (long long)gridDim.x * blockDim.x;
  long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x;

  QP p;
  p.qmin = qmin;
  p.qmax = qmax;
  p.s = 1.f;
  p.zp = 0.f;
  p.rs = 1.0;
  if (DOQ && MODE == MODE_TENSOR) p.set(__ldg(scale), __ldg(zero_point));
  // Channel bookkeeping: one division per thread, increments afterwards.
  long long pos = 0;
  int c = 0, c_loaded = -1;
  if (DOQ && MODE == MODE_CHANNEL) {
    const long long e = v * VEC;
    const long long row = e / g.inner;
    pos = e - row * g.inner;
    c = (int)(row % g.channels);
  }

  MinMaxAcc acc;
  if (STATS) acc.init();

  for (; v < nvec; v += (long long)kUnroll * T) {
    float a[kUnroll][VEC];
    float m[kUnroll][VEC];
    bool ok[kUnroll];
#pragma unroll
    for (int u = 0; u < kUnroll; ++u) {
      ok[u] = (v + (long long)u * T) < nvec;
      if (ok[u]) {
        load_vec<VEC>(x, v + (long long)u * T, a[u]);
        if (MASK) load_mask<VEC>(mask, v + (long long)u * T, m[u]);
      }
    }
#pragma unroll
    for (int u = 0; u < kUnroll; ++u) {
      if (ok[u]) {
        if (STATS) {
#pragma unroll
          for (int j = 0; j < VEC; ++j) acc.add(a[u][j]);
        }
        if (MASK) {
#pragma unroll
          for (int j = 0; j < VEC; ++j) a[u][j] = __fmul_rn(a[u][j], m[u][j]);
        }
        if (DOQ) {
          if (MODE == MODE_TENSOR) {
#pragma unroll
            for (int j = 0; j < VEC; ++j) a[u][j] = qdq1<ROUNDING>(a[u][j], p, rounding);
          } else {  // MODE_CHANNEL
            if (use_tab) {
              // Warp-uniform choice: with short rows (7 x 7 maps: inner = 49) one lane in sixteen holds a vector that
              // straddles a channel boundary, i.e. nearly every warp does -- a per-lane branch would run the whole
              // warp through both paths.  When any lane straddles, all lanes take the two-entry select path below.
              const bool cross = pos + (VEC - 1) >= g.inner;
              const bool any_cross = __any_sync(__activemask(), cross);
              if (!any_cross) {  // whole vector inside one channel row
                const float4 t = s_tab[c];
                p.s = t.x; p.r = t.y; p.zp = t.z; p.fast = t.w != 0.f;
#pragma unroll
                for (int j = 0; j < VEC; ++j) a[u][j] = qdq1<ROUNDING, true>(a[u][j], p, rounding);
              } else if (g.inner >= VEC) {  // at most ONE boundary inside the vector: this channel's entry or the next one's
                const float4 t0 = s_tab[c];
                const float4 t1 = s_tab[(c + 1 == g.channels) ? 0 : c + 1];
#pragma unroll
                for (int j = 0; j < VEC; ++j) {
                  const bool nx = pos + j >= g.inner;
                  p.s = nx ? t1.x : t0.x; p.r = nx ? t1.y : t0.y; p.zp = nx ? t1.z : t0.z; p.fast = (nx ? t1.w : t0.w) != 0.f;
                  a[u][j] = qdq1<ROUNDING, true>(a[u][j], p, rounding);
                }
              } else {
#pragma unroll
                for (int j = 0; j < VEC; ++j) {
                  long long pj = pos + j;
                  int cj = c;
                  while (pj >= g.inner) {
                    pj -= g.inner;
                    cj = (cj + 1 == g.channels) ? 0 : cj + 1;
                  }
                  const float4 t = s_tab[cj];
                  p.s = t.x; p.r = t.y; p.zp = t.z; p.fast = t.w != 0.f;
                  a[u][j] = qdq1<ROUNDING, true>(a[u][j], p, rounding);
                }
              }
            } else if (pos + (VEC - 1) < g.inner) {  // whole vector inside one channel row (fast path)
              if (c != c_loaded) {
                p.set(__ldg(scale + c), __ldg(zero_point + c));
                c_loaded = c;
              }
#pragma unroll
              for (int j = 0; j < VEC; ++j) a[u][j] = qdq1<ROUNDING>(a[u][j], p, rounding);
            } else {  // vector straddles a row boundary: per-element channel
#pragma unroll
              for (int j = 0; j < VEC; ++j) {
                long long pj = pos + j;
                int cj = c;
                while (pj >= g.inner) {
                  pj -= g.inner;
                  cj = (cj + 1 == g.channels) ? 0 : cj + 1;
                }
                if (cj != c_loaded) {
                  p.set(__ldg(scale + cj), __ldg(zero_point + cj));
                  c_loaded = cj;
                }
                a[u][j] = qdq1<ROUNDING>(a[u][j], p, rounding);
              }
            }
          }
        }
        if (STORE) store_vec<VEC>(out, v + (long long)u * T, a[u]);
      }
      // advance the channel cursor by one step (T vectors) -- also for !ok lanes, harmless
      if (DOQ && MODE == MODE_CHANNEL) {
        pos += g.dpos;
        c += g.dc;
        if (pos >= g.inner) {
          pos -= g.inner;
          c += 1;
        }
        if (c >= g.channels) c -= g.channels;
      }
    }
  }

  // Scalar tail (n % 4 elements) for the vector instantiation.
  if (VEC == 4) {
    const long long rem = n & 3;
    const long long gtid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (gtid < rem) {
      const long long e = (nvec << 2) + gtid;
      float val = ld_stream1(x + e);
      if (STATS) acc.add(val);
      if (MASK) val = __fmul_rn(val, __ldcs(mask + e) ? 1.f : 0.f);
      if (DOQ) {
        if (MODE != MODE_TENSOR) {
          const int ce = (int)((e / g.inner) % g.channels);
          p.set(__ldg(scale + ce), __ldg(zero_point + ce));
        }
        val = qdq1<ROUNDING>(val, p, rounding);
      }
      if (STORE) st_stream1(out + e, val);
    }
  }

  if (STATS) {
    __shared__ float red[64];
    block_reduce_minmax(acc, red);
    if (threadIdx.x == 0) acc.publish(mm);
  }
}

// ------------------------------------------------------------------------------------------
// TMA variant of the per-tensor kernel.  The LDG version above is latency bound (ncu: ~all stalls
// are long_scoreboard with DRAM ~70 % busy) because the bytes in flight are capped by registers
// (1024 threads x 4 x 16 B = 64 KB / SM).  Here the loads do not touch registers at all: one elected
// thread keeps a ring of kTmaStages x 16 KB bulk copies (cp.async.bulk -> shared memory, completion
// on an mbarrier) in flight per CTA, two CTAs per SM = 192 KB in flight per SM.  Consumers pull a
// landed tile into registers (conflict-free LDS.128), release the slot with one __syncthreads so
// the producer refills it immediately, compute, and write 128-bit streaming stores straight from
// registers (stores are fire-and-forget and need no staging).
constexpr int kTmaTile = 4096;   // floats per stage (16 KB)
constexpr int kTmaStages = 6;    // 96 KB of shared memory per CTA
constexpr int kTmaCtasPerSm = 2;
constexpr int kTmaPerThread = kTmaTile / kThreads / 4;  // float4 per thread per tile

template <bool STATS, int ROUNDING>
__global__ void __launch_bounds__(kThreads, kTmaCtasPerSm)
stream_tma_kernel(const float* __restrict__ x, float* __restrict__ out, const float* __restrict__ scale,
                  const float* __restrict__ zero_point, long long n, float qmin, float qmax, int rounding,
                  uint32_t* __restrict__ mm) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float* ring = reinterpret_cast<float*>(smem_raw);
  __shared__ __align__(8) uint64_t full[kTmaStages];
  const int tid = threadIdx.x;
  const long long nbody = n & ~3LL;                       // bulk copies move whole float4s
  const long long ntiles = (nbody + kTmaTile - 1) / kTmaTile;
  QP p;
  p.qmin = qmin;
  p.qmax = qmax;
  p.set(__ldg(scale), __ldg(zero_point));
  MinMaxAcc acc;
  if (STATS) acc.init();

  if (tid == 0) {
#pragma unroll
    for (int s = 0; s < kTmaStages; ++s) mbar_init(&full[s], 1);
    mbar_fence_init();
  }
  __syncthreads();
  auto issue = [&](long long tile, int s) {  // called by tid 0 only
    const long long off = tile * kTmaTile;
    const uint32_t bytes = (uint32_t)(((nbody - off) < kTmaTile ? (nbody - off) : (long long)kTmaTile) * 4);
    mbar_expect_tx(&full[s], bytes);
    tma_bulk_g2s(ring + (size_t)s * kTmaTile, x + off, bytes, &full[s]);
  };
  if (tid == 0) {
#pragma unroll
    for (int s = 0; s < kTmaStages; ++s) {
      const long long t = (long long)blockIdx.x + (long long)s * gridDim.x;
      if (t < ntiles) issue(t, s);
    }
  }
  int s = 0;
  uint32_t parity = 0;
  for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const long long off = tile * kTmaTile;
    const int len4 = (int)(((nbody - off) < kTmaTile ? (nbody - off) : (long long)kTmaTile) >> 2);
    mbar_wait(&full[s], parity);
    const float4* src = reinterpret_cast<const float4*>(ring + (size_t)s * kTmaTile);
    float4 v[kTmaPerThread];
#pragma unroll
    for (int k = 0; k < kTmaPerThread; ++k) {
      const int i = tid + k * kThreads;
      if (i < len4) v[k] = src[i];
    }
    __syncthreads();  // every thread holds its part of the tile in registers: slot s is free
    if (tid == 0) {
      const long long nt = tile + (long long)kTmaStages * gridDim.x;
      if (nt < ntiles) issue(nt, s);
    }
    float4* dst = reinterpret_cast<float4*>(out + off);
#pragma unroll
    for (int k = 0; k < kTmaPerThread; ++k) {
      const int i = tid + k * kThreads;
      if (i < len4) {
        if (STATS) acc.add4(v[k]);
        float4 r;
        r.x = qdq1<ROUNDING>(v[k].x, p, rounding);
        r.y = qdq1<ROUNDING>(v[k].y, p, rounding);
        r.z = qdq1<ROUNDING>(v[k].z, p, rounding);
        r.w = qdq1<ROUNDING>(v[k].w, p, rounding);
        st_stream4(dst + i, r);
      }
    }
    if (++s == kTmaStages) {
      s = 0;
      parity ^= 1;
    }
  }
  // scalar tail (n % 4 elements)
  if (blockIdx.x == 0 && tid < (int)(n - nbody)) {
    const float val = ld_stream1(x + nbody + tid);
    if (STATS) acc.add(val);
    st_stream1(out + nbody + tid, qdq1<ROUNDING>(val, p, rounding));
  }
  if (STATS) {
    __shared__ float red[64];
    block_reduce_minmax(acc, red);
    if (tid == 0) acc.publish(mm);
  }
}

template <bool STATS>
static int launch_stream_tma(const float* x, float* out, const float* scale, const float* zp, long long n, int qmin,
                             int qmax, int rounding, uint32_t* mm, cudaStream_t st) {
  const size_t smem = (size_t)kTmaStages * kTmaTile * sizeof(float);
  static std::atomic<int> attr_done[2][64];  // [rounding variant][device]
  const long long ntiles = ((n & ~3LL) + kTmaTile - 1) / kTmaTile;
  long long grid = (long long)sm_count() * kTmaCtasPerSm;
  if (grid > ntiles) grid = ntiles < 1 ? 1 : ntiles;
#define SB_GO(R_)                                                                                              \
  do {                                                                                                         \
    SB_CUDA(ensure_dyn_smem(stream_tma_kernel<STATS, R_>, (int)smem, attr_done[R_ == 0 ? 0 : 1]));            \
    stream_tma_kernel<STATS, R_><<<(unsigned)grid, kThreads, smem, st>>>(x, out, scale, zp, n, (float)qmin,    \
                                                                         (float)qmax, rounding, mm);           \
  } while (0)
  if (rounding == 0) SB_GO(0); else SB_GO(-1);
#undef SB_GO
  SB_LAUNCHED();
  return SB200_OK;
}

// Which implementation serves a per-tensor QDQ: sb200_set_variant 1 = LDG, 2 = TMA, 0 = auto.
static inline bool use_tma(const float* x, const float* out, long long n) {
  if (g_variant == 1) return false;
  const bool ok = aligned16(x) && aligned16(out) && n >= 4 * kTmaTile;
  if (g_variant == 2) return ok;
  // auto: measured on an H100 (400 W limit) the LDG register pipeline and the TMA ring take the same 115 us on the
  // 154 MB headline tensor (0.80 of the 3.35 TB/s data-sheet bandwidth) -> the simpler LDG path unless selected.
  return false;
}

// Channel-last ([R, C], inner == 1, e.g. NLC activations with ch_axis = 2): a thread owns VEC
// adjacent channels for the whole kernel (reciprocals computed once) and walks a block of rows;
// adjacent threads touch adjacent 16-byte columns, so every row is read with full coalescing.
template <int VEC, int ROUNDING>
__global__ void __launch_bounds__(128) qdq_cols_kernel(const float* __restrict__ x, float* __restrict__ out,
                                                       const float* __restrict__ scale,
                                                       const float* __restrict__ zero_point, long long R,
                                                       int channels, long long rows_per_block, float qmin,
                                                       float qmax, int rounding) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  const int nq = channels / VEC;
  if (q >= nq) return;
  QP p[VEC];
#pragma unroll
  for (int j = 0; j < VEC; ++j) {
    p[j].qmin = qmin;
    p[j].qmax = qmax;
    p[j].set(__ldg(scale + q * VEC + j), __ldg(zero_point + q * VEC + j));
  }
  const long long r0 = (long long)blockIdx.y * rows_per_block;
  const long long r1 = r0 + rows_per_block < R ? r0 + rows_per_block : R;
  if (VEC == 4) {
    const float4* xi = reinterpret_cast<const float4*>(x) + q;
    float4* oi = reinterpret_cast<float4*>(out) + q;
    long long r = r0;
    for (; r + 3 < r1; r += 4) {
      float4 t[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) t[u] = ld_stream4(xi + (r + u) * nq);
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        t[u].x = qdq1<ROUNDING>(t[u].x, p[0], rounding);
        t[u].y = qdq1<ROUNDING>(t[u].y, p[1 % VEC], rounding);
        t[u].z = qdq1<ROUNDING>(t[u].z, p[2 % VEC], rounding);
        t[u].w = qdq1<ROUNDING>(t[u].w, p[3 % VEC], rounding);
        st_stream4(oi + (r + u) * nq, t[u]);
      }
    }
    for (; r < r1; ++r) {
      float4 t = ld_stream4(xi + r * nq);
      t.x = qdq1<ROUNDING>(t.x, p[0], rounding);
      t.y = qdq1<ROUNDING>(t.y, p[1 % VEC], rounding);
      t.z = qdq1<ROUNDING>(t.z, p[2 % VEC], rounding);
      t.w = qdq1<ROUNDING>(t.w, p[3 % VEC], rounding);
      st_stream4(oi + r * nq, t);
    }
  } else {
    for (long long r = r0; r < r1; ++r)
      st_stream1(out + r * channels + q, qdq1<ROUNDING>(ld_stream1(x + r * channels + q), p[0], rounding));
  }
}

// ------------------------------------------------------------------------------------------
static inline int grid_for(long long nvec) {
  long long want = (nvec + (long long)kThreads * kUnroll - 1) / ((long long)kThreads * kUnroll);
  long long cap = (long long)sm_count() * kCtasPerSm;
  if (want < 1) want = 1;
  return (int)(want < cap ? want : cap);
}

template <int MODE, bool DOQ, bool STORE, bool STATS, bool MASK>
static int launch_stream(const float* x, const uint8_t* mask, float* out, const float* scale,
                         const float* zp, long long n, long long outer, long long channels,
                         long long inner, int qmin, int qmax, int rounding, uint32_t* mm,
                         cudaStream_t st) {
  const bool vec = aligned16(x) && (!STORE || aligned16(out)) && n >= 4 &&
                   (!MASK || (reinterpret_cast<uintptr_t>(mask) & 3u) == 0);
  const long long nvec = vec ? (n >> 2) : n;
  const int grid = grid_for(nvec);
  const long long step = (long long)grid * kThreads * (vec ? 4 : 1);
  ChanGeom g;
  g.inner = inner > 0 ? inner : 1;
  g.channels = (int)(channels > 0 ? channels : 1);
  g.dpos = step % g.inner;
  g.dc = (int)((step / g.inner) % g.channels);
  const int use_tab = (MODE == MODE_CHANNEL && DOQ && channels <= 2048) ? 1 : 0;
  const size_t tab_bytes = use_tab ? (size_t)channels * sizeof(float4) : 0;  // <= 32 KB
#define SB_GO(VEC_, R_)                                                                         \
  stream_kernel<MODE, VEC_, DOQ, STORE, STATS, MASK, R_><<<grid, kThreads, tab_bytes, st>>>(    \
      x, mask, out, scale, zp, n, (float)qmin, (float)qmax, rounding, g, mm, use_tab)
  if (vec) {
    if (rounding == 0) SB_GO(4, 0); else SB_GO(4, -1);
  } else {
    if (rounding == 0) SB_GO(1, 0); else SB_GO(1, -1);
  }
#undef SB_GO
  SB_LAUNCHED();
  return SB200_OK;
}

static int check_common(const void* x, const void* scale, const void* zp, const void* out,
                        long long n, int qmin, int qmax, int rounding, const char* who) {
  SB_REQUIRE(x && scale && zp && out, "%s: null pointer argument", who);
  // The reference rejects empty tensors (torch_extensions/common.cuh:51-54).
  SB_REQUIRE(n > 0, "%s: Kernel Failure, Tensor is empty: data", who);
  SB_REQUIRE(qmin <= qmax, "%s: qmin (%d) > qmax (%d)", who, qmin, qmax);
  SB_REQUIRE(rounding >= 0 && rounding <= 2, "%s: rounding must be 0, 1 or 2 (got %d)", who, rounding);
  return SB200_OK;
}

static int launch_cols(const float* x, const float* scale, const float* zp, float* out, long long outer,
                       long long channels, int qmin, int qmax, int rounding, cudaStream_t st) {
  const bool vec = (channels % 4 == 0) && aligned16(x) && aligned16(out);
  const long long nq = vec ? channels / 4 : channels;
  const unsigned gx = (unsigned)((nq + 127) / 128);
  long long want_y = ((long long)sm_count() * 8 + gx - 1) / gx;
  if (want_y > outer) want_y = outer;
  if (want_y > 65535) want_y = 65535;
  if (want_y < 1) want_y = 1;
  const long long rpb = (outer + want_y - 1) / want_y;
  const dim3 grid(gx, (unsigned)((outer + rpb - 1) / rpb));
#define SB_GO(VEC_, R_) \
  qdq_cols_kernel<VEC_, R_><<<grid, 128, 0, st>>>(x, out, scale, zp, outer, (int)channels, rpb, (float)qmin, (float)qmax, rounding)
  if (vec) {
    if (rounding == 0) SB_GO(4, 0); else SB_GO(4, -1);
  } else {
    if (rounding == 0) SB_GO(1, 0); else SB_GO(1, -1);
  }
#undef SB_GO
  SB_LAUNCHED();
  return SB200_OK;
}

// Per-channel dispatch shared by the plain and the mask-fused entry points.
template <bool MASK>
static int perchannel_fwd(const float* x, const uint8_t* mask, const float* scale, const float* zp,
                          float* out, long long outer, long long channels, long long inner,
                          int qmin, int qmax, int rounding, cudaStream_t st) {
  const long long n = outer * channels * inner;
  if (channels == 1) {
    return launch_stream<MODE_TENSOR, true, true, false, MASK>(x, mask, out, scale, zp, n, 1, 1, n, qmin,
                                                               qmax, rounding, nullptr, st);
  }
  if (!MASK && inner == 1 && channels < (1LL << 31)) {
    return launch_cols(x, scale, zp, out, outer, channels, qmin, qmax, rounding, st);
  }
  return launch_stream<MODE_CHANNEL, true, true, false, MASK>(x, mask, out, scale, zp, n, outer,
                                                              channels, inner, qmin, qmax, rounding,
                                                              nullptr, st);
}

// ------------------------------------------------------------------------------------------
// mask_gt / mask_apply_f32 / minmax state helpers: small dedicated kernels.
__global__ void __launch_bounds__(kThreads) mask_gt_kernel(const float* __restrict__ w,
                                                            const float* __restrict__ thresh,
                                                            uint8_t* __restrict__ mask, long long n) {
  const float t = __ldg(thresh);
  const long long T = (long long)gridDim.x * blockDim.x;
  const long long nvec = n >> 2;
  const bool vec = ((reinterpret_cast<uintptr_t>(w) & 15u) == 0) && ((reinterpret_cast<uintptr_t>(mask) & 3u) == 0);
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (vec) {
    for (long long v = i; v < nvec; v += T) {
      const float4 a = ld_stream4(reinterpret_cast<const float4*>(w) + v);
      uchar4 r;
      r.x = fabsf(a.x) > t; r.y = fabsf(a.y) > t; r.z = fabsf(a.z) > t; r.w = fabsf(a.w) > t;
      reinterpret_cast<uchar4*>(mask)[v] = r;
    }
    for (long long e = (nvec << 2) + i; e < n; e += T) mask[e] = fabsf(w[e]) > t;
  } else {
    for (long long e = i; e < n; e += T) mask[e] = fabsf(w[e]) > t;
  }
}

__global__ void __launch_bounds__(kThreads) mul_f32_kernel(const float* __restrict__ w,
                                                            const float* __restrict__ m,
                                                            float* __restrict__ out, long long n) {
  const long long T = (long long)gridDim.x * blockDim.x;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += T)
    out[e] = __fmul_rn(w[e], m[e]);
}

__global__ void minmax_init_kernel(uint32_t* st, long long channels) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < channels) {
    st[2 * i] = SB_MM_EMPTY_MIN;
    st[2 * i + 1] = SB_MM_EMPTY_MAX;
  }
}
__global__ void minmax_read_kernel(const uint32_t* __restrict__ st, long long channels,
                                   float* __restrict__ mn, float* __restrict__ mx) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < channels) {
    mn[i] = dec_f32(st[2 * i]);
    mx[i] = dec_f32(st[2 * i + 1]);
  }
}

}  // namespace sb200

using namespace sb200;

extern "C" {

int sb200_qdq_pertensor_fwd(const float* x, const float* scale, const float* zero_point, float* out,
                            int64_t n, int qmin, int qmax, int rounding, void* stream) {
  int rc = check_common(x, scale, zero_point, out, n, qmin, qmax, rounding, "sb200_qdq_pertensor_fwd");
  if (rc) return rc;
  if (use_tma(x, out, n))
    return launch_stream_tma<false>(x, out, scale, zero_point, n, qmin, qmax, rounding, nullptr, (cudaStream_t)stream);
  return launch_stream<MODE_TENSOR, true, true, false, false>(x, nullptr, out, scale, zero_point, n, 1, 1,
                                                              n, qmin, qmax, rounding, nullptr,
                                                              (cudaStream_t)stream);
}

int sb200_qdq_stats_pertensor_fwd(const float* x, const float* scale, const float* zero_point,
                                  float* out, uint32_t* minmax_state, int64_t n, int qmin, int qmax,
                                  int rounding, void* stream) {
  int rc = check_common(x, scale, zero_point, out, n, qmin, qmax, rounding, "sb200_qdq_stats_pertensor_fwd");
  if (rc) return rc;
  SB_REQUIRE(minmax_state, "sb200_qdq_stats_pertensor_fwd: null minmax_state");
  if (use_tma(x, out, n))
    return launch_stream_tma<true>(x, out, scale, zero_point, n, qmin, qmax, rounding, minmax_state, (cudaStream_t)stream);
  return launch_stream<MODE_TENSOR, true, true, true, false>(x, nullptr, out, scale, zero_point, n, 1, 1, n,
                                                             qmin, qmax, rounding, minmax_state,
                                                             (cudaStream_t)stream);
}

int sb200_qdq_perchannel_fwd(const float* x, const float* scale, const float* zero_point, float* out,
                             int64_t outer, int64_t channels, int64_t inner, int qmin, int qmax,
                             int rounding, void* stream) {
  SB_REQUIRE(outer > 0 && channels > 0 && inner > 0,
             "sb200_qdq_perchannel_fwd: Kernel Failure, Tensor is empty: data (outer=%lld C=%lld inner=%lld)",
             (long long)outer, (long long)channels, (long long)inner);
  int rc = check_common(x, scale, zero_point, out, outer * channels * inner, qmin, qmax, rounding,
                        "sb200_qdq_perchannel_fwd");
  if (rc) return rc;
  return perchannel_fwd<false>(x, nullptr, scale, zero_point, out, outer, channels, inner, qmin, qmax,
                               rounding, (cudaStream_t)stream);
}

int sb200_mask_apply_qdq_perchannel(const float* w, const uint8_t* mask, const float* scale,
                                    const float* zero_point, float* out, int64_t outer,
                                    int64_t channels, int64_t inner, int qmin, int qmax, int rounding,
                                    void* stream) {
  SB_REQUIRE(outer > 0 && channels > 0 && inner > 0, "sb200_mask_apply_qdq_perchannel: empty tensor");
  SB_REQUIRE(mask, "sb200_mask_apply_qdq_perchannel: null mask");
  int rc = check_common(w, scale, zero_point, out, outer * channels * inner, qmin, qmax, rounding,
                        "sb200_mask_apply_qdq_perchannel");
  if (rc) return rc;
  return perchannel_fwd<true>(w, mask, scale, zero_point, out, outer, channels, inner, qmin, qmax,
                              rounding, (cudaStream_t)stream);
}

int sb200_mask_apply(const float* w, const uint8_t* mask, float* out, int64_t n, void* stream) {
  SB_REQUIRE(w && mask && out, "sb200_mask_apply: null pointer argument");
  SB_REQUIRE(n > 0, "sb200_mask_apply: empty tensor");
  return launch_stream<MODE_TENSOR, false, true, false, true>(w, mask, out, nullptr, nullptr, n, 1, 1, n, 0,
                                                              0, 0, nullptr, (cudaStream_t)stream);
}

int sb200_mask_apply_f32(const float* w, const float* mask, float* out, int64_t n, void* stream) {
  SB_REQUIRE(w && mask && out, "sb200_mask_apply_f32: null pointer argument");
  SB_REQUIRE(n > 0, "sb200_mask_apply_f32: empty tensor");
  mul_f32_kernel<<<grid_for(n), kThreads, 0, (cudaStream_t)stream>>>(w, mask, out, n);
  SB_LAUNCHED();
  return SB200_OK;
}

int sb200_mask_gt(const float* w, const float* thresh, uint8_t* mask, int64_t n, void* stream) {
  SB_REQUIRE(w && thresh && mask, "sb200_mask_gt: null pointer argument");
  SB_REQUIRE(n > 0, "sb200_mask_gt: empty tensor");
  mask_gt_kernel<<<grid_for(n >> 2), kThreads, 0, (cudaStream_t)stream>>>(w, thresh, mask, n);
  SB_LAUNCHED();
  return SB200_OK;
}

int sb200_minmax_init(uint32_t* state, int64_t channels, void* stream) {
  SB_REQUIRE(state && channels > 0, "sb200_minmax_init: bad arguments");
  minmax_init_kernel<<<(unsigned)((channels + 255) / 256), 256, 0, (cudaStream_t)stream>>>(state, channels);
  SB_LAUNCHED();
  return SB200_OK;
}

int sb200_minmax_read(const uint32_t* state, int64_t channels, float* out_min, float* out_max,
                      void* stream) {
  SB_REQUIRE(state && out_min && out_max && channels > 0, "sb200_minmax_read: bad arguments");
  minmax_read_kernel<<<(unsigned)((channels + 255) / 256), 256, 0, (cudaStream_t)stream>>>(state, channels,
                                                                                          out_min, out_max);
  SB_LAUNCHED();
  return SB200_OK;
}

int sb200_observe_minmax(const float* x, int64_t n, uint32_t* state, void* stream) {
  SB_REQUIRE(x && state, "sb200_observe_minmax: null pointer argument");
  SB_REQUIRE(n > 0, "sb200_observe_minmax: empty tensor");
  return launch_stream<MODE_TENSOR, false, false, true, false>(x, nullptr, nullptr, nullptr, nullptr, n, 1, 1,
                                                               n, 0, 0, 0, state, (cudaStream_t)stream);
}

}  // extern "C"
