// bwd.cu -- STE backward of the fake-quant op for sm_90a.
//
// Replaces (reference, megvii-research/Sparsebit):
//   sparsebit/quantization/torch_extensions/fake_quant_tensor.cu:97-167   per-tensor backward
//   sparsebit/quantization/torch_extensions/fake_quant_tensor.cu:227-314  per-channel backward
//   formula restated from quantizers/quant_tensor.py:46-71 (MySTE.backward)
//
//   vq  = round(x/s) + zp
//   gx  = gy            if qmin <= vq <= qmax else 0
//   gs  = sum gy * (round(x/s) - x/s)   inside ;  gy * (qmin - zp) below ;  gy * (qmax - zp) above
//   gzp = sum -s * gy                   outside the range, 0 inside
//
// 12 B/elem (x, gy in; gx out).  The reference reduces gs/gzp with a block reduce + float
// atomicAdd *per grid-stride iteration* and has __syncthreads() under divergent control flow
// (fake_quant_tensor.cu:123,128,260,265); here every tile produces one fp64 partial that a second
// tiny kernel sums in a fixed order -> deterministic, no atomics.  Zero-point gradient rule: the reference's
// per-tensor kernel and MySTE.backward treat qmin <= vq <= qmax as inside; its per-channel kernel uses
// qmin <= vq < qmax (fake_quant_tensor.cu:264, SURVEY.md Q4).  sb200_qdq_perchannel_bwd reproduces the
// reference's per-channel kernel; sb200_qdq_perchannel_bwd_ex(flags = SB200_BWD_GZP_CLOSED) selects the
// MySTE / per-tensor rule.
#include "common.cuh"

namespace sb200 {

constexpr int kThreads = 256;
constexpr long long kTile = 8192;  // elements per reduction tile

struct BwdAcc {
  float gs, gzp;
};

template <int ROUNDING>
__device__ __forceinline__ float bwd1(float x, float gy, const QP& p, float lo_term, float hi_term, BwdAcc& a,
                                      int rounding) {
  const float q = div_exact(x, p);
  float r;
  if (ROUNDING == 0) r = rintf(q);
  else r = rounding == 1 ? floorf(__fadd_rn(q, 0.5f)) : (rounding == 2 ? ceilf(__fsub_rn(q, 0.5f)) : rintf(q));
  const float vq = __fadd_rn(r, p.zp);
  const bool below = vq < p.qmin;
  const bool inside = (vq >= p.qmin) && (vq <= p.qmax);
  const float term = inside ? __fsub_rn(r, q) : (below ? lo_term : hi_term);
  a.gs = fmaf(term, gy, a.gs);
  a.gzp += ((vq >= p.qmin) && (vq <= p.gz_hi)) ? 0.f : __fmul_rn(-p.s, gy);
  return inside ? gy : 0.f;
}

// Process `len` contiguous elements cooperatively (thread rank t of nthr).
template <int ROUNDING>
__device__ __forceinline__ void span_bwd(const float* __restrict__ x, const float* __restrict__ gy,
                                         float* __restrict__ gx, long long len, int t, int nthr, const QP& p,
                                         BwdAcc& a, int rounding) {
  const float lo_term = __fsub_rn(p.qmin, p.zp), hi_term = __fsub_rn(p.qmax, p.zp);
  const uintptr_t ax = reinterpret_cast<uintptr_t>(x) & 15u;
  const bool vec = (ax == (reinterpret_cast<uintptr_t>(gy) & 15u)) && (ax == (reinterpret_cast<uintptr_t>(gx) & 15u));
  if (!vec) {
    for (long long i = t; i < len; i += nthr) gx[i] = bwd1<ROUNDING>(__ldcs(x + i), __ldcs(gy + i), p, lo_term, hi_term, a, rounding);
    return;
  }
  long long head = ((16 - ax) & 15u) >> 2;
  if (head > len) head = len;
  for (long long i = t; i < head; i += nthr) gx[i] = bwd1<ROUNDING>(__ldcs(x + i), __ldcs(gy + i), p, lo_term, hi_term, a, rounding);
  const float4* x4 = reinterpret_cast<const float4*>(x + head);
  const float4* g4 = reinterpret_cast<const float4*>(gy + head);
  float4* o4 = reinterpret_cast<float4*>(gx + head);
  const long long nv = (len - head) >> 2;
  long long i = t;
  for (; i + nthr < nv; i += 2LL * nthr) {
    const float4 xa = ld_stream4(x4 + i), ga = ld_stream4(g4 + i);
    const float4 xb = ld_stream4(x4 + i + nthr), gb = ld_stream4(g4 + i + nthr);
    float4 r;
    r.x = bwd1<ROUNDING>(xa.x, ga.x, p, lo_term, hi_term, a, rounding);
    r.y = bwd1<ROUNDING>(xa.y, ga.y, p, lo_term, hi_term, a, rounding);
    r.z = bwd1<ROUNDING>(xa.z, ga.z, p, lo_term, hi_term, a, rounding);
    r.w = bwd1<ROUNDING>(xa.w, ga.w, p, lo_term, hi_term, a, rounding);
    st_stream4(o4 + i, r);
    r.x = bwd1<ROUNDING>(xb.x, gb.x, p, lo_term, hi_term, a, rounding);
    r.y = bwd1<ROUNDING>(xb.y, gb.y, p, lo_term, hi_term, a, rounding);
    r.z = bwd1<ROUNDING>(xb.z, gb.z, p, lo_term, hi_term, a, rounding);
    r.w = bwd1<ROUNDING>(xb.w, gb.w, p, lo_term, hi_term, a, rounding);
    st_stream4(o4 + i + nthr, r);
  }
  for (; i < nv; i += nthr) {
    const float4 xa = ld_stream4(x4 + i), ga = ld_stream4(g4 + i);
    float4 r;
    r.x = bwd1<ROUNDING>(xa.x, ga.x, p, lo_term, hi_term, a, rounding);
    r.y = bwd1<ROUNDING>(xa.y, ga.y, p, lo_term, hi_term, a, rounding);
    r.z = bwd1<ROUNDING>(xa.z, ga.z, p, lo_term, hi_term, a, rounding);
    r.w = bwd1<ROUNDING>(xa.w, ga.w, p, lo_term, hi_term, a, rounding);
    st_stream4(o4 + i, r);
  }
  for (long long e = head + (nv << 2) + t; e < len; e += nthr)
    gx[e] = bwd1<ROUNDING>(__ldcs(x + e), __ldcs(gy + e), p, lo_term, hi_term, a, rounding);
}

// Tiles: x viewed as rows of `inner` elements; tile = (row, j-th chunk of kTile).  A CTA (CTA_TILE) or
// a warp handles one tile and writes partial[tile] = {gs, gzp} in fp64.
template <bool CTA_TILE, int ROUNDING>
__global__ void __launch_bounds__(kThreads) bwd_rows_kernel(const float* __restrict__ x, const float* __restrict__ gy,
                                                            float* __restrict__ gx, const float* __restrict__ scale,
                                                            const float* __restrict__ zero_point, long long rows,
                                                            long long inner, int channels, float qmin, float qmax,
                                                            float gz_hi, int rounding, double2* __restrict__ partial) {
  __shared__ double s_red[2][kThreads / 32];
  const long long tpr = (inner + kTile - 1) / kTile;
  const long long total = rows * tpr;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const long long first = CTA_TILE ? blockIdx.x : (((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  const long long stride = CTA_TILE ? gridDim.x : (((long long)gridDim.x * blockDim.x) >> 5);
  for (long long tile = first; tile < total; tile += stride) {
    const long long row = tile / tpr, j = tile - row * tpr;
    const long long off = row * inner + j * kTile;
    const long long len = (inner - j * kTile) < kTile ? (inner - j * kTile) : kTile;
    const int c = (int)(row % channels);
    QP p;
    p.set(__ldg(scale + c), __ldg(zero_point + c));
    p.qmin = qmin;
    p.qmax = qmax;
    p.gz_hi = gz_hi;
    BwdAcc a = {0.f, 0.f};
    span_bwd<ROUNDING>(x + off, gy + off, gx + off, len, CTA_TILE ? threadIdx.x : lane, CTA_TILE ? blockDim.x : 32,
                       p, a, rounding);
    if (partial) {
      const double gs = warp_sum((double)a.gs), gz = warp_sum((double)a.gzp);
      if (CTA_TILE) {
        if (lane == 0) {
          s_red[0][wid] = gs;
          s_red[1][wid] = gz;
        }
        __syncthreads();
        if (threadIdx.x == 0) {
          double t0 = 0.0, t1 = 0.0;
#pragma unroll
          for (int w = 0; w < kThreads / 32; ++w) {
            t0 += s_red[0][w];
            t1 += s_red[1][w];
          }
          partial[tile] = make_double2(t0, t1);
        }
        __syncthreads();
      } else if (lane == 0) {
        partial[tile] = make_double2(gs, gz);
      }
    }
  }
}

// Stage 2 for row tiles: channel c sums partial[(o*C + c)*tpr + j] over o, j.  One CTA per channel,
// fixed thread -> item mapping and a fixed-order tree, so the result is deterministic.
__global__ void __launch_bounds__(kThreads) bwd_rows_finish_kernel(const double2* __restrict__ partial, long long outer,
                                                                   int channels, long long tpr,
                                                                   float* __restrict__ gs, float* __restrict__ gzp) {
  __shared__ double s_red[2][kThreads / 32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const long long c = blockIdx.x;
  const long long cnt = outer * tpr;
  double t0 = 0.0, t1 = 0.0;
  if (tpr == 1) {
    for (long long o = threadIdx.x; o < outer; o += kThreads) {
      const double2 v = partial[o * channels + c];
      t0 += v.x;
      t1 += v.y;
    }
  } else {
    for (long long i = threadIdx.x; i < cnt; i += kThreads) {
      const long long o = i / tpr, j = i - o * tpr;
      const double2 v = partial[(o * channels + c) * tpr + j];
      t0 += v.x;
      t1 += v.y;
    }
  }
  t0 = warp_sum(t0);
  t1 = warp_sum(t1);
  if (lane == 0) {
    s_red[0][wid] = t0;
    s_red[1][wid] = t1;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double a0 = 0.0, a1 = 0.0;
#pragma unroll
    for (int w = 0; w < kThreads / 32; ++w) {
      a0 += s_red[0][w];
      a1 += s_red[1][w];
    }
    if (gs) gs[c] = (float)a0;
    if (gzp) gzp[c] = (float)a1;
  }
}

// Channel-last ([R, C], inner == 1): a thread owns VEC adjacent channels (128-bit loads of x, gy and
// stores of gx, adjacent threads -> adjacent 16-byte columns) and walks a block of rows two at a time.
template <int VEC, int ROUNDING>
__global__ void __launch_bounds__(128) bwd_cols_kernel(const float* __restrict__ x, const float* __restrict__ gy,
                                                       float* __restrict__ gx, const float* __restrict__ scale,
                                                       const float* __restrict__ zero_point, long long R, int channels,
                                                       long long rows_per_block, float qmin, float qmax, float gz_hi,
                                                       int rounding, double2* __restrict__ partial) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  const int nq = channels / VEC;
  if (q >= nq) return;
  QP p[VEC];
  float lo_term[VEC], hi_term[VEC];
  BwdAcc a[VEC];
  double d0[VEC], d1[VEC];
#pragma unroll
  for (int j = 0; j < VEC; ++j) {
    p[j].set(__ldg(scale + q * VEC + j), __ldg(zero_point + q * VEC + j));
    p[j].qmin = qmin;
    p[j].qmax = qmax;
    p[j].gz_hi = gz_hi;
    lo_term[j] = __fsub_rn(qmin, p[j].zp);
    hi_term[j] = __fsub_rn(qmax, p[j].zp);
    a[j].gs = a[j].gzp = 0.f;
    d0[j] = d1[j] = 0.0;
  }
  const long long r0 = (long long)blockIdx.y * rows_per_block;
  const long long r1 = r0 + rows_per_block < R ? r0 + rows_per_block : R;
  int k = 0;
  if (VEC == 4) {
    const float4* x4 = reinterpret_cast<const float4*>(x) + q;
    const float4* g4 = reinterpret_cast<const float4*>(gy) + q;
    float4* o4 = reinterpret_cast<float4*>(gx) + q;
    long long r = r0;
    auto row = [&](const float4& xv, const float4& gv, long long rr) {
      float4 o;
      o.x = bwd1<ROUNDING>(xv.x, gv.x, p[0], lo_term[0], hi_term[0], a[0], rounding);
      o.y = bwd1<ROUNDING>(xv.y, gv.y, p[1 % VEC], lo_term[1 % VEC], hi_term[1 % VEC], a[1 % VEC], rounding);
      o.z = bwd1<ROUNDING>(xv.z, gv.z, p[2 % VEC], lo_term[2 % VEC], hi_term[2 % VEC], a[2 % VEC], rounding);
      o.w = bwd1<ROUNDING>(xv.w, gv.w, p[3 % VEC], lo_term[3 % VEC], hi_term[3 % VEC], a[3 % VEC], rounding);
      st_stream4(o4 + rr * nq, o);
    };
    for (; r + 3 < r1; r += 4) {  // eight independent 128-bit loads in flight per thread (12 B/elem of traffic to cover)
      const float4 xa = ld_stream4(x4 + r * nq), ga = ld_stream4(g4 + r * nq);
      const float4 xb = ld_stream4(x4 + (r + 1) * nq), gb = ld_stream4(g4 + (r + 1) * nq);
      const float4 xc = ld_stream4(x4 + (r + 2) * nq), gc = ld_stream4(g4 + (r + 2) * nq);
      const float4 xd = ld_stream4(x4 + (r + 3) * nq), gd = ld_stream4(g4 + (r + 3) * nq);
      row(xa, ga, r);
      row(xb, gb, r + 1);
      row(xc, gc, r + 2);
      row(xd, gd, r + 3);
      if ((k += 4) >= 256) {  // bound the fp32 accumulation length
#pragma unroll
        for (int j = 0; j < VEC; ++j) { d0[j] += a[j].gs; d1[j] += a[j].gzp; a[j].gs = a[j].gzp = 0.f; }
        k = 0;
      }
    }
    for (; r + 1 < r1; r += 2) {
      const float4 xa = ld_stream4(x4 + r * nq), ga = ld_stream4(g4 + r * nq);
      const float4 xb = ld_stream4(x4 + (r + 1) * nq), gb = ld_stream4(g4 + (r + 1) * nq);
      float4 o;
      o.x = bwd1<ROUNDING>(xa.x, ga.x, p[0], lo_term[0], hi_term[0], a[0], rounding);
      o.y = bwd1<ROUNDING>(xa.y, ga.y, p[1 % VEC], lo_term[1 % VEC], hi_term[1 % VEC], a[1 % VEC], rounding);
      o.z = bwd1<ROUNDING>(xa.z, ga.z, p[2 % VEC], lo_term[2 % VEC], hi_term[2 % VEC], a[2 % VEC], rounding);
      o.w = bwd1<ROUNDING>(xa.w, ga.w, p[3 % VEC], lo_term[3 % VEC], hi_term[3 % VEC], a[3 % VEC], rounding);
      st_stream4(o4 + r * nq, o);
      o.x = bwd1<ROUNDING>(xb.x, gb.x, p[0], lo_term[0], hi_term[0], a[0], rounding);
      o.y = bwd1<ROUNDING>(xb.y, gb.y, p[1 % VEC], lo_term[1 % VEC], hi_term[1 % VEC], a[1 % VEC], rounding);
      o.z = bwd1<ROUNDING>(xb.z, gb.z, p[2 % VEC], lo_term[2 % VEC], hi_term[2 % VEC], a[2 % VEC], rounding);
      o.w = bwd1<ROUNDING>(xb.w, gb.w, p[3 % VEC], lo_term[3 % VEC], hi_term[3 % VEC], a[3 % VEC], rounding);
      st_stream4(o4 + (r + 1) * nq, o);
      if ((k += 2) >= 256) {  // bound the fp32 accumulation length
#pragma unroll
        for (int j = 0; j < VEC; ++j) { d0[j] += a[j].gs; d1[j] += a[j].gzp; a[j].gs = a[j].gzp = 0.f; }
        k = 0;
      }
    }
    for (; r < r1; ++r) {
      const float4 xa = ld_stream4(x4 + r * nq), ga = ld_stream4(g4 + r * nq);
      float4 o;
      o.x = bwd1<ROUNDING>(xa.x, ga.x, p[0], lo_term[0], hi_term[0], a[0], rounding);
      o.y = bwd1<ROUNDING>(xa.y, ga.y, p[1 % VEC], lo_term[1 % VEC], hi_term[1 % VEC], a[1 % VEC], rounding);
      o.z = bwd1<ROUNDING>(xa.z, ga.z, p[2 % VEC], lo_term[2 % VEC], hi_term[2 % VEC], a[2 % VEC], rounding);
      o.w = bwd1<ROUNDING>(xa.w, ga.w, p[3 % VEC], lo_term[3 % VEC], hi_term[3 % VEC], a[3 % VEC], rounding);
      st_stream4(o4 + r * nq, o);
    }
  } else {
    for (long long r = r0; r < r1; ++r) {
      const long long e = r * channels + q;
      gx[e] = bwd1<ROUNDING>(__ldcs(x + e), __ldcs(gy + e), p[0], lo_term[0], hi_term[0], a[0], rounding);
      if (++k == 256) { d0[0] += a[0].gs; d1[0] += a[0].gzp; a[0].gs = a[0].gzp = 0.f; k = 0; }
    }
  }
  if (partial) {
#pragma unroll
    for (int j = 0; j < VEC; ++j)
      partial[(long long)blockIdx.y * channels + q * VEC + j] = make_double2(d0[j] + a[j].gs, d1[j] + a[j].gzp);
  }
}

// gs[c] / gzp[c] = sum over the row blocks b of partial[b * channels + c], fixed order.  32 channels x 32 slices per
// CTA: thread (s, c) sums the blocks b = s, s + 32, ... (two accumulators), the 32 slice sums of a channel are combined in
// slice order.  (One thread per channel walking all ~600 row blocks serially took as long as the streaming pass itself.)
__global__ void __launch_bounds__(1024) bwd_cols_finish_kernel(const double2* __restrict__ partial, int nblocks, int channels,
                                                               float* __restrict__ gs, float* __restrict__ gzp) {
  __shared__ double2 s_part[32][33];
  const int lc = threadIdx.x & 31, s = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + lc;
  double a0 = 0.0, a1 = 0.0, b0 = 0.0, b1 = 0.0;
  if (c < channels) {
    int b = s;
    for (; b + 32 < nblocks; b += 64) {
      const double2 v = partial[(long long)b * channels + c], w = partial[(long long)(b + 32) * channels + c];
      a0 += v.x; a1 += v.y; b0 += w.x; b1 += w.y;
    }
    if (b < nblocks) {
      const double2 v = partial[(long long)b * channels + c];
      a0 += v.x; a1 += v.y;
    }
  }
  s_part[s][lc] = make_double2(a0 + b0, a1 + b1);
  __syncthreads();
  if (s == 0 && c < channels) {
    double t0 = 0.0, t1 = 0.0;
    for (int q = 0; q < 32; ++q) { t0 += s_part[q][lc].x; t1 += s_part[q][lc].y; }
    if (gs) gs[c] = (float)t0;
    if (gzp) gzp[c] = (float)t1;
  }
}

static inline int persistent_grid(long long tiles, int ctas_per_sm) {
  long long cap = (long long)sm_count() * ctas_per_sm;
  if (tiles < 1) tiles = 1;
  return (int)(tiles < cap ? tiles : cap);
}

// Threads per CTA of the channel-last kernels: 64 when that leaves fewer idle lanes in the last CTA of a row (192 vector
// columns of a 768-channel tensor: 2 x 128 wastes a quarter of the threads, 3 x 64 none), else 128.
static inline int cols_block_threads(long long channels) {
  const long long nq = (channels % 4 == 0) ? channels / 4 : channels;
  const long long w128 = (nq + 127) / 128 * 128 - nq, w64 = (nq + 63) / 64 * 64 - nq;
  return w64 < w128 ? 64 : 128;
}
static inline long long cols_row_blocks(long long outer, long long channels) {
  const int bt = cols_block_threads(channels);
  const long long gx = (((channels % 4 == 0) ? channels / 4 : channels) + bt - 1) / bt;
  long long want = ((long long)sm_count() * 8 * (128 / bt) + gx - 1) / gx;
  if (want > outer) want = outer;
  if (want > 65535) want = 65535;
  if (want < 1) want = 1;
  const long long rpb = (outer + want - 1) / want;
  return (outer + rpb - 1) / rpb;
}

static size_t bwd_ws_bytes(long long outer, long long channels, long long inner) {
  if (outer <= 0 || channels <= 0 || inner <= 0) return 0;
  if (inner == 1 && channels > 1) return (size_t)(cols_row_blocks(outer, channels) * channels) * sizeof(double2);
  const long long tpr = (inner + kTile - 1) / kTile;
  return (size_t)(outer * channels * tpr) * sizeof(double2);
}

static int bwd_dispatch(const float* x, const float* scale, const float* zp, const float* gy, float* gx, float* gs,
                        float* gzp, long long outer, long long channels, long long inner, int qmin, int qmax,
                        int rounding, bool gzp_open_top, void* workspace, size_t workspace_bytes, cudaStream_t st,
                        const char* who) {
  const float gz_hi = gzp_open_top ? (float)qmax - 1.f : (float)qmax;
  SB_REQUIRE(x && scale && zp && gy && gx, "%s: null pointer argument", who);
  SB_REQUIRE(outer > 0 && channels > 0 && inner > 0, "%s: Kernel Failure, Tensor is empty: data", who);
  SB_REQUIRE(qmin <= qmax, "%s: qmin > qmax", who);
  SB_REQUIRE(rounding >= 0 && rounding <= 2, "%s: rounding must be 0, 1 or 2", who);
  SB_REQUIRE(channels < (1LL << 31), "%s: too many channels", who);
  const bool need_red = gs || gzp;
  const size_t need = need_red ? bwd_ws_bytes(outer, channels, inner) : 0;
  if (need_red && (!workspace || workspace_bytes < need)) {
    set_error("%s: workspace too small (%zu < %zu bytes)", who, workspace_bytes, need);
    return SB200_E_WORKSPACE;
  }
  double2* partial = need_red ? (double2*)workspace : nullptr;
  if (inner == 1 && channels > 1) {
    const long long nb = cols_row_blocks(outer, channels);
    const long long rpb = (outer + nb - 1) / nb;
    const bool vec = (channels % 4 == 0) && aligned16(x) && aligned16(gy) && aligned16(gx);
    // cols_row_blocks sizes the grid for the vector layout when C % 4 == 0; the scalar fallback only
    // gets more thread blocks along x, the partial layout [row block][C] is the same.
    const long long nqv = vec ? channels / 4 : channels;
    const int bt = cols_block_threads(channels);
    const dim3 grid((unsigned)((nqv + bt - 1) / bt), (unsigned)nb);
#define SB_GOC(V_, R_) \
  bwd_cols_kernel<V_, R_><<<grid, bt, 0, st>>>(x, gy, gx, scale, zp, outer, (int)channels, rpb, (float)qmin, (float)qmax, gz_hi, rounding, partial)
    if (vec) {
      if (rounding == 0) SB_GOC(4, 0); else SB_GOC(4, -1);
    } else {
      if (rounding == 0) SB_GOC(1, 0); else SB_GOC(1, -1);
    }
#undef SB_GOC
    SB_LAUNCHED();
    if (need_red) {
      bwd_cols_finish_kernel<<<(unsigned)((channels + 31) / 32), 1024, 0, st>>>(partial, (int)nb, (int)channels, gs, gzp);
      SB_LAUNCHED();
    }
    return SB200_OK;
  }
  const long long rows = outer * channels;
  const long long tpr = (inner + kTile - 1) / kTile;
  const long long tiles = rows * tpr;
  const bool cta_tile = inner >= 1024;
#define SB_GO(CT_, R_)                                                                                   \
  bwd_rows_kernel<CT_, R_><<<persistent_grid(CT_ ? tiles : (tiles + 7) / 8, 8), kThreads, 0, st>>>(     \
      x, gy, gx, scale, zp, rows, inner, (int)channels, (float)qmin, (float)qmax, gz_hi, rounding, partial)
  if (cta_tile) {
    if (rounding == 0) SB_GO(true, 0); else SB_GO(true, -1);
  } else {
    if (rounding == 0) SB_GO(false, 0); else SB_GO(false, -1);
  }
#undef SB_GO
  SB_LAUNCHED();
  if (need_red) {
    bwd_rows_finish_kernel<<<(unsigned)channels, kThreads, 0, st>>>(partial, outer, (int)channels, tpr, gs, gzp);
    SB_LAUNCHED();
  }
  return SB200_OK;
}

}  // namespace sb200

using namespace sb200;

extern "C" {

size_t sb200_qdq_bwd_workspace_bytes(int64_t outer, int64_t channels, int64_t inner) {
  return bwd_ws_bytes(outer, channels, inner);
}

int sb200_qdq_pertensor_bwd(const float* x, const float* scale, const float* zero_point, const float* grad_y,
                            float* grad_x, float* grad_scale, float* grad_zp, int64_t n, int qmin, int qmax,
                            int rounding, void* workspace, size_t workspace_bytes, void* stream) {
  return bwd_dispatch(x, scale, zero_point, grad_y, grad_x, grad_scale, grad_zp, 1, 1, n, qmin, qmax, rounding, false,
                      workspace, workspace_bytes, (cudaStream_t)stream, "sb200_qdq_pertensor_bwd");
}

int sb200_qdq_perchannel_bwd(const float* x, const float* scale, const float* zero_point, const float* grad_y,
                             float* grad_x, float* grad_scale, float* grad_zp, int64_t outer, int64_t channels,
                             int64_t inner, int qmin, int qmax, int rounding, void* workspace, size_t workspace_bytes,
                             void* stream) {
  return bwd_dispatch(x, scale, zero_point, grad_y, grad_x, grad_scale, grad_zp, outer, channels, inner, qmin, qmax,
                      rounding, true, workspace, workspace_bytes, (cudaStream_t)stream, "sb200_qdq_perchannel_bwd");
}

int sb200_qdq_perchannel_bwd_ex(const float* x, const float* scale, const float* zero_point, const float* grad_y,
                                float* grad_x, float* grad_scale, float* grad_zp, int64_t outer, int64_t channels,
                                int64_t inner, int qmin, int qmax, int rounding, int flags, void* workspace,
                                size_t workspace_bytes, void* stream) {
  SB_REQUIRE((flags & ~SB200_BWD_GZP_CLOSED) == 0, "sb200_qdq_perchannel_bwd_ex: unknown flags 0x%x", flags);
  return bwd_dispatch(x, scale, zero_point, grad_y, grad_x, grad_scale, grad_zp, outer, channels, inner, qmin, qmax,
                      rounding, (flags & SB200_BWD_GZP_CLOSED) == 0, workspace, workspace_bytes, (cudaStream_t)stream,
                      "sb200_qdq_perchannel_bwd_ex");
}

}  // extern "C"
