// int8_group_conv.cu -- integer-grid inference of a calibrated grouped or depthwise QConv2d (groups >= 2):
//   y[img, n, oh, ow] = fp32(fp64(I) * (fp64(s_x) * fp64(s_w[n])))  (+ bias[n] in fp32)
//   I = sum over the C_g channels of group g(n) = n / (C_out / groups) and the KH x KW taps of (v_x - Z_x)(v_w[n] - Z_w[n])
// computed directly, without a lowered copy of the input: the fake-quant conv reads x for the QDQ pass, writes it,
// and reads it again for cuDNN; here x is read once and y written once.
//
// A CTA owns one image, a block of output channels and a TH x TW tile of output pixels.  It stages the stored grid
// values (stored_grid of int8_grid.cuh, the quantizer of every integer-grid kernel) of the input window of its
// channels, halo and padding included, in shared memory, and its weight rows next to them; a padding tap holds
// rint(zp) - off, the grid point of the fake-quant input's zero padding, as in the conv2d lowering (int8_linear.cu).
// Each thread then keeps a register tile of outputs and accumulates, per output, sum a b and the window sum sum a in
// int32, and the zero points come out in int64 with the epilogue of int8_linear_gemm_kernel, operation for operation:
//   I = sum a b - Z_w sum a + (K_g Z_x Z_w - Z_x sum_k b),   y = fp32(fp64(I) * (s_x * s_w[n])),   y + bias[n]
// so that a group is bit-identical to sb200_int8_conv2d run on that group's channel slice.  |a|, |b| <= 128:
// |sum a b| <= K_g 2^14 fits int32 for K_g < 2^17, the limit of the linear.
//
// Paths (chosen per call on the host, gc_plan):
//   kDepthwise  C_g = 1: tile [CB channels][TIH][TIW] of s8; plain integer MACs, 4 outputs per thread per round.
//   kGrouped    C_g >= 2: tile [C4 = ceil(C_g / 4)][TIH][TIW] of words holding 4 channels (channels past C_g are 0);
//               weights [MB][KH KW][C4] words; __dp4a, 4 output channels x 2 pixels per thread per round.
//   kDirect     the staged tile with halo, or the weight rows, would not fit kGcSmemMax: one thread per output reads
//               its window from x (stored_grid per tap) and w_q; no shared memory.
// The staged paths load x with 16-byte loads when W % 4 == 0 and x is 16-byte aligned (rows of x then start on 16
// bytes and a 4-aligned column quad is wholly inside or outside the row), else with coalesced scalar loads.
// NaN: a CTA whose tile holds a NaN (__syncthreads_or) re-reads each output's window from x to mark the outputs whose
// group's window covers it; other CTAs pay nothing.  No workspace, no atomics, no state between calls: deterministic
// and graph-capturable with nothing to pin.  Every offset into x and out is 64-bit.
#include "int8_grid.cuh"

namespace sb200 {
namespace {

constexpr int kGcThreads = 256;
constexpr int kGcSmemMax = 48 * 1024;    // the staged tile + weights; above it the call takes the direct path
constexpr int kGcTarget = 2048;          // outputs per CTA aimed at (depthwise); kGrouped aims at 2 x as many
constexpr int kGcMaxTW = 128;            // output columns per tile
constexpr int kGcMaxMB = 64;             // output channels per CTA (kGrouped)
constexpr long long kGcMaxGrid = 1 << 16;  // CTAs launched; a larger call loops (grid-stride over CTA tiles)

enum GcMode { kDepthwise = 0, kGrouped = 1, kDirect = 2 };

struct GcDims {
  long long N, C, H, W, OH, OW, Cout;
  int Cg, Mg, KH, KW, sh, sw, dh, dw, pt, pl, Kg, Kp;
  // staged paths: the CTA tile
  int TH, TW, TIH, TIW, tiles_h, tiles_w;
  int OB;        // output channels per CTA: CB m (depthwise, CB channels of multiplier m = Mg) or MB (grouped)
  int CB, C4;    // staged input channels per CTA (depthwise), channel words (grouped)
  int oblocks;   // output-channel blocks per image (depthwise: ceil(C / CB); grouped: groups ceil(Mg / MB))
  int mblocks;   // grouped: blocks per group
  long long ctas;
  int vec;
};

// The per-output epilogue, operation for operation that of int8_linear_gemm_kernel<true>.
__device__ __forceinline__ float gc_epilogue(int acc, int sa, int n, long long zx, float sx, int K,
                                             const int* __restrict__ w_sum, const float* __restrict__ w_scale,
                                             const int* __restrict__ w_zero, const float* __restrict__ bias, bool nan) {
  const int zw = __ldg(w_zero + n);
  const long long cn = (long long)K * zx * zw - zx * (long long)__ldg(w_sum + n);
  const double sxw = (double)sx * (double)__ldg(w_scale + n);
  const long long I = (long long)acc - (long long)zw * (long long)sa + cn;
  float y = __double2float_rn((double)I * sxw);
  if (bias) y = __fadd_rn(y, __ldg(bias + n));
  if (nan) y = __int_as_float(0x7fc00000);
  return y;
}

// Does the window of output (img, oh, ow) over channels [c0, c0 + cn) hold an element whose grid value is NaN?
template <bool kDoReFa>
__device__ bool gc_window_nan(const float* __restrict__ x, const GcDims& d, const QP& p, int off, double xm, long long img,
                              long long c0, int cn, long long oh, long long ow) {
  bool nan = false;
  for (int c = 0; c < cn; ++c) {
    const float* xc = x + ((img * d.C + c0 + c) * d.H) * d.W;
    for (int kh = 0; kh < d.KH; ++kh) {
      const long long ih = oh * d.sh - d.pt + (long long)kh * d.dh;
      if ((unsigned long long)ih >= (unsigned long long)d.H) continue;
      for (int kw = 0; kw < d.KW; ++kw) {
        const long long iw = ow * d.sw - d.pl + (long long)kw * d.dw;
        if ((unsigned long long)iw < (unsigned long long)d.W)
          (void)input_grid<kDoReFa>(__ldg(xc + ih * d.W + iw), xm, p, off, nan);
      }
    }
  }
  return nan;
}

// Stage the stored grid of the input window [ih_lo, ih_lo + TIH) x [iw_lo, iw_lo + TIW) of `cq` channels: put(cl, r,
// col, value) stores one element; channel cl is real when cl < creal (else it stores 0); c0 is the first channel.
template <bool kDoReFa, typename Put>
__device__ __forceinline__ bool gc_stage(const float* __restrict__ x, const GcDims& d, const QP& p, int off, double xm,
                                         int pad, long long img, long long c0, int cq, int creal, long long ih_lo, long long iw_lo,
                                         Put put) {
  bool nan = false;
  if (d.vec) {
    const long long q0 = iw_lo >= 0 ? iw_lo & ~3LL : -((3 - iw_lo) & ~3LL);  // floor to a multiple of 4
    const int nq = (int)((iw_lo + d.TIW - q0 + 3) >> 2);
    const int total = cq * d.TIH * nq;
    for (int i = threadIdx.x; i < total; i += kGcThreads) {
      const int cl = i / (d.TIH * nq), rem = i - cl * (d.TIH * nq), r = rem / nq, qi = rem - r * nq;
      const long long ih = ih_lo + r, gc = q0 + 4LL * qi;
      int e[4];
      if (cl >= creal) {
        e[0] = e[1] = e[2] = e[3] = 0;
      } else if ((unsigned long long)ih < (unsigned long long)d.H && gc >= 0 && gc < d.W) {
        const float4 f = __ldg(reinterpret_cast<const float4*>(x + ((img * d.C + c0 + cl) * d.H + ih) * d.W + gc));
        e[0] = input_grid<kDoReFa>(f.x, xm, p, off, nan), e[1] = input_grid<kDoReFa>(f.y, xm, p, off, nan);
        e[2] = input_grid<kDoReFa>(f.z, xm, p, off, nan), e[3] = input_grid<kDoReFa>(f.w, xm, p, off, nan);
      } else {
        e[0] = e[1] = e[2] = e[3] = pad;
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const long long col = gc + j - iw_lo;
        if (col >= 0 && col < d.TIW) put(cl, r, (int)col, e[j]);
      }
    }
  } else {
    const int total = cq * d.TIH * d.TIW;
    for (int i = threadIdx.x; i < total; i += kGcThreads) {
      const int cl = i / (d.TIH * d.TIW), rem = i - cl * (d.TIH * d.TIW), r = rem / d.TIW, col = rem - r * d.TIW;
      const long long ih = ih_lo + r, iw = iw_lo + col;
      int e = 0;
      if (cl < creal) {
        if ((unsigned long long)ih < (unsigned long long)d.H && (unsigned long long)iw < (unsigned long long)d.W)
          e = input_grid<kDoReFa>(__ldg(x + ((img * d.C + c0 + cl) * d.H + ih) * d.W + iw), xm, p, off, nan);
        else
          e = pad;
      }
      put(cl, r, col, e);
    }
  }
  return nan;
}

// kDoReFa: x is a DoReFa input normalised by *x_absmax (input_grid of int8_grid.cuh), in every path.
// The DoReFa kGrouped instantiation asks for 4 CTAs per SM (64 registers, as the plain one): without the hint ptxas
// spills a few words of it to reach its own occupancy target.  Every other instantiation has no hint.
template <int kMode, bool kDoReFa>
__global__ void __launch_bounds__(kGcThreads, kDoReFa && kMode == kGrouped ? 4 : 0) int8_group_conv_kernel(const float* __restrict__ x, GcDims d,
                                                                     const float* __restrict__ x_scale,
                                                                     const float* __restrict__ x_zero, float qmin,
                                                                     float qmax, int off, const int8_t* __restrict__ w_q,
                                                                     const int* __restrict__ w_sum,
                                                                     const float* __restrict__ w_scale,
                                                                     const int* __restrict__ w_zero,
                                                                     const float* __restrict__ bias,
                                                                     float* __restrict__ out,
                                                                     const float* __restrict__ x_absmax) {
  extern __shared__ __align__(16) unsigned char gc_smem[];
  QP p;
  p.set(__ldg(x_scale), __ldg(x_zero));
  p.qmin = qmin;
  p.qmax = qmax;
  const int pad = (int)p.zp - off;  // the grid point v = 0 of the fake-quant input's zero padding
  const float sx = __ldg(x_scale);
  const long long zx = (long long)rintf(__ldg(x_zero)) - off;
  const double xm = kDoReFa ? dorefa_rcp(__ldg(x_absmax)) : 0.0;  // 1 / m of a DoReFa input
  const int taps = d.KH * d.KW;
  const long long plane = d.OH * d.OW;

  if constexpr (kMode == kDirect) {
    // one output per thread, grid-stride over every output; out is NCHW, so consecutive threads store consecutive ow
    const long long total = d.N * d.Cout * plane;
    for (long long o = (long long)blockIdx.x * kGcThreads + threadIdx.x; o < total; o += (long long)gridDim.x * kGcThreads) {
      const long long img = o / (d.Cout * plane), rem = o - img * (d.Cout * plane);
      const int n = (int)(rem / plane);
      const long long pix = rem - (long long)n * plane, oh = pix / d.OW, ow = pix - oh * d.OW;
      const long long c0 = (long long)(n / d.Mg) * d.Cg;
      const int8_t* wr = w_q + (long long)n * d.Kp;
      int acc = 0, sa = 0;
      bool nan = false;
      for (int c = 0; c < d.Cg; ++c) {
        const float* xc = x + ((img * d.C + c0 + c) * d.H) * d.W;
        for (int kh = 0; kh < d.KH; ++kh) {
          const long long ih = oh * d.sh - d.pt + (long long)kh * d.dh;
          for (int kw = 0; kw < d.KW; ++kw) {
            const long long iw = ow * d.sw - d.pl + (long long)kw * d.dw;
            int a = pad;
            if ((unsigned long long)ih < (unsigned long long)d.H && (unsigned long long)iw < (unsigned long long)d.W)
              a = input_grid<kDoReFa>(__ldg(xc + ih * d.W + iw), xm, p, off, nan);
            a = (int)(int8_t)a;  // the s8 the staged paths and the conv2d lowering store
            acc += a * (int)__ldg(wr + c * taps + kh * d.KW + kw);
            sa += a;
          }
        }
      }
      out[o] = gc_epilogue(acc, sa, n, zx, sx, d.Kg, w_sum, w_scale, w_zero, bias, nan);
    }
    return;
  } else {
    const int tile_pix = d.TH * d.TW;
    for (long long t = blockIdx.x; t < d.ctas; t += gridDim.x) {
      // spatial tile fastest: neighbouring CTAs share their halo rows in L2
      const int tw = (int)(t % d.tiles_w);
      long long u = t / d.tiles_w;
      const int th = (int)(u % d.tiles_h);
      u /= d.tiles_h;
      const int ob = (int)(u % d.oblocks);
      const long long img = u / d.oblocks;
      const long long oh0 = (long long)th * d.TH, ow0 = (long long)tw * d.TW;
      const long long ih_lo = oh0 * d.sh - d.pt, iw_lo = ow0 * d.sw - d.pl;
      const int tplane = d.TIH * d.TIW;
      long long n0, c0;  // first output channel, first input channel of the CTA
      int nout, creal;   // live output channels, real input channels staged
      if constexpr (kMode == kDepthwise) {
        c0 = (long long)ob * d.CB;
        creal = (int)min((long long)d.CB, d.C - c0);
        n0 = c0 * d.Mg;
        nout = creal * d.Mg;
      } else {
        const int g = ob / d.mblocks, mb = ob - g * d.mblocks;
        c0 = (long long)g * d.Cg;
        creal = d.Cg;
        n0 = (long long)g * d.Mg + (long long)mb * d.OB;
        nout = min(d.OB, d.Mg - mb * d.OB);
      }
      __syncthreads();  // the previous tile's shared memory has been read
      bool nan;
      if constexpr (kMode == kDepthwise) {
        int8_t* xs = reinterpret_cast<int8_t*>(gc_smem);
        int8_t* ws = xs + (size_t)d.CB * tplane;
        for (int i = threadIdx.x; i < nout * taps; i += kGcThreads) {
          const int ol = i / taps, k = i - ol * taps;
          ws[i] = __ldg(w_q + (n0 + ol) * d.Kp + k);
        }
        nan = gc_stage<kDoReFa>(x, d, p, off, xm, pad, img, c0, d.CB, creal, ih_lo, iw_lo,
                       [&](int cl, int r, int col, int e) { xs[cl * tplane + r * d.TIW + col] = (int8_t)e; });
      } else {
        uint32_t* xs = reinterpret_cast<uint32_t*>(gc_smem);
        uint32_t* ws = xs + (size_t)d.C4 * tplane;
        // ws[(ol taps + k) C4 + c4] packs channels 4 c4 .. 4 c4 + 3 of tap k of output ol; w_q's K order is (c, kh, kw)
        for (int i = threadIdx.x; i < (d.OB + 3) / 4 * 4 * taps * d.C4; i += kGcThreads) {  // rows past nout are 0
          const int ol = i / (taps * d.C4), rem = i - ol * (taps * d.C4), k = rem / d.C4, c4 = rem - k * d.C4;
          uint32_t wv = 0u;
          if (ol < nout) {
            const int8_t* wr = w_q + (n0 + ol) * d.Kp + k;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const int c = 4 * c4 + j;
              if (c < d.Cg) wv |= ((uint32_t)(uint8_t)__ldg(wr + c * taps)) << (8 * j);
            }
          }
          ws[i] = wv;
        }
        unsigned char* xb = gc_smem;
        nan = gc_stage<kDoReFa>(x, d, p, off, xm, pad, img, c0, 4 * d.C4, creal, ih_lo, iw_lo,
                                [&](int cl, int r, int col, int e) {
          xb[(((cl >> 2) * tplane + r * d.TIW + col) << 2) + (cl & 3)] = (unsigned char)e;
        });
      }
      const bool any_nan = __syncthreads_or(nan) != 0;

      if constexpr (kMode == kDepthwise) {
        const int8_t* xs = reinterpret_cast<const int8_t*>(gc_smem);
        const int8_t* ws = xs + (size_t)d.CB * tplane;
        const int items = nout * tile_pix;
        for (int base = threadIdx.x; base < items; base += 4 * kGcThreads) {
          int acc[4], sa[4], ol[4], pix[4], xo[4];
#pragma unroll
          for (int r = 0; r < 4; ++r) {
            const int i = min(base + r * kGcThreads, items - 1);  // a dead slot recomputes the last item
            ol[r] = i / tile_pix;
            pix[r] = i - ol[r] * tile_pix;
            const int ph = pix[r] / d.TW, pw = pix[r] - ph * d.TW;
            xo[r] = (ol[r] / d.Mg) * tplane + ph * d.sh * d.TIW + pw * d.sw;  // the window's top-left tap in the tile
            acc[r] = 0, sa[r] = 0;
          }
          for (int kh = 0; kh < d.KH; ++kh) {
            for (int kw = 0; kw < d.KW; ++kw) {
              const int k = kh * d.KW + kw, to = kh * d.dh * d.TIW + kw * d.dw;
#pragma unroll
              for (int r = 0; r < 4; ++r) {
                const int a = xs[xo[r] + to];
                acc[r] += a * (int)ws[ol[r] * taps + k];
                sa[r] += a;
              }
            }
          }
#pragma unroll
          for (int r = 0; r < 4; ++r) {
            if (base + r * kGcThreads >= items) continue;
            const int ph = pix[r] / d.TW, pw = pix[r] - ph * d.TW;
            const long long oh = oh0 + ph, ow = ow0 + pw;
            if (oh >= d.OH || ow >= d.OW) continue;
            const long long n = n0 + ol[r];
            const bool wn = any_nan && gc_window_nan<kDoReFa>(x, d, p, off, xm, img, c0 + ol[r] / d.Mg, 1, oh, ow);
            out[((img * d.Cout + n) * d.OH + oh) * d.OW + ow] =
                gc_epilogue(acc[r], sa[r], (int)n, zx, sx, d.Kg, w_sum, w_scale, w_zero, bias, wn);
          }
        }
      } else {
        const uint32_t* xs = reinterpret_cast<const uint32_t*>(gc_smem);
        const uint32_t* ws = xs + (size_t)d.C4 * tplane;
        const int quads = (nout + 3) >> 2;
        const int items = quads * tile_pix;
        for (int base = threadIdx.x; base < items; base += 2 * kGcThreads) {
          int acc[2][4], sa[2], oq[2], xo[2];
#pragma unroll
          for (int r = 0; r < 2; ++r) {
            const int i = min(base + r * kGcThreads, items - 1);  // a dead slot recomputes the last item
            oq[r] = i / tile_pix;
            const int px = i - oq[r] * tile_pix, ph = px / d.TW, pw = px - ph * d.TW;
            xo[r] = ph * d.sh * d.TIW + pw * d.sw;  // the window's top-left tap in the tile
            sa[r] = 0;
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[r][j] = 0;
          }
          for (int kh = 0; kh < d.KH; ++kh) {
            for (int kw = 0; kw < d.KW; ++kw) {
              const int k = kh * d.KW + kw, to = kh * d.dh * d.TIW + kw * d.dw;
              for (int c4 = 0; c4 < d.C4; ++c4) {
#pragma unroll
                for (int r = 0; r < 2; ++r) {
                  const int a4 = (int)xs[c4 * tplane + xo[r] + to];
                  sa[r] = __dp4a(a4, 0x01010101, sa[r]);
#pragma unroll
                  for (int j = 0; j < 4; ++j)
                    acc[r][j] = __dp4a(a4, (int)ws[((4 * oq[r] + j) * taps + k) * d.C4 + c4], acc[r][j]);
                }
              }
            }
          }
#pragma unroll
          for (int r = 0; r < 2; ++r) {
            const int i = base + r * kGcThreads;
            if (i >= items) continue;
            const int px = i - oq[r] * tile_pix, ph = px / d.TW, pw = px - ph * d.TW;
            const long long oh = oh0 + ph, ow = ow0 + pw;
            if (oh >= d.OH || ow >= d.OW) continue;
            const bool wn = any_nan && gc_window_nan<kDoReFa>(x, d, p, off, xm, img, c0, d.Cg, oh, ow);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const int ol = 4 * oq[r] + j;
              if (ol >= nout) continue;
              const long long n = n0 + ol;
              out[((img * d.Cout + n) * d.OH + oh) * d.OW + ow] =
                  gc_epilogue(acc[r][j], sa[r], (int)n, zx, sx, d.Kg, w_sum, w_scale, w_zero, bias, wn);
            }
          }
        }
      }
    }
  }
}

long long cdiv(long long a, long long b) { return (a + b - 1) / b; }

// Shared memory of a staged tile: the input window (halo included) and the weight rows, each 16-byte aligned.
// Saturated at 2^40: a window of a huge dilation must not wrap around.
long long gc_smem_bytes(int mode, const GcDims& d) {
  const __int128 tile = (__int128)d.TIH * d.TIW, taps = (__int128)d.KH * d.KW;
  const __int128 b = mode == kDepthwise ? d.CB * tile + 16 + d.OB * taps : 4 * d.C4 * tile + 4 * ((d.OB + 3) / 4 * 4) * taps * d.C4;
  return b > ((__int128)1 << 40) ? (1LL << 40) : (long long)b;
}

void gc_tile(GcDims* d, int th, int tw) {
  d->TH = th, d->TW = tw;
  d->TIH = (int)min((long long)INT32_MAX / 2, (long long)(th - 1) * d->sh + (long long)(d->KH - 1) * d->dh + 1);
  d->TIW = (int)min((long long)INT32_MAX / 2, (long long)(tw - 1) * d->sw + (long long)(d->KW - 1) * d->dw + 1);
}

// The launch plan: path, tile, channel block.  Returns the path.
int gc_plan(GcDims* d, const float* x) {
  const long long OH = d->OH, OW = d->OW;
  const int mode = d->Cg == 1 ? kDepthwise : kGrouped;
  d->C4 = (d->Cg + 3) / 4;
  const int tw = (int)min(OW, (long long)kGcMaxTW);
  int th, cb = 1, mb = 1;
  if (mode == kDepthwise) {
    th = (int)max(1LL, min(OH, (long long)kGcTarget / tw));
    cb = (int)max(1LL, min(d->C, (long long)kGcTarget / ((long long)th * tw * d->Mg)));
  } else {
    mb = (int)min((long long)d->Mg, (long long)kGcMaxMB);
    th = (int)max(1LL, min(OH, 2LL * kGcTarget / ((long long)mb * tw)));
  }
  int twc = tw;
  for (;;) {
    gc_tile(d, th, twc);
    d->CB = cb;
    d->OB = mode == kDepthwise ? cb * d->Mg : mb;
    if (gc_smem_bytes(mode, *d) <= kGcSmemMax) break;
    if (mode == kDepthwise && cb > 1) cb = (cb + 1) / 2;
    else if (mode == kGrouped && mb > 1) mb = (mb + 1) / 2;
    else if (th > 1) th = (th + 1) / 2;
    else if (twc > 1) twc = (twc + 1) / 2;
    else return kDirect;
  }
  d->tiles_h = (int)cdiv(OH, d->TH);
  d->tiles_w = (int)cdiv(OW, d->TW);
  if (mode == kDepthwise) {
    d->mblocks = 1;
    d->oblocks = (int)cdiv(d->C, d->CB);
  } else {
    d->mblocks = (int)cdiv(d->Mg, d->OB);
    d->oblocks = (int)(d->C / d->Cg) * d->mblocks;
  }
  d->ctas = d->N * d->oblocks * (long long)d->tiles_h * d->tiles_w;
  d->vec = (d->W % 4 == 0) && aligned16(x);
  return mode;
}

// ---------------------------------------------------------------------------------- NHWC
// x [n, h, w, c] and out [n, OH, OW, c_out] stored NHWC: the channels of one pixel are contiguous, so a thread owns a
// quad of 4 adjacent output channels n0 .. n0 + 3 at a few output pixels and reads each tap's channels with vector
// loads, straight from x (L1 / L2 serve the overlap of neighbouring windows); no staged input tile.  A CTA covers a
// block of 4 QB output channels (QB quads, QB a power of two <= 16) and 256 / QB x kNhRounds consecutive output
// pixels; its weights are staged in shared memory, re-laid out from w_q [c_out, Kp] for the path:
//   kNhDw    C_g = 1, M_g = 1 (depthwise): word [tap][quad] packs the quad's 4 weights of the tap; the quad's 4
//            channels are one float4 (vec) and 4 independent outputs, plain integer MACs.
//   kNhQuad  M_g % 4 = 0: the quad lies in one group and shares its window; word [output][tap][c4] packs channels
//            4 c4 .. 4 c4 + 3 (0 past C_g) and a float4 of the group's channels (vec: C_g % 4 = 0) quantizes straight
//            into one __dp4a word.
//   kNhAny   any other grouping, or weights that do not fit kGcSmemMax: each output of the quad reads its own group's
//            window and w_q directly.
// An output's NaN flag is set by exactly the elements of its group's window, its epilogue is gc_epilogue: outputs are
// bit-identical to the NCHW kernel.  No workspace, no atomics: deterministic and graph-capturable.
constexpr int kNhMaxQuads = 16;
constexpr int kNhRounds = 4;  // pixels per thread

enum NhMode { kNhDw = 0, kNhQuad = 1, kNhAny = 2 };

struct NhDims {
  long long M, P, OW, H, W, C, Cout;
  int Cg, Mg, KH, KW, sh, sw, dh, dw, pt, pl, Kg, Kp, C4;
  int QB, pix;                     // output-channel quads, output pixels per CTA
  long long pblocks, nblocks, ctas;
  int vec, vec_out;
};

__device__ __forceinline__ void nh_store(float* __restrict__ out, const NhDims& d, long long m, long long n0,
                                         const float (&y)[4]) {
  float* o = out + m * d.Cout + n0;
  if (d.vec_out && n0 + 3 < d.Cout) {
    *reinterpret_cast<float4*>(o) = make_float4(y[0], y[1], y[2], y[3]);
  } else {
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (n0 + j < d.Cout) o[j] = y[j];
  }
}

// The DoReFa kNhAny instantiation asks for 3 CTAs per SM (72 registers, as the plain one), which keeps ptxas from
// spilling it to a smaller register count; every other instantiation has no hint.
template <int kMode, bool kDoReFa>
__global__ void __launch_bounds__(kGcThreads, kDoReFa && kMode == kNhAny ? 3 : 0) int8_group_conv_nhwc_kernel(const float* __restrict__ x, NhDims d,
                                                                          const float* __restrict__ x_scale,
                                                                          const float* __restrict__ x_zero, float qmin,
                                                                          float qmax, int off,
                                                                          const int8_t* __restrict__ w_q,
                                                                          const int* __restrict__ w_sum,
                                                                          const float* __restrict__ w_scale,
                                                                          const int* __restrict__ w_zero,
                                                                          const float* __restrict__ bias,
                                                                          float* __restrict__ out,
                                                                          const float* __restrict__ x_absmax) {
  extern __shared__ __align__(16) unsigned char gc_smem[];
  uint32_t* ws = reinterpret_cast<uint32_t*>(gc_smem);
  QP p;
  p.set(__ldg(x_scale), __ldg(x_zero));
  p.qmin = qmin;
  p.qmax = qmax;
  const int pad = (int)p.zp - off;  // the grid point v = 0 of the fake-quant input's zero padding
  const float sx = __ldg(x_scale);
  const long long zx = (long long)rintf(__ldg(x_zero)) - off;
  const double xm = kDoReFa ? dorefa_rcp(__ldg(x_absmax)) : 0.0;  // 1 / m of a DoReFa input
  const int taps = d.KH * d.KW;
  const int ql = threadIdx.x % d.QB, slot = threadIdx.x / d.QB, pstride = kGcThreads / d.QB;
  long long staged = -1;
  for (long long tile = blockIdx.x; tile < d.ctas; tile += gridDim.x) {
    // pixel block fastest: neighbouring CTAs share the weight block and their windows' rows in L2
    const long long pb = tile % d.pblocks, nb = tile / d.pblocks;
    const long long nbase = nb * 4 * d.QB;
    if constexpr (kMode != kNhAny) {
      if (nb != staged) {
        __syncthreads();  // the previous block's weights have been read
        if constexpr (kMode == kNhDw) {
          for (int i = threadIdx.x; i < taps * d.QB; i += kGcThreads) {
            const int k = i / d.QB, qq = i - k * d.QB;
            uint32_t wv = 0u;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const long long n = nbase + 4 * qq + j;
              if (n < d.Cout) wv |= (uint32_t)(uint8_t)__ldg(w_q + n * d.Kp + k) << (8 * j);
            }
            ws[i] = wv;
          }
        } else {
          for (int i = threadIdx.x; i < 4 * d.QB * taps * d.C4; i += kGcThreads) {
            const int ol = i / (taps * d.C4), rem = i - ol * (taps * d.C4), k = rem / d.C4, c4 = rem - k * d.C4;
            const long long n = nbase + ol;
            uint32_t wv = 0u;
            if (n < d.Cout) {
#pragma unroll
              for (int j = 0; j < 4; ++j) {
                const int c = 4 * c4 + j;
                if (c < d.Cg) wv |= (uint32_t)(uint8_t)__ldg(w_q + n * d.Kp + c * taps + k) << (8 * j);
              }
            }
            ws[i] = wv;
          }
        }
        __syncthreads();
        staged = nb;
      }
    }
    const long long n0 = nbase + 4 * ql;  // the thread's quad of output channels
    if (n0 >= d.Cout) continue;
    for (int r = 0; r < kNhRounds; ++r) {
      const long long m = pb * d.pix + slot + (long long)r * pstride;
      if (m >= d.M) break;
      const long long img = m / d.P, pp = m - img * d.P, oh = pp / d.OW, ow = pp - oh * d.OW;
      const long long ih0 = oh * d.sh - d.pt, iw0 = ow * d.sw - d.pl;
      const float* xi = x + img * d.H * d.W * d.C;
      float y[4];
      if constexpr (kMode == kNhDw) {
        int acc[4] = {0, 0, 0, 0}, sa[4] = {0, 0, 0, 0};
        bool nan[4] = {false, false, false, false};
        for (int kh = 0; kh < d.KH; ++kh) {
          const long long ih = ih0 + (long long)kh * d.dh;
          for (int kw = 0; kw < d.KW; ++kw) {
            const long long iw = iw0 + (long long)kw * d.dw;
            int a[4];
            if ((unsigned long long)ih < (unsigned long long)d.H && (unsigned long long)iw < (unsigned long long)d.W) {
              const float* xp = xi + (ih * d.W + iw) * d.C + n0;
              float v[4];
              if (d.vec) {
                const float4 f = __ldg(reinterpret_cast<const float4*>(xp));
                v[0] = f.x, v[1] = f.y, v[2] = f.z, v[3] = f.w;
              } else {
#pragma unroll
                for (int j = 0; j < 4; ++j) v[j] = n0 + j < d.C ? __ldg(xp + j) : 0.f;
              }
#pragma unroll
              for (int j = 0; j < 4; ++j) a[j] = (int)(int8_t)input_grid<kDoReFa>(v[j], xm, p, off, nan[j]);
            } else {
#pragma unroll
              for (int j = 0; j < 4; ++j) a[j] = (int)(int8_t)pad;
            }
            const uint32_t wv = ws[(kh * d.KW + kw) * d.QB + ql];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              acc[j] += a[j] * (int)(int8_t)(wv >> (8 * j));
              sa[j] += a[j];
            }
          }
        }
#pragma unroll
        for (int j = 0; j < 4; ++j)
          y[j] = n0 + j < d.Cout ? gc_epilogue(acc[j], sa[j], (int)(n0 + j), zx, sx, d.Kg, w_sum, w_scale, w_zero, bias,
                                               nan[j])
                                 : 0.f;
      } else if constexpr (kMode == kNhQuad) {
        const long long c0 = n0 / d.Mg * d.Cg;  // M_g % 4 = 0: the quad's one group
        const uint32_t* wt = ws + (size_t)4 * ql * taps * d.C4;
        const int wstride = taps * d.C4;
        int acc[4] = {0, 0, 0, 0}, sa = 0;
        bool nan = false;
        for (int kh = 0; kh < d.KH; ++kh) {
          const long long ih = ih0 + (long long)kh * d.dh;
          for (int kw = 0; kw < d.KW; ++kw) {
            const long long iw = iw0 + (long long)kw * d.dw;
            const bool in = (unsigned long long)ih < (unsigned long long)d.H && (unsigned long long)iw < (unsigned long long)d.W;
            const float* xp = xi + (ih * d.W + iw) * d.C + c0;
            const int k = kh * d.KW + kw;
            for (int c4 = 0; c4 < d.C4; ++c4) {
              uint32_t a4 = 0u;
              const int live = min(4, d.Cg - 4 * c4);  // channels of the quad inside the group
              if (in) {
                float4 f;
                if (d.vec) {
                  f = __ldg(reinterpret_cast<const float4*>(xp + 4 * c4));
                } else {
                  f.x = __ldg(xp + 4 * c4);
                  f.y = live > 1 ? __ldg(xp + 4 * c4 + 1) : 0.f;
                  f.z = live > 2 ? __ldg(xp + 4 * c4 + 2) : 0.f;
                  f.w = live > 3 ? __ldg(xp + 4 * c4 + 3) : 0.f;
                }
                a4 = ((uint32_t)input_grid<kDoReFa>(f.x, xm, p, off, nan) & 0xFFu);
                if (live > 1) a4 |= ((uint32_t)input_grid<kDoReFa>(f.y, xm, p, off, nan) & 0xFFu) << 8;
                if (live > 2) a4 |= ((uint32_t)input_grid<kDoReFa>(f.z, xm, p, off, nan) & 0xFFu) << 16;
                if (live > 3) a4 |= ((uint32_t)input_grid<kDoReFa>(f.w, xm, p, off, nan) & 0xFFu) << 24;
              } else {
                a4 = ((uint32_t)pad & 0xFFu) * 0x01010101u;
                if (live < 4) a4 &= 0xFFFFFFFFu >> (8 * (4 - live));
              }
              sa = __dp4a((int)a4, 0x01010101, sa);
#pragma unroll
              for (int j = 0; j < 4; ++j) acc[j] = __dp4a((int)a4, (int)wt[j * wstride + k * d.C4 + c4], acc[j]);
            }
          }
        }
#pragma unroll
        for (int j = 0; j < 4; ++j)
          y[j] = n0 + j < d.Cout ? gc_epilogue(acc[j], sa, (int)(n0 + j), zx, sx, d.Kg, w_sum, w_scale, w_zero, bias, nan)
                                 : 0.f;
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const long long n = n0 + j;
          y[j] = 0.f;
          if (n >= d.Cout) continue;
          const long long c0 = n / d.Mg * d.Cg;
          const int8_t* wr = w_q + n * d.Kp;
          int acc = 0, sa = 0;
          bool nan = false;
          for (int kh = 0; kh < d.KH; ++kh) {
            const long long ih = ih0 + (long long)kh * d.dh;
            for (int kw = 0; kw < d.KW; ++kw) {
              const long long iw = iw0 + (long long)kw * d.dw;
              const bool in = (unsigned long long)ih < (unsigned long long)d.H && (unsigned long long)iw < (unsigned long long)d.W;
              const float* xp = xi + (ih * d.W + iw) * d.C + c0;
              const int k = kh * d.KW + kw;
              for (int c = 0; c < d.Cg; ++c) {
                const int a = (int)(int8_t)(in ? input_grid<kDoReFa>(__ldg(xp + c), xm, p, off, nan) : pad);
                acc += a * (int)__ldg(wr + c * taps + k);
                sa += a;
              }
            }
          }
          y[j] = gc_epilogue(acc, sa, (int)n, zx, sx, d.Kg, w_sum, w_scale, w_zero, bias, nan);
        }
      }
      nh_store(out, d, m, n0, y);
    }
  }
}

long long nh_smem_bytes(int mode, const NhDims& d) {
  const long long taps = (long long)d.KH * d.KW;
  if (mode == kNhDw) return 4 * taps * d.QB;
  if (mode == kNhQuad) return 16LL * d.QB * taps * d.C4;
  return 0;
}

// The NHWC launch plan: path and channel block.  Returns the path.
int nh_plan(NhDims* d, const float* x, const float* out) {
  int mode = d->Cg == 1 && d->Mg == 1 ? kNhDw : d->Mg % 4 == 0 ? kNhQuad : kNhAny;
  d->C4 = (d->Cg + 3) / 4;
  int qb = 1;
  while (qb < kNhMaxQuads && 4LL * qb < d->Cout) qb *= 2;
  if (mode != kNhAny) {
    for (;;) {
      d->QB = qb;
      if (nh_smem_bytes(mode, *d) <= kGcSmemMax) break;
      if (qb == 1) {
        mode = kNhAny;
        break;
      }
      qb /= 2;
    }
  }
  d->QB = qb;
  d->pix = kGcThreads / qb * kNhRounds;
  d->pblocks = cdiv(d->M, d->pix);
  d->nblocks = cdiv(d->Cout, 4LL * qb);
  d->ctas = d->pblocks * d->nblocks;
  d->vec = (mode == kNhDw ? d->C % 4 == 0 : d->Cg % 4 == 0) && aligned16(x);
  d->vec_out = d->Cout % 4 == 0 && aligned16(out);
  return mode;
}

}  // namespace
}  // namespace sb200

using namespace sb200;

// The checks of sb200_int8_group_conv2d{,_nhwc}, in order, then (dorefa) check_absmax; fills the conv geometry and K_g.
static int group_conv_checks(const char* fn, const char* dense_fn, bool dorefa, const float* x,
                             const sb200_conv2d_geom* geom, int64_t groups, const float* x_scale,
                             const float* x_zero_point, const float* x_absmax, int qmin_x, int qmax_x, const int8_t* w_q,
                             const int32_t* w_rowsum, const float* w_scale, const int32_t* w_zero, const float* out,
                             int64_t c_out, ConvDims* cd, long long* kg) {
  SB_REQUIRE(x && geom && x_scale && x_zero_point && w_q && w_rowsum && w_scale && w_zero && out,
             "%s: null pointer argument", fn);
  SB_REQUIRE(c_out > 0, "%s: empty operand (c_out=%lld)", fn, (long long)c_out);
  SB_REQUIRE(c_out < (1LL << 31), "%s: dimension too large (c_out=%lld)", fn, (long long)c_out);
  SB_REQUIRE(groups >= 2, "%s: groups = %lld; a conv with groups = 1 runs on %s", fn, (long long)groups, dense_fn);
  if (const int rc = check_conv(fn, geom, cd)) return rc;
  const sb200_conv2d_geom& g = *geom;
  SB_REQUIRE(g.c % groups == 0 && c_out % groups == 0, "%s: groups = %lld does not divide c = %lld and c_out = %lld", fn,
             (long long)groups, (long long)g.c, (long long)c_out);
  if (const int rc = check_range(fn, qmin_x, qmax_x)) return rc;
  *kg = (g.c / groups) * g.kh * g.kw;  // c, kh, kw < 2^31 each: c / groups * kh stays far below 2^63 / kw
  if ((__int128)(g.c / groups) * g.kh * g.kw >= kI8MaxK) {
    set_error("%s: K_g = c / groups kh kw = %lld x %lld x %lld >= 2^17, the integer path supports K_g < 2^17 (|sum| <= "
              "K_g * 2^14 must fit int32)", fn, (long long)(g.c / groups), (long long)g.kh, (long long)g.kw);
    return SB200_E_UNSUPPORTED;
  }
  return check_absmax(fn, dorefa, x_absmax);
}

// sb200_int8_group_conv2d_nhwc (dorefa = false) and sb200_int8_group_conv2d_nhwc_dorefa
static int group_conv_nhwc_entry(const char* fn, bool dorefa, const float* x, const sb200_conv2d_geom* geom,
                                 int64_t groups, const float* x_scale, const float* x_zero_point, const float* x_absmax,
                                 int qmin_x, int qmax_x, const int8_t* w_q, const int32_t* w_rowsum,
                                 const float* w_scale, const int32_t* w_zero, const float* bias, float* out,
                                 int64_t c_out, void* stream) {
  ConvDims cd;
  long long kg;
  if (const int rc = group_conv_checks(fn, "sb200_int8_conv2d_nhwc", dorefa, x, geom, groups, x_scale, x_zero_point,
                                       x_absmax, qmin_x, qmax_x, w_q, w_rowsum, w_scale, w_zero, out, c_out, &cd, &kg))
    return rc;
  const sb200_conv2d_geom& g = *geom;
  NhDims d{};
  d.M = cd.M, d.P = cd.P, d.OW = cd.OW, d.H = g.h, d.W = g.w, d.C = g.c, d.Cout = c_out;
  d.Cg = (int)(g.c / groups), d.Mg = (int)(c_out / groups);
  d.KH = (int)g.kh, d.KW = (int)g.kw, d.sh = (int)g.stride_h, d.sw = (int)g.stride_w;
  d.dh = (int)g.dilation_h, d.dw = (int)g.dilation_w, d.pt = (int)g.pad_top, d.pl = (int)g.pad_left;
  d.Kg = (int)kg, d.Kp = (int)padded_k(kg);
  const int mode = nh_plan(&d, x, out);
  const unsigned grid = (unsigned)min(d.ctas, kGcMaxGrid);
  const size_t smem = (size_t)nh_smem_bytes(mode, d);
  const bool df = x_absmax != nullptr;
  const auto kernel = mode == kNhDw    ? (df ? int8_group_conv_nhwc_kernel<kNhDw, true> : int8_group_conv_nhwc_kernel<kNhDw, false>)
                      : mode == kNhQuad ? (df ? int8_group_conv_nhwc_kernel<kNhQuad, true> : int8_group_conv_nhwc_kernel<kNhQuad, false>)
                                        : (df ? int8_group_conv_nhwc_kernel<kNhAny, true> : int8_group_conv_nhwc_kernel<kNhAny, false>);
  kernel<<<grid, kGcThreads, smem, (cudaStream_t)stream>>>(x, d, x_scale, x_zero_point, (float)qmin_x, (float)qmax_x,
                                                           grid_offset(qmin_x), w_q, reinterpret_cast<const int*>(w_rowsum),
                                                           w_scale, reinterpret_cast<const int*>(w_zero), bias, out,
                                                           x_absmax);
  SB_LAUNCHED();
  return SB200_OK;
}

// sb200_int8_group_conv2d (dorefa = false) and sb200_int8_group_conv2d_dorefa
static int group_conv_entry(const char* fn, bool dorefa, const float* x, const sb200_conv2d_geom* geom, int64_t groups,
                            const float* x_scale, const float* x_zero_point, const float* x_absmax, int qmin_x,
                            int qmax_x, const int8_t* w_q, const int32_t* w_rowsum, const float* w_scale,
                            const int32_t* w_zero, const float* bias, float* out, int64_t c_out, void* stream) {
  ConvDims cd;
  long long kg;
  if (const int rc = group_conv_checks(fn, "sb200_int8_conv2d", dorefa, x, geom, groups, x_scale, x_zero_point, x_absmax,
                                       qmin_x, qmax_x, w_q, w_rowsum, w_scale, w_zero, out, c_out, &cd, &kg))
    return rc;
  const sb200_conv2d_geom& g = *geom;
  GcDims d{};
  d.N = g.n, d.C = g.c, d.H = g.h, d.W = g.w, d.Cout = c_out, d.OH = cd.P / cd.OW, d.OW = cd.OW;
  d.Cg = (int)(g.c / groups), d.Mg = (int)(c_out / groups);
  d.KH = (int)g.kh, d.KW = (int)g.kw, d.sh = (int)g.stride_h, d.sw = (int)g.stride_w;
  d.dh = (int)g.dilation_h, d.dw = (int)g.dilation_w, d.pt = (int)g.pad_top, d.pl = (int)g.pad_left;
  d.Kg = (int)kg, d.Kp = (int)padded_k(kg);
  const int mode = gc_plan(&d, x);
  unsigned grid;
  size_t smem = 0;
  if (mode == kDirect) {
    grid = (unsigned)min(cdiv(d.N * d.Cout * d.OH * d.OW, kGcThreads), kGcMaxGrid);
  } else {
    grid = (unsigned)min(d.ctas, kGcMaxGrid);
    smem = (size_t)gc_smem_bytes(mode, d);
  }
  const bool df = x_absmax != nullptr;
  const auto kernel = mode == kDirect      ? (df ? int8_group_conv_kernel<kDirect, true> : int8_group_conv_kernel<kDirect, false>)
                      : mode == kDepthwise ? (df ? int8_group_conv_kernel<kDepthwise, true> : int8_group_conv_kernel<kDepthwise, false>)
                                           : (df ? int8_group_conv_kernel<kGrouped, true> : int8_group_conv_kernel<kGrouped, false>);
  kernel<<<grid, kGcThreads, smem, (cudaStream_t)stream>>>(x, d, x_scale, x_zero_point, (float)qmin_x, (float)qmax_x,
                                                           grid_offset(qmin_x), w_q, reinterpret_cast<const int*>(w_rowsum),
                                                           w_scale, reinterpret_cast<const int*>(w_zero), bias, out,
                                                           x_absmax);
  SB_LAUNCHED();
  return SB200_OK;
}

int sb200_int8_group_conv2d_nhwc(const float* x, const sb200_conv2d_geom* geom, int64_t groups, const float* x_scale,
                                 const float* x_zero_point, int qmin_x, int qmax_x, const int8_t* w_q,
                                 const int32_t* w_rowsum, const float* w_scale, const int32_t* w_zero, const float* bias,
                                 float* out, int64_t c_out, void* stream) {
  return group_conv_nhwc_entry("sb200_int8_group_conv2d_nhwc", false, x, geom, groups, x_scale, x_zero_point, nullptr,
                               qmin_x, qmax_x, w_q, w_rowsum, w_scale, w_zero, bias, out, c_out, stream);
}

int sb200_int8_group_conv2d_nhwc_dorefa(const float* x, const sb200_conv2d_geom* geom, int64_t groups,
                                        const float* x_scale, const float* x_zero_point, const float* x_absmax,
                                        int qmin_x, int qmax_x, const int8_t* w_q, const int32_t* w_rowsum,
                                        const float* w_scale, const int32_t* w_zero, const float* bias, float* out,
                                        int64_t c_out, void* stream) {
  return group_conv_nhwc_entry("sb200_int8_group_conv2d_nhwc_dorefa", true, x, geom, groups, x_scale, x_zero_point,
                               x_absmax, qmin_x, qmax_x, w_q, w_rowsum, w_scale, w_zero, bias, out, c_out, stream);
}

int sb200_int8_group_conv2d(const float* x, const sb200_conv2d_geom* geom, int64_t groups, const float* x_scale,
                            const float* x_zero_point, int qmin_x, int qmax_x, const int8_t* w_q, const int32_t* w_rowsum,
                            const float* w_scale, const int32_t* w_zero, const float* bias, float* out, int64_t c_out,
                            void* stream) {
  return group_conv_entry("sb200_int8_group_conv2d", false, x, geom, groups, x_scale, x_zero_point, nullptr, qmin_x,
                          qmax_x, w_q, w_rowsum, w_scale, w_zero, bias, out, c_out, stream);
}

int sb200_int8_group_conv2d_dorefa(const float* x, const sb200_conv2d_geom* geom, int64_t groups, const float* x_scale,
                                   const float* x_zero_point, const float* x_absmax, int qmin_x, int qmax_x,
                                   const int8_t* w_q, const int32_t* w_rowsum, const float* w_scale,
                                   const int32_t* w_zero, const float* bias, float* out, int64_t c_out, void* stream) {
  return group_conv_entry("sb200_int8_group_conv2d_dorefa", true, x, geom, groups, x_scale, x_zero_point, x_absmax,
                          qmin_x, qmax_x, w_q, w_rowsum, w_scale, w_zero, bias, out, c_out, stream);
}
