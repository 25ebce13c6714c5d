// tc_common.cuh -- pieces shared by the wgmma GPTQ kernels (gptq_tc.cu, gptq_ts.cu): mbarrier / TMA / wgmma PTX
// wrappers, setmaxnreg, the in-register int4 -> fp16 fragment unpack, the TMA producer role, cuTensorMapEncodeTiled.
//
// Both kernels compute the transposed product D[n, m] = sum_k W[n, k] * x'[m, k] with one warpgroup-wide
// wgmma.m64n128k16 per 16 K: the weights are the A operand, unpacked by every consumer thread straight into its own
// register fragment (no shared-memory round trip for the fp16 weights), the activations x' (fp16 planes, every 8 K
// permuted as 0,4,1,5,2,6,3,7) are the B operand, TMA-loaded as 128-token x 64-K SWIZZLE_128B tiles.
// CTA = one 128-feature x 128-token output tile: warpgroup 0 = TMA producer (one thread), warpgroups 1 and 2 = 64
// features each.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>

#include <mutex>

#include "common.cuh"

namespace sb200 {

constexpr int kWgFeat = 128;                                 // features per CTA (two consumer warpgroups x 64)
constexpr int kWgTok = 128;                                  // tokens per CTA = wgmma N
constexpr int kWgBK = 64;                                    // K per stage = one 128-byte swizzle atom of fp16
constexpr int kWgThreads = 384;                              // producer warpgroup + two consumer warpgroups
constexpr int kWgXBytes = kWgTok * kWgBK * 2;                // 16 KB  x_hi or x_lo tile
constexpr int kWgQBytes = (kWgBK / 8) * kWgFeat * 4;         // 4 KB   packed words [8][128]
constexpr int kWgStageBytes = 2 * kWgXBytes + kWgQBytes;     // 36 KB  (a multiple of 1024: every tile stays aligned)

// ---------------------------------------------------------------------------------- PTX wrappers
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(
          smem_u32(dst)),
      "l"(map), "r"(c0), "r"(c1), "r"(smem_u32(bar))
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

// Register re-balancing between warpgroups (384 threads launch with 168 registers each; the producer needs few, the
// consumers hold two 64-float accumulators plus the weight fragments).
template <int N>
__device__ __forceinline__ void reg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void reg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
// wait for every outstanding wgmma of this warpgroup; the accumulators are threaded through the statement so that no
// use of them can be scheduled above the wait
__device__ __forceinline__ void wgmma_wait_all(float (&d)[64]) {
#pragma unroll
  for (int i = 0; i < 64; ++i) asm volatile("" : "+f"(d[i])::"memory");
  asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
#pragma unroll
  for (int i = 0; i < 64; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// K-major SWIZZLE_128B shared-memory matrix descriptor (sm_90 GMMA form): [0,14) start address >> 4 | [16,30) LBO >> 4
// (unused for swizzled K-major, 1) | [32,46) SBO >> 4 = 1024 B between 8-row groups | [62,64) layout 1 = SWIZZLE_128B.
// Advancing 16 K inside the 128-byte atom adds 32 bytes (2) to the start address field.
__device__ __forceinline__ uint64_t gmma_desc_sw128(uint32_t smem_addr) {
  return (uint64_t)((smem_addr >> 4) & 0x3FFFu) | (1ull << 16) | ((uint64_t)(1024 >> 4) << 32) | (1ull << 62);
}

// D[64 x 128] (+)= A[64 x 16] * B[16 x 128]: A = fp16 fragments in registers (the m16n8k16 layout per warp, warp w of the
// warpgroup holding rows 16w..16w+15), B = 128 x 16 fp16 K-major in shared memory (SWIZZLE_128B descriptor), fp32 D in
// registers.  accumulate == 0 overwrites D.
__device__ __forceinline__ void wgmma_m64n128k16_rs(float (&d)[64], const uint32_t (&a)[4], uint64_t bdesc, int accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %69, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, "
      "{%64,%65,%66,%67}, %68, p, 1, 1, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accumulate));
}

// ---------------------------------------------------------------------------------- int4 -> fp16 fragment unpack
// One packed word = 8 nibbles along K.  With the activations permuted inside every 8 K as 0,4,1,5,2,6,3,7, the two
// fp16 values a thread with (lane & 3) == q needs from a word (K positions 2q, 2q+1 of the fragment layout) are the
// nibbles q and q + 4: one shift, one (x & mask) | bias, one HFMA2.  0x6400 | v is the fp16 number 1024 + v; the odd
// pairs are extracted in place (bits 4..7, i.e. 1024 + 16 q) and brought back by the multiplier 1/16.
struct NibblePair {
  uint32_t shift, mask;
  __half2 mul;
  float base;  // 1024 or 64: the bias the extraction leaves after the multiplier
  __device__ __forceinline__ explicit NibblePair(int q) {
    shift = (uint32_t)(q >> 1) * 8u;
    mask = (q & 1) ? 0x00F000F0u : 0x000F000Fu;
    mul = __float2half2_rn((q & 1) ? 0.0625f : 1.f);
    base = (q & 1) ? 64.f : 1024.f;
  }
  // -(base + zero) for an integer zero point |zero| <= 1024 (exact in fp16)
  __device__ __forceinline__ __half2 offset(float zero) const { return __float2half2_rn(-(base + zero)); }
  // (q - zero) for the two nibbles, exact
  __device__ __forceinline__ __half2 operator()(uint32_t w, __half2 off) const {
    const uint32_t v = ((w >> shift) & mask) | 0x64006400u;
    return __hfma2(*reinterpret_cast<const __half2*>(&v), mul, off);
  }
};
__device__ __forceinline__ uint32_t h2u(__half2 v) { return *reinterpret_cast<const uint32_t*>(&v); }

// ---------------------------------------------------------------------------------- TMA producer role
// Stage s of a tile: x_hi [128 tok][64 K] | x_lo [128 tok][64 K] (only when need_lo) | packed words [8][128 features].
__device__ __forceinline__ void wg_produce(unsigned char* stage_base, uint64_t* full, uint64_t* empty, int stages,
                                           const CUtensorMap* map_hi, const CUtensorMap* map_lo, const CUtensorMap* map_q,
                                           int m0, int n0, int num_kb, bool need_lo, int backoff_ns) {
  const uint32_t tx = (uint32_t)(kWgXBytes + kWgQBytes + (need_lo ? kWgXBytes : 0));
  for (int kb = 0; kb < num_kb; ++kb) {
    const int s = kb % stages;
    const uint32_t ph = (uint32_t)(kb / stages) & 1u;
    mbar_wait_relaxed(&empty[s], ph ^ 1u, backoff_ns);
    unsigned char* st = stage_base + (size_t)s * kWgStageBytes;
    mbar_expect_tx(&full[s], tx);
    tma_load_2d(st, map_hi, kb * kWgBK, m0, &full[s]);
    if (need_lo) tma_load_2d(st + kWgXBytes, map_lo, kb * kWgBK, m0, &full[s]);
    tma_load_2d(st + 2 * kWgXBytes, map_q, n0, kb * (kWgBK / 8), &full[s]);
  }
}

// ---------------------------------------------------------------------------------- tensor maps (host)
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static inline EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

static inline bool make_map_2d(CUtensorMap* map, CUtensorMapDataType dt, const void* base, uint64_t inner, uint64_t outer,
                               uint64_t row_bytes, uint32_t box_inner, uint32_t box_outer, CUtensorMapSwizzle sw) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return false;
  const cuuint64_t dims[2] = {inner, outer};
  const cuuint64_t strides[1] = {row_bytes};
  const cuuint32_t box[2] = {box_inner, box_outer};
  const cuuint32_t estr[2] = {1, 1};
  return enc(map, dt, 2, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
             CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// the three maps of a launch: activation planes (128-token x 64-K boxes, SWIZZLE_128B) and packed words (128 x 8)
static inline bool make_wg_maps(CUtensorMap* hi, CUtensorMap* lo, CUtensorMap* q, const __half* a_hi, const __half* a_lo,
                                const int32_t* qweight, long long M, long long K, long long N, long long KW) {
  return make_map_2d(hi, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, a_hi, (uint64_t)K, (uint64_t)M, (uint64_t)K * 2, kWgBK, kWgTok,
                     CU_TENSOR_MAP_SWIZZLE_128B) &&
         make_map_2d(lo, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, a_lo, (uint64_t)K, (uint64_t)M, (uint64_t)K * 2, kWgBK, kWgTok,
                     CU_TENSOR_MAP_SWIZZLE_128B) &&
         make_map_2d(q, CU_TENSOR_MAP_DATA_TYPE_INT32, qweight, (uint64_t)N, (uint64_t)KW, (uint64_t)N * 4, kWgFeat,
                     kWgBK / 8, CU_TENSOR_MAP_SWIZZLE_NONE);
}

static inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

}  // namespace sb200
