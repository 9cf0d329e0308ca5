// rx_common.cuh -- shared definitions of the sm_90a Gen2 receive path:
// derived configuration, the numerical contract (how each libm/libgcc call the
// reference makes is evaluated on the device), mbarrier / TMA-bulk PTX wrappers,
// the capture kernels' raw-tile loader and running-sum replay.
//
// Numerical contract (SURVEY.md Appendix A.5; every item is exercised by the
// parity tests against the compiled reference):
//   * no FMA contraction anywhere: this translation unit is built with
//     -fmad=false and all arithmetic that must round like the reference uses
//     the explicit _rn intrinsics;
//   * std::abs(complex<float>) = glibc cabsf = (float)sqrt((double)re*re + (double)im*im)
//     (gate_impl.cc:130);
//   * z / complex<float>(N,0) = one IEEE float division per component
//     (libgcc __divsc3 with a zero imaginary divisor; gate_impl.cc:141, tag_decoder_impl.cc:103);
//   * std::norm = re*re + im*im with three roundings (libstdc++ 13);
//   * complex * complex = (ac - bd, ad + bc) with separately rounded products.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/rfid_b200.h"

namespace rfid_b200 {

// ---- protocol constants: include/rfid/global_vars.h:72-143 of the reference ----
constexpr int kT1_D = 240;                // us
constexpr int kPW_D = 12;                 // us
constexpr int kT2_D = 480, kCW_D = 250, kP_DOWN_D = 2000, kDELIM_D = 12, kTRCAL_D = 200;  // us, reader TX (global_vars.h:88-97)
constexpr int kNumPulsesCommand = 5;
constexpr int kTagPreambleBits = 6;
constexpr int kRN16Bits = 17;
constexpr int kEPCBits = 129;
constexpr int kWinSizeD = 250;            // us
constexpr int kDcSizeD = 120;             // us
constexpr int kReaderFreq = 40000;        // BLF
constexpr float kThreshFraction = 0.75f;
constexpr unsigned kPreambleMask = 0xC4B; // TAG_PREAMBLE {1,1,0,1,0,0,1,0,0,0,1,1}: bit j = P[j]

// Derived sample counts (gate_impl.cc:48-53,115,121; tag_decoder_impl.cc:60), computed on the
// host with the reference's own double/float expression order.
struct RxConfig {
  int adc_rate, decim, ntaps;
  int fs_dec;
  int n_T1, n_PW, n_tag_bit_i;
  float n_tag_bit_f;
  int win_length, dc_length;
  int len_rn16, len_epc;
  int fixed_q, max_queries, max_tags;
  int mf_q, mf_rem;        // ntaps / decim, ntaps % decim
  int sync_range;          // number of i with i < 1.5 * n_tag_bit_f   (tag_decoder_impl.cc:85)
  float t_min, t_max;      // EPC period search bounds (tag_decoder_impl.cc:151-152)
  // division by the two ring lengths: reciprocal + "fast" flag when the multiply-correct sequence of
  // f_div_const has been verified exhaustively for this divisor (tools/micro/verify_constdiv.c)
  float win_recip, dc_recip;
  int win_div_fast, dc_div_fast;
};

// ---------------------------------------------------------------- arithmetic primitives
__device__ __forceinline__ float f_add(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float f_sub(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float f_mul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float f_div(float a, float b) { return __fdiv_rn(a, b); }

// IEEE-exact x / d for a constant d whose reciprocal c = RN(1/d) passed the exhaustive check: q = RN(x*c),
// r = x - q*d (exact, fused), result = RN(q + r*c).  Three instructions instead of the ~10 of div.rn.  Only
// applied where no intermediate can underflow / overflow; everything else takes the general division.
__device__ __noinline__ float f_div_general(float x, float d) { return __fdiv_rn(x, d); }

// branch-free halves of f_div_const, so that several divisions can be in flight together:
// the multiply-correct quotient, and whether x is inside the range for which it is verified
__device__ __forceinline__ float f_div_fast(float x, float d, float c)
{
  const float q = __fmul_rn(x, c);
  return __fmaf_rn(__fmaf_rn(-q, d, x), c, q);
}
constexpr float kDivFastMin = 7.9e-31f, kDivFastMax = 1.2e30f;  // verified dividend range of f_div_fast
__device__ __forceinline__ bool f_div_fast_ok(float x)
{
  const float ax = fabsf(x);
  return ax >= kDivFastMin && ax <= kDivFastMax;
}

__device__ __forceinline__ float f_div_const(float x, float d, float c, int fast)
{
  const float ax = fabsf(x);
  if (fast && ax >= 7.9e-31f && ax <= 1.2e30f) {
    const float q = __fmul_rn(x, c);
    const float r = __fmaf_rn(-q, d, x);
    return __fmaf_rn(r, c, q);
  }
  return f_div_general(x, d);  // rare: out of the verified range, or an unverified divisor
}

// glibc cabsf(re + i*im): products are exact in double, one rounding for the sum, correctly
// rounded double sqrt, one rounding to float.
__device__ __forceinline__ float cabsf_ref(float re, float im)
{
  double dr = (double)re, di = (double)im;
  double s = __fma_rn(di, di, __dmul_rn(dr, dr));  // dr*dr exact (48 bits) => fma == round(dr*dr + di*di)
  return __double2float_rn(__dsqrt_rn(s));
}

// rare paths kept out of the callers' instruction stream (the capture kernels are instruction-cache sensitive)
__device__ __noinline__ float cabsf_ref_call(float re, float im) { return cabsf_ref(re, im); }
__device__ __noinline__ float f_div_const_call(float x, float d, float c, int fast) { return f_div_const(x, d, c, fast); }

// The same value without the branches of __dsqrt_rn, so that several evaluations interleave: s as above, one Newton step
// on rsqrt.approx.f64 (relative error after the step < 2^-40), rounded to float.  That equals
// (float)sqrt_rn(s) whenever the approximation is farther than its own error bound from every float rounding boundary
// (the mid-points between adjacent floats, 29 bits below the double's leading bit); `risky` reports the rest -- values
// within 2^-38 of a boundary (one sample in 2^13), zero, and magnitudes where the float result would be subnormal or
// infinite -- for which the caller evaluates cabsf_ref.  tools/micro/cabs_check.cu compares the pair against cabsf_ref.
__device__ __forceinline__ float cabsf_quick(float re, float im, bool& risky)
{
  const double dr = (double)re, di = (double)im;
  const double s = __fma_rn(di, di, __dmul_rn(dr, dr));
  double y;
  asm("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(s));
  double g = __dmul_rn(s, y);
  const double h = __dmul_rn(0.5, y);
  const double r = __fma_rn(-g, h, 0.5);
  g = __fma_rn(g, r, g);
  const unsigned long long bits = (unsigned long long)__double_as_longlong(g);
  const unsigned low = (unsigned)bits & 0x1FFFFFFFu;                 // the 29 bits a float does not keep
  const unsigned hi = (unsigned)(bits >> 32);
  const bool near_mid = (unsigned)(low - 0x10000000u + 0x8000u) < 0x10000u;   // |low - mid| < 2^15  (2^-38 relative)
  const bool range_ok = hi > 0x38200000u && hi < 0x47E00000u;       // 2^-125 < g < 2^127: normal float, finite, not NaN
  risky = near_mid || !range_ok;
  return __double2float_rn(g);
}

__device__ __forceinline__ float2 c_add(float2 a, float2 b) { return make_float2(f_add(a.x, b.x), f_add(a.y, b.y)); }
__device__ __forceinline__ float2 c_sub(float2 a, float2 b) { return make_float2(f_sub(a.x, b.x), f_sub(a.y, b.y)); }
__device__ __forceinline__ float c_norm(float2 a) { return f_add(f_mul(a.x, a.x), f_mul(a.y, a.y)); }
// std::real((a - b) * std::conj(h)): (x+iy)(c+id) with d = -h.y, real = x*c - y*d
__device__ __forceinline__ float c_proj(float2 a, float2 b, float2 h)
{
  float x = f_sub(a.x, b.x), y = f_sub(a.y, b.y);
  return f_sub(f_mul(x, h.x), f_mul(y, -h.y));
}

// ---------------------------------------------------------------- mbarrier / TMA (sm_90+ PTX)
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count)
{
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init()
{
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar)
{
  asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.shared::cta.b64 st, [%0];\n\t}" ::"r"(smem_u32(bar)) : "memory");
}
// arrive without release semantics (the default .release.cta makes the arriving thread's earlier writes visible first)
__device__ __forceinline__ void mbar_arrive_relaxed(uint64_t* bar)
{
  asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.relaxed.cta.shared::cta.b64 st, [%0];\n\t}" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes)
{
  asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.expect_tx.shared::cta.b64 st, [%0], %1;\n\t}" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity)
{
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// non-blocking test (try_wait may park the thread for a system-dependent time when the phase is not complete): for a
// warp that watches more than one barrier
__device__ __forceinline__ bool mbar_test_wait(uint64_t* bar, uint32_t parity)
{
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\tmbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// spin a few times (the phase is usually complete or about to be), then back off so that a waiting warp
// does not take issue slots away from the latency-critical warps of the co-resident CTAs
#ifndef RFID_B200_MBAR_BACKOFF_NS
#define RFID_B200_MBAR_BACKOFF_NS 200
#endif
#ifndef RFID_B200_MBAR_SPINS
#define RFID_B200_MBAR_SPINS 4
#endif
constexpr unsigned kMbarBackoffNs = RFID_B200_MBAR_BACKOFF_NS;
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity)
{
  for (int i = 0; i < RFID_B200_MBAR_SPINS; i++)
    if (mbar_try_wait(bar, parity)) return;
  while (!mbar_try_wait(bar, parity)) __nanosleep(kMbarBackoffNs);
}
// wait for a phase that is not on this warp's critical path: let the hardware park the warp
// (suspend-time hint, ns) instead of burning issue slots that the sequencer warps need
__device__ __forceinline__ void mbar_wait_relaxed(uint64_t* bar, uint32_t parity, uint32_t hint_ns = 20000)
{
  uint32_t ok = 0;
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\tselp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity), "r"(hint_ns)
        : "memory");
  } while (!ok);
}
// wait of a warp that has nothing else to do: test, sleep, test ... (the suspend-time hint of try_wait returns after a few
// dozen cycles on this part, so a hinted loop spins; an explicit sleep keeps an idle warp out of the issue slots)
__device__ __forceinline__ void mbar_wait_idle(uint64_t* bar, uint32_t parity, unsigned sleep_ns)
{
  while (!mbar_try_wait(bar, parity)) __nanosleep(sleep_ns);
}
// 1-D bulk copy global -> shared through the TMA engine; completion is signalled on `bar`
// (SASS: UBLKCP).  dst/src 16-byte aligned, bytes a multiple of 16.
__device__ __forceinline__ void tma_load_1d(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar)
{
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(smem_dst)),
               "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
// same, with an L2 eviction hint for data that is read exactly once (the raw capture): evict-first keeps the streaming
// input from displacing the kernel's L2-resident scratch
__device__ __forceinline__ unsigned long long l2_policy_evict_first()
{
  unsigned long long pol;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
__device__ __forceinline__ void tma_load_1d_hint(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar, unsigned long long pol)
{
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(
                   smem_u32(smem_dst)),
               "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar)), "l"(pol)
               : "memory");
}
__device__ __forceinline__ void named_bar_sync(int id, int nthreads)
{
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// ---- what every capture kernel does with its tiles: raw-tile copies, running-sum replay ----
constexpr int kTT = 128;          // decimated samples per tile (rx_pack_kernel: per half-tile)

__device__ __forceinline__ void chain8(float4& u, float4& v, float& acc)
{
  acc = f_add(acc, u.x); u.x = acc;
  acc = f_add(acc, u.y); u.y = acc;
  acc = f_add(acc, u.z); u.z = acc;
  acc = f_add(acc, u.w); u.w = acc;
  acc = f_add(acc, v.x); v.x = acc;
  acc = f_add(acc, v.y); v.y = acc;
  acc = f_add(acc, v.z); v.z = acc;
  acc = f_add(acc, v.w); v.w = acc;
}

// Sequential in-place running sum: acc = acc + buf[i]; buf[i] = acc (one rounding per step, the order of
// the reference's recurrences).  The next 8 inputs are always in flight while 8 dependent adds retire, so
// the loop runs at the FADD dependency latency.  May READ up to 16 floats past buf[n-1] (callers pad).
__device__ __forceinline__ void chain_inplace(float* buf, int n, float& acc)
{
  int i = 0;
  if (n >= 16) {
    float4 a0 = *reinterpret_cast<const float4*>(buf), a1 = *reinterpret_cast<const float4*>(buf + 4);
    for (; i + 16 <= n; i += 16) {
      float4 b0 = *reinterpret_cast<const float4*>(buf + i + 8), b1 = *reinterpret_cast<const float4*>(buf + i + 12);
      chain8(a0, a1, acc);
      *reinterpret_cast<float4*>(buf + i) = a0;
      *reinterpret_cast<float4*>(buf + i + 4) = a1;
      a0 = *reinterpret_cast<const float4*>(buf + i + 16);
      a1 = *reinterpret_cast<const float4*>(buf + i + 20);
      chain8(b0, b1, acc);
      *reinterpret_cast<float4*>(buf + i + 8) = b0;
      *reinterpret_cast<float4*>(buf + i + 12) = b1;
    }
  }
  for (; i < n; i++) {
    acc = f_add(acc, buf[i]);
    buf[i] = acc;
  }
}

// ---- raw sample formats.  Every capture kernel is instantiated for each: its raw stages hold the capture's own elements,
// and every sample is converted to float2 as P1 reads it, so the stages move the capture's bytes and no more.
struct RawFc32 {               // interleaved float32 I, Q (8 B per sample)
  typedef float2 T;
  static constexpr int kBytes = 8;
  static __device__ __forceinline__ float2 cvt(float2 v, float) { return v; }
  static __device__ __forceinline__ float2 ldcs(const float2* p) { return __ldcs(p); }
};
struct RawSc16 {               // interleaved int16 I, Q (UHD "sc16", 4 B per sample): I in the low half-word
  typedef uint32_t T;
  static constexpr int kBytes = 4;
  // ((float)I * scale, (float)Q * scale): one round-to-nearest multiply per component, as np.float32(i) * np.float32(scale)
  // (int16 -> float is exact; I2F measured faster than the exact IADD + FADD form, tests/cuda/sc16_harness.cu)
  static __device__ __forceinline__ float2 cvt(uint32_t v, float scale)
  {
    const int i = (short)(v & 0xFFFFu), q = (int)v >> 16;
    return make_float2(f_mul((float)i, scale), f_mul((float)q, scale));
  }
  static __device__ __forceinline__ uint32_t ldcs(const uint32_t* p) { return __ldcs(p); }
};
// samples per 16-byte TMA granule: a stage starts at a multiple of this absolute sample index
template <class RAW>
__host__ __device__ constexpr int raw_granule() { return 16 / RAW::kBytes; }

// N consecutive sc16 samples stage[st .. st + N) of one lane (st mod 4 the same for the whole warp): the aligned 16-byte
// loads of the words around them, then a shift by st mod 4 words in two select steps (by 2, by 1), so that every stage
// residue takes the vector path.  Reads up to 6 words past the run (the stages have that room: kSc16StagePad).
template <int N>
__device__ __forceinline__ void sc16_run(const uint32_t* stage, int st, uint32_t (&x)[N])
{
  constexpr int NQ = (N + 6) / 4;   // granules covering words st & ~3 .. (st & ~3) + 3 + N
  const int r = st & 3;
  uint32_t w[4 * NQ];
  const uint4* p = reinterpret_cast<const uint4*>(stage + (st & ~3));
#pragma unroll
  for (int j = 0; j < NQ; j++) {
    const uint4 v = p[j];
    w[4 * j] = v.x; w[4 * j + 1] = v.y; w[4 * j + 2] = v.z; w[4 * j + 3] = v.w;
  }
  uint32_t s[N + 1];
#pragma unroll
  for (int j = 0; j < N + 1; j++) s[j] = (r & 2) ? w[j + 2] : w[j];
#pragma unroll
  for (int j = 0; j < N; j++) x[j] = (r & 1) ? s[j + 1] : s[j];
}
constexpr int kSc16StagePad = 8;    // samples of an sc16 raw stage beyond a tile's D*kTT: granule alignment + read-ahead

// raw tile geometry: segment-relative index of the first sample held in the stage buffer (moved down to a 16-byte
// aligned absolute index)
template <int DECIM, class RAW>
__device__ __forceinline__ long long tile_load_start(unsigned long long seg_off, int k)
{
  long long lo = (long long)DECIM * k * kTT - (DECIM - 1);
  if (lo < 0) lo = 0;
  long long abs_lo = (long long)seg_off + lo;
  abs_lo &= ~(long long)(raw_granule<RAW>() - 1);  // 16-byte aligned source
  return abs_lo - (long long)seg_off;
}

// the copy of raw tile k of segment sg (any tile; iq holds n_raw samples)
template <int DECIM, class RAW>
__device__ __forceinline__ void issue_tile_load(const typename RAW::T* iq, unsigned long long n_raw, const rfid_b200_segment& sg,
                                                int k, typename RAW::T* stage, uint64_t* bar)
{
  constexpr int E = raw_granule<RAW>();
  const long long start = tile_load_start<DECIM, RAW>(sg.offset, k);  // may be up to E-1 below the segment
  long long hi = (long long)DECIM * ((long long)k * kTT + kTT - 1);
  if (hi > (long long)sg.length - 1) hi = (long long)sg.length - 1;
  long long count = hi - start + 1;  // samples start..hi
  long long count_al = (count + E - 1) & ~(long long)(E - 1);
  const long long abs_start = (long long)sg.offset + start;
  if ((unsigned long long)(abs_start + count_al) > n_raw) {
    // the rounded-up copy would run past the capture buffer: copy whole granules and fetch the last (at most E-1)
    // samples with plain loads
    count_al = count & ~(long long)(E - 1);
#pragma unroll
    for (int j = 0; j < E - 1; j++)
      if (count_al + j < count) stage[count_al + j] = iq[abs_start + count_al + j];
  }
  const uint32_t bytes = (uint32_t)(count_al * RAW::kBytes);
  mbar_arrive_expect_tx(bar, bytes);
  if (bytes) tma_load_1d(stage, iq + abs_start, bytes, bar);
}

// Tile k >= 1 starts at raw sample D*kTT*k - (D-1) of the segment, moved down to a 16-byte aligned absolute index (by
// r = offset mod E samples, E = raw_granule); tile 0 starts at the segment's first (aligned) sample.  Tiles 1 .. n-1 are
// interior: their last sample D*(k*kTT + kTT-1) exists and the rounded-up copy stays inside the capture, so each is
// `bytes` bytes from src + D*kTT*k.  The other tiles go through issue_tile_load.
template <class T>
struct InteriorTiles {
  const T* src;
  uint32_t bytes;
  int n;
};
template <int DECIM, class RAW>
__device__ __forceinline__ InteriorTiles<typename RAW::T> interior_tiles(const typename RAW::T* iq, unsigned long long n_raw,
                                                                         const rfid_b200_segment& sg, int ntiles)
{
  constexpr int E = raw_granule<RAW>();
  static_assert((DECIM - 1) % E == 0, "interior tiles start on a granule");
  const int r = (int)(sg.offset & (unsigned long long)(E - 1));
  const int span = DECIM * kTT + ((r + E - 1) & ~(E - 1));   // samples copied per interior tile
  InteriorTiles<typename RAW::T> t;
  t.src = iq + sg.offset - (DECIM - 1) - r;
  t.bytes = (uint32_t)(span * RAW::kBytes);
  const long long by_len = ((long long)sg.length - 1 - (long long)DECIM * (kTT - 1)) / ((long long)DECIM * kTT);
  const long long room = (long long)n_raw - (long long)sg.offset + (DECIM - 1) + r - span;
  const long long by_buf = room >= 0 ? room / ((long long)DECIM * kTT) : -1;
  long long f = (by_len < by_buf ? by_len : by_buf) + 1;
  if (sg.length < (unsigned)(DECIM * kTT)) f = 0;
  t.n = f < 0 ? 0 : (f > ntiles ? ntiles : (int)f);
  return t;
}

}  // namespace rfid_b200
