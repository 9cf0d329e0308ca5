// rx_decode.cuh -- one warp decodes one ungated window held in shared memory.
// Replaces tag_decoder_impl::general_work and its helpers
// (reference gr-rfid/lib/tag_decoder_impl.cc:78-193, 223-393, 401-445).
#pragma once

#include "rx_common.cuh"

namespace rfid_b200 {

struct WindowDecode {
  int sync_index;
  float score;
  float2 h;
  float T;
  int crc_ok;
  int tag_id;
  uint32_t bits[4];  // bit j of the message at word j/32, bit position 31 - j%32 (MSB first)
};

// warp argmax with the reference's tie rule: first (lowest index) strict maximum
__device__ __forceinline__ void warp_argmax_first(float& v, int& idx)
{
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    float ov = __shfl_xor_sync(0xffffffffu, v, off);
    int oi = __shfl_xor_sync(0xffffffffu, idx, off);
    bool take = (ov > v) || (ov == v && oi < idx);
    v = take ? ov : v;
    idx = take ? oi : idx;
  }
}

// CRC-16/CCITT (poly 0x1021, init 0xFFFF, final complement) over the first 14 bytes = what check_crc computes bit
// by bit (tag_decoder_impl.cc:424-440), here a byte per step with the standard shift/xor identity for this polynomial
__device__ __forceinline__ int crc16_check(const uint32_t bits[4])
{
  unsigned crc = 0xFFFF;
#pragma unroll
  for (int i = 0; i < 14; i++) {
    const unsigned byte = (bits[i >> 2] >> (24 - 8 * (i & 3))) & 0xFFu;
    unsigned x = ((crc >> 8) ^ byte) & 0xFFu;
    x ^= x >> 4;
    crc = ((crc << 8) ^ (x << 12) ^ (x << 5) ^ x) & 0xFFFFu;
  }
  crc = (~crc) & 0xFFFFu;
  unsigned rcvd = bits[3] & 0xFFFFu;  // bytes 14,15
  return rcvd == crc ? 1 : 0;
}

// ---------------------------------------------------------------------------------------------------------
// The decoder of one window (tag_decoder_impl.cc:78-191, 223-393), ONE copy for every kernel: the window lives in global
// memory (a capture kernel's L2-resident scratch / history, or the block-mode input buffer); the warp copies the part of
// the window it is about to use into a small shared-memory stage with coalesced loads and gathers from there.
// w = y - dc_est: dc is subtracted as the samples are loaded (one exact float subtraction, gate_impl.cc:173,187).
// All 32 lanes of the warp must call; the result is valid in every lane.  The stage must hold the window head (sync range +
// 6 symbols); with room for a chunk of the symbol-period search the search runs from the stage, else it gathers from L2.
__host__ __device__ inline int decode_stage_samples(float n_tag_bit)
{
  // one chunk = 32 consecutive bit pairs: 31 symbols + one half symbol at the longest candidate period, + slack
  return ((int)(32.5f * n_tag_bit * 1.0101f) + 16 + 7) & ~7;
}

// `progress` (may be null): number of window samples the producer has published so far; the fill waits until
// the range it is about to read exists.  This is what lets the decoder work on a window WHILE it is still being
// gated (streaming decode), instead of starting when the window closes.
#ifndef RFID_B200_PROGRESS_NS
#define RFID_B200_PROGRESS_NS 300
#endif
// How the decoder waits for window samples that are still being gated: `counter` = samples published so far.  With a
// doorbell (an mbarrier the producer arrives on after every publication) the waiting warp is parked by the hardware;
// without one it polls the counter with a sleep in between.  The counter, not the doorbell's phase, decides: every wait
// is bounded (suspend hint), so a phase that was rung before the warp looked only costs one time-out.
struct ProgressWait {
  const volatile int* counter;
  uint64_t* bell;
  uint32_t seen;
};
__device__ __forceinline__ void progress_wait(ProgressWait* pw, int need)
{
  if (!pw || !pw->counter) return;
  while (*pw->counter < need) {
    if (pw->bell) { if (mbar_try_wait_hint(pw->bell, pw->seen & 1u, 2000)) pw->seen++; }
    else __nanosleep(RFID_B200_PROGRESS_NS);
  }
  asm volatile("fence.acq_rel.cta;" ::: "memory");  // the samples were written (and fenced, CTA scope) before the counter moved
}

// dc: subtracted from every sample as it is staged (x - (+0.0f) == x for every x, so the default changes nothing).
// All loads of a fill are issued before the first store (kFillBatch per lane): the fill costs one trip to L2, not one per
// 32 samples.
// Where a window lives in global memory: sample g of the window is base[(ofs + g) & mask].  mask = -1: a plain array; the
// pack kernel's windows lie in a circular per-segment history of y (mask = its size - 1, ofs = the window's first sample).
struct WinSrc {
  const float2* base;
  int ofs, mask;
  __device__ __forceinline__ const float2* at(int g) const { return base + ((ofs + g) & mask); }
};
constexpr int kFillBatch = 12;
__device__ __forceinline__ float2 ld_ca_f2(const float2* p)
{
  float2 v;
  asm volatile("ld.global.ca.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "l"(p));
  return v;
}
// touch the cache lines of window samples [lo, lo + count) (clamped to the window): lane l loads one word of line l.
// Returns a value the caller must keep alive (asm volatile("" :: "f"(x))) until it no longer minds waiting for the loads.
__device__ __forceinline__ float l1_touch_span(const WinSrc gw, int lo, int count, int n_avail)
{
  const int lane = threadIdx.x & 31;
  const int first = max(lo, 0), last = min(lo + count, n_avail) - 1;   // samples; a line holds 16 of them
  float d = 0.0f;
  const int smp = min(first + 16 * lane, last);
  if (last >= first && first + 16 * lane < last + 16) asm volatile("ld.global.ca.f32 %0, [%1];" : "=f"(d) : "l"(gw.at(smp)));
  return d;
}
__device__ __forceinline__ void stage_fill(float2* stage, const WinSrc gw, int lo, int count, int n_avail,
                                           ProgressWait* progress = nullptr, float2 dc = make_float2(0.f, 0.f))
{
  const int lane = threadIdx.x & 31;
  __syncwarp();
  progress_wait(progress, min(n_avail, lo + count));
  for (int p0 = 0; p0 < count; p0 += 32 * kFillBatch) {
    float2 v[kFillBatch];
#pragma unroll
    for (int k = 0; k < kFillBatch; k++) {
      const int p = p0 + 32 * k + lane, g = lo + p;
      v[k] = (p < count && g >= 0 && g < n_avail) ? __ldcg(gw.at(g)) : make_float2(0.f, 0.f);
    }
#pragma unroll
    for (int k = 0; k < kFillBatch; k++) {
      const int p = p0 + 32 * k + lane, g = lo + p;
      if (p < count) stage[p] = (g >= 0 && g < n_avail) ? c_sub(v[k], dc) : make_float2(0.f, 0.f);
    }
  }
  __syncwarp();
}

// same, storing |w|^2 (std::norm: re*re + im*im, separately rounded) instead of the sample
// L1: load through the SM's L1 (ld.global.ca) instead of L2 only -- for callers that touched the lines beforehand
template <bool L1 = false>
__device__ __forceinline__ void stage_fill_norm(float* stage_m, const WinSrc gw, int lo, int count, int n_avail,
                                                ProgressWait* progress = nullptr, float2 dc = make_float2(0.f, 0.f))
{
  const int lane = threadIdx.x & 31;
  __syncwarp();
  progress_wait(progress, min(n_avail, lo + count));
  for (int p0 = 0; p0 < count; p0 += 32 * kFillBatch) {
    float2 v[kFillBatch];
#pragma unroll
    for (int k = 0; k < kFillBatch; k++) {
      const int p = p0 + 32 * k + lane, g = lo + p;
      v[k] = (p < count && g >= 0 && g < n_avail) ? (L1 ? ld_ca_f2(gw.at(g)) : __ldcg(gw.at(g))) : make_float2(0.f, 0.f);
    }
#pragma unroll
    for (int k = 0; k < kFillBatch; k++) {
      const int p = p0 + 32 * k + lane, g = lo + p;
      if (p < count) stage_m[p] = (g >= 0 && g < n_avail) ? c_norm(c_sub(v[k], dc)) : 0.0f;
    }
  }
  __syncwarp();
}

// Whole window present (nobody to wait for): optionally touch the span's cache lines (L2 -> this SM's L1, one load per
// lane), then fill in rolled batches of four loads per lane through L1.  Small code, and one trip to L2 per fill.  The
// window was written by this SM before the decode began; an SM's own stores keep its L1 coherent.
template <bool NORM>
__device__ __forceinline__ void stage_fill_l1(void* stage_v, const WinSrc gw, int lo, int count, int n_avail, float2 dc, bool touch)
{
  const int lane = threadIdx.x & 31;
  __syncwarp();
  float sink = 0.0f;
  if (touch) sink = l1_touch_span(gw, lo, count, n_avail);
#pragma unroll 1
  for (int p0 = 0; p0 < count; p0 += 128) {
    float2 v[4];
#pragma unroll
    for (int k = 0; k < 4; k++) {
      const int p = p0 + 32 * k + lane, g = lo + p;
      v[k] = (p < count && g >= 0 && g < n_avail) ? ld_ca_f2(gw.at(g)) : make_float2(0.f, 0.f);
    }
#pragma unroll
    for (int k = 0; k < 4; k++) {
      const int p = p0 + 32 * k + lane, g = lo + p;
      const bool in = g >= 0 && g < n_avail;
      if (p < count) {
        if (NORM) reinterpret_cast<float*>(stage_v)[p] = in ? c_norm(c_sub(v[k], dc)) : 0.0f;
        else reinterpret_cast<float2*>(stage_v)[p] = in ? c_sub(v[k], dc) : make_float2(0.f, 0.f);
      }
    }
  }
  asm volatile("" ::"f"(sink));
  __syncwarp();
}

// ---- the staged decode as a resumable sequence of phases ---------------------------------------------------------------
// head (tag_sync, h_est, tag_decoder_impl.cc:78-109) -> kSearchChunks chunks of the symbol-period search (:151-165) ->
// finish (argmax, 128 bit decisions :171-191, CRC).  Each phase needs the window only up to a known position, so a
// caller that is still receiving the window (rx_pack.cuh: warp C copies it tile by tile) runs the phases as the samples
// arrive; decode_window_staged below runs them back to back.  One copy of the arithmetic either way.
constexpr int kChunkSteps = 64;                       // steps of the symbol-period search per phase (one stage fill each)
constexpr int kSearchChunks = 256 / kChunkSteps;
struct WinStream {
  int phase;     // 0: head pending, 1..kSearchChunks: search chunk (phase - 1) pending, kSearchChunks + 1: search complete
  int index;     // first data sample: sync index + 6.5 symbols (:107)
  int head;      // samples the head staged (an RN16 window is staged whole)
  float e;       // this lane's running energy of candidate period `lane` (lanes 0..19)
  float Tt;      // this lane's candidate period
  float2 h;
};

// lane t's candidate period of the symbol-period search, t_min + t (t_max - t_min) / 19 (:151-156; lanes 20..31 carry
// t_min and are never read).  A caller that resumes a search from saved state recomputes it with this.
__device__ __forceinline__ float win_stream_period(const RxConfig& c, int lane)
{
  const int number_steps = 20;
  return f_add(c.t_min, f_div(f_mul((float)(lane < number_steps ? lane : 0), f_sub(c.t_max, c.t_min)), (float)(number_steps - 1)));
}

__device__ __forceinline__ int win_head_samples(const RxConfig& c, int kind, int n_total, int stage_cap)
{
  return min(stage_cap, kind == RFID_B200_RN16 ? n_total : (int)(c.sync_range + 6.0f * c.n_tag_bit_f) + 2);
}

// window samples a search chunk reads (exclusive upper bound, clamped to the window)
__device__ __forceinline__ int win_chunk_need(const RxConfig& c, const WinStream& S, int chunk, int n_total, int stage_cap)
{
  const int span = min(2 * stage_cap, (int)((float)kChunkSteps * c.t_max + 256.0f * (c.t_max - c.t_min)) + 8);
  const int lo = (int)f_add(f_mul((float)(kChunkSteps * chunk), c.t_min), (float)S.index);
  return min(n_total, lo + span);
}

// tag_sync + h_est; fills sync_index / score / h of `out` and the stream state.  progress = null: the whole window is
// present, the head is loaded through L1.  A ProgressWait without a counter: the head's samples are present but the
// window is still being written -- the head is loaded through L2 only, so that L1 keeps no line of the unwritten part.
__device__ __forceinline__ void win_stream_head(const RxConfig& c, int kind, const WinSrc gw, int n_total,
                                                float2* __restrict__ stage, int stage_cap, float2 dc, WinStream& S,
                                                WindowDecode& out, ProgressWait* progress = nullptr)
{
  const int lane = threadIdx.x & 31;
  const float n = c.n_tag_bit_f;
  const float half = f_mul(n, 0.5f);   // (x / 2 == x * 0.5 exactly, every x)
  const int head = win_head_samples(c, kind, n_total, stage_cap);
  if (progress) stage_fill(stage, gw, 0, head, n_total, progress, dc);
  else stage_fill_l1<false>(stage, gw, 0, head, n_total, dc, true);
  // (whole window present: start the first search chunk's lines towards L1 now; it begins 6.5 symbols after the sync index)
  float sink = 0.0f;
  if (!progress && kind != RFID_B200_RN16) sink = l1_touch_span(gw, (int)(6.5f * n), 32 * 16, n_total);
  float best = -1.0f;
  int best_i = 0x7fffffff;
  for (int i = lane; i < c.sync_range; i += 32) {
    float2 acc = make_float2(0.0f, 0.0f);
#pragma unroll 2
    for (int j = 0; j < 2 * kTagPreambleBits; j++) {
      int k = (int)f_add((float)i, f_mul(f_mul((float)j, n), 0.5f));
      float2 s = stage[k];
      float cr = (float)((kPreambleMask >> j) & 1u);
      float pr = f_sub(f_mul(s.x, cr), f_mul(s.y, 0.0f));
      float pi = f_add(f_mul(s.x, 0.0f), f_mul(s.y, cr));
      acc.x = f_add(acc.x, pr);
      acc.y = f_add(acc.y, pi);
    }
    float corr = c_norm(acc);
    if (corr > best) { best = corr; best_i = i; }
  }
  warp_argmax_first(best, best_i);
  int max_index = 0;
  float max_corr = 0.0f;
  if (best > 0.0f) { max_index = best_i; max_corr = best; }
  {
    int t1 = (int)f_add((float)max_index, half);
    int t3 = (int)f_add((float)max_index, f_mul(f_mul(3.0f, n), 0.5f));
    int t6 = (int)f_add((float)max_index, f_mul(f_mul(6.0f, n), 0.5f));
    int t10 = (int)f_add((float)max_index, f_mul(f_mul(10.0f, n), 0.5f));
    int t11 = (int)f_add((float)max_index, f_mul(f_mul(11.0f, n), 0.5f));
    float2 s = stage[max_index];
    s = c_add(s, stage[t1]);
    s = c_add(s, stage[t3]);
    s = c_add(s, stage[t6]);
    s = c_add(s, stage[t10]);
    s = c_add(s, stage[t11]);
    out.h = make_float2(f_div(s.x, 6.0f), f_div(s.y, 6.0f));
  }
  out.sync_index = max_index;
  out.score = max_corr;
  out.bits[0] = out.bits[1] = out.bits[2] = out.bits[3] = 0u;
  S.index = (int)f_add(f_add((float)max_index, f_mul((float)kTagPreambleBits, n)), half);
  S.head = head;
  S.h = out.h;
  S.e = 0.0f;
  S.Tt = win_stream_period(c, lane);
  S.phase = 1;
  asm volatile("" ::"f"(sink));
}

// kChunkSteps steps of the symbol-period search: E_t += M[(int)(i * T_t + index)], i ascending
__device__ __forceinline__ void win_stream_chunk(const RxConfig& c, const WinSrc gw, int n_total,
                                                 float2* __restrict__ stage, int stage_cap, float2 dc, WinStream& S,
                                                 ProgressWait* progress = nullptr)
{
  const int lane = threadIdx.x & 31;
  const int number_steps = 20;
  const int chunk = S.phase - 1;
  const int i0 = kChunkSteps * chunk;
  // Only |w|^2 is needed here (magn_squared_samples, gate_impl.cc:176,186), so the stage holds one float per sample.
  float* stage_m = reinterpret_cast<float*>(stage);
  const int span = min(2 * stage_cap, (int)((float)kChunkSteps * c.t_max + 256.0f * (c.t_max - c.t_min)) + 8);
  const int lo = (int)f_add(f_mul((float)i0, c.t_min), (float)S.index);  // smallest index any candidate touches
  stage_fill_norm(stage_m, gw, lo, span, n_total, progress, dc);
  if (lane < number_steps) {
    const float findex = (float)S.index, Tt = S.Tt;
    float fi = (float)i0;                          // (float)i, advanced by exact +1.0f steps
    float e = S.e;
#pragma unroll 8
    for (int i = i0; i < i0 + kChunkSteps; i++) {
      const int p = (int)f_add(f_mul(fi, Tt), findex);  // (int)(i * T + index), :161; fi == (float)i exactly
      e = f_add(e, stage_m[p - lo]);
      fi = f_add(fi, 1.0f);
    }
    S.e = e;
  }
  S.phase++;
}

// EPC, the symbol-period search complete: argmax, 128 bit decisions, CRC-16 (the end of win_stream_finish)
__device__ __forceinline__ void win_stream_decide(const RxConfig& c, const WinSrc gw, int n_avail, float2* __restrict__ stage,
                                                  int stage_cap, float2 dc, const WinStream& S, WindowDecode& out,
                                                  ProgressWait* progress = nullptr, long long* pp = nullptr)
{
  const int lane = threadIdx.x & 31;
  const int index = S.index;
  const float2 h = S.h;
  if (pp && lane == 0) pp[2] = clock64();
  const int number_steps = 20;
  const float min_val = c.t_min, max_val = c.t_max;
  float energy = lane < number_steps ? S.e : -1.0f;
  int e_idx = lane < number_steps ? lane : 0x7fffffff;
  warp_argmax_first(energy, e_idx);
  const int index_T = e_idx;
  const float T = f_add(min_val, f_div(f_mul((float)index_T, f_sub(max_val, min_val)), (float)(number_steps - 1)));
  out.T = T;
  // ---- 128 bit decisions (:171-191), 32 pairs per stage fill
  const float twoT = f_mul(2.0f, T);
  unsigned Sg[4];
  if (!progress) {
    // the whole window is present: every lane gathers its eight samples straight from L2, all loads in flight together
    float2 wa[4], wb[4];
#pragma unroll
    for (int r = 0; r < 4; r++) {
      const int j = r * 32 + lane;
      const int a = (int)f_add(f_mul((float)j, twoT), (float)index);
      const int b = (int)f_add(f_add(f_mul((float)(j * 2), T), T), (float)index);
      const bool ia = a >= 0 && a < n_avail, ib = b >= 0 && b < n_avail;   // (outside the window: 0, as the stage fill does)
      wa[r] = ia ? __ldcg(gw.at(a)) : dc;
      wb[r] = ib ? __ldcg(gw.at(b)) : dc;
    }
#pragma unroll
    for (int r = 0; r < 4; r++) {
      const int j = r * 32 + lane;
      const int a = (int)f_add(f_mul((float)j, twoT), (float)index);
      const int b = (int)f_add(f_add(f_mul((float)(j * 2), T), T), (float)index);
      const float2 sa = (a >= 0 && a < n_avail) ? c_sub(wa[r], dc) : make_float2(0.f, 0.f);
      const float2 sb = (b >= 0 && b < n_avail) ? c_sub(wb[r], dc) : make_float2(0.f, 0.f);
      const float res = c_proj(sa, sb, h);
      Sg[r] = __ballot_sync(0xffffffffu, res > 0.0f);
    }
  } else {
#pragma unroll
    for (int r = 0; r < 4; r++) {
      const int j0 = r * 32;
      const int lo = (int)f_add(f_mul((float)j0, twoT), (float)index);
      stage_fill(stage, gw, lo, stage_cap, n_avail, progress, dc);
      int j = j0 + lane;
      int a = (int)f_add(f_mul((float)j, twoT), (float)index);
      int b = (int)f_add(f_add(f_mul((float)(j * 2), T), T), (float)index);
      float res = c_proj(stage[a - lo], stage[b - lo], h);
      Sg[r] = __ballot_sync(0xffffffffu, res > 0.0f);
    }
  }
  if (pp && lane == 0) pp[3] = clock64();
  unsigned carry = 1u;
#pragma unroll
  for (int r = 0; r < 4; r++) {
    unsigned prev = (Sg[r] << 1) | carry;
    carry = Sg[r] >> 31;
    unsigned Bv = Sg[r] ^ prev;
    out.bits[r] = __brev(Bv);
  }
  out.crc_ok = crc16_check(out.bits);
  out.tag_id = (int)((out.bits[3] >> 16) & 0xFFu);
  if (pp && lane == 0) pp[4] = clock64();
}

// RN16: half-bit sampling + tag_detection_RN16 (:114-142, :237-253); EPC: remaining search chunks, argmax, 128 bit
// decisions, CRC-16.  The whole window must be present.
__device__ __forceinline__ void win_stream_finish(const RxConfig& c, int kind, const WinSrc gw, int n_avail,
                                                  float2* __restrict__ stage, int stage_cap, float2 dc, WinStream& S,
                                                  WindowDecode& out, ProgressWait* progress = nullptr, long long* pp = nullptr)
{
  const int lane = threadIdx.x & 31;
  const float n = c.n_tag_bit_f;
  const float half = f_mul(n, 0.5f);
  const int index = S.index;
  const float2 h = S.h;
  if (kind == RFID_B200_RN16) {
    float jm = (float)index;
    for (int m = 0; m < lane; m++) jm = f_add(jm, half);
    bool have = jm < (float)n_avail;
    unsigned have_mask = __ballot_sync(0xffffffffu, have);
    float2 s = make_float2(0.0f, 0.0f);
    if (have) {
      const int k = (int)roundf(jm);
      s = k < S.head ? stage[k] : c_sub(__ldcg(gw.at(k)), dc);
    }
    out.T = 0.0f;
    out.crc_ok = -1;
    if (have_mask == 0xffffffffu) {
      float2 s_next = make_float2(__shfl_down_sync(0xffffffffu, s.x, 1), __shfl_down_sync(0xffffffffu, s.y, 1));
      float res = c_proj(s, s_next, h);
      unsigned pos = __ballot_sync(0xffffffffu, res > 0.0f);
      unsigned Sg = 0;
#pragma unroll
      for (int j = 0; j < 16; j++) Sg |= ((pos >> (2 * j)) & 1u) << j;
      unsigned Bv = (Sg ^ ((Sg << 1) | 1u)) & 0xFFFFu;
      unsigned msb = 0;
#pragma unroll
      for (int j = 0; j < 16; j++) msb |= ((Bv >> j) & 1u) << (31 - j);
      out.bits[0] = msb;
      out.tag_id = (int)(msb >> 16);
    } else {
      out.crc_ok = -2;
      out.tag_id = -1;
    }
    if (pp && lane == 0) { pp[2] = pp[3] = pp[4] = clock64(); }
    return;
  }
  if (!progress) {
    // ---- remaining chunks of the symbol-period search, whole window present (nobody to wait for): while chunk k's 64
    // steps run from the stage, chunk k+1's samples travel from L2 into registers; 16 gathers in flight, added in order.
    // (Tried: all 32 lanes gathering 16 steps x 20 candidates into a table that lane t then adds up in order -- fewer
    // instructions, but slower than the plain loop below: 19.6 k vs 15.6 k cycles per window.)
    float* stage_m = reinterpret_cast<float*>(stage);
    const int span_full = (int)((float)kChunkSteps * c.t_max + 256.0f * (c.t_max - c.t_min)) + 8;
    const int span = min(2 * stage_cap, span_full);
    if (span_full > 2 * stage_cap || span > 32 * kFillBatch) {
      // the stage holds the head only (kernels whose shared memory is spoken for), or a chunk is longer than one load
      // batch: |w|^2 straight from global memory, eight gathers in flight, added in order
      if (lane < 20) {
        const float findex = (float)index, Tt = S.Tt;
        float e = S.e;
#pragma unroll 1
        for (int i = kChunkSteps * (S.phase - 1); i < kChunkSteps * kSearchChunks; i += 8) {
          const float fi = (float)i;
          float2 g8[8];
          bool in8[8];
#pragma unroll
          for (int u = 0; u < 8; u++) {
            const int p = (int)f_add(f_mul(f_add(fi, (float)u), Tt), findex);  // (int)(i * T + index), :161
            in8[u] = p >= 0 && p < n_avail;
            g8[u] = in8[u] ? __ldcg(gw.at(p)) : dc;
          }
#pragma unroll
          for (int u = 0; u < 8; u++) e = f_add(e, in8[u] ? c_norm(c_sub(g8[u], dc)) : 0.0f);
        }
        S.e = e;
      }
      S.phase = kSearchChunks + 1;
    } else {
      // chunk k+1's samples travel from L2 into registers while chunk k's 64 steps run from the stage
      float2 v[kFillBatch];
      int lo = (int)f_add(f_mul((float)(kChunkSteps * (S.phase - 1)), c.t_min), (float)index);
      auto issue = [&](int lo_) {
#pragma unroll
        for (int k = 0; k < kFillBatch; k++) {
          const int p = 32 * k + lane, g = lo_ + p;
          v[k] = (p < span && g >= 0 && g < n_avail) ? __ldcg(gw.at(g)) : make_float2(0.f, 0.f);
        }
      };
      issue(lo);
      while (S.phase <= kSearchChunks) {
        const int i0 = kChunkSteps * (S.phase - 1);
        __syncwarp();  // the previous chunk's reads of the stage are complete
#pragma unroll
        for (int k = 0; k < kFillBatch; k++) {
          const int p = 32 * k + lane, g = lo + p;
          if (p < span) stage_m[p] = (g >= 0 && g < n_avail) ? c_norm(c_sub(v[k], dc)) : 0.0f;
        }
        __syncwarp();
        const float* sm = stage_m - lo;
        if (S.phase < kSearchChunks) {
          lo = (int)f_add(f_mul((float)(i0 + kChunkSteps), c.t_min), (float)index);
          issue(lo);
        }
        if (lane < 20) {
          const float findex = (float)index, Tt = S.Tt;
          float e = S.e;
#pragma unroll 1
          for (int i = i0; i < i0 + kChunkSteps; i += 16) {
            // sixteen gathers in flight, then their sixteen additions in order
            const float fi = (float)i;
            float u16[16];
#pragma unroll
            for (int u = 0; u < 16; u++) u16[u] = sm[(int)f_add(f_mul(f_add(fi, (float)u), Tt), findex)];  // (int)(i * T + index), :161
#pragma unroll
            for (int u = 0; u < 16; u++) e = f_add(e, u16[u]);
          }
          S.e = e;
        }
        S.phase++;
      }
      __syncwarp();
    }
  } else {
    while (S.phase <= kSearchChunks) win_stream_chunk(c, gw, n_avail, stage, stage_cap, dc, S, progress);
  }
  win_stream_decide(c, gw, n_avail, stage, stage_cap, dc, S, out, progress, pp);
}

__device__ __forceinline__ void decode_window_staged(const RxConfig& c, int kind, const WinSrc gw, int n_avail,
                                                     float2* __restrict__ stage, int stage_cap, WindowDecode& out,
                                                     const volatile int* progress_counter = nullptr, uint64_t* bell = nullptr,
                                                     float2 dc = make_float2(0.f, 0.f), long long* pp = nullptr)
{
  ProgressWait pw_{progress_counter, bell, 0u};
  ProgressWait* const progress = progress_counter ? &pw_ : nullptr;
  WinStream S;
  if (pp && (threadIdx.x & 31) == 0) pp[0] = clock64();
  win_stream_head(c, kind, gw, n_avail, stage, stage_cap, dc, S, out, progress);
  if (pp && (threadIdx.x & 31) == 0) pp[1] = clock64();
  win_stream_finish(c, kind, gw, n_avail, stage, stage_cap, dc, S, out, progress, pp);
}

__device__ __forceinline__ void decode_window_staged(const RxConfig& c, int kind, const float2* __restrict__ w, int n_avail,
                                                     float2* __restrict__ stage, int stage_cap, WindowDecode& out,
                                                     const volatile int* progress_counter = nullptr, uint64_t* bell = nullptr,
                                                     float2 dc = make_float2(0.f, 0.f))
{
  decode_window_staged(c, kind, WinSrc{w, 0, -1}, n_avail, stage, stage_cap, out, progress_counter, bell, dc);
}

__device__ __forceinline__ void store_result(rfid_b200_window_result* dst, const WindowDecode& d, int segment, int window,
                                             int open_index, int length, int kind)
{
  // one lane writes the 64-byte record as four 16-byte stores
  int4 q0 = make_int4(segment, window, open_index, length);
  int4 q1 = make_int4(kind, d.sync_index, __float_as_int(d.score), __float_as_int(d.h.x));
  int4 q2 = make_int4(__float_as_int(d.h.y), __float_as_int(d.T), d.crc_ok, d.tag_id);
  // bits[]: byte k = message bits 8k..8k+7, MSB first => big-endian words
  int4 q3 = make_int4((int)__byte_perm(d.bits[0], 0, 0x0123), (int)__byte_perm(d.bits[1], 0, 0x0123),
                      (int)__byte_perm(d.bits[2], 0, 0x0123), (int)__byte_perm(d.bits[3], 0, 0x0123));
  int4* p = reinterpret_cast<int4*>(dst);
  p[0] = q0;
  p[1] = q1;
  p[2] = q2;
  p[3] = q3;
}

}  // namespace rfid_b200
