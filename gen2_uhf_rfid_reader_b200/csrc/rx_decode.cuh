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
// the window it is about to gather from many times into a small shared-memory stage with coalesced loads and gathers from
// there; the 256 samples of the bit decisions are gathered from L2 directly.
// w = y - dc_est: dc is subtracted as the samples are loaded (one exact float subtraction, gate_impl.cc:173,187).
// All 32 lanes of the warp must call; the result is valid in every lane.  The stage must hold the window head (sync range +
// 6 symbols); with room for a chunk of the symbol-period search the search runs from the stage, else it gathers from L2
// (win_stream_chunk).

// `progress` (may be null): how the decoder waits for window samples that are still being gated.  `counter` = number of
// window samples the producer has published so far; a reader polls it, with a sleep in between, until the range it is
// about to read exists.  This is what lets the decoder work on a window WHILE it is still being gated (streaming decode),
// instead of starting when the window closes.
constexpr unsigned kProgressPollNs = 300;
struct ProgressWait {
  const volatile int* counter;
};
__device__ __forceinline__ void progress_wait(const ProgressWait* pw, int need)
{
  if (!pw || !pw->counter) return;
  while (*pw->counter < need) __nanosleep(kProgressPollNs);
  asm volatile("fence.acq_rel.cta;" ::: "memory");  // the samples were written (and fenced, CTA scope) before the counter moved
}

// dc: subtracted from every sample as it is staged (x - (+0.0f) == x for every x: a window that holds w already passes 0).
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
                                           const ProgressWait* progress, float2 dc)
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

// same, storing |w|^2 (std::norm: re*re + im*im, separately rounded) instead of the sample; the range must be present
__device__ __forceinline__ void stage_fill_norm(float* stage_m, const WinSrc gw, int lo, int count, int n_avail, float2 dc)
{
  const int lane = threadIdx.x & 31;
  __syncwarp();
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
      if (p < count) stage_m[p] = (g >= 0 && g < n_avail) ? c_norm(c_sub(v[k], dc)) : 0.0f;
    }
  }
  __syncwarp();
}

// Whole window present (nobody to wait for): optionally touch the span's cache lines (L2 -> this SM's L1, one load per
// lane), then fill in rolled batches of four loads per lane through L1.  Small code, and one trip to L2 per fill.  The
// window was written by this SM before the decode began; an SM's own stores keep its L1 coherent.
__device__ __forceinline__ void stage_fill_l1(float2* stage, const WinSrc gw, int lo, int count, int n_avail, float2 dc, bool touch)
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
      if (p < count) stage[p] = (g >= 0 && g < n_avail) ? c_sub(v[k], dc) : make_float2(0.f, 0.f);
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
constexpr int kChunkSteps = 64;                       // steps of the symbol-period search per phase
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

// The decoder's sample positions, shared with the window-quality kernel (rx_quality.cuh), which projects the same samples.
// First data sample: sync index + 6.5 symbols (:107).
__device__ __forceinline__ int win_data_index(const RxConfig& c, int sync_index)
{
  const float n = c.n_tag_bit_f;
  return (int)f_add(f_add((float)sync_index, f_mul((float)kTagPreambleBits, n)), f_mul(n, 0.5f));
}
// RN16 half-bit m (:237-253): the float position index + half + ... + half (m additions, each rounded); the sample is
// roundf of it.  win_stream_finish writes the same loop out.
__device__ __forceinline__ float win_rn16_halfbit(int index, float half, int m)
{
  float jm = (float)index;
  for (int i = 0; i < m; i++) jm = f_add(jm, half);
  return jm;
}
// EPC bit j's pair (:173): a = (int)(j * (2T) + index), b = (int)(j * 2 * T + T + index)
__device__ __forceinline__ int win_epc_pos_a(int j, float twoT, int index) { return (int)f_add(f_mul((float)j, twoT), (float)index); }
__device__ __forceinline__ int win_epc_pos_b(int j, float T, int index)
{
  return (int)f_add(f_add(f_mul((float)(j * 2), T), T), (float)index);
}

__device__ __forceinline__ int win_head_samples(const RxConfig& c, int kind, int n_total, int stage_cap)
{
  return min(stage_cap, kind == RFID_B200_RN16 ? n_total : (int)(c.sync_range + 6.0f * c.n_tag_bit_f) + 2);
}

// Samples a search chunk reads, from the smallest index any candidate touches in it (win_chunk_lo): kChunkSteps steps at
// the longest candidate period, plus how far the longest candidate has drifted from the shortest by the last chunk, plus
// slack.  Also the host's decoder-stage rule (rfid_b200.cu), so host and device agree on which stages hold a chunk.
__host__ __device__ inline int win_chunk_span(const RxConfig& c)
{
  return (int)((float)kChunkSteps * c.t_max + 256.0f * (c.t_max - c.t_min)) + 8;
}
__device__ __forceinline__ int win_chunk_lo(const RxConfig& c, int index, int chunk)
{
  return (int)f_add(f_mul((float)(kChunkSteps * chunk), c.t_min), (float)index);
}

// window samples a search chunk reads (exclusive upper bound, clamped to the window)
__device__ __forceinline__ int win_chunk_need(const RxConfig& c, int index, int chunk, int n_total)
{
  return min(n_total, win_chunk_lo(c, index, chunk) + win_chunk_span(c));
}

// tag_sync + h_est; fills sync_index / score / h of `out` and the stream state.  progress = null: the whole window is
// present, the head is loaded through L1.  A ProgressWait without a counter: the head's samples are present but the
// window is still being written -- the head is loaded through L2 only, so that L1 keeps no line of the unwritten part.
__device__ __forceinline__ void win_stream_head(const RxConfig& c, int kind, const WinSrc gw, int n_total,
                                                float2* __restrict__ stage, int stage_cap, float2 dc, WinStream& S,
                                                WindowDecode& out, const ProgressWait* progress = nullptr)
{
  const int lane = threadIdx.x & 31;
  const float n = c.n_tag_bit_f;
  const float half = f_mul(n, 0.5f);   // (x / 2 == x * 0.5 exactly, every x)
  const int head = win_head_samples(c, kind, n_total, stage_cap);
  if (progress) stage_fill(stage, gw, 0, head, n_total, progress, dc);
  else stage_fill_l1(stage, gw, 0, head, n_total, dc, true);
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
  S.index = win_data_index(c, max_index);
  S.head = head;
  S.h = out.h;
  S.e = 0.0f;
  S.Tt = win_stream_period(c, lane);
  S.phase = 1;
  asm volatile("" ::"f"(sink));
}

// One chunk (kChunkSteps steps) of the symbol-period search: E_t += M[(int)(i * T_t + index)], i ascending, eight gathers
// in flight and then their eight additions in order.  Only M = |w|^2 is needed (magn_squared_samples,
// gate_impl.cc:176,186).  STAGED: the kernel's stage holds a chunk's span at one float per sample (rfid_b200.cu,
// chunk_stage_samples); it is filled with M and the steps gather from there.  Else (rx_fused_kernel, whose stage holds
// the head only) the steps gather the samples straight from L2.  The source is fixed per kernel at compile time: a kernel
// that carries both loops pays in registers for the one it never runs (spills in its other roles; rx_fused_kernel took
// 2-5 % longer at 4-8 MS/s on an H100 SXM at a 400 W power limit).
template <bool STAGED>
__device__ __forceinline__ void win_stream_chunk(const RxConfig& c, const WinSrc gw, int n_total,
                                                 float2* __restrict__ stage, int stage_cap, float2 dc, WinStream& S,
                                                 const ProgressWait* progress = nullptr)
{
  const int lane = threadIdx.x & 31;
  const int number_steps = 20;
  const int i0 = kChunkSteps * (S.phase - 1);
  const int span = win_chunk_span(c);
  const int lo = win_chunk_lo(c, S.index, S.phase - 1);
  float* stage_m = reinterpret_cast<float*>(stage);
  progress_wait(progress, min(n_total, lo + span));
  if (STAGED) {
    if (span > 2 * stage_cap) __trap();   // a stage below the host's rule: fail rather than read stale entries
    stage_fill_norm(stage_m, gw, lo, span, n_total, dc);
  }
  if (lane < number_steps) {
    const float findex = (float)S.index, Tt = S.Tt;
    float e = S.e;
#pragma unroll 1
    for (int i = i0; i < i0 + kChunkSteps; i += 8) {
      const float fi = (float)i;
      float2 g[8];                                   // STAGED: M in .x; else the sample (dc outside the window)
      bool in[8];
#pragma unroll
      for (int u = 0; u < 8; u++) {
        const int p = (int)f_add(f_mul(f_add(fi, (float)u), Tt), findex);  // (int)(i * T + index), :161 (exact: i < 256)
        in[u] = p >= 0 && p < n_total;
        if (STAGED) g[u].x = stage_m[p - lo];
        else g[u] = in[u] ? __ldcg(gw.at(p)) : dc;
      }
#pragma unroll
      for (int u = 0; u < 8; u++) e = f_add(e, STAGED ? g[u].x : in[u] ? c_norm(c_sub(g[u], dc)) : 0.0f);
    }
    S.e = e;
  }
  S.phase++;
}

// EPC, the symbol-period search complete: argmax, 128 bit decisions, CRC-16 (the end of win_stream_finish).  The whole
// window must be present.
__device__ __forceinline__ void win_stream_decide(const RxConfig& c, const WinSrc gw, int n_avail, float2 dc,
                                                  const WinStream& S, WindowDecode& out, long long* pp)
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
  // ---- 128 bit decisions (:171-191): every lane gathers its eight samples straight from L2, all loads in flight
  // together (outside the window a sample is 0, as a stage fill makes it)
  const float twoT = f_mul(2.0f, T);
  float2 wa[4], wb[4];
  bool ia[4], ib[4];
#pragma unroll
  for (int r = 0; r < 4; r++) {
    const int j = r * 32 + lane;
    const int a = win_epc_pos_a(j, twoT, index);
    const int b = win_epc_pos_b(j, T, index);
    ia[r] = a >= 0 && a < n_avail;
    ib[r] = b >= 0 && b < n_avail;
    wa[r] = ia[r] ? __ldcg(gw.at(a)) : dc;
    wb[r] = ib[r] ? __ldcg(gw.at(b)) : dc;
  }
  unsigned Sg[4];
#pragma unroll
  for (int r = 0; r < 4; r++) {
    const float2 sa = ia[r] ? c_sub(wa[r], dc) : make_float2(0.f, 0.f);
    const float2 sb = ib[r] ? c_sub(wb[r], dc) : make_float2(0.f, 0.f);
    Sg[r] = __ballot_sync(0xffffffffu, c_proj(sa, sb, h) > 0.0f);
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

// RN16: half-bit sampling + tag_detection_RN16 (:114-142, :237-253); the whole window must be present.  EPC: remaining
// search chunks (each waits for the samples it reads), then, the whole window present, argmax, 128 bit decisions, CRC-16.
template <bool STAGED>
__device__ __forceinline__ void win_stream_finish(const RxConfig& c, int kind, const WinSrc gw, int n_avail,
                                                  float2* __restrict__ stage, int stage_cap, float2 dc, WinStream& S,
                                                  WindowDecode& out, const ProgressWait* progress = nullptr,
                                                  long long* pp = nullptr)
{
  const int lane = threadIdx.x & 31;
  const float n = c.n_tag_bit_f;
  const float half = f_mul(n, 0.5f);
  const int index = S.index;
  const float2 h = S.h;
  if (kind == RFID_B200_RN16) {
    float jm = (float)index;   // win_rn16_halfbit(index, half, lane), written out: called, it moves spills in rx_pack_kernel<sc16>
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
  while (S.phase <= kSearchChunks) win_stream_chunk<STAGED>(c, gw, n_avail, stage, stage_cap, dc, S, progress);
  progress_wait(progress, n_avail);
  win_stream_decide(c, gw, n_avail, dc, S, out, pp);
}

// The decode of one window held in w[0, n_avail), its phases back to back.  progress_counter (may be null): window
// samples published so far, for a window that is still being gated.  STAGED: as win_stream_chunk.
template <bool STAGED>
__device__ __forceinline__ void decode_window_staged(const RxConfig& c, int kind, const float2* __restrict__ w, int n_avail,
                                                     float2* __restrict__ stage, int stage_cap, WindowDecode& out,
                                                     const volatile int* progress_counter = nullptr)
{
  const WinSrc gw{w, 0, -1};
  const float2 dc = make_float2(0.f, 0.f);
  const ProgressWait pw{progress_counter};
  const ProgressWait* const progress = progress_counter ? &pw : nullptr;
  WinStream S;
  win_stream_head(c, kind, gw, n_avail, stage, stage_cap, dc, S, out, progress);
  win_stream_finish<STAGED>(c, kind, gw, n_avail, stage, stage_cap, dc, S, out, progress);
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
