// rx_cmd.cuh -- capture mode, the reader's side: PIE command decoding (rfid_b200_decode_commands).
//
// In a monostatic capture the reader's TX leaks into the RX at full carrier level, so every segment holds the reader's
// commands as well as the tag's replies.  A command is a burst of low pulses (PW = 12 us of near-zero envelope at the end
// of every PIE symbol, reader_impl.cc:55-71); the fall-to-fall intervals are the symbol lengths: delimiter + data-0
// (Tari), RTcal, TRcal (preamble only), then one interval per data bit.  The rule, per segment and independent of
// everything outside it (include/rfid_b200.h states it in full; tests/command_model.py restates it in numpy):
//   p = re*re + im*im (three roundings), P = max p, thr2 = (level_frac*level_frac) * P (or level_abs^2), low = p < thr2;
//   fall = low sample whose predecessor in the segment is high; a burst starts at a fall whose previous low sample lies
//   >= gap samples back (or that has none); bursts of >= 4 falls are decoded.
//
// rx_cmd_kernel: one CTA per segment, two passes over it.
//   pass 1  the peak P (a max: exact in any order, so the block reduction needs no fixed order);
//   pass 2  chunks of kCmdChunk samples: every warp builds 32 low-mask words by ballot (as ingest_mask does), every
//           thread takes one word, falls = word & ~((word << 1) | prev_top); a block scan gives each fall its index and
//           its previous low sample, the falls are compacted into shared memory, and thread 0 walks them in order,
//           carrying the open burst (intervals, bits) across chunks, and writes a record when a burst closes.  The
//           other warps load the next chunk meanwhile.
// The CTA reads its segment twice, the second time meant to hit L2 (DESIGN.md 4.5 and 6 on how far that holds).
// Samples are read one per lane (8 B fc32 / 4 B sc16, coalesced across the warp): no 16-byte granules, so no odd-offset
// or capture-end case exists here; the capture kernels' tile loader (rx_common.cuh) copies decimated tiles with their
// matched-filter history, a geometry this pass does not have.
#pragma once

#include <cstdint>

#include "rx_common.cuh"
#include "tx_synth.cuh"

namespace rfid_b200 {

// 256 threads, 4 CTAs per SM: measured faster than 512 x 2 and 1024 x 1 (DESIGN.md section 6)
constexpr int kCmdThreads = 256;
constexpr int kCmdWarps = kCmdThreads / 32;
constexpr int kCmdWords = 256;                // low-mask words per pass-2 chunk
constexpr int kCmdChunk = kCmdWords * 32;     // samples per pass-2 chunk
constexpr int kCmdScanWarps = kCmdWords / 32; // warps that scan a chunk (one word per thread)
constexpr int kCmdWarpWords = kCmdWords / kCmdWarps;   // words each warp builds
constexpr int kCmdMaxFalls = kCmdChunk / 2;   // falls in a chunk (every other sample at most)
constexpr int kCmdBits = 128;                 // data bits stored per record
constexpr int kCmdLoads = kCmdWarpWords < 16 ? kCmdWarpWords : 16;   // loads in flight per lane in pass 2
constexpr int kCmdMinBlocks = 1024 / kCmdThreads;                    // 64 registers per thread
static_assert(kCmdWords % kCmdWarps == 0 && kCmdWarpWords <= 32 && kCmdWarpWords % kCmdLoads == 0, "chunk geometry");

struct CmdArgs {
  const void* iq;
  float scale;                 // sc16 only
  unsigned long long n_raw;
  const rfid_b200_segment* segs;
  int nseg;
  int max_cmds;
  rfid_b200_command* cmds;
  int32_t* counts;
  float frac2;                 // level_frac * level_frac
  float abs2;                  // level_abs * level_abs
  int use_abs;                 // level_abs > 0
  int gap;                     // raw samples
};

// thread 0's view of the burst being decoded
struct CmdBurst {
  int nf;                      // falls so far (0: no burst open)
  int start, last;             // first / latest fall
  int tari, rtcal, trcal;
  int n_bits;
};

__device__ __forceinline__ int cmd_bit(const uint8_t* b, int i) { return (b[i >> 3] >> (7 - (i & 7))) & 1; }
__device__ __forceinline__ int cmd_field(const uint8_t* b, int lo, int hi)
{
  int v = 0;
  for (int i = lo; i < hi; i++) v = (v << 1) | cmd_bit(b, i);
  return v;
}

// kind / arg / crc_ok of a closed burst (include/rfid_b200.h, table of rfid_b200_decode_commands)
__device__ void cmd_classify(const CmdBurst& B, const uint8_t* bits, rfid_b200_command& r)
{
  const int n = B.n_bits;
  r.kind = RFID_B200_CMD_OTHER;
  r.arg = -1;
  r.crc_ok = -1;
  if (B.trcal > 0) {
    if (n == 22 && cmd_field(bits, 0, 4) == 0x8) {  // 1000 DR M TRext Sel Session Target Q CRC-5 (reader_impl.cc:131-162)
      int b17[17];
      for (int i = 0; i < 17; i++) b17[i] = cmd_bit(bits, i);
      r.kind = RFID_B200_TX_QUERY;
      r.arg = cmd_field(bits, 13, 17);
      r.crc_ok = tx_crc5(b17) == cmd_field(bits, 17, 22) ? 1 : 0;
    }
    return;
  }
  if (n == 4 && cmd_field(bits, 0, 2) == 0x0) {
    r.kind = RFID_B200_TX_QUERY_REP;
    r.arg = cmd_field(bits, 2, 4);
  } else if (n == 18 && cmd_field(bits, 0, 2) == 0x1) {
    r.kind = RFID_B200_TX_ACK;
    r.arg = cmd_field(bits, 2, 18);
  } else if (n == 9 && cmd_field(bits, 0, 4) == 0x9) {
    r.kind = RFID_B200_TX_QUERY_ADJUST;
    r.arg = cmd_field(bits, 4, 6);
  } else if (n == 8 && cmd_field(bits, 0, 8) == 0xC0) {
    r.kind = RFID_B200_TX_NAK;
  }
}

template <class RAW>
__global__ void __launch_bounds__(kCmdThreads, kCmdMinBlocks) rx_cmd_kernel(const CmdArgs A)
{
  __shared__ unsigned int s_mask[kCmdWords];
  __shared__ int s_pos[kCmdMaxFalls];
  __shared__ int s_prev[kCmdMaxFalls];          // last low sample before each fall (-1: none)
  __shared__ int s_wsum[kCmdScanWarps], s_wmax[kCmdScanWarps];
  __shared__ float s_peak[kCmdWarps];
  __shared__ int s_carry_last, s_nfalls;
  __shared__ unsigned int s_carry_top;
  __shared__ uint8_t s_bits[kCmdBits / 8];

  const int s = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const rfid_b200_segment sg = A.segs[s];
  if (sg.length > 0x7fffffffu) {               // start / end are int32
    if (tid == 0) A.counts[s] = RFID_B200_EINVAL;
    return;
  }
  long long len_ll = (long long)sg.length;     // a segment is cut at the end of the capture
  if (sg.offset >= A.n_raw) len_ll = 0;
  else if ((unsigned long long)len_ll > A.n_raw - sg.offset) len_ll = (long long)(A.n_raw - sg.offset);
  const int len = (int)len_ll;
  const typename RAW::T* x = static_cast<const typename RAW::T*>(A.iq) + sg.offset;

  // ---- pass 1: the peak (NaN samples never win a comparison)
  float peak = 0.f;
  if (!A.use_abs) {
    constexpr int U = 8;
    for (long long b = 0; b < len; b += U * kCmdThreads) {   // (64-bit indices: len may be INT32_MAX)
      typename RAW::T v[U];
#pragma unroll
      for (int j = 0; j < U; j++) {
        const long long i = b + j * kCmdThreads + tid;
        if (i < len) v[j] = x[i];
      }
#pragma unroll
      for (int j = 0; j < U; j++) {
        const long long i = b + j * kCmdThreads + tid;
        if (i < len) {
          const float p = c_norm(RAW::cvt(v[j], A.scale));
          peak = p > peak ? p : peak;
        }
      }
    }
    for (int o = 16; o; o >>= 1) {
      const float q = __shfl_xor_sync(0xffffffffu, peak, o);
      peak = q > peak ? q : peak;
    }
    if (lane == 0) s_peak[warp] = peak;
  }
  if (tid == 0) { s_carry_last = -1; s_carry_top = 0u; }
  __syncthreads();
  float thr2 = A.abs2;
  if (!A.use_abs) {
    peak = s_peak[0];
    for (int w = 1; w < kCmdWarps; w++) peak = s_peak[w] > peak ? s_peak[w] : peak;
    thr2 = f_mul(A.frac2, peak);
  }

  // ---- pass 2: masks, falls, bursts
  CmdBurst B = {0, 0, 0, 0, 0, 0, 0};
  int n_cmd = 0;
  rfid_b200_command* out = A.cmds + (size_t)s * (size_t)A.max_cmds;
  auto close = [&](int end) {                  // thread 0: the open burst ends; its last low sample is end - 1
    if (B.nf >= 4) {
      if (n_cmd < A.max_cmds) {
        rfid_b200_command r;
        r.segment = s;
        r.index = n_cmd;
        r.start = B.start;
        r.end = end;
        r.n_bits = B.n_bits;
        r.tari = B.tari;
        r.rtcal = B.rtcal;
        r.trcal = B.trcal;
        r.reserved = 0;
        cmd_classify(B, s_bits, r);
        for (int k = 0; k < kCmdBits / 8; k++) r.bits[k] = s_bits[k];
        out[n_cmd] = r;
      }
      n_cmd++;
    }
    B.nf = 0;
  };

  for (long long c0 = 0; c0 < len; c0 += kCmdChunk) {
    // masks: warp w builds words w*kCmdWarpWords + k (lane k keeps word k), word j = samples c0 + 32j .. +31
    {
      const long long wb = c0 + (long long)warp * kCmdWarpWords * 32;
      unsigned int word = 0;
#pragma unroll
      for (int h = 0; h < kCmdWarpWords; h += kCmdLoads) {
        typename RAW::T v[kCmdLoads];
#pragma unroll
        for (int k = 0; k < kCmdLoads; k++) {
          const long long i = wb + (h + k) * 32 + lane;
          if (i < len) v[k] = RAW::ldcs(x + i);
        }
#pragma unroll
        for (int k = 0; k < kCmdLoads; k++) {
          const long long i = wb + (h + k) * 32 + lane;
          const bool low = i < len && c_norm(RAW::cvt(v[k], A.scale)) < thr2;
          const unsigned int b = __ballot_sync(0xffffffffu, low);
          if (lane == h + k) word = b;
        }
      }
      if (lane < kCmdWarpWords) s_mask[warp * kCmdWarpWords + lane] = word;
    }
    __syncthreads();
    // the first kCmdScanWarps warps, one word per thread: falls, last low sample; block scans of both
    const bool scan = tid < kCmdWords;   // (warp-uniform)
    unsigned int word = 0, fall = 0;
    int base = 0, nf = 0, inc_n = 0, before = -1;
    if (scan) {
      word = s_mask[tid];
      const unsigned int prev_top = tid ? s_mask[tid - 1] >> 31 : s_carry_top;
      fall = word & ~((word << 1) | prev_top);
      base = (int)(c0 + tid * 32);      // (a word past the segment's end has no bits: base is unused there)
      const int last = word ? base + 31 - __clz(word) : -1;
      nf = __popc(fall);
      inc_n = nf;
      int inc_last = last;
      for (int o = 1; o < 32; o <<= 1) {
        const int on = __shfl_up_sync(0xffffffffu, inc_n, o);
        const int ol = __shfl_up_sync(0xffffffffu, inc_last, o);
        if (lane >= o) { inc_n += on; inc_last = ol > inc_last ? ol : inc_last; }
      }
      before = __shfl_up_sync(0xffffffffu, inc_last, 1);
      if (lane == 0) before = -1;
      if (lane == 31) { s_wsum[warp] = inc_n; s_wmax[warp] = inc_last; }
    }
    const int carry_last = s_carry_last;
    __syncthreads();
    if (scan) {
      int off = inc_n - nf;
      before = before > carry_last ? before : carry_last;
      int tot = 0, tot_last = carry_last;
      for (int w = 0; w < kCmdScanWarps; w++) {
        if (w < warp) { off += s_wsum[w]; before = s_wmax[w] > before ? s_wmax[w] : before; }
        tot += s_wsum[w];
        tot_last = s_wmax[w] > tot_last ? s_wmax[w] : tot_last;
      }
      while (fall) {
        const int p = __ffs(fall) - 1;
        fall &= fall - 1;
        const unsigned int below = word & ((1u << p) - 1u);
        s_pos[off] = base + p;
        s_prev[off] = below ? base + 31 - __clz(below) : before;
        off++;
      }
      if (tid == kCmdWords - 1) { s_carry_top = word >> 31; s_carry_last = tot_last; s_nfalls = tot; }
    }
    __syncthreads();
    if (tid == 0) {
      const int n = s_nfalls;
      for (int j = 0; j < n; j++) {
        const int pos = s_pos[j], prev = s_prev[j];
        if (prev < 0 || pos - prev - 1 >= A.gap) {
          close(prev + 1);
          B.nf = 1; B.start = pos; B.last = pos; B.n_bits = 0; B.trcal = 0;
          for (int k = 0; k < kCmdBits / 8; k++) s_bits[k] = 0;
          continue;
        }
        const int d = pos - B.last;
        B.last = pos;
        bool data = B.nf >= 4;
        if (B.nf == 1) B.tari = d;
        else if (B.nf == 2) B.rtcal = d;
        else if (B.nf == 3) {
          if (d > B.rtcal) B.trcal = d;
          else data = true;
        }
        if (data) {
          if (B.n_bits < kCmdBits && 2ll * d > (long long)B.rtcal) s_bits[B.n_bits >> 3] |= (uint8_t)(0x80u >> (B.n_bits & 7));
          B.n_bits++;
        }
        B.nf++;
      }
    }
  }
  if (tid == 0) {
    close(s_carry_last + 1);
    A.counts[s] = n_cmd;
  }
}

}  // namespace rfid_b200
