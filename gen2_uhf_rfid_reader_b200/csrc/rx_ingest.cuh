// rx_ingest.cuh -- capture ingest: CW-gap segmenter (SURVEY.md section 8f, rank 2).
//
// The reference has no segmenter: its offline mode (apps/reader.py:101-112) pushes the whole file through
// one sequential gate.  Capture mode decodes *segments* in parallel, so a recorded capture first has to be
// cut at places where nothing is happening.  The reader's commands are bursts of low pulses (PW = 12 us of
// near-zero envelope per PIE symbol, reader_impl.cc:55-71) separated by long stretches of CW during which the
// tag replies; every command with more than NUM_PULSES_COMMAND pulses makes the reference gate arm exactly one
// window (gate_impl.cc:150-180), and the window kinds alternate RN16 / EPC (SURVEY.md 3.5).  A segment is
// therefore "two consecutive commands and the CW that follows each", starting a lead-in before the first.
//
// Device work (all passes stream over HBM or over a 1 bit/sample mask; no atomics on the data path):
//   ingest_level_*   CW level = mean |x| of the head of the capture  -> threshold^2 = (level_frac * level)^2
//   ingest_mask      1 bit per raw sample (|x|^2 < threshold^2), per-1024-sample-chunk summary
//                    (last low sample, number of falling edges)
//   ingest_scan      exclusive max / sum scan of the chunk summaries (one CTA)
//   ingest_bursts    every falling edge whose preceding low sample lies at least `gap` samples back starts a
//                    burst; emits (position, rank among all falling edges) -- the host turns ranks into pulse
//                    counts, drops bursts that are not commands and pairs the rest into segments.
#pragma once

#include <cstdint>

#include "rx_common.cuh"

namespace rfid_b200 {

constexpr int kIngestChunk = 1024;       // raw samples per warp pass (32 mask words)
constexpr int kLevelBlocks = 128;        // fixed geometry => reproducible sum
constexpr int kLevelThreads = 256;

struct IngestBurst {
  unsigned long long pos;   // raw index of the burst's first falling edge
  unsigned long long rank;  // number of falling edges before it in the capture
};

struct IngestTotals {
  unsigned int n_bursts;          // bursts emitted (may exceed capacity; only capacity are stored)
  unsigned int pad;
  unsigned long long n_falls;     // falling edges in the capture
  float thr2;                     // threshold^2 in use
  float level;                    // CW level estimate
};

// RAW: the capture's sample format (rx_common.cuh); every sample is converted (RAW::cvt, `scale`) before it is used, so
// an sc16 capture gives the level, masks and segment table of its fc32 conversion
template <class RAW>
__global__ void __launch_bounds__(kLevelThreads) ingest_level_partial(const typename RAW::T* __restrict__ iq, float scale,
                                                                     unsigned long long n0, double* __restrict__ partial)
{
  __shared__ double s_w[kLevelThreads / 32];
  double acc = 0.0;
  for (unsigned long long i = (unsigned long long)blockIdx.x * kLevelThreads + threadIdx.x; i < n0;
       i += (unsigned long long)kLevelBlocks * kLevelThreads) {
    const float2 v = RAW::cvt(iq[i], scale);
    acc += (double)sqrtf(v.x * v.x + v.y * v.y);
  }
  for (int o = 16; o; o >>= 1) acc += __shfl_down_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < kLevelThreads / 32; w++) t += s_w[w];
    partial[blockIdx.x] = t;
  }
}

__global__ void ingest_level_final(const double* __restrict__ partial, unsigned long long n0, float level_frac,
                                   IngestTotals* __restrict__ tot)
{
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    double t = 0.0;
    for (int b = 0; b < kLevelBlocks; b++) t += partial[b];
    const float level = n0 ? (float)(t / (double)n0) : 0.f;
    const float thr = level_frac * level;
    tot->level = level;
    tot->thr2 = thr * thr;
    tot->n_bursts = 0;
    tot->n_falls = 0;
  }
}

// One warp per chunk of 1024 raw samples [first_chunk, first_chunk + n_chunks).
template <class RAW>
__global__ void __launch_bounds__(256) ingest_mask(const typename RAW::T* __restrict__ iq, float scale, unsigned long long n_raw, long long first_chunk,
                                                   long long n_chunks, const IngestTotals* __restrict__ tot,
                                                   unsigned int* __restrict__ mask, long long* __restrict__ chunk_last,
                                                   unsigned int* __restrict__ chunk_falls)
{
  const int lane = threadIdx.x & 31;
  const long long warp = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const long long nwarps = (long long)gridDim.x * (blockDim.x >> 5);
  const float thr2 = tot->thr2;
  for (long long cc = warp; cc < n_chunks; cc += nwarps) {
    const long long c = first_chunk + cc;
    const unsigned long long base = (unsigned long long)c * kIngestChunk;
    unsigned int word = 0;
#pragma unroll 8
    for (int k = 0; k < 32; k++) {
      const unsigned long long i = base + (unsigned)(k * 32 + lane);
      bool low = false;
      if (i < n_raw) {
        const float2 v = RAW::cvt(RAW::ldcs(iq + i), scale);
        low = v.x * v.x + v.y * v.y < thr2;
      }
      const unsigned int b = __ballot_sync(0xffffffffu, low);
      if (lane == k) word = b;
    }
    // previous sample's bit for each word
    unsigned int prev_top = __shfl_up_sync(0xffffffffu, word, 1) >> 31;
    if (lane == 0) {
      prev_top = 0;
      if (base > 0) {
        const float2 v = RAW::cvt(iq[base - 1], scale);
        prev_top = v.x * v.x + v.y * v.y < thr2 ? 1u : 0u;
      }
    }
    const unsigned int fall = word & ~((word << 1) | prev_top);
    long long last = word ? (long long)(base + (unsigned)(lane * 32 + 31 - __clz(word))) : -1;
    unsigned int nf = __popc(fall);
    for (int o = 16; o; o >>= 1) {
      const long long other = __shfl_xor_sync(0xffffffffu, last, o);
      last = other > last ? other : last;
      nf += __shfl_xor_sync(0xffffffffu, nf, o);
    }
    mask[c * 32 + lane] = word;
    if (lane == 0) { chunk_last[c] = last; chunk_falls[c] = nf; }
  }
}

// Exclusive scans over the chunk summaries (one CTA of 1024 threads): prev_low[c] = last low sample before
// chunk c (-1: none), falls_before[c] = falling edges before chunk c.
__global__ void __launch_bounds__(1024) ingest_scan(long long n_chunks, const long long* __restrict__ chunk_last,
                                                    const unsigned int* __restrict__ chunk_falls,
                                                    long long* __restrict__ prev_low, unsigned long long* __restrict__ falls_before,
                                                    IngestTotals* __restrict__ tot)
{
  __shared__ long long s_max[1024];
  __shared__ unsigned long long s_sum[1024];
  const int t = threadIdx.x;
  const long long per = (n_chunks + 1023) / 1024;
  const long long lo = (long long)t * per, hi = lo + per < n_chunks ? lo + per : n_chunks;
  long long m = -1;
  unsigned long long s = 0;
  for (long long c = lo; c < hi; c++) {
    const long long v = chunk_last[c];
    m = v > m ? v : m;
    s += chunk_falls[c];
  }
  s_max[t] = m;
  s_sum[t] = s;
  __syncthreads();
  for (int o = 1; o < 1024; o <<= 1) {  // Hillis-Steele inclusive scan
    long long om = -1;
    unsigned long long os = 0;
    if (t >= o) { om = s_max[t - o]; os = s_sum[t - o]; }
    __syncthreads();
    if (t >= o) { s_max[t] = om > s_max[t] ? om : s_max[t]; s_sum[t] += os; }
    __syncthreads();
  }
  long long run_m = t ? s_max[t - 1] : -1;
  unsigned long long run_s = t ? s_sum[t - 1] : 0;
  for (long long c = lo; c < hi; c++) {
    prev_low[c] = run_m;
    falls_before[c] = run_s;
    const long long v = chunk_last[c];
    run_m = v > run_m ? v : run_m;
    run_s += chunk_falls[c];
  }
  if (t == 1023) tot->n_falls = s_sum[1023];
}

// One warp per chunk: burst starts.
__global__ void __launch_bounds__(256) ingest_bursts(long long n_chunks, const unsigned int* __restrict__ mask,
                                                     const long long* __restrict__ prev_low,
                                                     const unsigned long long* __restrict__ falls_before, unsigned int gap,
                                                     IngestBurst* __restrict__ bursts, unsigned int capacity,
                                                     IngestTotals* __restrict__ tot)
{
  const int lane = threadIdx.x & 31;
  const long long warp = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const long long nwarps = (long long)gridDim.x * (blockDim.x >> 5);
  for (long long c = warp; c < n_chunks; c += nwarps) {
    const unsigned long long base = (unsigned long long)c * kIngestChunk + (unsigned)(lane * 32);
    const unsigned int word = mask[c * 32 + lane];
    unsigned int prev_top = __shfl_up_sync(0xffffffffu, word, 1) >> 31;
    if (lane == 0) prev_top = c > 0 ? mask[c * 32 - 1] >> 31 : 0u;
    unsigned int fall = word & ~((word << 1) | prev_top);
    // last low sample before this word / falling edges before this word (warp exclusive scans)
    long long last = word ? (long long)(base + (unsigned)(31 - __clz(word))) : -1;
    unsigned int nf = __popc(fall);
    long long inc_last = last;
    unsigned int inc_nf = nf;
    for (int o = 1; o < 32; o <<= 1) {
      const long long ol = __shfl_up_sync(0xffffffffu, inc_last, o);
      const unsigned int on = __shfl_up_sync(0xffffffffu, inc_nf, o);
      if (lane >= o) { inc_last = ol > inc_last ? ol : inc_last; inc_nf += on; }
    }
    long long before = __shfl_up_sync(0xffffffffu, inc_last, 1);
    if (lane == 0) before = -1;
    const long long chunk_prev = prev_low[c];
    before = chunk_prev > before ? chunk_prev : before;
    unsigned long long rank = falls_before[c] + (inc_nf - nf);
    while (fall) {
      const int p = __ffs(fall) - 1;
      fall &= fall - 1;
      const unsigned int below = p ? word & ((1u << p) - 1u) : 0u;
      const long long prev = below ? (long long)(base + (unsigned)(31 - __clz(below))) : before;
      const unsigned long long pos = base + (unsigned)p;
      if (prev < 0 || pos - (unsigned long long)prev - 1ull >= gap) {
        const unsigned int slot = atomicAdd(&tot->n_bursts, 1u);
        if (slot < capacity) { bursts[slot].pos = pos; bursts[slot].rank = rank; }
      }
      rank++;
    }
  }
}

}  // namespace rfid_b200
