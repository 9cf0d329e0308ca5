// rx_report.cuh -- the tag inventory report (rfid_b200_tag_report; the rule is stated in include/rfid_b200.h): a
// group-by of the reads of a decode_capture call over their 128-bit keys.  Three steps, four kernels:
//   1. rx_report_insert_kernel: a warp takes kReportIter rounds of 32 consecutive slots.  Each lane classifies its slot;
//      the reads of a round are grouped by key (leader = lowest lane, full 16-byte compare), and each group is merged into
//      a per-warp cache of 32 keys held one per lane.  A key the cache misses is inserted into an open-addressing table
//      (owner = slot + 1, set by atomicCAS; the owner's key is read back from its record or fix, which are in memory
//      before the kernel starts), and the entry it evicts is flushed into the owner's aggregate with four atomics.  So one
//      tag read 320,000 times costs one flush per warp, and 320,000 distinct keys one insert each.  Every slot's owner
//      (or its class) goes to rep[].  Lanes map to consecutive slots, so a group's first and last slot are its lowest
//      and highest lane.
//   2. rx_report_count_kernel / rx_report_scan_kernel: a read whose slot is its tag's first slot starts a tag; the flags
//      are counted per block of kReportBlockSlots slots and the counts scanned by one CTA.
//   3. rx_report_write_kernel numbers the tags of a block (ballot prefix in slot order), writes their records and, with
//      d_read_tag, every stored slot's tag index (a second launch of the same kernel, once every tag has its number).
// tests/report_model.py restates the rule in numpy.
#pragma once

#include "rx_common.cuh"

namespace rfid_b200 {

constexpr int kReportIter = 8;                                       // rounds of 32 slots per warp (insert kernel)
constexpr int kReportWarps = 4;                                      // warps per CTA of the insert kernel
constexpr int kReportBlockSlots = 32 * kReportIter * kReportWarps;   // slots per CTA of every per-slot kernel (1024)
constexpr int kReportThreads = 256;                                  // threads per CTA of the count and write kernels
constexpr int kReportScanThreads = 1024;

// rep[] codes besides an owner slot (>= 0)
constexpr int kRepNotCandidate = -1, kRepRejected = -2, kRepNotStored = -3;

// aggregate of one tag, at its owner's slot index; all-zero bytes are the empty aggregate
struct __align__(32) ReportAgg {
  unsigned long long counts;       // reads | recovered << 32
  unsigned first_inv;              // max of ~slot = ~(smallest slot)
  unsigned last1;                  // max of slot + 1
  unsigned long long peak;         // max of (power key << 32) | ~slot
  int tag;                         // tag index (step 3)
  int pad;
};
static_assert(sizeof(ReportAgg) == 32, "ReportAgg layout");

struct ReportArgs {
  const rfid_b200_segment* segs;
  const rfid_b200_window_result* results;
  const int32_t* counts;
  const rfid_b200_quality* quality;  // may be null
  const rfid_b200_epc_fix* fix;      // may be null
  rfid_b200_tag* tags;
  rfid_b200_tag_summary* summary;
  int32_t* read_tag;                 // may be null
  ReportAgg* agg;                    // [n_slots]
  unsigned* table;                   // [table_mask + 1]: owner slot + 1, 0 = empty
  int32_t* rep;                      // [n_slots]
  int32_t* block_count;              // [n_blocks]: tags starting in the block, then their exclusive prefix
  int max_windows, n_slots, n_blocks, max_tags, check_length, decim;
  unsigned table_mask;
};

__device__ __forceinline__ uint4 report_load_key(const uint8_t* bits) { return *reinterpret_cast<const uint4*>(bits); }

// the key of slot i, which is a read: the record's bits when the record passes, else the fix's
__device__ __forceinline__ uint4 report_key_of(const ReportArgs& A, int i)
{
  const rfid_b200_window_result& r = A.results[i];
  if (r.kind == RFID_B200_EPC && r.crc_ok == 1) return report_load_key(r.bits);
  return report_load_key(A.fix[i].bits);
}

__device__ __forceinline__ bool report_key_eq(uint4 a, uint4 b)
{
  return a.x == b.x && a.y == b.y && a.z == b.z && a.w == b.w;
}

__device__ __forceinline__ unsigned report_mix(unsigned h)   // murmur3's finaliser
{
  h ^= h >> 16; h *= 0x85ebca6bu; h ^= h >> 13; h *= 0xc2b2ae35u; h ^= h >> 16;
  return h;
}

__device__ __forceinline__ unsigned report_hash(uint4 k)
{
  return report_mix(k.w ^ report_mix(k.z ^ report_mix(k.y ^ report_mix(k.x ^ 0x9e3779b9u))));
}

// p = (float)(re*re + im*im in double); its order key: 0 for NaN, else bits + 1 (p >= +0, so its bits order like it)
__device__ __forceinline__ unsigned report_power_key(float re, float im)
{
  const double x = re, y = im;
  const float p = __double2float_rn(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)));
  return p != p ? 0u : __float_as_uint(p) + 1u;
}

// the owner slot of key k, inserting it with owner `slot` when it is new (one lane).  The table has at least twice as
// many buckets as there are slots, so the probe ends.
__device__ __forceinline__ int report_insert(const ReportArgs& A, uint4 k, int slot)
{
  unsigned b = report_hash(k) & A.table_mask;
  for (;;) {
    const unsigned old = atomicCAS(A.table + b, 0u, (unsigned)slot + 1u);
    if (old == 0u) return slot;
    if (report_key_eq(report_key_of(A, (int)(old - 1u)), k)) return (int)(old - 1u);
    b = (b + 1u) & A.table_mask;
  }
}

__device__ __forceinline__ void report_flush(const ReportArgs& A, int owner, unsigned cnt, unsigned rcnt, int first,
                                             int last, unsigned long long peak)
{
  ReportAgg* g = A.agg + owner;
  atomicAdd(&g->counts, (unsigned long long)cnt | ((unsigned long long)rcnt << 32));
  atomicMax(&g->first_inv, ~(unsigned)first);
  atomicMax(&g->last1, (unsigned)last + 1u);
  atomicMax(&g->peak, peak);
}

__global__ void __launch_bounds__(32 * kReportWarps) rx_report_insert_kernel(const ReportArgs A)
{
  const unsigned full = 0xffffffffu;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long warp_base = ((long long)blockIdx.x * kReportWarps + warp) * (32 * kReportIter);
  // the cache: lane c holds entry c (key, owner; owner -1 = empty) and the aggregate not yet flushed
  uint4 ck = make_uint4(0u, 0u, 0u, 0u);
  int c_owner = -1, c_first = 0, c_last = 0;
  unsigned c_cnt = 0u, c_rcnt = 0u;
  unsigned long long c_peak = 0ull;
  unsigned victim = 0u;                                          // round-robin eviction (warp-uniform)
  unsigned n_reads = 0u, n_rec = 0u, n_len = 0u, n_empty = 0u;   // the warp's summary counts (every lane)
  for (int it = 0; it < kReportIter && warp_base + it * 32 < A.n_slots; it++) {
    const long long li = warp_base + it * 32 + lane;
    const int i = (int)li;
    int code = kRepNotStored;
    bool read = false, from_fix = false, rej_len = false, rej_empty = false;
    uint4 key = make_uint4(0u, 0u, 0u, 0u);
    unsigned pkey = 0u;
    if (li < A.n_slots) {
      const int s = i / A.max_windows, k = i - s * A.max_windows;
      if (k < min(max(A.counts[s], 0), A.max_windows)) {
        code = kRepNotCandidate;
        const rfid_b200_window_result& r = A.results[i];
        const bool rec_ok = r.kind == RFID_B200_EPC && r.crc_ok == 1;
        from_fix = !rec_ok && A.fix != nullptr && A.fix[i].status == RFID_B200_FIX_RECOVERED;
        if (rec_ok || from_fix) {
          key = report_load_key(rec_ok ? r.bits : A.fix[i].bits);
          code = kRepRejected;
          if (A.check_length && ((key.x & 0xffu) >> 3) != 6u) {
            rej_len = true;
          } else if (A.quality != nullptr && A.quality[i].outcome == RFID_B200_SLOT_EMPTY) {
            rej_empty = true;
          } else {
            read = true;
            pkey = report_power_key(r.h_re, r.h_im);
          }
        }
      }
    }
    const unsigned reads = __ballot_sync(full, read);
    n_reads += __popc(reads);
    n_rec += __popc(__ballot_sync(full, read && from_fix));
    n_len += __popc(__ballot_sync(full, rej_len));
    n_empty += __popc(__ballot_sync(full, rej_empty));
    // group the round's reads by key and merge each group into the cache
    for (unsigned pending = reads; pending;) {
      const int L = __ffs(pending) - 1;
      const uint4 lk = make_uint4(__shfl_sync(full, key.x, L), __shfl_sync(full, key.y, L), __shfl_sync(full, key.z, L),
                                  __shfl_sync(full, key.w, L));
      const bool same = read && report_key_eq(key, lk);
      const unsigned G = __ballot_sync(full, same);
      const unsigned gcnt = __popc(G), grc = __popc(__ballot_sync(full, same && from_fix));
      const int gfirst = i - lane + L, glast = i - lane + (31 - __clz(G));
      const unsigned gp = __reduce_max_sync(full, same ? pkey : 0u);
      const int gpl = __ffs(__ballot_sync(full, same && pkey == gp)) - 1;   // ties: the lowest slot
      const unsigned long long gpeak = ((unsigned long long)gp << 32) | (unsigned)~(unsigned)(i - lane + gpl);
      const unsigned hit = __ballot_sync(full, c_owner >= 0 && report_key_eq(ck, lk));
      int gowner;
      if (hit) {
        const int h = __ffs(hit) - 1;
        if (lane == h) {
          c_cnt += gcnt; c_rcnt += grc;
          c_first = min(c_first, gfirst); c_last = max(c_last, glast);
          c_peak = gpeak > c_peak ? gpeak : c_peak;
        }
        gowner = __shfl_sync(full, c_owner, h);
      } else {
        int owner = 0;
        if (lane == L) owner = report_insert(A, lk, gfirst);
        gowner = __shfl_sync(full, owner, L);
        if (lane == (int)(victim & 31u)) {
          if (c_owner >= 0) report_flush(A, c_owner, c_cnt, c_rcnt, c_first, c_last, c_peak);
          ck = lk; c_owner = gowner; c_cnt = gcnt; c_rcnt = grc; c_first = gfirst; c_last = glast; c_peak = gpeak;
        }
        victim++;
      }
      if (same) code = gowner;
      pending &= ~G;
    }
    if (li < A.n_slots) A.rep[i] = code;
  }
  if (c_owner >= 0) report_flush(A, c_owner, c_cnt, c_rcnt, c_first, c_last, c_peak);
  __shared__ unsigned s_sum[kReportWarps][4];
  if (lane == 0) { s_sum[warp][0] = n_reads; s_sum[warp][1] = n_rec; s_sum[warp][2] = n_len; s_sum[warp][3] = n_empty; }
  __syncthreads();
  if (threadIdx.x < 4) {
    unsigned t = 0u;
    for (int w = 0; w < kReportWarps; w++) t += s_sum[w][threadIdx.x];
    // reads, recovered, rejected_length, rejected_empty: the summary's int32 fields 1..4
    if (t) atomicAdd(reinterpret_cast<int*>(A.summary) + 1 + threadIdx.x, (int)t);
  }
}

// does slot i start a tag (a read at its tag's first slot)?  slot i < n_slots
__device__ __forceinline__ bool report_starts_tag(const ReportArgs& A, int i, int& owner)
{
  owner = A.rep[i];
  return owner >= 0 && ~A.agg[owner].first_inv == (unsigned)i;
}

__global__ void __launch_bounds__(kReportThreads) rx_report_count_kernel(const ReportArgs A)
{
  int n = 0;
  for (int r = 0; r < kReportBlockSlots / kReportThreads; r++) {
    const long long i = (long long)blockIdx.x * kReportBlockSlots + r * kReportThreads + threadIdx.x;
    int owner;
    if (i < A.n_slots && report_starts_tag(A, (int)i, owner)) n++;
  }
  __shared__ int s_n[kReportThreads / 32];
  for (int off = 16; off > 0; off >>= 1) n += __shfl_xor_sync(0xffffffffu, n, off);
  if ((threadIdx.x & 31) == 0) s_n[threadIdx.x >> 5] = n;
  __syncthreads();
  if (threadIdx.x == 0) {
    int t = 0;
    for (int w = 0; w < kReportThreads / 32; w++) t += s_n[w];
    A.block_count[blockIdx.x] = t;
  }
}

// exclusive prefix over the block of one int per thread (all kReportScanThreads or kReportThreads threads); *total
// receives the block's sum
template <int NT>
__device__ __forceinline__ int report_block_exclusive(int v, int* s_w, int* total)
{
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int x = v;
  for (int off = 1; off < 32; off <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, x, off);
    if (lane >= off) x += y;
  }
  if (lane == 31) s_w[warp] = x;
  __syncthreads();
  int before = 0, t = 0;
  for (int w = 0; w < NT / 32; w++) {
    const int sw = s_w[w];
    if (w < warp) before += sw;
    t += sw;
  }
  __syncthreads();   // s_w may be reused
  *total = t;
  return before + x - v;
}

__global__ void __launch_bounds__(kReportScanThreads) rx_report_scan_kernel(const ReportArgs A)
{
  __shared__ int s_w[kReportScanThreads / 32];
  int carry = 0;
  for (int base = 0; base < A.n_blocks; base += kReportScanThreads) {
    const int b = base + (int)threadIdx.x;
    const int v = b < A.n_blocks ? A.block_count[b] : 0;
    int total;
    const int ex = report_block_exclusive<kReportScanThreads>(v, s_w, &total);
    if (b < A.n_blocks) A.block_count[b] = carry + ex;
    carry += total;
  }
  if (threadIdx.x == 0) A.summary->n_tags = carry;
}

__device__ __forceinline__ long long report_time(const ReportArgs& A, int i, const rfid_b200_window_result& r)
{
  const unsigned long long t = A.segs[i / A.max_windows].offset +
                               (unsigned long long)((long long)A.decim * ((long long)r.open_index + (long long)r.sync_index));
  return (long long)t;
}

// read_tags == false: number the tags starting in this block and write their records; true: write every stored slot's
// tag index (after the first launch has numbered every tag)
__global__ void __launch_bounds__(kReportThreads) rx_report_write_kernel(const ReportArgs A, bool read_tags)
{
  __shared__ int s_w[kReportThreads / 32];
  int run = read_tags ? 0 : A.block_count[blockIdx.x];
  for (int r = 0; r < kReportBlockSlots / kReportThreads; r++) {
    const long long li = (long long)blockIdx.x * kReportBlockSlots + r * kReportThreads + threadIdx.x;
    const int i = (int)li;
    if (read_tags) {
      if (li < A.n_slots) {
        const int code = A.rep[i];
        if (code != kRepNotStored) A.read_tag[i] = code >= 0 ? A.agg[code].tag : code;
      }
      continue;
    }
    int owner = -1;
    const bool starts = li < A.n_slots && report_starts_tag(A, i, owner);
    int total;
    const int tag = run + report_block_exclusive<kReportThreads>(starts ? 1 : 0, s_w, &total);
    run += total;
    if (!starts) continue;
    A.agg[owner].tag = tag;
    if (tag >= A.max_tags) continue;
    const ReportAgg g = A.agg[owner];
    const int last = (int)g.last1 - 1;
    const unsigned pk = (unsigned)(g.peak >> 32);
    const rfid_b200_window_result& rf = A.results[i];
    const rfid_b200_window_result& rl = A.results[last];
    int4* o = reinterpret_cast<int4*>(A.tags + tag);
    const uint4 key = report_key_of(A, i);
    o[0] = make_int4((int)key.x, (int)key.y, (int)key.z, (int)key.w);
    o[1] = make_int4((int)(unsigned)g.counts, (int)(unsigned)(g.counts >> 32), i, last);
    o[2] = make_int4((int)~(unsigned)g.peak, pk == 0u ? 0x7fc00000 : (int)(pk - 1u), __float_as_int(rl.h_re),
                     __float_as_int(rl.h_im));
    reinterpret_cast<longlong2*>(o)[3] = make_longlong2(report_time(A, i, rf), report_time(A, last, rl));
  }
}

}  // namespace rfid_b200
