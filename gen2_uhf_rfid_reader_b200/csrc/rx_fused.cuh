// rx_fused.cuh -- the fused capture-mode kernel: matched filter + decimation,
// gate (reader-command detection, windowing) and tag_decoder for one capture
// segment per CTA, streaming the segment through shared memory in tiles so the
// only HBM traffic is one read of every raw sample (8 B/sample) plus 64-byte
// result records.
//
// Replaces (reference gr-rfid/): filter.fir_filter_ccc(5,[1]*25) (apps/reader.py:65,75),
// gate_impl::general_work (lib/gate_impl.cc:85-200) and
// tag_decoder_impl::general_work (lib/tag_decoder_impl.cc:196-397).
//
// CTA = 4 warps with fixed roles (rotated over the hardware warps by blockIdx so that the
// latency-critical warps of co-resident CTAs spread over the four SM sub-partitions):
//   sequencer   everything that is order-dependent in the reference.  Per 128-sample tile it runs ONE
//               pass of three simultaneous float running sums -- lane 0: avg_ampl over tile k
//               (gate_impl.cc:131), lanes 1,2: dc_est.re/.im over the closed samples of tile k-1
//               (gate_impl.cc:141) -- then finishes tile k-1 (window emission with the now-known DC
//               estimate, window hand-off to the decoder) and runs thresholds + the edge/pulse state
//               machine of tile k (rx_gate.cuh) on its 128-bit masks.
//   workers x2  wait for the TMA bulk copy of the next raw tile, block-sum matched filter, |y|
//               (exact cabsf), amplitude-ring difference / win_length  -> tile stage.
//   decoder     decodes each closed window from shared memory (preamble correlation, channel
//               estimate, FM0 decisions, period search, CRC-16) and writes the result record.
// Hand-offs use named barriers (bar.arrive / bar.sync): a waiting warp is parked by the hardware
// and costs no issue slots; only the TMA completion uses an mbarrier (transaction count).
#pragma once

#include "rx_common.cuh"
#include "rx_decode.cuh"
#include "rx_gate.cuh"

namespace rfid_b200 {

#ifdef RFID_B200_PHASE_PROFILE
// developer aid: per-phase clock64() sums of the sequencer / worker warp of CTA 0..N, written to the window tap
#define PH_DECL long long ph_t0 = clock64(), ph_acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
#define PH_MARK(i) { long long ph_t1 = clock64(); ph_acc[i] += ph_t1 - ph_t0; ph_t0 = ph_t1; }
#define PH_DUMP(base) if (lane == 0 && A.window_tap) { long long* o = reinterpret_cast<long long*>(A.window_tap) + (size_t)blockIdx.x * 24 + (base); for (int i = 0; i < 8; i++) o[i] = ph_acc[i]; }
#else
#define PH_DECL
#define PH_MARK(i)
#define PH_DUMP(base)
#endif

constexpr int kRawStages = 2;
constexpr int kTileStages = 3;    // >= 3: tile k-1 is still being finished while tile k+1 is produced
constexpr int kWorkerWarps = 2;
constexpr int kWorkerThreads = kWorkerWarps * 32;
constexpr int kFusedThreads = 32 * (2 + kWorkerWarps);
constexpr int kMaxTileEvents = 6;

// named barrier ids (immediates, so that ptxas reserves 8 and not all 16 hardware barriers per CTA)
enum : int {
  BAR_WORKERS = 1,      // the two worker warps (64)
  BAR_TILE_FULL = 2,    // +stage: workers arrive (64), sequencer syncs (32)
  BAR_TILE_EMPTY = 5    // +stage: sequencer arrives (32), workers sync (64)
};

template <int BASE>
__device__ __forceinline__ void bar_sync_stage(int s, int n)
{
  if (s == 0) asm volatile("bar.sync %0, %1;" ::"n"((int)BASE), "r"(n) : "memory");
  else if (s == 1) asm volatile("bar.sync %0, %1;" ::"n"((int)(BASE + 1)), "r"(n) : "memory");
  else asm volatile("bar.sync %0, %1;" ::"n"((int)(BASE + 2)), "r"(n) : "memory");
}
template <int BASE>
__device__ __forceinline__ void bar_arrive_stage(int s, int n)
{
  if (s == 0) asm volatile("bar.arrive %0, %1;" ::"n"((int)BASE), "r"(n) : "memory");
  else if (s == 1) asm volatile("bar.arrive %0, %1;" ::"n"((int)(BASE + 1)), "r"(n) : "memory");
  else asm volatile("bar.arrive %0, %1;" ::"n"((int)(BASE + 2)), "r"(n) : "memory");
}
__device__ __forceinline__ void bar_sync_workers()
{
  asm volatile("bar.sync 1, 64;" ::: "memory");
}

struct FusedArgs {
  const void* iq;                // raw capture (device, RAW::T[n_raw]), 16-byte aligned
  unsigned long long n_raw;      // total samples in the capture buffer
  const rfid_b200_segment* segs;
  int nseg;
  int seg_base;                  // added to the segment index stored in the records (a call that decodes a slice of a table)
  int max_windows;               // record slots per segment
  rfid_b200_window_result* results;
  int32_t* counts;
  float2* window_tap;            // optional: ungated samples of every stored window (stride len_epc)
  float2* win_scratch;           // [nseg][win_stride]: the window being decoded (RN16 at 0, EPC at rn16_pad); L2-resident
  int win_stride, rn16_pad;
  int off_dstage, dstage_samples; // decoder staging buffer
  RxConfig cfg;
  // shared-memory carve-up (bytes from the dynamic smem base), computed on the host
  int off_raw, raw_stage_samples;
  int off_bhist, bhist_size;     // float2[bhist_size] (+ partial-block ring right after it when mf_rem > 0)
  int off_ahist, ahist_size;     // float[ahist_size]
  int off_tile_y, off_tile_a, off_tile_d;
  int off_ycl, ycl_size;         // float2[ycl_size]                       (generic path)
  int off_e;                     // float[2][kTT + 16]                      (generic path)
  int off_etile;                 // float[kTileStages][2][kTT] (+pad)       (fast path: workers' DC-ring differences)
  int off_snap;                  // float2[dc_length]: dc ring snapshot taken when the gate opens (fast path)
  int smem_bytes;
  float scale;                   // sc16 captures: the int16 -> float factor (RawSc16::cvt)
};

struct TileEvent {
  int type;  // 1 = gate opens at tile position pos (trigger sample), 2 = window ends before position pos
  int pos;
  int a, b, c, d;  // open: a = index of the trigger in the tile's closed-sample list, b = open index, c = store
                   // close: a = kind, b = ordinal, c = length, d = open index
};

struct FusedShared {
  uint64_t raw_full[kRawStages];
  uint64_t win_ready[2], win_free[2];  // alternate per hand-off: the sequencer may run two hand-offs ahead
  int meta_kind[2], meta_open[2], meta_ordinal[2], meta_len[2];  // double-buffered by hand-off parity
  int n_ev;
  TileEvent ev[kMaxTileEvents];
};

// MFQ > 0: ntaps == MFQ * DECIM (compile-time unrolled block sums); MFQ == 0: generic ntaps.
// This kernel keeps explicit amplitude / closed-sample rings of any length: it serves every rate whose 250 us window is
// longer than a tile (raw rates of 2.6 MS/s and up); rx_fused_split_kernel is the fast path below that.
template <int DECIM, int MFQ, class RAW>
__global__ void __launch_bounds__(kFusedThreads, 8) rx_fused_kernel(const FusedArgs A)
{
  extern __shared__ __align__(128) unsigned char smem[];
  __shared__ FusedShared B;

  const int seg = blockIdx.x;
  const int lane = threadIdx.x & 31;
  const int warp = ((threadIdx.x >> 5) + blockIdx.x) & 3;  // role: 0 sequencer, 1..2 workers, 3 decoder
  const RxConfig& C = A.cfg;
  const rfid_b200_segment sg = A.segs[seg];
  const int n_out = (int)(sg.length / DECIM);
  const int ntiles = (n_out + kTT - 1) / kTT;

  typedef typename RAW::T RawT;
  const RawT* const iq = static_cast<const RawT*>(A.iq);
  RawT* raw = reinterpret_cast<RawT*>(smem + A.off_raw);
  float2* bhist = reinterpret_cast<float2*>(smem + A.off_bhist);
  float2* phist = bhist + A.bhist_size;
  float* ahist = reinterpret_cast<float*>(smem + A.off_ahist);
  float2* tile_y = reinterpret_cast<float2*>(smem + A.off_tile_y);
  float* tile_a = reinterpret_cast<float*>(smem + A.off_tile_a);
  float* tile_d = reinterpret_cast<float*>(smem + A.off_tile_d);
  float2* ycl = reinterpret_cast<float2*>(smem + A.off_ycl);
  float* e_re = reinterpret_cast<float*>(smem + A.off_e);
  float* e_im = e_re + kTT + 16;
  // ungated window samples go to a per-segment global scratch (written once, read once by the decoder warp
  // of the same CTA a few microseconds later: L2 traffic, not shared memory -- that is what lets 8 CTAs fit an SM)
  float2* const win_base = A.win_scratch + (size_t)seg * A.win_stride;
  float2* const dstage = reinterpret_cast<float2*>(smem + A.off_dstage);  // decoder's staging buffer

  // ---- init: zero the history rings (win_samples / dc_samples start at 0, gate_impl.cc:55-56;
  //      x[<0] = +0 for the matched filter), set up the TMA barriers
  for (int i = threadIdx.x; i < A.bhist_size * (C.mf_rem ? 2 : 1); i += kFusedThreads) bhist[i] = make_float2(0.f, 0.f);
  for (int i = threadIdx.x; i < A.ahist_size; i += kFusedThreads) ahist[i] = 0.f;
  for (int i = threadIdx.x; i < A.ycl_size; i += kFusedThreads) ycl[i] = make_float2(0.f, 0.f);
  if (threadIdx.x == 0) {
    for (int s = 0; s < kRawStages; s++) mbar_init(&B.raw_full[s], 1);
    for (int s = 0; s < 2; s++) { mbar_init(&B.win_ready[s], 1); mbar_init(&B.win_free[s], 1); }
    B.n_ev = 0;
    mbar_fence_init();
  }
  __syncthreads();

  if (warp >= 1 && warp <= kWorkerWarps) {
    // =========================================================== workers
    const int wt = (warp - 1) * 32 + lane;
    if (wt == 0) {
      for (int k = 0; k < kRawStages && k < ntiles; k++)
        issue_tile_load<DECIM, RAW>(iq, A.n_raw, sg, k, raw + (size_t)k * A.raw_stage_samples, &B.raw_full[k]);
    }
    const int bmask = A.bhist_size - 1, amask = A.ahist_size - 1;
    const float winlen_f = (float)C.win_length;
    PH_DECL
    for (int k = 0; k < ntiles; k++) {
      const int rs = k % kRawStages, ts = k % kTileStages;
      const RawT* stage = raw + (size_t)rs * A.raw_stage_samples;
      // stage index of raw sample x[D*n - (D-1) + j] for tile-local output t:  D*t - (D-1) + j - delta
      const int delta = (int)(tile_load_start<DECIM, RAW>(sg.offset, k) - (long long)DECIM * k * kTT);
      const int nvalid = min(kTT, n_out - k * kTT);
      PH_MARK(0)
      mbar_wait(&B.raw_full[rs], (k / kRawStages) & 1);
      PH_MARK(1)
      // ---- block sums B(n) = x[D*n-D+1 .. D*n], ascending (and the partial block when ntaps % D != 0)
#pragma unroll
      for (int r = 0; r < kTT / kWorkerThreads; r++) {
        const int t = wt + r * kWorkerThreads;
        if (t < nvalid) {
          const int n = k * kTT + t;
          const int base = DECIM * t - (DECIM - 1) - delta;
          float2 x[DECIM];
#pragma unroll
          for (int j = 0; j < DECIM; j++) {
            // only the very first block of a segment reaches before sample 0 (reads as +0)
            const bool before = (k == 0) && (DECIM * t - (DECIM - 1) + j < 0);
            x[j] = before ? make_float2(0.f, 0.f) : RAW::cvt(stage[base + j], A.scale);
          }
          float2 b = x[0];
#pragma unroll
          for (int j = 1; j < DECIM; j++) b = c_add(b, x[j]);
          bhist[n & bmask] = b;
          if (MFQ == 0 && C.mf_rem) {  // P(n): newest mf_rem samples of the block, ascending (static indexing only)
            float2 p = make_float2(0.f, 0.f);
            bool started = false;
#pragma unroll
            for (int j = 0; j < DECIM; j++) {
              if (j >= DECIM - C.mf_rem) {
                p = started ? c_add(p, x[j]) : x[j];
                started = true;
              }
            }
            phist[n & bmask] = p;
          }
        }
      }
      PH_MARK(2)
      bar_sync_workers();  // raw stage rs fully consumed, block sums visible
      if (wt == 0 && k + kRawStages < ntiles)
        issue_tile_load<DECIM, RAW>(iq, A.n_raw, sg, k + kRawStages, raw + (size_t)rs * A.raw_stage_samples, &B.raw_full[rs]);
      PH_MARK(3)
      if (k >= kTileStages) bar_sync_stage<BAR_TILE_EMPTY>(ts, 96);  // the sequencer is done with tile k - 3
      PH_MARK(4)
      // ---- y[n] = ((P(n-q) + B(n-q+1)) + ...) + B(n);  a = |y|
      float a_reg[kTT / kWorkerThreads];
      float2 y_reg[kTT / kWorkerThreads];
#pragma unroll
      for (int r = 0; r < kTT / kWorkerThreads; r++) {
        const int t = wt + r * kWorkerThreads;
        a_reg[r] = 0.f;
        y_reg[r] = make_float2(0.f, 0.f);
        if (t < nvalid) {
          const int n = k * kTT + t;
          float2 y;
          if (MFQ > 0) {
            y = bhist[(n - MFQ + 1) & bmask];
#pragma unroll
            for (int m = MFQ - 2; m >= 0; m--) y = c_add(y, bhist[(n - m) & bmask]);
          } else {
            int m = n - C.mf_q + 1;
            if (C.mf_rem) {
              y = phist[(n - C.mf_q) & bmask];
            } else {
              y = bhist[m & bmask];
              m++;
            }
            for (; m <= n; m++) y = c_add(y, bhist[m & bmask]);
          }
          const float a = cabsf_ref(y.x, y.y);  // gate_impl.cc:130
          tile_y[ts * kTT + t] = y;
          tile_a[ts * kTT + t] = a;
          ahist[n & amask] = a;
          a_reg[r] = a;
          y_reg[r] = y;
        }
      }
      PH_MARK(5)
      bar_sync_workers();  // this tile's amplitudes / filtered samples visible
      PH_MARK(6)
      // ---- (a - win_samples[win_index]) / win_length   (gate_impl.cc:131)
#pragma unroll
      for (int r = 0; r < kTT / kWorkerThreads; r++) {
        const int t = wt + r * kWorkerThreads;
        if (t < nvalid) {
          const int n = k * kTT + t;
          tile_d[ts * kTT + t] = f_div(f_sub(a_reg[r], ahist[(n - C.win_length) & amask]), winlen_f);
        }
      }
      __threadfence_block();
      bar_arrive_stage<BAR_TILE_FULL>(ts, 96);
      PH_MARK(7)
    }
    if (wt == 0) { PH_DUMP(8) }
  } else if (warp == 0) {
    // =========================================================== sequencer
    float acc = 0.f;  // lane 0: avg_ampl, lane 1: dc_est.re, lane 2: dc_est.im
    // --- gate state machine (runs one tile ahead of the window emission)
    GateFsm gs = {false, 0, 0};    // signal_state starts NEG_EDGE (gate_impl.cc:45)
    bool gate_open = false;
    int to_ungate = C.len_rn16;    // first SEEK is for an RN16 (global_vars.cc:47, reader_impl.cc:262)
    int wcount = 0;
    int n_closed = 0;              // closed-sample ordinal (index into the DC ring stream)
    int open_idx = 0;
    bool cur_store = false;
    int nq = 1;                    // n_queries_sent after START -> SEND_QUERY (reader_impl.cc:259)
    bool terminated = false;
    int n_e = 0;                   // closed samples of the tile whose DC chain is still to run
    // --- emission state (tile k-1)
    bool f_open = false, f_store = false;
    int f_wpos = 0, n_signalled = 0, n_freed = 0;
    float2* win = win_base;
    int closed_since = C.dc_length;  // closed samples since the last window (>= dc_length: ring lookback is time-contiguous)
    float2 dc_open = make_float2(0.f, 0.f);
    const int ymask = A.ycl_size - 1;
    const float dclen_f = (float)C.dc_length;
    const int half_pw = C.n_PW / 2;
    PH_DECL

    for (int k = 0; k <= ntiles; k++) {
      const int ts = k % kTileStages;
      const int nvalid = k < ntiles ? min(kTT, n_out - k * kTT) : 0;
      float* davg = tile_d + ts * kTT;
      PH_MARK(0)
      if (k < ntiles) bar_sync_stage<BAR_TILE_FULL>(ts, 96);
      PH_MARK(1)
      // ---- 1. the three recurrences, one pass: avg_ampl over tile k, dc_est over tile k-1's closed samples
      float* pe_re = e_re;  // tile k-1's list
      float* pe_im = e_im;
      if (lane < 3) chain_inplace(lane == 0 ? davg : (lane == 1 ? pe_re : pe_im), lane == 0 ? nvalid : n_e, acc);
      __syncwarp();
      PH_MARK(2)
      // ---- 2. finish tile k-1: window emission (gate_impl.cc:173,187) and hand-off to the decoder
      if (k >= 1) {
        const int pts = (k - 1) % kTileStages;
        const float2* py = tile_y + pts * kTT;
        const int pvalid = min(kTT, n_out - (k - 1) * kTT);
        const int nev = B.n_ev;
        int pos = 0;
        for (int e = 0; e <= nev; e++) {
          const bool last = e == nev;
          const int etype = last ? 0 : B.ev[e].type;
          const int epos = last ? pvalid : B.ev[e].pos;
          if (f_open) {
            const int take = epos - pos;  // an open event cannot occur while the gate is open
            if (f_store)
              for (int j = lane; j < take; j += 32) win[f_wpos + j] = c_sub(py[pos + j], dc_open);
            f_wpos += take;
            pos = epos;
          }
          if (etype == 2) {
            // window complete: hand it to the decoder
            f_open = false;
            if (f_store) {
              __syncwarp();
              if (lane == 0) {
                const int ms = n_signalled & 1;  // the slot of hand-off n-2 is free: at most one window is outstanding
                B.meta_kind[ms] = B.ev[e].a; B.meta_ordinal[ms] = B.ev[e].b; B.meta_len[ms] = B.ev[e].c; B.meta_open[ms] = B.ev[e].d;
              }
              __threadfence();  // window samples were written to global memory
              __syncwarp();
              if (lane == 0) mbar_arrive(&B.win_ready[n_signalled & 1]);
              n_signalled++;
            }
            pos = epos;
          } else if (etype == 1) {
            // READER COMMAND DETECTED (gate_impl.cc:164-180): dc_est right after the trigger sample
            const int j = B.ev[e].a;
            dc_open = make_float2(pe_re[j], pe_im[j]);
            f_store = B.ev[e].c != 0;
            f_open = true;
            win = win_base + (B.ev[e].d ? A.rn16_pad : 0);  // RN16 and EPC windows have their own scratch areas
            if (f_store) {
              // the area is reused two windows later: at most one window may still be with the decoder
              while (n_signalled - n_freed >= 2) { mbar_wait(&B.win_free[n_freed & 1], (n_freed >> 1) & 1); n_freed++; }
              if (lane == 0) win[0] = c_sub(py[epos], dc_open);
            }
            f_wpos = 1;
            pos = epos + 1;
          }
        }
        __syncwarp();
      }
      PH_MARK(3)
      // ---- 3. thresholds + state machine of tile k; collect its closed samples for the DC chain
      n_e = 0;
      int nev = 0;
      if (k < ntiles && !terminated) {
        const float* ta = tile_a + ts * kTT;
        const float2* ty = tile_y + ts * kTT;
        unsigned ltw, gtw;   // word (lane & 3) of the threshold masks
        gate_masks<4>(davg, ta, nvalid, ltw, gtw);
        PH_MARK(4)

        int pos = 0;
        while (pos < nvalid) {
          if (!gate_open) {
            // ---- closed: edges, pulse counting and the open test of this run (gate_impl.cc:145-180)
            const int run_start = pos;
            const int p_open = gate_closed_run<4>(ltw, gtw, run_start, nvalid, C.n_T1, half_pw, gs);
            const bool opened = p_open >= 0;
            pos = opened ? p_open + 1 : nvalid;
            // ---- DC tracker inputs for the closed run [run_start, pos) (gate_impl.cc:141-143); the run
            //      includes the trigger sample, as in the reference (the update precedes the open test)
            const int len = pos - run_start;
            for (int j = lane; j < len; j += 32) ycl[(n_closed + j) & ymask] = ty[run_start + j];
            __syncwarp();
            for (int j = lane; j < len; j += 32) {
              const float2 yv = ty[run_start + j];
              const float2 old = ycl[(n_closed + j - C.dc_length) & ymask];
              e_re[n_e + j] = f_div(f_sub(yv.x, old.x), dclen_f);
              e_im[n_e + j] = f_div(f_sub(yv.y, old.y), dclen_f);
            }
            n_closed += len;
            n_e += len;
            if (opened) {
              gate_open = true;
              open_idx = k * kTT + pos - 1;
              cur_store = wcount < A.max_windows;
              if (lane == 0 && nev < kMaxTileEvents) {
                TileEvent& ev = B.ev[nev];
                ev.type = 1; ev.pos = pos - 1; ev.a = n_e - 1; ev.b = open_idx; ev.c = cur_store ? 1 : 0; ev.d = wcount & 1;
              }
              nev++;
            }
          } else {
            // ---- open: the samples pass through (gate_impl.cc:182-195); emitted one tile later
            const int take = min(to_ungate - gs.n_samples, nvalid - pos);
            gs.n_samples += take; pos += take;
            if (gs.n_samples >= to_ungate) {
              gate_open = false;
              const int kind = wcount & 1;  // windows alternate RN16, EPC (SURVEY.md 3.5)
              if (lane == 0 && nev < kMaxTileEvents) {
                TileEvent& ev = B.ev[nev];
                ev.type = 2; ev.pos = pos; ev.a = kind; ev.b = wcount; ev.c = to_ungate; ev.d = open_idx;
              }
              nev++;
              wcount++;
              closed_since = 0;
              // the Gen2 logic answers (ACK after RN16 -> GATE_SEEK_EPC, Query/QueryRep after EPC ->
              // GATE_SEEK_RN16) and the next gate call applies it (gate_impl.cc:112-123)
              to_ungate = kind ? C.len_rn16 : C.len_epc;
              gs.n_samples = 0;
              if (kind) {
                nq++;
                if (nq > C.max_queries) { terminated = true; break; }  // gate_impl.cc:101-109
              }
            }
          }
        }
      }
      if (lane == 0) B.n_ev = min(nev, kMaxTileEvents);
      __syncwarp();
      // the stage of tile k-1 (its samples fed the ring lookbacks / snapshot above) may be refilled now
      if (k >= 1 && k - 1 + kTileStages < ntiles) {
        __threadfence_block();
        bar_arrive_stage<BAR_TILE_EMPTY>((k - 1) % kTileStages, 96);
      }
      PH_MARK(5)
    }
    PH_DUMP(0)
    // ---- shut the decoder down, publish the window count
    // the exit message needs the meta slot of hand-off n-2 only
    while (n_signalled - n_freed >= 2) { mbar_wait(&B.win_free[n_freed & 1], (n_freed >> 1) & 1); n_freed++; }
    if (lane == 0) {
      B.meta_kind[n_signalled & 1] = -1;
      A.counts[seg] = wcount;
    }
    __threadfence_block();
    __syncwarp();
    if (lane == 0) mbar_arrive(&B.win_ready[n_signalled & 1]);
  } else {
    // =========================================================== decoder
    for (int j = 0;; j++) {
      while (!mbar_try_wait(&B.win_ready[j & 1], (j >> 1) & 1)) __nanosleep(400);  // idle most of the time: poll slowly
      const int kind = B.meta_kind[j & 1];
      if (kind < 0) break;
      const int ordinal = B.meta_ordinal[j & 1], open_idx = B.meta_open[j & 1], len = B.meta_len[j & 1];
      WindowDecode wd;
      const float2* win = win_base + (kind ? A.rn16_pad : 0);
      decode_window_staged<false>(C, kind, win, len, dstage, A.dstage_samples, wd);
      rfid_b200_window_result* dst = A.results + (size_t)seg * A.max_windows + ordinal;
      if (lane == 0) store_result(dst, wd, seg + A.seg_base, ordinal, open_idx, len, kind);
#ifndef RFID_B200_PHASE_PROFILE
      if (A.window_tap) {
        float2* tap = A.window_tap + ((size_t)(seg + A.seg_base) * A.max_windows + ordinal) * C.len_epc;
        for (int p = lane; p < len; p += 32) tap[p] = __ldcg(win + p);
      }
#endif
      __syncwarp();
      if (lane == 0) mbar_arrive(&B.win_free[j & 1]);
    }
  }
}

}  // namespace rfid_b200
