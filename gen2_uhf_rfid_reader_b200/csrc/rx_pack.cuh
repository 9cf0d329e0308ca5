// rx_pack.cuh -- the roofline kernel of the reference configuration (decimation 5, 25 taps, rings inside one tile):
// same arithmetic as rx_fused_split.cuh (the gate of rx_gate.cuh, the raw-tile loader and running-sum replay of
// rx_common.cuh, the decoder of rx_decode.cuh), re-scheduled around three measurements (tools/pack_profile.py, ncu):
//   * the exact replay of the gate's float running sums (avg_ampl, gate_impl.cc:131; dc_est, gate_impl.cc:141) is a
//     dependent FADD chain -- it costs the same whether 3 or 24 lanes of the warp carry a chain;
//   * everything else of a segment is one warp's worth of *latency*, not of issue slots: a warp that walks a tile through
//     matched filter, |y|, ring differences (or thresholds + the edge / pulse state machine) needs 2-3 thousand cycles per
//     pass almost independently of how many samples the pass covers;
//   * the stages of a segment have very different costs from tile to tile (the state machine costs 1 k cycles on a
//     carrier-only tile and 6 k on a tile full of reader pulses), so a lockstep hand-off per tile runs at the sum of the
//     worst stages.
// So a CTA owns G <= kPMaxSeg capture segments, one warp per role and segment (the decoders: D <= G warps for the CTA),
// ONE chain warp for all of them, and the stages are coupled only through small rings with full / free barriers
// (mbarriers, one phase per slot use):
//   warp A0/A1[g] P1: waits for the raw half-tile (TMA bulk copies issued by the loader warp), block-sum matched filter,
//               exact |y|, amplitude / DC ring differences of 4 outputs per lane.  Writes |y| and the amplitude quotients
//               into pas-slot rings, the DC quotients into a pds-slot ring, and y itself into the segment's circular
//               history in global memory (L2 resident, kYW samples).  May run up to pas tiles ahead of warp B.
//   chain warp  lane 8*c + g replays running sum c (0 avg_ampl, 1 dc_est.re, 2 dc_est.im) of segment g: avg_ampl of tile i
//               as soon as every segment's P1(i) is in, dc_est of tile j once every segment's P3(j) has fixed its list --
//               whichever is ready, both in one pass when both are; then hands dc_est at every window's trigger sample
//               to warp C.
//   warp B[g]   P3: thresholds by ballot (one mask word per lane), the edge / pulse state machine on the 256-bit masks, the
//               DC-tracker inputs of the 48 samples after a window (y read back from the history), -0.0f for the samples
//               inside windows.  Frees the |y| / quotient slot as soon as its masks are made.  Queues opening windows.
//   warps C     D decoder warps, ONE pool over the queued windows of all G segments, straight from the history
//               (rx_decode.cuh): any idle warp runs the next runnable phase of any segment's next window -- an EPC
//               window's head and search chunks as soon as their samples and its dc_est exist, the rest once the whole
//               window does; an RN16 window in one piece.  The state between phases is in shared memory (PackWinState).
//               dc_est is subtracted as the decoder reads the samples -- the same exact float subtraction,
//               gate_impl.cc:173,187.  D = G while the CTA has room for 4G + 2 warps, D = 6 at G = 8; warp A1[g] joins
//               the pool once segment g is through P1, with the segment's raw stages as its decoder stage.
//   loader      lane g streams segment g's raw samples through its two half-tile stages as warp A frees them.
// The history is indexed by the SM (one CTA per SM: the shared-memory request guarantees it), so its size does not depend
// on the number of segments of the launch; warp A never overwrites a sample a queued window still needs.
// Shared memory per segment: 2 raw half-tile stages (10 KB; 5 KB for sc16 captures), the last dc_length outputs of either half-tile (P1's DC
// lookback is a lane shuffle plus this tail), a pas-tile ring of |y| (1 KB per tile), the decode state of its next
// window (112 B, static); per decoder warp C its stage (2 KB; a warp A1 in the pool uses its segment's raw stages); per CTA
// the running-sum buffers (pas + pds x 2 per segment, 1072 B each, skewed so the chain warp's 128-bit accesses are
// bank-conflict free).  HBM traffic: every raw sample is read once (evict-first), 64 B are written per window; the history
// (8 B per decimated sample, rewritten in place) lives in L2.
//
// Phase safety (an mbarrier wait names a phase by its parity, so no barrier may complete the phase after the awaited one
// before the waiter looks; no producer may arrive twice in one phase).  Tile i of a segment with work:
//   freeA[i % pas]    warps A wait for warp B's release of tile i - pas; B releases tile i only after A wrote it.
//   dcdone[i % pds]   warps A wait for the chain's DC pass of tile i - pds; the DC pass of tile i needs p3done(i), hence
//                      avgdone(i), hence fullA(i): A's arrival for tile i, after its wait.
//   fullA[i % pas]    (2G arrivals) an A warp's arrival for tile i comes after freeA(i - pas) or, for a warp without work,
//                      after avgdone(i - pas): either way the phase of tile i - pas is complete.
//   p3done[t % pds]   (G arrivals) warp B's arrival for tile t + pds needs avgdone(t + pds), hence fullA(t + pds), hence
//                      (some segment has work in every tile below max_tiles) dcdone(t): the chain is through with tile t.
//                      The DC-list side slots (n_e, trig_*) of tile t are reused under the same argument.
//   avgdone[t % pas]  the chain's pass of tile t + pas needs fullA(t + pas): a warp B with work has released tile t, so it
//                      is past its wait; a warp B without work (it "keeps step") is only known to have arrived at
//                      p3done(t - 1), through the dcdone(t + pas - pds) wait of a warp A with work (pds = pas + 1).
//                      Its next instructions are the wait for tile t, against pas tiles of P1 of the other warps.
#pragma once

#include "rx_decode.cuh"
#include "rx_gate.cuh"

namespace rfid_b200 {

constexpr int kT2 = 2 * kTT;                 // decimated samples per tile (two half-tiles of kTT)
constexpr int kPMaxSeg = 8;                  // segments per CTA (chain lanes 8*c + g, g < 8)
// ring depths of a launch (PackArgs::pas / pds): slots of the |y| ring and of the amplitude quotient / avg_ampl lists
// (P1 runs up to pas tiles ahead), and pds = pas + 1 DC-list slots (P1 ahead, P3 fix-ups, chain).  Four and five; three
// and four at G = kPMaxSeg, where the deeper rings do not fit the shared memory.
constexpr int kPASMax = 4;
constexpr int kPDSMax = kPASMax + 1;
__host__ __device__ constexpr int pack_ring_slots(int G) { return G < kPMaxSeg ? kPASMax : kPASMax - 1; }
constexpr int kPChainBuf = kT2 + 12;         // floats per running-sum buffer: read-ahead pad; 1072 B = 48 mod 128
constexpr int kPackMaxThreads = 1024;        // A0, A1, B per segment + loader + chain + decoders
// decoder warps of a CTA with G segments: one per segment while 4G + 2 warps fit, else whatever the CTA has left
__host__ __device__ constexpr int pack_decoders(int G)
{
  return G < kPackMaxThreads / 32 - 3 * G - 2 ? G : kPackMaxThreads / 32 - 3 * G - 2;
}
__host__ __device__ constexpr int pack_threads(int G) { return 32 * (3 * G + 2 + pack_decoders(G)); }
static_assert(pack_decoders(kPMaxSeg) >= 1 && pack_threads(kPMaxSeg) <= kPackMaxThreads, "pack kernel: warp budget");
constexpr int kYW = 4096;                    // samples of y history per segment (power of two)
constexpr int kPQ = 8;                       // queue of windows that will be decoded (opened, not yet decoded)
constexpr int kPTrig = 2;                    // windows that may open within one tile (host: len_rn16 >= kT2 / 2)
constexpr int kPackMinSmem = 116 * 1024;     // request at least this much: two CTAs never share an SM (and its history)

struct PackArgs {
  const void* iq;                            // raw capture (device, RAW::T[n_raw]), 16-byte aligned
  unsigned long long n_raw;
  const rfid_b200_segment* segs;
  int nseg;
  int seg_base;                              // added to the segment index stored in the records
  int max_windows;
  rfid_b200_window_result* results;
  int32_t* counts;
  float2* window_tap;
  float2* y_hist;                            // [%nsmid][kPMaxSeg][kYW]
  RxConfig cfg;
  int G;                                     // segments per CTA of this launch
  int pas, pds;                              // ring depths (pack_ring_slots)
  int raw_stage_samples;
  int seg_bytes;                             // per-segment shared-memory region
  int o_raw, o_tail_y, o_ring_a;             // offsets inside a segment region
  int dstage_samples;                        // per decoder warp
  int off_dA, off_dD, off_dstage, off_seg;   // offsets from the dynamic shared-memory base
  int smem_bytes;
  float scale;                               // sc16 captures: the int16 -> float factor (RawSc16::cvt)
};

// The decode of a segment's next window (sequence number n_decoded) between two of its phases (rx_decode.cuh: head,
// search chunks, finish), which the decoder warps may run one after the other on different warps.  `ctl` = window
// sequence number * 16 + next phase * 2 (+ 1 while a warp runs that phase); the candidate periods are recomputed
// (win_stream_period), the energies e[] of candidates 0..19 are the only per-lane part.
struct PackWinState {
  volatile int ctl;
  int index, head, sync_index;
  float score;
  float2 h;
  float e[20];
};
__device__ __forceinline__ int pws_ctl(int k, int phase) { return k * 16 + phase * 2; }

struct PackSegCtl {
  rfid_b200_segment seg;     // the segment's table entry (length 0: none), read from global memory once per CTA
  uint64_t raw_full[2];      // loader (TMA transaction count) -> warp A
  uint64_t raw_empty[2];     // warps A (stage 0: A0 and A1's halo read, stage 1: A1) -> loader
  uint64_t half_rdy;         // warp A0 -> warp A1: y and |y| of the first half-tile are in the rings
  uint64_t tail_rdy;         // warp A1 -> warp A0 (next tile): second half-tile in the rings, block-sum halo in `keep`
  uint64_t freeA[kPASMax];      // warp B -> warps A: masks of the tile in this slot are made, the slot may be rewritten
  float2 keep[2][4];         // the tile's last MFQ-1 block sums, by tile parity
  // windows that will be decoded, by sequence number k (slot k & (kPQ-1)): written by warp B, dc_val by the chain warp
  int q_open[kPQ], q_kind[kPQ], q_ord[kPQ];
  float2 dc_val[kPQ];
  volatile int n_opened, n_dc, n_decoded, seg_done;
  volatile int y_tiles;      // tiles whose y is complete in the history (written by warp A1, or A0 for a lone first half)
  // warp B's state that only changes at gate events (kept out of its registers)
  int b_wcount, b_nq, b_snap_base, b_queued;
  int n_e[kPDSMax];           // closed samples of the tile in DC-list slot (written by P3)
  int trig_n[kPDSMax];        // queued windows that opened in that tile: index of the trigger in the list, sequence number
  int trig_j[kPDSMax][kPTrig], trig_k[kPDSMax][kPTrig];
  PackWinState w;            // the decode of window n_decoded (warps C)
};
struct PackCtaCtl {
  uint64_t fullA[kPASMax];    // 2G warps A -> chain: P1 of the tile is in
  uint64_t avgdone[kPASMax];    // chain -> warps B: avg_ampl of the tile is final
  uint64_t p3done[kPDSMax];     // G warps B -> chain: the tile's DC list is final
  uint64_t dcdone[kPDSMax];     // chain -> warps A: the DC-list slot may be rewritten
};

#ifdef RFID_B200_PHASE_PROFILE
// developer aid (tools/pack_profile.py): absolute clock64() stamps (since CTA start) of warps A, B, C, chain of CTA 0
#define PP_DECL long long* pp_log = nullptr;
#define PP_AT(i) { if (pp_log && lane == 0) pp_log[pp_step * 8 + (i)] = clock64() - pp_cta_t0; }
#else
#define PP_DECL
#define PP_AT(i)
#endif

// hand-off waits on the critical path: the hardware parks the warp for a few dozen cycles per try
__device__ __forceinline__ void pwait(uint64_t* bar, uint32_t parity) { mbar_wait_relaxed(bar, parity, 2000); }

// One claimed phase of a window's decode (decoder pool): act 1 the head, 2 one chunk of the symbol-period search, 3 the
// rest (the head if not yet run, the remaining chunks, bit decisions, CRC) and the record.  The decode's state comes
// from and goes back to W (rx_decode.cuh's WinStream / WindowDecode: the arithmetic of decode_window_staged, resumed).
__device__ __forceinline__ void pack_decode_phase(const RxConfig& C, PackWinState& W, int kind, const WinSrc wv, int len,
                                               float2* dstage, int stage_cap, float2 dc, int phase, int act,
                                               rfid_b200_window_result* dst, int seg_id, int ord, int wopen, float2* tap,
                                               long long* pe)
{
  const int lane = threadIdx.x & 31;
  WinStream S;
  WindowDecode wd;
  if (phase == 0) {
    // the whole window present: the head through L1, as decode_window_staged; else through L2 only
    const ProgressWait l2_only{nullptr};
    win_stream_head(C, kind, wv, len, dstage, stage_cap, dc, S, wd, act == 3 ? nullptr : &l2_only);
    if (pe && lane == 0) pe[1] = clock64();
  } else {
    S.phase = phase; S.index = W.index; S.head = W.head; S.h = W.h;
    S.e = lane < 20 ? W.e[lane] : 0.0f;
    S.Tt = win_stream_period(C, lane);
    wd.sync_index = W.sync_index; wd.score = W.score; wd.h = W.h;
    wd.bits[0] = wd.bits[1] = wd.bits[2] = wd.bits[3] = 0u;
  }
  if (act == 2) {
    const long long t = pe ? clock64() : 0;
    win_stream_chunk<true>(C, wv, len, dstage, stage_cap, dc, S);
    if (pe && lane == 0) { pe[5] += clock64() - t; pe[7]++; }
  }
  if (act == 3) {
    if (pe && lane == 0) pe[6] = clock64();
    win_stream_finish<true>(C, kind, wv, len, dstage, stage_cap, dc, S, wd, nullptr, pe);
    if (lane == 0) store_result(dst, wd, seg_id, ord, wopen, len, kind);
    if (tap)
      for (int p2 = lane; p2 < len; p2 += 32) tap[p2] = c_sub(__ldcg(wv.at(p2)), dc);
  } else {
    if (lane < 20) W.e[lane] = S.e;
    if (lane == 0) { W.index = S.index; W.head = S.head; W.h = S.h; W.sync_index = wd.sync_index; W.score = wd.score; }
  }
}

// PAS = pack_ring_slots(G) of the launch (PackArgs::pas): the ring indices stay compile-time divisions
template <int DECIM, int MFQ, int PAS, class RAW>
__global__ void __launch_bounds__(kPackMaxThreads, 1) rx_pack_kernel(const PackArgs A)
{
  typedef typename RAW::T RawT;
  extern __shared__ __align__(128) unsigned char smem[];
  __shared__ PackSegCtl ctl_all[kPMaxSeg];
  __shared__ PackCtaCtl cta;
#ifdef RFID_B200_PHASE_PROFILE
  __shared__ long long pp_cta_t0;
  if (threadIdx.x == 0) pp_cta_t0 = clock64();
  int pp_step = 0;
  // per CTA on the global timer (ns), rows 512.. of the log: start, last decode done, last window closed by a gate
  unsigned long long* pp_cta = A.window_tap ? reinterpret_cast<unsigned long long*>(A.window_tap) + 512 * 8 + 4 * blockIdx.x : nullptr;
  if (pp_cta && threadIdx.x == 0) { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); pp_cta[0] = t; }
#endif

  static_assert(MFQ >= 2, "pack kernel: block-sum matched filter");
  constexpr int Q = kTT / 32;                // outputs per lane and half-tile
  static_assert(MFQ - 1 <= Q, "block-sum halo comes from the neighbouring lane only");
  static_assert(Q == 4, "four consecutive outputs per lane and half-tile");

  const int G = A.G;
  constexpr int PDS = PAS + 1;
  static_assert(PAS >= 2 && PAS <= kPASMax, "pack kernel: ring depth");
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int seg0 = blockIdx.x * G;
  const int g_act = min(G, A.nseg - seg0);   // segments this CTA really has
  const RxConfig& C = A.cfg;
  unsigned smid;
  asm("mov.u32 %0, %%smid;" : "=r"(smid));
  float2* const y_cta = A.y_hist + (size_t)smid * kPMaxSeg * kYW;

  float* const dA = reinterpret_cast<float*>(smem + A.off_dA);   // [PAS][G][kPChainBuf]
  float* const dD = reinterpret_cast<float*>(smem + A.off_dD);   // [PDS][2][G][kPChainBuf]

  // ---- init.  The loader warp initialises the raw-stage barriers itself and sends the first two half-tiles of every
  // segment on their way before it joins the start-up barrier; meanwhile the other warps initialise the hand-off barriers,
  // zero the rings (win_samples / dc_samples start at 0, gate_impl.cc:55-56) and read the segment lengths.
  int max_tiles = 0;
  if (warp == 3 * G) {
    if (lane < G) {
      PackSegCtl& c = ctl_all[lane];
      for (int s = 0; s < 2; s++) { mbar_init(&c.raw_full[s], 1); mbar_init(&c.raw_empty[s], s == 0 ? 2 : 1); }
      mbar_fence_init();
    }
    __syncwarp();
  } else {
    rfid_b200_segment sg0;       // (threads 0..G-1: the load is in flight while the barriers are initialised and the rings zeroed)
    sg0.offset = 0; sg0.length = 0; sg0.reserved = 0;
    if ((int)threadIdx.x < g_act) sg0 = A.segs[seg0 + threadIdx.x];
    if (threadIdx.x < G) {
      PackSegCtl& c = ctl_all[threadIdx.x];
      mbar_init(&c.half_rdy, 1); mbar_init(&c.tail_rdy, 1);
      for (int s = 0; s < PAS; s++) mbar_init(&c.freeA[s], 1);
      for (int m = 0; m < 4; m++) { c.keep[0][m] = make_float2(0.f, 0.f); c.keep[1][m] = make_float2(0.f, 0.f); }
      for (int s = 0; s < PDS; s++) { c.n_e[s] = 0; c.trig_n[s] = 0; }
      c.n_opened = 0; c.n_dc = 0; c.n_decoded = 0; c.seg_done = 0; c.y_tiles = 0;
      c.b_wcount = 0; c.b_nq = 1; c.b_snap_base = 0; c.b_queued = 0;
      c.w.ctl = pws_ctl(0, 0);
      mbar_fence_init();
    }
    if (threadIdx.x == 32) {
      for (int s = 0; s < PAS; s++) { mbar_init(&cta.fullA[s], 2 * G); mbar_init(&cta.avgdone[s], 1); }
      for (int s = 0; s < PDS; s++) { mbar_init(&cta.p3done[s], G); mbar_init(&cta.dcdone[s], 1); }
      mbar_fence_init();
    }
    for (int g = 0; g < G; g++) {
      unsigned char* sb = smem + A.off_seg + (size_t)g * A.seg_bytes;
      float4* ry = reinterpret_cast<float4*>(sb + A.o_tail_y);
      float4* ra = reinterpret_cast<float4*>(sb + A.o_ring_a);
      const int tid = threadIdx.x - (warp > 3 * G ? 32 : 0), nth = blockDim.x - 32;
      for (int i = tid; i < C.dc_length; i += nth) ry[i] = make_float4(0.f, 0.f, 0.f, 0.f);   // two tails of dc_length samples
      for (int i = tid; i < PAS * kT2 / 4; i += nth) ra[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    if (threadIdx.x < G) ctl_all[threadIdx.x].seg = sg0;
    asm volatile("bar.sync 14, %0;" ::"r"((int)blockDim.x) : "memory");   // start-up barrier (the loader joins it below)
    // the CTA's barriers count every warp A / B for every tile of the longest segment
    for (int g = 0; g < g_act; g++) {
      const int n_out_g = (int)(ctl_all[g].seg.length / DECIM);
      max_tiles = max(max_tiles, (n_out_g + kT2 - 1) / kT2);
    }
  }

  // the decoder pool (below): warps C from the start, each with its stage; warp A1[g] once segment g is through P1
  float2* pool_stage = nullptr;
  int pool_id = 0;
  if (warp < 3 * G) {
    // ======================================================================================= warps A0 / A1 (P1) and B (P3)
    const bool is_a = warp < 2 * G;
    const int ahalf = warp < G ? 0 : 1;       // which half-tile a P1 warp owns
    const int g = warp < G ? warp : (warp < 2 * G ? warp - G : warp - 2 * G);
    const bool have = g < g_act;
    const int seg = seg0 + g;
    rfid_b200_segment sg;
    sg.offset = 0; sg.length = 0; sg.reserved = 0;
    if (have) sg = ctl_all[g].seg;
    const int n_out = (int)(sg.length / DECIM);
    const int ntiles = (n_out + kT2 - 1) / kT2;
    PackSegCtl& B = ctl_all[g];
    unsigned char* sb = smem + A.off_seg + (size_t)g * A.seg_bytes;
    RawT* raw = reinterpret_cast<RawT*>(sb + A.o_raw);
    float2* tail_y = reinterpret_cast<float2*>(sb + A.o_tail_y);   // [2][dc_length]: the last outputs of either half-tile
    float* ring_a = reinterpret_cast<float*>(sb + A.o_ring_a);
    float2* const y_seg = y_cta + (size_t)g * kYW;
    auto bufA = [&](int tile) { return dA + (size_t)((tile % PAS) * G + g) * kPChainBuf; };
    auto bufD = [&](int tile, int comp) { return dD + (size_t)(((tile % PDS) * 2 + comp) * G + g) * kPChainBuf; };
    const float dclen_f = (float)C.dc_length;
    PP_DECL

    if (is_a) {
      // ------------------------------------------------------------------------------------- warps A0 / A1: P1 of one half-tile
      const int odd = (int)(sg.offset & (unsigned long long)(raw_granule<RAW>() - 1));   // residue of the 16-byte granule
      const float winlen_f = (float)C.win_length;
      const int h2 = ahalf;
#ifdef RFID_B200_PHASE_PROFILE
      if (seg == 0 && A.window_tap) pp_log = reinterpret_cast<long long*>(A.window_tap) + (h2 ? 256 * 8 : 0);
#endif
      for (int i = 0; i < max_tiles; i++) {
#ifdef RFID_B200_PHASE_PROFILE
        pp_step = i;
#endif
        PP_AT(0)
        const int k = 2 * i + h2;                      // half-tile index = tile index of the 128-sample kernels
        if (have && i < ntiles) {
          // the slots this tile is written into are free: warp B made the masks of tile i - PAS, the chain warp is through
          // with the DC list of tile i - PDS, and no queued window still needs the history samples about to be replaced
          if (i >= PAS) pwait(&B.freeA[i % PAS], (uint32_t)((i / PAS - 1) & 1));
          if (i >= PDS) pwait(&cta.dcdone[i % PDS], (uint32_t)((i / PDS - 1) & 1));
          if ((i + 1) * kT2 > kYW) {
            const int lowest = (i + 1) * kT2 - kYW;     // oldest history sample that survives this tile
            while (true) {
              const int nd = B.n_decoded, no = B.n_opened;
              const int need = nd < no ? B.q_open[nd & (kPQ - 1)] : 0x7fffffff;
              if (B.n_decoded == nd && need >= lowest) break;
              __nanosleep(200);
            }
          }
        } else if (i >= PAS) {
          // nothing to compute (segment over, or no segment): keep step with the CTA so that this warp's arrival can never
          // fall into an earlier phase of the barrier
          pwait(&cta.avgdone[i % PAS], (uint32_t)((i / PAS - 1) & 1));
        }
        if (k * kTT < n_out) {
          const int nvalid = min(kTT, n_out - k * kTT);  // outputs of this half-tile
          const int t0 = Q * lane;
          const RawT* stage = raw + (size_t)h2 * A.raw_stage_samples;
          const int delta = -odd - (k > 0 ? DECIM - 1 : 0);
          const int base = DECIM * t0 - (DECIM - 1) - delta;
          // ---- block sums B(n) = x[D*n-D+1 .. D*n], ascending
          float2 w[MFQ - 1 + Q];
          mbar_wait(&B.raw_full[h2], (uint32_t)(i & 1));
#pragma unroll
          for (int h = 0; h < Q; h += 2) {
            float2 x[2 * DECIM];
            if constexpr (RAW::kBytes == 4) {
              uint32_t xs[2 * DECIM];   // interior half-tiles: two outputs' raw samples, one vector run
              if (k > 0) sc16_run(stage, base + DECIM * h, xs);
#pragma unroll
              for (int j = 0; j < 2 * DECIM; j++) {
                const bool before = (k == 0) && (DECIM * (t0 + h) - (DECIM - 1) + j < 0);  // before sample 0 of the segment: +0
                x[j] = before ? make_float2(0.f, 0.f)
                              : RAW::cvt(k > 0 ? xs[j] : stage[base + DECIM * h + j], A.scale);
              }
            } else if (odd == 0 && k > 0) {
              const float4* p4 = reinterpret_cast<const float4*>(stage + base + DECIM * h);
#pragma unroll
              for (int j = 0; j < DECIM; j++) {
                const float4 v = p4[j];
                x[2 * j] = make_float2(v.x, v.y);
                x[2 * j + 1] = make_float2(v.z, v.w);
              }
            } else {   // (first half-tile of a segment, odd offsets: one pass in 28 at most)
#pragma unroll
              for (int j = 0; j < 2 * DECIM; j++) {
                const bool before = (k == 0) && (DECIM * (t0 + h) - (DECIM - 1) + j < 0);  // before sample 0 of the segment: +0
                x[j] = before ? make_float2(0.f, 0.f) : stage[base + DECIM * h + j];
              }
            }
#pragma unroll
            for (int q = 0; q < 2; q++) {
              float2 b = x[DECIM * q];
#pragma unroll
              for (int j = 1; j < DECIM; j++) b = c_add(b, x[DECIM * q + j]);
              w[MFQ - 1 + h + q] = b;
            }
          }
          // ---- the MFQ-1 block sums before this half-tile (lane 0's halo)
          float2 halo[MFQ - 1];
          if (h2 == 0) {
            // ... are the last ones of the previous tile: warp A1 left them in the keep slot (and the tile's second half in
            // the time rings, which the lookbacks below reach into)
            if (i >= 1) pwait(&B.tail_rdy, (uint32_t)((i - 1) & 1));
#pragma unroll
            for (int m = 0; m < MFQ - 1; m++) halo[m] = B.keep[(i + 1) & 1][m];
          } else {
            // ... are the last ones of the first half-tile: lanes 0..MFQ-2 recompute them from the tail of stage 0
            mbar_wait(&B.raw_full[0], (uint32_t)(i & 1));
            const RawT* stage0 = raw;
            const int delta0 = -odd - (k - 1 > 0 ? DECIM - 1 : 0);
            const int tl = kTT - (MFQ - 1) + min(lane, MFQ - 2);          // output kTT-4 .. kTT-1 of half-tile 0
            const int b0 = DECIM * tl - (DECIM - 1) - delta0;
            float2 hb = RAW::cvt(stage0[b0], A.scale);
#pragma unroll
            for (int j = 1; j < DECIM; j++) hb = c_add(hb, RAW::cvt(stage0[b0 + j], A.scale));
#pragma unroll
            for (int m = 0; m < MFQ - 1; m++) halo[m] = make_float2(__shfl_sync(0xffffffffu, hb.x, m), __shfl_sync(0xffffffffu, hb.y, m));
          }
          __syncwarp();  // raw stages consumed: the loader may refill them
          if (lane == 0) { mbar_arrive(&B.raw_empty[h2]); if (h2 == 1) mbar_arrive(&B.raw_empty[0]); }
          PP_AT(1)
#pragma unroll
          for (int m = 0; m < MFQ - 1; m++) {
            const float2 mine = w[Q + m];
            const float ux = __shfl_up_sync(0xffffffffu, mine.x, 1), uy = __shfl_up_sync(0xffffffffu, mine.y, 1);
            w[m] = lane ? make_float2(ux, uy) : halo[m];
            if (h2 == 1) {  // hand the tile's last block sums to warp A0 (read after tail_rdy)
              const float ex = __shfl_sync(0xffffffffu, mine.x, 31), ey = __shfl_sync(0xffffffffu, mine.y, 31);
              if (lane == 0) B.keep[i & 1][m] = make_float2(ex, ey);
            }
          }
          // ---- y = sum of MFQ block sums (canonical order), a = |y| (gate_impl.cc:130)
          float2 y[Q];
          float a[Q];
          bool risky = false;
#pragma unroll
          for (int q = 0; q < Q; q++) {
            y[q] = w[q];
#pragma unroll
            for (int m = 1; m < MFQ; m++) y[q] = c_add(y[q], w[q + m]);
            // outputs past the end of the segment (last, partial tile) are computed from stale shared memory: give them
            // a harmless value so that they cannot push the whole warp onto the rare exact-evaluation paths below
            if (nvalid < kTT && t0 + q >= nvalid) y[q] = make_float2(1.0f, 0.0f);
            bool rq;
            a[q] = cabsf_quick(y[q].x, y[q].y, rq);
            risky = risky || rq;
          }
          if (__any_sync(0xffffffffu, risky)) {  // rare (about one tile in 60): the exact evaluation for the whole warp
#pragma unroll
            for (int q = 0; q < Q; q++) a[q] = cabsf_ref_call(y[q].x, y[q].y);
          }
          const int ba = (i % PAS) * kT2 + h2 * kTT;   // this half-tile's place in the |y| ring
          {
            const float4 y01 = make_float4(y[0].x, y[0].y, y[1].x, y[1].y), y23 = make_float4(y[2].x, y[2].y, y[3].x, y[3].y);
            *reinterpret_cast<float4*>(ring_a + ba + t0) = make_float4(a[0], a[1], a[2], a[3]);
            float4* hy = reinterpret_cast<float4*>(y_seg + ((i * kT2 + h2 * kTT + t0) & (kYW - 1)));   // the history
            hy[0] = y01;
            hy[1] = y23;
          }
          PP_AT(2)
          __syncwarp();  // this half-tile's |y| visible to the lookback below
          if (h2 == 1) pwait(&B.half_rdy, (uint32_t)(i & 1));   // the lookbacks reach into the first half
          // ---- ring differences (gate_impl.cc:131,141).  |y| from the time ring; y from dc_length samples back: the lane
          // dc_length / 4 below (same output slot), or -- for the first lanes -- the tail the previous half-tile left.
          // (host: window / DC lengths are multiples of 4, so the groups are aligned and never straddle the ring's end)
          float xd[Q], xr[Q], xi[Q];
          {
            int ia = ba + t0 - C.win_length;
            if (ia < 0) ia += PAS * kT2;
            const float4 oa = *reinterpret_cast<const float4*>(ring_a + ia);
            xd[0] = f_sub(a[0], oa.x); xd[1] = f_sub(a[1], oa.y); xd[2] = f_sub(a[2], oa.z); xd[3] = f_sub(a[3], oa.w);
            const int dl = C.dc_length >> 2;                                   // lanes
            const float2* tprev = tail_y + (h2 ? 0 : C.dc_length);             // A0 reads A1's tail (previous tile), A1 reads A0's
            float4 t01 = make_float4(0.f, 0.f, 0.f, 0.f), t23 = t01;
            if (lane < dl) {
              t01 = *reinterpret_cast<const float4*>(tprev + 4 * lane);
              t23 = *reinterpret_cast<const float4*>(tprev + 4 * lane + 2);
            }
            float2 oy[Q];
#pragma unroll
            for (int q = 0; q < Q; q++) {
              oy[q].x = __shfl_up_sync(0xffffffffu, y[q].x, dl);
              oy[q].y = __shfl_up_sync(0xffffffffu, y[q].y, dl);
            }
            if (lane < dl) { oy[0] = make_float2(t01.x, t01.y); oy[1] = make_float2(t01.z, t01.w); oy[2] = make_float2(t23.x, t23.y); oy[3] = make_float2(t23.z, t23.w); }
#pragma unroll
            for (int q = 0; q < Q; q++) { xr[q] = f_sub(y[q].x, oy[q].x); xi[q] = f_sub(y[q].y, oy[q].y); }
            // this half-tile's own tail (the previous reader of that buffer is through: tail_rdy / half_rdy above)
            if (lane >= 32 - dl) {
              float4* tw = reinterpret_cast<float4*>(tail_y + (h2 ? C.dc_length : 0) + 4 * (lane - (32 - dl)));
              tw[0] = make_float4(y[0].x, y[0].y, y[1].x, y[1].y);
              tw[1] = make_float4(y[2].x, y[2].y, y[3].x, y[3].y);
            }
          }
          if (nvalid < kTT) {
#pragma unroll
            for (int q = 0; q < Q; q++)
              if (t0 + q >= nvalid) { xd[q] = 1.0f; xr[q] = 1.0f; xi[q] = 1.0f; }
          }
          // all twelve divisions in flight together; the multiply-correct quotients need every dividend in the verified range
          float mx = fabsf(xd[0]), mn = mx;
#pragma unroll
          for (int q = 0; q < Q; q++) {
            mx = fmaxf(fmaxf(mx, fabsf(xd[q])), fmaxf(fabsf(xr[q]), fabsf(xi[q])));
            mn = fminf(fminf(mn, fabsf(xd[q])), fminf(fabsf(xr[q]), fabsf(xi[q])));
          }
          const bool all_ok = C.win_div_fast && C.dc_div_fast && mn >= kDivFastMin && mx <= kDivFastMax;
          const bool warp_ok = __all_sync(0xffffffffu, all_ok);
          __syncwarp();
          // (every lane's lookback values have arrived, this half's tail is written: warp A1 may go on to the second half)
          if (h2 == 0 && lane == 0 && (k + 1) * kTT < n_out) mbar_arrive(&B.half_rdy);
          float qd[Q], qr[Q], qi[Q];
          if (warp_ok) {
#pragma unroll
            for (int q = 0; q < Q; q++) {
              qd[q] = f_div_fast(xd[q], winlen_f, C.win_recip);
              qr[q] = f_div_fast(xr[q], dclen_f, C.dc_recip);
              qi[q] = f_div_fast(xi[q], dclen_f, C.dc_recip);
            }
          } else {  // an exact zero, a denormal, or an unverified divisor somewhere in the warp: IEEE division
#pragma unroll
            for (int q = 0; q < Q; q++) {
              qd[q] = f_div_const_call(xd[q], winlen_f, C.win_recip, C.win_div_fast);
              qr[q] = f_div_const_call(xr[q], dclen_f, C.dc_recip, C.dc_div_fast);
              qi[q] = f_div_const_call(xi[q], dclen_f, C.dc_recip, C.dc_div_fast);
            }
          }
          if (nvalid < kTT) {
            // the segment's last, partial half-tile: the chain warp runs whole groups of 16 steps, so the slots past the
            // end hold -0.0f (x + -0.0f == x for every x, including both zeros: the running sum is carried unchanged)
#pragma unroll
            for (int q = 0; q < Q; q++)
              if (t0 + q >= nvalid) { qd[q] = -0.0f; qr[q] = -0.0f; qi[q] = -0.0f; }
          }
          *reinterpret_cast<float4*>(bufA(i) + h2 * kTT + t0) = make_float4(qd[0], qd[1], qd[2], qd[3]);
          *reinterpret_cast<float4*>(bufD(i, 0) + h2 * kTT + t0) = make_float4(qr[0], qr[1], qr[2], qr[3]);
          *reinterpret_cast<float4*>(bufD(i, 1) + h2 * kTT + t0) = make_float4(qi[0], qi[1], qi[2], qi[3]);
          __syncwarp();
          // second half-tile (and the halo) handed to warp A0's next tile
          if (h2 == 1 && lane == 0 && (k + 1) * kTT < n_out) mbar_arrive(&B.tail_rdy);
          // the tile's y is in the history (warp A1 got here after warp A0's half_rdy; a lone first half is the segment's last)
          if (lane == 0 && (h2 == 1 || (k + 1) * kTT >= n_out)) { __threadfence_block(); B.y_tiles = i + 1; }
        }
        PP_AT(3)
        __syncwarp();
        if (lane == 0) mbar_arrive(&cta.fullA[i % PAS]);   // this half of tile i is ready for the chain warp
      }
    } else {
      // ------------------------------------------------------------------------------------- warp B: P3
      // the gate (gate_impl.cc:45, global_vars.cc:47, reader_impl.cc:259,262)
      GateFsm gs = {false, 0, 0};
      bool gate_open = false;
      int to_ungate = C.len_rn16;
      bool terminated = false;
      bool was_quiet = true;      // the last tile with a closed run had no sample below its threshold
      int closed_since = C.dc_length;
      // (window count, queries, queue counters, ...: PackSegCtl::b_*, touched at gate events only.  b_snap_base = history
      // index of the DC ring's oldest entry when the last window opened)
      // y from the history; before the segment's first sample the rings hold +0 (gate_impl.cc:55-56)
      auto y_at = [&](int idx) { return idx >= 0 ? __ldcg(y_seg + (idx & (kYW - 1))) : make_float2(0.f, 0.f); };
#ifdef RFID_B200_PHASE_PROFILE
      if (seg == 0 && A.window_tap) pp_log = reinterpret_cast<long long*>(A.window_tap) + 64 * 8;
#endif
      for (int t = 0; t < max_tiles; t++) {
#ifdef RFID_B200_PHASE_PROFILE
        pp_step = t;
#endif
        PP_AT(0)
        pwait(&cta.avgdone[t % PAS], (uint32_t)((t / PAS) & 1));  // avg_ampl of tile t is final
        PP_AT(1)
        // ================================================================= P3(t): thresholds, state machine, DC list
        if (have && t < ntiles) {
          // room in the window queue for every window this tile can open (the oldest queued window has closed and its
          // dc_est is out or on its way: warp C does not depend on this warp to get through it)
          while (B.b_queued - B.n_decoded > kPQ - 1 - kPTrig) __nanosleep(200);
          const int s = t % PDS;
          int n_e = 0, ntrig = 0;
          const int nvalid = min(kT2, n_out - t * kT2);
          const int tb = t * kT2;                     // history index of the tile's first sample
          const float* davg = bufA(t);
          const float* ta = ring_a + (t % PAS) * kT2;
          float* er = bufD(t, 0);
          float* ei = bufD(t, 1);
          bool freed = false;
          auto release_a = [&]() {   // this tile's |y| and avg_ampl have been read for the last time
            if (!freed) { __syncwarp(); if (lane == 0) mbar_arrive(&B.freeA[t % PAS]); freed = true; }
          };
          if (!terminated && gate_open && to_ungate - gs.n_samples > nvalid) {
            // the whole tile lies inside an open window (gate_impl.cc:182-195): nothing to detect, no DC update
            release_a();
            gs.n_samples += nvalid;   // (n_e = 0: the chain warp skips the tile)
          } else if (!terminated) {
            // thresholds (gate_impl.cc:136,148,154).  First a one-vote test in the lanes' natural 4-sample groups: while the
            // signal is high and no sample of the tile falls below its threshold, no edge can occur (carrier only).
            unsigned ltw = 0u, gtw = 0u;   // word (lane & 7) of the below- / above-threshold masks (gate_masks)
            // (only tried when the previous tile was edge-free too: inside a reader command the test would fail every time)
            bool quiet = false;
            if (gs.sig_pos && !gate_open && nvalid == kT2 && was_quiet) {
              bool below = false;
#pragma unroll
              for (int h2 = 0; h2 < 2; h2++) {
                const float4 av = *reinterpret_cast<const float4*>(davg + h2 * kTT + 4 * lane);
                const float4 aa = *reinterpret_cast<const float4*>(ta + h2 * kTT + 4 * lane);
                below = below || aa.x < f_mul(av.x, kThreshFraction) || aa.y < f_mul(av.y, kThreshFraction) ||
                        aa.z < f_mul(av.z, kThreshFraction) || aa.w < f_mul(av.w, kThreshFraction);
              }
              quiet = !__any_sync(0xffffffffu, below);
            }
            bool have_masks = false;
            int pos = 0;
            while (pos < nvalid) {
              if (!gate_open) {
                const int run_start = pos;
                // (the one-vote result only covers a run that starts the tile with the signal high)
                PP_AT(4)
                if (!have_masks && !(quiet && run_start == 0)) {
                  gate_masks<8>(davg, ta, nvalid, ltw, gtw);
                  have_masks = true;
                  release_a();
                }
                PP_AT(5)
                was_quiet = !__any_sync(0xffffffffu, ltw != 0u);
                const int p_open = gate_closed_run<8>(ltw, gtw, run_start, nvalid, C.n_T1, C.n_PW / 2, gs);
                PP_AT(6)
                const bool opened = p_open >= 0;
                pos = opened ? p_open + 1 : nvalid;
                // ---- DC tracker inputs of the closed run [run_start, pos) (gate_impl.cc:141-143; includes the trigger).
                // The list keeps the tile's natural positions: P1's time-contiguous differences are exact except for the
                // first dc_length samples after a window, whose ring entries date from before the window -- those are
                // recomputed here (y from the history); samples inside windows get -0.0f below (x + -0.0f == x).
                const int len = pos - run_start;
                if (closed_since < C.dc_length) {
                  const int nfix = min(len, C.dc_length - closed_since);
                  const int snap0 = B.b_snap_base;
#pragma unroll 1
                  for (int j0 = 0; j0 < nfix; j0 += 64) {
                    float2 yv[2], ov[2];
#pragma unroll
                    for (int u = 0; u < 2; u++) {
                      const int j = j0 + 32 * u + lane;
                      const bool valid = j < nfix;
                      yv[u] = y_at(tb + run_start + (valid ? j : 0));
                      ov[u] = y_at(snap0 + closed_since + (valid ? j : 0));
                    }
#pragma unroll
                    for (int u = 0; u < 2; u++) {
                      const int j = j0 + 32 * u + lane;
                      const bool valid = j < nfix;
                      const float xr = valid ? f_sub(yv[u].x, ov[u].x) : 1.0f, xi = valid ? f_sub(yv[u].y, ov[u].y) : 1.0f;
                      float qr, qi;
                      if (__all_sync(0xffffffffu, C.dc_div_fast && f_div_fast_ok(xr) && f_div_fast_ok(xi))) {
                        qr = f_div_fast(xr, dclen_f, C.dc_recip);
                        qi = f_div_fast(xi, dclen_f, C.dc_recip);
                      } else {
                        qr = f_div_const_call(xr, dclen_f, C.dc_recip, C.dc_div_fast);
                        qi = f_div_const_call(xi, dclen_f, C.dc_recip, C.dc_div_fast);
                      }
                      if (valid) { er[run_start + j] = qr; ei[run_start + j] = qi; }
                    }
                  }
                }
                PP_AT(7)
                closed_since = min(closed_since + len, 1 << 24);
                n_e = pos;
                if (opened) {
                  // READER COMMAND DETECTED (gate_impl.cc:164-180): the DC ring stands as it is now
                  gate_open = true;
                  const int open_idx = tb + pos - 1, wcount = B.b_wcount, n_queued = B.b_queued;
                  // a window is decoded when it closes inside the segment (its length is known now); windows beyond
                  // max_windows are not decoded
                  const bool cur_store = wcount < A.max_windows && ntrig < kPTrig && open_idx + to_ungate <= n_out;
                  __syncwarp();
                  if (lane == 0) {
                    B.b_snap_base = open_idx - C.dc_length + 1;
                    if (cur_store) {
                      // queue the window for warp C; dc_est right after the trigger sample follows from the chain warp
                      const int qs = n_queued & (kPQ - 1);
                      B.q_open[qs] = open_idx; B.q_kind[qs] = wcount & 1; B.q_ord[qs] = wcount;
                      B.trig_j[s][ntrig] = pos - 1; B.trig_k[s][ntrig] = n_queued;
                      B.b_queued = n_queued + 1;
                      __threadfence_block();
                      B.n_opened = n_queued + 1;
                    }
                  }
                  __syncwarp();
                  if (cur_store) ntrig++;
                }
              } else {
                // ---- open: samples pass through (gate_impl.cc:182-195); warp C reads them from the history.  They do not
                // enter the DC tracker: their list entries carry the running sums unchanged
                const int take = min(to_ungate - gs.n_samples, nvalid - pos);
                for (int j = lane; j < take; j += 32) { er[pos + j] = -0.0f; ei[pos + j] = -0.0f; }
                gs.n_samples += take; pos += take;
                n_e = pos;
                if (gs.n_samples >= to_ungate) {
                  gate_open = false;
#ifdef RFID_B200_PHASE_PROFILE
                  if (pp_cta && lane == 0) { unsigned long long tg; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(tg)); atomicMax(pp_cta + 2, tg); }
#endif
                  const int wcount = B.b_wcount, nq = B.b_nq;
                  const int kind = wcount & 1;  // windows alternate RN16, EPC (SURVEY.md 3.5)
                  __syncwarp();
                  if (lane == 0) {
                    B.b_wcount = wcount + 1;
                    if (kind) B.b_nq = nq + 1;
                  }
                  __syncwarp();
                  closed_since = 0;
                  // ACK after RN16 -> GATE_SEEK_EPC, Query/QueryRep after EPC -> GATE_SEEK_RN16 (gate_impl.cc:112-123)
                  to_ungate = kind ? C.len_rn16 : C.len_epc;
                  gs.n_samples = 0;
                  if (kind && nq + 1 > C.max_queries) { terminated = true; break; }  // gate_impl.cc:101-109
                }
              }
            }
          }
          release_a();
          if (terminated) {
            // the list ends where the reader stopped: pad its last group of 16 with -0.0f (see P1)
            const int n16 = (n_e + 15) & ~15;
            if (lane < 16 && n_e + lane < n16) { er[n_e + lane] = -0.0f; ei[n_e + lane] = -0.0f; }
          }
          if (lane == 0) { B.n_e[s] = n_e; B.trig_n[s] = ntrig; }
        } else if (have && lane == 0) {
          // segment over, the CTA's longer segments go on: an empty DC list, so that the chain warp does not replay this
          // slot's list of PDS tiles ago (and overwrite dc_val of a window still waiting for its decode)
          B.n_e[t % PDS] = 0; B.trig_n[t % PDS] = 0;
        }
        PP_AT(2)
        __syncwarp();
        if (lane == 0) mbar_arrive(&cta.p3done[t % PDS]);   // the tile's DC list is final
      }
      // ---- end of the segment
      if (have && lane == 0) A.counts[seg] = B.b_wcount;
      if (lane == 0) { __threadfence_block(); B.seg_done = 1; }
    }
  } else if (warp == 3 * G + 1) {
    // ======================================================================================= chain warp
    // lane 8*c + g: running sum c (0 avg_ampl, 1 dc_est.re, 2 dc_est.im) of segment g
    const int comp = lane >> 3, g = lane & 7;
    const bool active = comp < 3 && g < g_act;
    int n_out = 0;
    if (active) n_out = (int)(ctl_all[g].seg.length / DECIM);
    float acc = 0.f;
    PP_DECL
#ifdef RFID_B200_PHASE_PROFILE
    if (blockIdx.x == 0 && A.window_tap) pp_log = reinterpret_cast<long long*>(A.window_tap) + 128 * 8;
#endif
    // avg_ampl of tile ia as soon as every segment's P1(ia) is in, dc_est of tile id as soon as every segment's P3(id) has
    // fixed its list -- whichever is ready, both in ONE convergent loop when both are
    int ia = 0, id = 0;
    while (ia < max_tiles || id < max_tiles) {
      PP_AT(0)
      bool ra = false, rd = false;
      while (true) {
        ra = ia < max_tiles && mbar_test_wait(&cta.fullA[ia % PAS], (uint32_t)((ia / PAS) & 1));
        rd = id < ia && mbar_test_wait(&cta.p3done[id % PDS], (uint32_t)((id / PDS) & 1));
        if (ra || rd) break;
        __nanosleep(20);
      }
#ifdef RFID_B200_PHASE_PROFILE
      pp_step = ra ? ia : 32 + id;
#endif
      PP_AT(1)
      {
        // branch-free selection of this lane's buffer and length
        const int n_avg = ra ? min(kT2, max(0, n_out - ia * kT2)) : 0;
        const int n_dc = (rd && active && comp > 0) ? ctl_all[g].n_e[id % PDS] : 0;
        const int n = active ? (comp == 0 ? n_avg : n_dc) : 0;
        const int ofsA = ((ia % PAS) * G + g) * kPChainBuf;
        const int ofsD = (((id % PDS) * 2 + (comp - 1)) * G + g) * kPChainBuf;
        float* buf = comp == 0 ? dA + (ia < max_tiles ? ofsA : 0) : dD + (active && comp > 0 && id < max_tiles ? ofsD : 0);
        const int n16 = (n + 15) & ~15;
        __syncwarp();
        chain_inplace(buf, n16, acc);
        __syncwarp();
        if (ra) {
          if (lane == 0) mbar_arrive(&cta.avgdone[ia % PAS]);
          ia++;
        }
        // ---- dc_est right after the trigger sample of every queued window that opened in tile id: hand it to warp C
        if (rd) {
          if (active && comp > 0) {
            PackSegCtl& S = ctl_all[g];
            const int s = id % PDS;
            const int tn = S.trig_n[s];
            for (int e = 0; e < tn; e++) {
              const float v = buf[S.trig_j[s][e]];
              float* dst = reinterpret_cast<float*>(&S.dc_val[S.trig_k[s][e] & (kPQ - 1)]);
              dst[comp - 1] = v;
            }
          }
          __syncwarp();
          if (active && comp == 1) {
            PackSegCtl& S = ctl_all[g];
            const int tn = S.trig_n[id % PDS];
            if (tn > 0) { __threadfence_block(); S.n_dc = S.n_dc + tn; }
          }
          __syncwarp();
          if (lane == 0) mbar_arrive(&cta.dcdone[id % PDS]);
          id++;
        }
      }
      PP_AT(2)
    }
  } else if (warp == 3 * G) {
    // ======================================================================================= loader warp
    // lane g streams the raw half-tiles of segment g through its two stages (TMA bulk copies) as warp A frees them; the
    // first two go out before the start-up barrier
    const int g = lane;
    rfid_b200_segment sg;
    sg.offset = 0; sg.length = 0; sg.reserved = 0;
    if (g < g_act) sg = A.segs[seg0 + g];
    const int n_out = (int)(sg.length / DECIM);
    const int nhalf = g < g_act ? (n_out + kTT - 1) / kTT : 0;
    PackSegCtl& B = ctl_all[g < G ? g : 0];
    RawT* raw = reinterpret_cast<RawT*>(smem + A.off_seg + (size_t)(g < G ? g : 0) * A.seg_bytes + A.o_raw);
    const RawT* const iq = static_cast<const RawT*>(A.iq);
    const InteriorTiles<RawT> fast = interior_tiles<DECIM, RAW>(iq, A.n_raw, sg, nhalf);
    const unsigned long long pol = l2_policy_evict_first();   // every raw sample is read exactly once
    auto issue = [&](int k) {
      const int rs_ = k & 1;
      RawT* dst = raw + (size_t)rs_ * A.raw_stage_samples;
      if (k >= 1 && k < fast.n) {
        mbar_arrive_expect_tx(&B.raw_full[rs_], fast.bytes);
        tma_load_1d_hint(dst, fast.src + (size_t)k * (DECIM * kTT), fast.bytes, &B.raw_full[rs_], pol);
      } else {
        issue_tile_load<DECIM, RAW>(iq, A.n_raw, sg, k, dst, &B.raw_full[rs_]);
      }
    };
    for (int k = 0; k < 2 && k < nhalf; k++) issue(k);   // both stages are free at the start
    __syncwarp();
    asm volatile("bar.sync 14, %0;" ::"r"((int)blockDim.x) : "memory");   // start-up barrier
    for (int k = 2; k < nhalf; k++) {
      mbar_wait_idle(&B.raw_empty[k & 1], (uint32_t)(((k >> 1) - 1) & 1), 100);
      issue(k);
    }
  } else {
    pool_stage = reinterpret_cast<float2*>(smem + A.off_dstage) + (size_t)(warp - 3 * G - 2) * A.dstage_samples;
    pool_id = warp - 3 * G - 2;
  }
  if (warp >= G && warp < 2 * G) {
    // Warp A1[g] once segment g is through P1 (recomputed here: nothing of the pool stays live through P1's loop).  The
    // segment's raw stages are free once its last tile is in the history (y_tiles moves after the tile's last read of
    // them; a lone first half is warp A0's, and the loader's last copy went to it): warp A1 joins the decoder pool with
    // them as its stage -- the segments' last windows close towards the end of the CTA, when warps A are done.
    const int g = warp - G;
    if (g < g_act) {
      const int ntiles = ((int)(ctl_all[g].seg.length / DECIM) + kT2 - 1) / kT2;
      while (ctl_all[g].y_tiles < ntiles) __nanosleep(200);
    }
    pool_stage = reinterpret_cast<float2*>(smem + A.off_seg + (size_t)g * A.seg_bytes + A.o_raw);
    pool_id = pack_decoders(G) + g;
  }
  if (pool_stage) {
    // ======================================================================================= decoder pool: warps C, A1
    // The decoder warps are ONE pool over the phases of every segment's next window (rx_decode.cuh): the head of an EPC
    // window and the chunks of its symbol-period search may run as soon as the samples they read are in the history,
    // while the gate is still receiving the window (warp A runs ahead of it), and its finish (the remaining chunks, the
    // 128 bit decisions, the CRC) once the whole window is; an RN16 window is one unit (its finish reads the stage its
    // head filled).  Every phase needs dc_est right after the window's trigger sample, which the chain warp hands over
    // two tiles after the gate opened the window -- by then warp A is about a tile short of the window's end, so the head
    // usually runs early and the chunks rarely (tools/pack_profile.py).  An idle warp takes the runnable phase of the
    // window with the most phases left (lowest segment first among equals) and claims it by a compare-and-swap on the
    // window's ctl word: one phase of a window runs at a time, and its state between phases lives in PackSegCtl::w.  A
    // segment's windows finish in order and n_decoded moves only after the finish, so warp A's guard of the history
    // keeps its meaning.  Which warp runs a phase does not change its result: the records are the same bits.
    float2* const dstage = pool_stage;
    const unsigned FULL = 0xffffffffu;
#ifdef RFID_B200_PHASE_PROFILE
    // segment 0 of CTA 0: per window k, row k = opened seen, first phase starts, decoded, finish starts (cycles since
    // CTA start); rows 60 (EPC) / 61 (RN16): clock64() at head start, head end, search end, bit samples end, CRC end,
    // cycles spent in search chunks before the finish, finish start, number of those chunks
    long long* const pp_c0 = (seg0 == 0 && A.window_tap) ? reinterpret_cast<long long*>(A.window_tap) + 192 * 8 : nullptr;
#endif
    while (true) {
      // lane g looks at segment g: is its next window's next phase runnable (key > 0), is anything left (pending)
      bool pending = false;
      unsigned key = 0u;       // (phases left + 1) * 16 + 15 - g
      int st = 0, act = 0;     // the ctl word seen; what to run: 1 the head, 2 one search chunk, 3 the rest of the decode
      if (lane < g_act) {
        PackSegCtl& S = ctl_all[lane];
        const int done = S.seg_done;   // (read before the counters: once set, they are final)
        const int kg = S.n_decoded, no = S.n_opened;
        pending = no > kg || !done;
        if (no > kg) {
          __threadfence_block();
#ifdef RFID_B200_PHASE_PROFILE
          if (pp_c0 && lane == 0 && pp_c0[kg * 8] == 0) pp_c0[kg * 8] = clock64() - pp_cta_t0;
#endif
          st = S.w.ctl;
          if ((st >> 4) == kg && !(st & 1) && S.n_dc > kg) {
            const int qs = kg & (kPQ - 1);
            const int kind = S.q_kind[qs];
            const int len = kind ? C.len_epc : C.len_rn16;
            const int avail = S.y_tiles * kT2 - S.q_open[qs];   // the window's samples in the history
            const int phase = (st >> 1) & 7;
            if (avail >= len) {
              act = 3;
            } else if (kind && phase == 0) {
              act = avail >= win_head_samples(C, kind, len, A.dstage_samples) ? 1 : 0;
            } else if (kind && phase <= kSearchChunks) {
              act = avail >= win_chunk_need(C, S.w.index, phase - 1, len) ? 2 : 0;
            }
            if (act) key = (unsigned)(kind ? kSearchChunks + 3 - phase : 2) * 16u + 15u - (unsigned)lane;
          }
        }
      }
      if (!__any_sync(FULL, pending)) break;
      const unsigned best = __reduce_max_sync(FULL, key);
      if (best == 0u) { __nanosleep(200); continue; }
      const int g = 15 - (int)(best & 15u);
      int won = 0;
      if (lane == g) won = atomicCAS(const_cast<int*>(&ctl_all[g].w.ctl), st, st | 1) == st;
      if (!__shfl_sync(FULL, won, g)) continue;   // another warp was first
      st = __shfl_sync(FULL, st, g);
      act = __shfl_sync(FULL, act, g);
      __threadfence_block();
      const int k = st >> 4, phase = (st >> 1) & 7;
      const int seg = seg0 + g;
      PackSegCtl& B = ctl_all[g];
      PackWinState& W = B.w;
      const int qs = k & (kPQ - 1);
      const int kind = B.q_kind[qs], ord = B.q_ord[qs], wopen = B.q_open[qs];
      const float2 dc = B.dc_val[qs];
      const int len = kind ? C.len_epc : C.len_rn16;
      const WinSrc wv{y_cta + (size_t)g * kYW, wopen, kYW - 1};
#ifdef RFID_B200_PHASE_PROFILE
      long long* const pw = (pp_c0 && g == 0) ? pp_c0 : nullptr;
      long long* const pe = pw ? pw + (kind ? 60 : 61) * 8 : nullptr;
      const long long pp_t = clock64();
      // every claim of CTA 0 (rows 1024..; count at row 1023): warp | segment | window | what | phase, start, end
      long long* pp_claim = nullptr;
      if (pp_c0 && lane == 0) {
        const long long n = atomicAdd(reinterpret_cast<unsigned long long*>(pp_c0) + (1023 - 192) * 8, 1ull);
        if (n < 1024) pp_claim = pp_c0 + (1024 - 192) * 8 + 4 * n;
      }
      if (pp_claim) { pp_claim[0] = pool_id | g << 8 | k << 16 | act << 24 | phase << 28; pp_claim[1] = pp_t - pp_cta_t0; }
      if (pw && lane == 0 && phase == 0) { pw[k * 8 + 1] = pp_t - pp_cta_t0; pe[0] = pp_t; pe[5] = 0; pe[7] = 0; }
      if (pw && lane == 0 && act == 3) pw[k * 8 + 3] = pp_t - pp_cta_t0;
      float2* const tap = nullptr;   // (the profile log)
#else
      long long* const pe = nullptr;
      float2* const tap = A.window_tap ? A.window_tap + ((size_t)(seg + A.seg_base) * A.max_windows + ord) * C.len_epc : nullptr;
#endif
      pack_decode_phase(C, W, kind, wv, len, dstage, A.dstage_samples, dc, phase, act,
                        A.results + (size_t)seg * A.max_windows + ord, seg + A.seg_base, ord, wopen, tap, pe);
      __syncwarp();
      if (act == 3) {
#ifdef RFID_B200_PHASE_PROFILE
        if (pw && lane == 0) pw[k * 8 + 2] = clock64() - pp_cta_t0;
        if (pp_cta && lane == 0) { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); atomicMax(pp_cta + 1, t); }
#endif
        if (lane == 0) {
          // the next window's state first: a warp that still reads n_decoded == k sees a ctl word of window k + 1
          __threadfence_block();
          W.ctl = pws_ctl(k + 1, 0);
          __threadfence_block();
          B.n_decoded = k + 1;   // warp A may reuse the window's history samples
        }
      } else if (lane == 0) {
        __threadfence_block();
        W.ctl = pws_ctl(k, act == 1 ? 1 : phase + 1);
      }
#ifdef RFID_B200_PHASE_PROFILE
      if (pp_claim) pp_claim[2] = clock64() - pp_cta_t0;
#endif
    }
  }
}

}  // namespace rfid_b200
