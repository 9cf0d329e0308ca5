// rx_gate.cuh -- the gate's reader-command detection for every capture kernel: the threshold masks of a tile and the
// edge / pulse state machine of one closed run (gate_impl.cc:136-180), on the masks of a tile of 32 W samples held one
// 32-bit word per lane (W = 4: the 128-sample tiles of rx_fused_kernel and rx_fused_split_kernel; W = 8: the
// 256-sample tiles of rx_pack_kernel).
#pragma once

#include "rx_common.cuh"

namespace rfid_b200 {

__device__ __forceinline__ unsigned m_below(int n) { return n <= 0 ? 0u : (n >= 32 ? 0xffffffffu : ((1u << n) - 1u)); }

// Thresholds (gate_impl.cc:136,148,154): bit p of ltw / gtw is a[p] < 0.75 avg[p] / a[p] > 0.75 avg[p].  Lane l gets
// word l % W of both masks; samples at or past nvalid (the segment's end) compare nothing.
template <int W>
__device__ __forceinline__ void gate_masks(const float* avg, const float* a, int nvalid, unsigned& ltw, unsigned& gtw)
{
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int r = 0; r < W; r++) {
    const int p = r * 32 + lane;
    const float thr = f_mul(avg[p], kThreshFraction);
    const float av = a[p];
    const unsigned bl = __ballot_sync(0xffffffffu, av < thr), bg = __ballot_sync(0xffffffffu, av > thr);
    if ((lane & (W - 1)) == r) { ltw = bl; gtw = bg; }
  }
  const unsigned vm = m_below(nvalid - (lane & (W - 1)) * 32);
  ltw &= vm;
  gtw &= vm;
}

// The reference walks the closed samples one by one (gate_impl.cc:145-180):
//     n_samples++;  POS && a < thr -> NEG, n_samples = 0;  NEG && a > thr -> POS, n_samples = 0, a pulse when
//     n_samples > n_PW/2 (num_pulses++, else num_pulses = 0);  open when POS && n_samples > n_T1 && num_pulses > 5.
struct GateFsm {
  bool sig_pos;              // signal_state == POS_EDGE
  int n_samples, num_pulses;
};

// The same decisions for the closed samples [from, nvalid) of a tile, from its masks (gate_masks), all at once:
//   carrier    signal high and no sample of the tile below its threshold (the common case): only the open test remains
//   states     state' = rise | keep & state is the carry recurrence of a binary addition; inside a word one 64-bit add,
//              across the words the same recurrence once more (generate = the word's sum overflows with carry-in 0,
//              propagate = only with carry-in 1), i.e. one more addition on the two ballots
//   pulses     a rise at p is a valid pulse when the fall before it is more than half_pw back: no fall bit at p-1 .. p-half_pw
//   num_pulses valid rises since the last invalid one (plus the carried count while no invalid rise has occurred)
//   opening    the carried state reaches n_T1 before the first edge, or a rise r with num_pulses > 5 is followed by
//              n_T1 + 1 edge-free samples inside the tile (the gate opens at r + 1 + n_T1; a fall there wins)
// Positions and counts are combined with redux.sync / vote (one instruction each); the reductions of the common path
// (a tile full of reader pulses, no opening) do not depend on each other, so they are in flight together.
// Returns the position at which the gate opens (the trigger sample; st is then the open gate's) or -1 (st advanced to
// the end of the tile).
// Precondition: half_pw <= 24 (win_length <= kMaxWinLen = 1024, so fs_dec <= 4.096 MHz and n_PW <= 49): the falls that
// spoil a rise lie in its own mask word or the one below.
template <int W>
__device__ __forceinline__ int gate_closed_run(unsigned ltw, unsigned gtw, int from, int nvalid, int n_T1, int half_pw,
                                               GateFsm& st)
{
  const unsigned FULL = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  const int w = lane & (W - 1);
  const bool own = lane < W;
  const int base = 32 * w;
  if (st.sig_pos && !__any_sync(FULL, ltw != 0u)) {
    if (st.num_pulses > kNumPulsesCommand) {
      const int p_open = from + max(0, n_T1 - st.n_samples);
      if (p_open < nvalid) { st.num_pulses = 0; st.n_samples = 1; return p_open; }
    }
    st.n_samples += nvalid - from;
    return -1;
  }
  const unsigned live = own ? ~m_below(from - base) : 0u;   // (lanes W..31 carry empty words)
  const unsigned F = ltw & live, R = gtw & live;
  const unsigned Pk = ~(F | R);
  const unsigned long long sum0 = (unsigned long long)(R | Pk) + R, sum1 = sum0 + 1ull;
  const unsigned C0 = __ballot_sync(FULL, own && (sum0 >> 32) != 0ull);
  const unsigned C1 = __ballot_sync(FULL, own && (sum1 >> 32) != 0ull);
  const unsigned cv = (C1 + C0 + (st.sig_pos ? 1u : 0u)) ^ C1 ^ C0;   // bit k: carry into word k (C0 is a subset of C1)
  const unsigned X = Pk ^ (unsigned)(((cv >> w) & 1u) ? sum1 : sum0);   // state before each position
  const unsigned RS = ~X & R, FE = X & F, E = RS | FE;
  const int e_first = __reduce_min_sync(FULL, E ? base + __ffs(E) - 1 : 1024);
  const int e_last = __reduce_max_sync(FULL, E ? base + 31 - __clz(E) : -1);
  const int r_last = __reduce_max_sync(FULL, RS ? base + 31 - __clz(RS) : -1);
  const unsigned fe_prev = __shfl_up_sync(FULL, FE, 1);
  const int first_edge = e_first < nvalid ? e_first : nvalid;
  if (st.sig_pos && st.num_pulses > kNumPulsesCommand) {
    const int p_open = from + max(0, n_T1 - st.n_samples);
    if (p_open < first_edge && p_open < nvalid) {
      st.sig_pos = true; st.num_pulses = 0; st.n_samples = 1;
      return p_open;
    }
  }
  if (e_first >= nvalid) { st.n_samples += nvalid - from; return -1; }
  const unsigned fe_lo = w == 0 ? 0u : fe_prev;
  unsigned knock = 0u;
  for (int k = 1; k <= half_pw; k++) knock |= (FE << k) | (fe_lo >> (32 - k));
  unsigned VR = RS & ~knock;
  // the first edge, if it is a rise: its pulse began before the run
  if ((e_first >> 5) == w && ((RS >> (e_first & 31)) & 1u) && !(st.n_samples + (e_first - from + 1) > half_pw))
    VR &= ~(1u << (e_first & 31));
  const unsigned IR = RS & ~VR;
  const int lim = nvalid - 1 - n_T1;  // rises at or above lim cannot open the gate within this tile
  // An opening rise is followed by n_T1 + 1 edge-free positions; when that is 64 or more, the stretch covers a whole
  // mask word, so a tile without an edge-free word below nvalid has no candidate.
  if (lim > 0 && (n_T1 + 1 < 64 || __any_sync(FULL, own && base < nvalid && E == 0u))) {
    unsigned cand;   // the rises followed by n_T1 + 1 edge-free positions
    if (n_T1 + 1 < 32) {
      // the stretch ends in the rise's word or the one above: shift the edges of both down over it
      const unsigned e_up = __shfl_down_sync(FULL, E, 1);
      unsigned shadow = 0u;
      for (int k = 1; k <= n_T1 + 1; k++) shadow |= (E >> k) | (e_up << (32 - k));
      cand = RS & ~shadow & m_below(lim - base);
    } else {
      // the stretch covers the rest of the rise's word: the rise is the word's highest edge, and the first edge of the
      // words above it (suffix minimum over the lanes) decides
      const int hi = E ? 31 - __clz(E) : -1;
      int nx = __shfl_down_sync(FULL, E ? base + __ffs(E) - 1 : 1024, 1);
#pragma unroll
      for (int d = 1; d < W; d *= 2) nx = min(nx, __shfl_down_sync(FULL, nx, d));
      const int rr = base + hi;
      cand = hi >= 0 && ((RS >> hi) & 1u) && rr < lim && nx > rr + 1 + n_T1 ? 1u << hi : 0u;
    }
    // in order; at most nvalid / (n_T1 + 1) rises qualify
    while (true) {
      const int r = __reduce_min_sync(FULL, cand ? base + __ffs(cand) - 1 : 1024);
      if (r >= 1024) break;
      if ((r >> 5) == w) cand &= ~(1u << (r & 31));
      // num_pulses right after the rise at r
      const unsigned upto = m_below(r + 1 - base);
      const unsigned im = IR & upto;
      const int last = __reduce_max_sync(FULL, im ? base + 31 - __clz(im) : -1);
      const int cnt = __reduce_add_sync(FULL, __popc(VR & upto & ~m_below(last + 1 - base)));
      if ((last >= 0 ? cnt : st.num_pulses + cnt) > kNumPulsesCommand) {
        st.sig_pos = true; st.num_pulses = 0; st.n_samples = 1;
        return r + 1 + n_T1;
      }
    }
  }
  st.sig_pos = e_last == r_last;            // the last edge is a rise
  st.n_samples = nvalid - 1 - e_last;
  if (r_last >= 0) {
    // valid rises after the last invalid one: the words above the last word that holds an invalid rise, and that word's
    // bits above it
    const unsigned Lm = __ballot_sync(FULL, IR != 0u);
    unsigned mine = VR;
    if (Lm) {
      const int L = 31 - __clz(Lm);
      if (w < L) mine = 0u;
      else if (w == L && IR) mine = VR & ~((2u << (31 - __clz(IR))) - 1u);
    }
    const int cnt = __reduce_add_sync(FULL, own ? __popc(mine) : 0);
    st.num_pulses = Lm ? cnt : st.num_pulses + cnt;
  }
  return -1;
}

}  // namespace rfid_b200
