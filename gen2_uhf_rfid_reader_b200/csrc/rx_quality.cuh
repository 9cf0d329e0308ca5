// rx_quality.cuh -- reply energy, decision SNR and slot outcome of every stored window (rfid_b200_window_quality; the
// rule is stated in include/rfid_b200.h).  One warp per record slot reads the window back from the window tap (the
// DC-removed gate output the decoder read), projects the decoder's own samples (rx_decode.cuh positions, c_proj) and
// sums in float64 in one fixed order, so that tests/quality_model.py restates it bit for bit.
#pragma once

#include "rx_decode.cuh"

namespace rfid_b200 {

constexpr int kSlotWarps = 4;   // warps (= record slots) per CTA of the kernels that read the window tap

struct QualityArgs {
  const float2* windows;                    // window tap: slot s * max_windows + k at stride cfg.len_epc
  const rfid_b200_window_result* results;
  const int32_t* counts;
  rfid_b200_quality* quality;
  int nseg, max_windows;
  double empty_ratio, single_ratio;         // linear thresholds
  RxConfig cfg;
};

// sum over the warp of one float64 per lane, lane 0 first (the same value in every lane)
__device__ __forceinline__ double quality_lane_sum(double part)
{
  double t = 0.0;
#pragma unroll 4
  for (int l = 0; l < 32; l++) t = __dadd_rn(t, __shfl_sync(0xffffffffu, part, l));
  return t;
}

// sum of |w|^2 = re^2 + im^2 (both squares exact in float64) over window samples [0, h1) and then [t0, t1): the i-th of
// them goes to lane i % 32
__device__ __forceinline__ double quality_power_sum(const float2* w, int h1, int t0, int t1)
{
  double part = 0.0;
  const int count = h1 + (t1 - t0);
  for (int i = (int)(threadIdx.x & 31); i < count; i += 32) {
    const float2 v = __ldg(w + (i < h1 ? i : t0 + (i - h1)));
    const double x = v.x, y = v.y;
    part = __dadd_rn(part, __dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)));
  }
  return quality_lane_sum(part);
}

// A stored record and its window as the decoder read it back from the window tap
struct TapWindow {
  long long slot;                       // s * max_windows + k
  const rfid_b200_window_result* rec;
  const float2* w;                      // the window's samples in the tap
  int n;                                // rec.length clamped to [0, len_epc]
  int index;                            // the decoder's data index
  float2 h;
  float T, twoT;
};

// The record slot of this warp (kSlotWarps per CTA) and its window.  False for a slot beyond nseg * max_windows or
// beyond its segment's stored records.  ARGS: a stage's arguments (windows, results, counts, nseg, max_windows, cfg).
template <class ARGS>
__device__ __forceinline__ bool tap_window(const ARGS& A, TapWindow& t)
{
  const long long slot = (long long)blockIdx.x * kSlotWarps + (threadIdx.x >> 5);
  if (slot >= (long long)A.nseg * A.max_windows) return false;
  const int seg = (int)(slot / A.max_windows), k = (int)(slot % A.max_windows);
  if (k >= min(A.counts[seg], A.max_windows)) return false;
  const RxConfig& c = A.cfg;
  const rfid_b200_window_result& rec = A.results[slot];
  t.slot = slot;
  t.rec = &rec;
  t.w = A.windows + slot * c.len_epc;
  t.n = max(0, min(rec.length, c.len_epc));
  t.index = win_data_index(c, rec.sync_index);
  t.h = make_float2(rec.h_re, rec.h_im);
  t.T = rec.T;
  t.twoT = f_mul(2.0f, t.T);
  return true;
}

// EPC decision j's projection r_j = c_proj(s_a, s_b, h) at the decoder's positions, a sample outside [0, n) taken as 0
// (the window-quality, EPC-recovery and EPC-match rules all use it).  Each kernel calls it once per decision inside
// its own loop over a lane's decisions j = 32 q + l: gathering all four into an array first holds more loads in flight
// and costs the recovery kernel six registers.
__device__ __forceinline__ float epc_projection(const TapWindow& t, int j)
{
  const float2 zero = make_float2(0.0f, 0.0f);
  const int pa = win_epc_pos_a(j, t.twoT, t.index), pb = win_epc_pos_b(j, t.T, t.index);
  const float2 sa = (pa >= 0 && pa < t.n) ? __ldg(t.w + pa) : zero;
  const float2 sb = (pb >= 0 && pb < t.n) ? __ldg(t.w + pb) : zero;
  return c_proj(sa, sb, t.h);
}

__device__ __forceinline__ float quality_canonical(double v)
{
  return v != v ? __int_as_float(0x7fc00000) : __double2float_rn(v);   // (one NaN pattern, numpy's)
}

__global__ void __launch_bounds__(32 * kSlotWarps) rx_quality_kernel(const QualityArgs A)
{
  const int lane = threadIdx.x & 31;
  TapWindow t;
  if (!tap_window(A, t)) return;
  const RxConfig& c = A.cfg;
  const int kind = t.rec->kind, sync = t.rec->sync_index, n = t.n;
  const float2 zero = make_float2(0.0f, 0.0f);
  double a1 = 0.0, a2 = 0.0;   // this lane's sums of |r_j| and r_j^2
  int n_dec, reply_end;
  if (kind == RFID_B200_RN16) {
    const float half = f_mul(c.n_tag_bit_f, 0.5f);
    const float jm = win_rn16_halfbit(t.index, half, lane);
    if (__ballot_sync(0xffffffffu, jm < (float)n) != 0xffffffffu) {   // the decoder made no decision (crc_ok -2)
      if (lane == 0) {
        const float nan = __int_as_float(0x7fc00000);
        A.quality[t.slot] = rfid_b200_quality{nan, nan, RFID_B200_SLOT_EMPTY, 0};
      }
      return;
    }
    const int p = (int)roundf(jm);
    const float2 s = (p >= 0 && p < n) ? __ldg(t.w + p) : zero;
    const float2 s_next = make_float2(__shfl_down_sync(0xffffffffu, s.x, 1), __shfl_down_sync(0xffffffffu, s.y, 1));
    const float r = __shfl_sync(0xffffffffu, c_proj(s, s_next, t.h), 2 * (lane & 15));   // lane j < 16: r_j
    if (lane < 16) {
      const double d = r;
      a1 = fabs(d);
      a2 = __dmul_rn(d, d);
    }
    n_dec = 16;
    const float je = f_add(f_add(jm, half), half);   // half-bit 33 (on lane 31)
    reply_end = (int)roundf(__shfl_sync(0xffffffffu, je, 31)) + c.n_tag_bit_i / 5;
  } else {
#pragma unroll
    for (int q = 0; q < 4; q++) {
      const double d = epc_projection(t, q * 32 + lane);
      a1 = __dadd_rn(a1, fabs(d));
      a2 = __dadd_rn(a2, __dmul_rn(d, d));
    }
    n_dec = 128;
    reply_end = win_epc_pos_b(128, t.T, t.index) + c.n_tag_bit_i / 5;
  }
  const double s1 = quality_lane_sum(a1), s2 = quality_lane_sum(a2);
  const double m = __ddiv_rn(s1, (double)n_dec), num = __dmul_rn(m, m);
  const double den = __dsub_rn(__ddiv_rn(s2, (double)n_dec), num);
  const float snr = den == 0.0 ? __int_as_float(0x7f800000) : quality_canonical(__ddiv_rn(num, den));
  // reply [sync, r1); noise reference: the head [0, h1) before the reply (which begins about half a bit before the sync
  // index) and the tail [t0, n) after it, the tail moved back when the two hold fewer than one symbol
  const int n_i = c.n_tag_bit_i;
  const int h1 = min(max(sync - 2 * n_i / 5, 0), n);
  int t0 = min(reply_end, n);
  if (h1 + (n - t0) < n_i) t0 = max(n - (n_i - h1), h1);
  const int r1 = min(reply_end, t0), n_noise = h1 + (n - t0);
  float energy = __int_as_float(0x7fc00000);
  if (sync >= 0 && r1 > sync && n_noise > 0) {
    const double er = quality_power_sum(t.w, 0, sync, r1), en = quality_power_sum(t.w, h1, t0, n);
    energy = quality_canonical(__ddiv_rn(__ddiv_rn(er, (double)(r1 - sync)), __ddiv_rn(en, (double)n_noise)));
  }
  int outcome;
  if (!((double)energy >= A.empty_ratio)) outcome = RFID_B200_SLOT_EMPTY;
  else if (kind != RFID_B200_RN16 || (double)snr >= A.single_ratio) outcome = RFID_B200_SLOT_SINGLE;
  else outcome = RFID_B200_SLOT_COLLISION;
  if (lane == 0) A.quality[t.slot] = rfid_b200_quality{energy, snr, outcome, n_dec};
}

}  // namespace rfid_b200
