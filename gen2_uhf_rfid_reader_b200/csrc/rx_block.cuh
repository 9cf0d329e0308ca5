// rx_block.cuh -- block-mode kernels: what the thin GNU Radio host blocks call
// once per general_work().  They are per-call latency-bound (chunks of a few
// thousand samples), so they are deliberately simple: a literal device replay
// of the reference loop with the persistent members kept in a device-side
// state record between calls.  The throughput path is rx_fused.cuh.
#pragma once

#include "rx_common.cuh"
#include "rx_decode.cuh"

namespace rfid_b200 {

constexpr int kMaxWinLen = 1024;  // win_samples capacity (400 at 1.6 MS/s decimated)
constexpr int kMaxDcLen = 512;    // dc_samples capacity

// gate_impl's private members (gate_impl.h:34-44) + the gate-related part of reader_state
struct GateState {
  float avg_ampl;
  float2 dc_est;
  int win_index, dc_index, n_samples, num_pulses;
  int sig_pos, gate_open, to_ungate;
  float win_samples[kMaxWinLen];
  float2 dc_samples[kMaxDcLen];
};

struct GateCallOut {
  int consumed, written, closed;
};

// gate_impl::general_work (gate_impl.cc:85-200) on one chunk.  One warp: lanes compute |in| for
// 32 samples at a time, lane 0 replays the recurrences and the state machine literally.
__global__ void __launch_bounds__(32) gate_block_kernel(RxConfig C, GateState* st, int seek, const float2* __restrict__ in,
                                                        int n_items, float2* __restrict__ out,
                                                        float* __restrict__ magn2, GateCallOut* res)
{
  __shared__ float s_win[kMaxWinLen];
  __shared__ float2 s_dc[kMaxDcLen];
  __shared__ float s_amp[32];
  __shared__ int s_stop;
  const int lane = threadIdx.x;
  for (int i = lane; i < C.win_length; i += 32) s_win[i] = st->win_samples[i];
  for (int i = lane; i < C.dc_length; i += 32) s_dc[i] = st->dc_samples[i];
  if (lane == 0) s_stop = -1;
  __syncwarp();

  float avg = st->avg_ampl;
  float2 dc = st->dc_est;
  int win_index = st->win_index, dc_index = st->dc_index, n_samples = st->n_samples, num_pulses = st->num_pulses;
  bool sig_pos = st->sig_pos != 0, gate_open = st->gate_open != 0;
  int to_ungate = st->to_ungate;
  int written = 0, consumed = n_items, closed = 0;

  // Gate block is controlled by the Gen2 Logic block (gate_impl.cc:112-123)
  if (seek == 2) { gate_open = false; to_ungate = C.len_epc; n_samples = 0; }
  else if (seek == 1) { gate_open = false; to_ungate = C.len_rn16; n_samples = 0; }

  const float winlen_f = (float)C.win_length, dclen_f = (float)C.dc_length;
  for (int base = 0; base < n_items; base += 32) {
    const int i_l = base + lane;
    float2 x = i_l < n_items ? in[i_l] : make_float2(0.f, 0.f);
    s_amp[lane] = cabsf_ref(x.x, x.y);
    __syncwarp();
    if (lane == 0) {
      const int lim = min(32, n_items - base);
      for (int j = 0; j < lim; j++) {
        const int i = base + j;
        const float2 v = in[i];
        const float a = s_amp[j];
        avg = f_add(avg, f_div(f_sub(a, s_win[win_index]), winlen_f));  // :131
        s_win[win_index] = a;
        win_index = (win_index + 1) % C.win_length;
        const float thr = f_mul(avg, kThreshFraction);  // :136
        if (!gate_open) {
          const float2 o = s_dc[dc_index];  // :141-143
          dc.x = f_add(dc.x, f_div(f_sub(v.x, o.x), dclen_f));
          dc.y = f_add(dc.y, f_div(f_sub(v.y, o.y), dclen_f));
          s_dc[dc_index] = v;
          dc_index = (dc_index + 1) % C.dc_length;
          n_samples++;
          if (a < thr && sig_pos) { n_samples = 0; sig_pos = false; }
          else if (a > thr && !sig_pos) {
            sig_pos = true;
            num_pulses = (n_samples > C.n_PW / 2) ? num_pulses + 1 : 0;
            n_samples = 0;
          }
          if (n_samples > C.n_T1 && sig_pos && num_pulses > kNumPulsesCommand) {  // :164
            gate_open = true;
            const float2 w = c_sub(v, dc);
            if (magn2) magn2[written] = c_norm(w);
            out[written++] = w;
            num_pulses = 0;
            n_samples = 1;
          }
        } else {
          n_samples++;
          const float2 w = c_sub(v, dc);
          if (magn2) magn2[written] = c_norm(w);
          out[written++] = w;
          if (n_samples >= to_ungate) {  // :189-194
            gate_open = false;
            consumed = i + 1;
            closed = 1;
            s_stop = 1;
            break;
          }
        }
      }
    }
    __syncwarp();
    if (s_stop >= 0) break;
  }
  __syncwarp();
  for (int i = lane; i < C.win_length; i += 32) st->win_samples[i] = s_win[i];
  for (int i = lane; i < C.dc_length; i += 32) st->dc_samples[i] = s_dc[i];
  if (lane == 0) {
    st->avg_ampl = avg; st->dc_est = dc;
    st->win_index = win_index; st->dc_index = dc_index; st->n_samples = n_samples; st->num_pulses = num_pulses;
    st->sig_pos = sig_pos ? 1 : 0; st->gate_open = gate_open ? 1 : 0; st->to_ungate = to_ungate;
    res->consumed = consumed; res->written = written; res->closed = closed;
  }
}

// tag_decoder_impl::general_work on one window (tag_decoder_impl.cc:223-393)
__global__ void __launch_bounds__(32) decode_block_kernel(RxConfig C, int kind, const float2* __restrict__ win_g, int n,
                                                          int stage_cap, rfid_b200_window_result* res)
{
  extern __shared__ __align__(16) float2 dstage[];   // the decoder stage: stage_cap samples
  WindowDecode wd;
  decode_window_staged<true>(C, kind, win_g, n, dstage, stage_cap, wd);
  if (threadIdx.x == 0)
    store_result(res, wd, 0, 0, 0, kind == RFID_B200_RN16 ? C.len_rn16 : C.len_epc, kind);
}

// fir_filter_ccc(decim,[1]*ntaps): canonical block-sum order, one thread per output.
// buf[0] holds absolute sample index abs0; output n needs x[D*n-K+1 .. D*n]; indices < 0 read +0.
__global__ void mf_block_kernel(RxConfig C, const float2* __restrict__ buf, long long abs0, long long first_n, int n_out,
                                float2* __restrict__ out)
{
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_out) return;
  const long long n = first_n + t;
  const int D = C.decim, q = C.mf_q, rem = C.mf_rem;
  float2 y = make_float2(0.f, 0.f);
  bool have = false;
  if (rem) {
    float2 p = make_float2(0.f, 0.f);
    for (int j = 0; j < rem; j++) {
      long long idx = (long long)D * (n - q) - rem + 1 + j;
      float2 x = idx >= 0 ? buf[idx - abs0] : make_float2(0.f, 0.f);
      p = j ? c_add(p, x) : x;
    }
    y = p;
    have = true;
  }
  for (long long m = n - q + 1; m <= n; m++) {
    float2 b = make_float2(0.f, 0.f);
    for (int j = 0; j < D; j++) {
      long long idx = (long long)D * m - D + 1 + j;
      float2 x = idx >= 0 ? buf[idx - abs0] : make_float2(0.f, 0.f);
      b = j ? c_add(b, x) : x;
    }
    y = have ? c_add(y, b) : b;
    have = true;
  }
  out[t] = y;
}

}  // namespace rfid_b200
