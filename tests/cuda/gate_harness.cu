// gate_harness.cu -- TEST INFRASTRUCTURE: the gate's threshold masks (gate_masks) and closed-run state machine
// (gate_closed_run) from csrc/rx_gate.cuh, unchanged, driven one warp per case so that tests/test_gate_fsm.py can compare
// them with a per-sample replay of the reference gate.  Built by oracle/gate_harness.py with the library's nvcc flags.
//
// Every launcher takes device pointers, runs on the default stream and returns the launch's cudaError_t.
#include <cuda_runtime.h>

#include "rx_gate.cuh"

using namespace rfid_b200;

#define GH_API extern "C" __attribute__((visibility("default")))

namespace {

constexpr int kWarps = 4;   // cases (warps) per block
constexpr unsigned FULL = 0xffffffffu;

// case c: avg / a are 32 W floats each; out: the (ltw, gtw) word each lane holds, [c][lane]
template <int W>
__global__ void masks_kernel(const float* avg, const float* a, const int* nvalid, unsigned* ltw, unsigned* gtw, int n)
{
  const int c = blockIdx.x * kWarps + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (c >= n) return;   // (whole warps)
  unsigned l = 0u, g = 0u;
  gate_masks<W>(avg + (size_t)c * 32 * W, a + (size_t)c * 32 * W, nvalid[c], l, g);
  ltw[(size_t)c * 32 + lane] = l;
  gtw[(size_t)c * 32 + lane] = g;
}

// lane l holds word l % W of the case's masks, as gate_masks leaves them
template <int W>
__device__ __forceinline__ void load_words(const unsigned* lt, const unsigned* gt, size_t c, unsigned& l, unsigned& g)
{
  const int lane = threadIdx.x & 31;
  l = lt[c * W + (lane & (W - 1))];
  g = gt[c * W + (lane & (W - 1))];
}

__device__ __forceinline__ bool warp_uniform(int v) { return __all_sync(FULL, v == __shfl_sync(FULL, v, 0)); }

// case c: masks lt / gt [c][W]; in [c][7] = from, nvalid, n_T1, half_pw, sig_pos, n_samples, num_pulses;
// out [c][5] = return value, sig_pos, n_samples, num_pulses, 1 if every lane returned the same
template <int W>
__global__ void closed_run_kernel(const unsigned* lt, const unsigned* gt, const int* in, int* out, int n)
{
  const int c = blockIdx.x * kWarps + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (c >= n) return;
  const int* q = in + (size_t)c * 7;
  unsigned l, g;
  load_words<W>(lt, gt, c, l, g);
  GateFsm st = {q[4] != 0, q[5], q[6]};
  const int r = gate_closed_run<W>(l, g, q[0], q[1], q[2], q[3], st);
  const bool same = warp_uniform(r) && warp_uniform(st.sig_pos) && warp_uniform(st.n_samples) &&
                    warp_uniform(st.num_pulses);
  if (lane == 0) {
    int* o = out + (size_t)c * 5;
    o[0] = r; o[1] = st.sig_pos; o[2] = st.n_samples; o[3] = st.num_pulses; o[4] = same;
  }
}

// stream s: T tiles of masks lt / gt [s][T][W] and nvalid [s][T]; in [s][7] = n_T1, half_pw, the first and the second
// window length (windows alternate between them), sig_pos, n_samples, num_pulses.  Tile by tile as the capture kernels
// call the gate (rx_pack.cuh, rx_fused_split.cuh): a closed run from pos, and after an opening the window's samples by
// the reference's ungate rule (gate_impl.cc:182-195: n_samples counts up to n_samples_to_ungate; then GATE_SEEK_* sets
// it to 0), after which the next closed run starts inside the same tile.
// out: opens [s][max_open] (sample index of each trigger, the first max_open); meta [s][7] = number of openings, sig_pos,
// n_samples, num_pulses, gate open at the end, 1 if every lane agreed throughout, 1 if no tile needed more than its bound
// of runs
template <int W>
__global__ void stream_kernel(const unsigned* lt, const unsigned* gt, const int* nvalid, const int* in, int T,
                              int* opens, int max_open, int* meta, int n)
{
  const int s = blockIdx.x * kWarps + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (s >= n) return;
  const int* q = in + (size_t)s * 7;
  const int n_T1 = q[0], half_pw = q[1];
  GateFsm gs = {q[4] != 0, q[5], q[6]};
  bool gate_open = false, same = true, bounded = true;
  int to_ungate = q[2], wcount = 0, n_open = 0;
  for (int t = 0; t < T; t++) {
    const size_t tile = (size_t)s * T + t;
    const int nv = nvalid[tile];
    unsigned l, g;
    load_words<W>(lt, gt, tile, l, g);
    int pos = 0;
    // each step advances pos by at least one sample: a tile needs at most nv steps
    for (int step = 0; pos < nv; step++) {
      if (step > nv) { bounded = false; break; }
      if (!gate_open) {
        const int p_open = gate_closed_run<W>(l, g, pos, nv, n_T1, half_pw, gs);
        same = same && warp_uniform(p_open);
        if (p_open >= 0) {
          if (n_open < max_open && lane == 0) opens[(size_t)s * max_open + n_open] = t * 32 * W + p_open;
          n_open++;
          gate_open = true;
          pos = max(p_open + 1, pos + 1);
        } else {
          pos = nv;
        }
      } else {
        const int take = min(to_ungate - gs.n_samples, nv - pos);
        gs.n_samples += take;
        pos += max(take, 1);
        if (gs.n_samples >= to_ungate) {
          gate_open = false;
          wcount++;
          to_ungate = (wcount & 1) ? q[3] : q[2];
          gs.n_samples = 0;
        }
      }
    }
  }
  same = same && warp_uniform(gs.sig_pos) && warp_uniform(gs.n_samples) && warp_uniform(gs.num_pulses);
  if (lane == 0) {
    int* o = meta + (size_t)s * 7;
    o[0] = n_open; o[1] = gs.sig_pos; o[2] = gs.n_samples; o[3] = gs.num_pulses; o[4] = gate_open; o[5] = same;
    o[6] = bounded;
  }
}

inline dim3 grid_for(int n) { return dim3((unsigned)((n + kWarps - 1) / kWarps)); }

}  // namespace

GH_API int gate_harness_masks(int W, const float* avg, const float* a, const int* nvalid, unsigned* ltw, unsigned* gtw,
                              int n)
{
  if (n <= 0) return 0;
  if (W == 4) masks_kernel<4><<<grid_for(n), 32 * kWarps>>>(avg, a, nvalid, ltw, gtw, n);
  else if (W == 8) masks_kernel<8><<<grid_for(n), 32 * kWarps>>>(avg, a, nvalid, ltw, gtw, n);
  else return (int)cudaErrorInvalidValue;
  return (int)cudaGetLastError();
}

GH_API int gate_harness_closed_run(int W, const unsigned* lt, const unsigned* gt, const int* in, int* out, int n)
{
  if (n <= 0) return 0;
  if (W == 4) closed_run_kernel<4><<<grid_for(n), 32 * kWarps>>>(lt, gt, in, out, n);
  else if (W == 8) closed_run_kernel<8><<<grid_for(n), 32 * kWarps>>>(lt, gt, in, out, n);
  else return (int)cudaErrorInvalidValue;
  return (int)cudaGetLastError();
}

GH_API int gate_harness_stream(int W, const unsigned* lt, const unsigned* gt, const int* nvalid, const int* in, int T,
                               int* opens, int max_open, int* meta, int n)
{
  if (n <= 0) return 0;
  if (W == 4) stream_kernel<4><<<grid_for(n), 32 * kWarps>>>(lt, gt, nvalid, in, T, opens, max_open, meta, n);
  else if (W == 8) stream_kernel<8><<<grid_for(n), 32 * kWarps>>>(lt, gt, nvalid, in, T, opens, max_open, meta, n);
  else return (int)cudaErrorInvalidValue;
  return (int)cudaGetLastError();
}
