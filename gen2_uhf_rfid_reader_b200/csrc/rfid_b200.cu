// rfid_b200.cu -- C-ABI of the H100-native Gen2 receive chain (see include/rfid_b200.h).
// Host side: context, configuration derivation, launches, host<->device marshalling,
// READER_STATS reduction.  There is no CPU implementation of the signal path in this
// library: every entry point that produces samples or decisions launches a kernel.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <new>
#include <string>
#include <vector>

#include "rx_block.cuh"
#include "rx_cmd.cuh"
#include "rx_common.cuh"
#include "rx_fused.cuh"
#include "rx_fused_split.cuh"
#include "rx_ingest.cuh"
#include "rx_pack.cuh"
#include "rx_quality.cuh"
#include "rx_match.cuh"
#include "rx_recover.cuh"
#include "rx_report.cuh"
#include "tx_synth.cuh"

using namespace rfid_b200;

// A device buffer of the context, freed with it; grow() sizes the scratch buffers on demand.
struct DevBuf {
  void* p = nullptr;
  size_t bytes = 0;
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  ~DevBuf() { if (p) cudaFree(p); }
};

// Created by value-initialisation: every member not set by rfid_b200_create starts zero.
struct rfid_b200_ctx {
  rfid_b200_params params;
  RxConfig cfg;
  int device;
  cudaStream_t stream;  // own stream for block mode / host-mode capture calls
  cudaStream_t copy_stream;  // host-mode capture calls: uploads of the next slice run beside the decode of this one
  cudaEvent_t ev_slice[4];
  std::string last_error;
  // capture mode
  FusedArgs layout;     // shared-memory carve-up (pointers filled per call), fc32 captures
  FusedArgs layout_sc16;  // the same for sc16 captures (raw stages of 4-byte samples)
  float* window_tap;
  int last_launches;
  bool timing;
  std::vector<std::pair<cudaEvent_t, cudaEvent_t>> pending;
  std::vector<cudaEvent_t> ev_pool;  // timing events are created once and reused (no driver calls inside a timed loop)
  float kernel_ms;
  int kernel_launches;
  int sm_count;
  int pack_g_override;  // RFID_B200_PACK_G (developer aid): segments per CTA of the pack kernel, 0 = automatic
  bool pack_disabled;   // RFID_B200_KERNEL=split: keep the one-CTA-per-segment kernels for every configuration
  // host-mode staging buffers
  DevBuf d_iq, d_segs, d_res, d_cnt;
  DevBuf d_win;                      // per-segment window scratch of the one-CTA-per-segment kernels
  DevBuf d_yhist;                    // rx_pack_kernel: y history, [%nsmid][kPMaxSeg][kYW] float2
  cudaEvent_t ev_hist;               // recorded after every rx_pack_kernel launch: the history serves one launch at a time
  cudaStream_t hist_stream;          // stream of the last rx_pack_kernel launch
  bool hist_used;
  // block mode
  DevBuf d_gate;                     // GateState
  DevBuf d_in, d_out, d_m2;
  DevBuf d_blk;                      // block mode: [GateCallOut | out samples | |out|^2] in one block -> ONE D2H per work call
  void* h_blk; size_t h_blk_bytes;   // its pinned host mirror
  DevBuf d_one;                      // rfid_b200_window_result
  // mf block mode
  DevBuf d_mf; long long mf_abs0; long long mf_have; long long mf_next_n;
  // capture ingest (segmenter work buffers, pinned upload staging)
  DevBuf d_mask;
  DevBuf d_chunk;  // chunk_last | prev_low | falls_before | chunk_falls
  DevBuf d_bursts;
  DevBuf d_ing;    // level partials + totals
  void* h_stage[2]; cudaEvent_t ev_stage[2];
  std::vector<IngestBurst> h_bursts;
  // TX synthesiser / slot simulator
  DevBuf d_script, d_sim_res, d_sim_cnt;
  // host-mode command records
  DevBuf d_cmd;
  // tag report scratch: aggregates, hash table, per-slot owners, block counts
  DevBuf d_report;
  // EPC match scratch: row count, compact rows of the attempted windows
  DevBuf d_match;
};

namespace {

const char* kErrNames[] = {"ok", "invalid argument", "no usable sm_90 CUDA device", "out of memory", "CUDA runtime error",
                           "output buffer too small"};

int fail_cuda(rfid_b200_ctx* c, cudaError_t e, const char* what)
{
  if (c) c->last_error = std::string(what) + ": " + cudaGetErrorString(e);
  return RFID_B200_ECUDA;
}
#define CK(call)                                                   \
  do {                                                             \
    cudaError_t _e = (call);                                       \
    if (_e != cudaSuccess) return fail_cuda(ctx, _e, #call);       \
  } while (0)

int next_pow2(int v)
{
  int p = 1;
  while (p < v) p <<= 1;
  return p;
}

// The reference's decoder takes every read index from the float n_samples_TAG_BIT, while the gate sizes its windows
// from the truncated integer (gate_impl.cc:115,121).  Where the two differ too much the EPC symbol-period search and bit
// decisions read past the end of the window (undefined behaviour in the reference, so there is no answer to reproduce),
// and an RN16 window can end before its 32 half-bits, after which the reference no longer alternates RN16 / EPC windows.
// A configuration is well defined when, for every sync index tag_sync can return, every read of the decoder stays
// inside its window and the RN16 loop reaches 32 half-bits.  Same expressions and types as tag_decoder_impl.cc.
bool well_defined(const RxConfig& c)
{
  const float n = c.n_tag_bit_f;
  for (int s = 0; s < c.sync_range; s++) {
    for (int j = 0; j < 2 * kTagPreambleBits; j++)  // tag_sync's correlation and h_est (:92,103)
      if ((int)(s + j * n / 2) >= c.len_rn16) return false;
    const int index = (int)(s + kTagPreambleBits * n + n / 2);  // :107
    int half_bits = 0;
    for (float j = (float)index; j < c.len_rn16; j += n / 2) {   // :237-253
      if ((int)std::round(j) >= c.len_rn16) return false;
      if (++half_bits == 2 * (kRN16Bits - 1)) break;
    }
    if (half_bits != 2 * (kRN16Bits - 1)) return false;
    for (int t = 0; t < 20; t++) {
      const float T = c.t_min + t * (c.t_max - c.t_min) / (20 - 1);  // :161,166
      for (int i = 0; i < 256; i++)
        if ((int)(i * T + index) >= c.len_epc) return false;
      for (int j = 0; j < 128; j++)  // :173
        if ((int)(j * (2 * T) + index) >= c.len_epc || (int)(j * 2 * T + T + index) >= c.len_epc) return false;
    }
  }
  return true;
}

// Derived counts with the reference's own expression order and types
// (gate_impl.cc:48-53,115,121; tag_decoder_impl.cc:60,85,151-152; global_vars.h:110-111).
int derive_config(const rfid_b200_params& p, RxConfig& c)
{
  if (p.adc_rate <= 0 || p.decim <= 0 || p.ntaps <= 0 || p.fixed_q < 0 || p.fixed_q > 15) return RFID_B200_EINVAL;
  memset(&c, 0, sizeof(c));
  c.adc_rate = p.adc_rate; c.decim = p.decim; c.ntaps = p.ntaps;
  const int sample_rate = p.adc_rate / p.decim;  // apps/reader.py:76
  c.fs_dec = sample_rate;
  const float TAG_BIT_D = (float)(1.0 / kReaderFreq * std::pow(10, 6));
  c.n_T1 = (int)(kT1_D * (sample_rate / std::pow(10, 6)));
  c.n_PW = (int)(kPW_D * (sample_rate / std::pow(10, 6)));
  c.n_tag_bit_i = (int)(TAG_BIT_D * (sample_rate / std::pow(10, 6)));
  c.win_length = (int)(kWinSizeD * (sample_rate / std::pow(10, 6)));
  c.dc_length = (int)(kDcSizeD * (sample_rate / std::pow(10, 6)));
  c.n_tag_bit_f = (float)(TAG_BIT_D * sample_rate / std::pow(10, 6));
  c.len_epc = (kEPCBits + kTagPreambleBits) * c.n_tag_bit_i + 2 * c.n_tag_bit_i;
  c.len_rn16 = (kRN16Bits + kTagPreambleBits) * c.n_tag_bit_i + 2 * c.n_tag_bit_i;
  c.fixed_q = p.fixed_q; c.max_queries = p.max_queries; c.max_tags = p.max_tags;
  c.mf_q = p.ntaps / p.decim; c.mf_rem = p.ntaps % p.decim;
  int sr = 0;
  for (int i = 0; i < 1.5 * c.n_tag_bit_f; i++) sr++;  // tag_decoder_impl.cc:85
  c.sync_range = sr;
  const float n = c.n_tag_bit_f;
  c.t_min = (float)(n / 2.0 - n / 2.0 / 100);  // :151
  c.t_max = (float)(n / 2.0 + n / 2.0 / 100);  // :152
  // divisors for which RN(x/d) == fma(fma(-RN(x*c), d, x), c, RN(x*c)) holds for every binary32 x (exhaustive
  // check: tools/micro/verify_constdiv.c, run by tests/test_host_logic.py)
  static const int kVerifiedDivisors[] = {6, 24, 48, 50, 60, 96, 100, 125, 144, 192, 200, 300, 400};
  c.win_recip = 1.0f / (float)c.win_length;
  c.dc_recip = 1.0f / (float)c.dc_length;
  c.win_div_fast = c.dc_div_fast = 0;
  for (int d : kVerifiedDivisors) {
    if (d == c.win_length) c.win_div_fast = 1;
    if (d == c.dc_length) c.dc_div_fast = 1;
  }
  if (c.win_length < 1 || c.dc_length < 1 || c.n_tag_bit_i < 1 || c.win_length > kMaxWinLen || c.dc_length > kMaxDcLen)
    return RFID_B200_EINVAL;
  if (!well_defined(c)) return RFID_B200_EINVAL;
  return RFID_B200_OK;
}

int align_up(int v, int a) { return (v + a - 1) / a * a; }

bool fast_path_ok(const RxConfig& c) { return c.win_length <= kTT && c.dc_length <= kTT; }

// Decoder stage (float2 samples) of one decoder warp of the pack, split and block-mode kernels (rx_decode.cuh, STAGED):
// the window's head (sync range + 6 symbols), one chunk of the symbol-period search (win_chunk_span samples at one float
// each) and an RN16 window whole.  The bit decisions read global memory directly.
int head_stage_samples(const RxConfig& c) { return align_up(c.sync_range + (int)(6.0f * c.n_tag_bit_f) + 2, 8); }
int chunk_stage_samples(const RxConfig& c)
{
  return align_up(std::max({head_stage_samples(c), (win_chunk_span(c) + 1) / 2, c.len_rn16}), 8);
}
// rx_fused_kernel stages the head only (head_stage_samples): its long rings leave little shared memory, so its search
// chunks and the rest of its RN16 windows gather from L2.

// shared-memory carve-up of rx_fused_split_kernel: five tile stages forming one time-indexed ring
// Raw stages hold a tile's samples in the capture's format (raw_bytes per sample, 8 fc32 or 4 sc16) plus the alignment of
// its 16-byte granule (rx_common.cuh: issue_tile_load) and, for sc16, the read-ahead of the vector loads (sc16_run).
int raw_stage_samples(const RxConfig& c, int raw_bytes) { return c.decim * kTT + (raw_bytes == 8 ? 2 : kSc16StagePad); }

void make_layout_split(const RxConfig& c, int raw_bytes, FusedArgs& L)
{
  int off = 0;
  L.raw_stage_samples = raw_stage_samples(c, raw_bytes);
  L.off_raw = off; off = align_up(off + kRawStages * L.raw_stage_samples * raw_bytes, 16);
  L.bhist_size = next_pow2(kTT + c.mf_q + 2);
  L.off_bhist = off; off = align_up(off + L.bhist_size * 8 * (c.mf_rem ? 2 : 1), 16);
  L.off_tile_y = off; off += kRing * 8;
  L.off_tile_a = off; off += kRing * 4;
  L.off_tile_d = off; off += kRing * 4 + 64;          // + read-ahead pad of the running-sum loop
  L.off_etile = off; off += kS * 2 * kTT * 4 + 64;
  L.off_snap = off; off = align_up(off + c.dc_length * 8, 16);
  L.dstage_samples = chunk_stage_samples(c);
  L.off_dstage = off; off = align_up(off + L.dstage_samples * 8, 16);
  L.ahist_size = L.ycl_size = 0;
  L.off_ahist = L.off_ycl = L.off_e = 0;
  L.rn16_pad = align_up(c.len_rn16, 16);
  L.win_stride = L.rn16_pad + align_up(c.len_epc, 16);
  L.smem_bytes = off;
}

void make_layout(const RxConfig& c, int raw_bytes, FusedArgs& L)
{
  if (fast_path_ok(c)) { make_layout_split(c, raw_bytes, L); return; }
  const bool spec = false;
  int off = 0;
  L.raw_stage_samples = raw_stage_samples(c, raw_bytes);
  L.off_raw = off; off = align_up(off + kRawStages * L.raw_stage_samples * raw_bytes, 16);
  L.bhist_size = next_pow2(kTT + c.mf_q + 2);
  L.off_bhist = off; off = align_up(off + L.bhist_size * 8 * (c.mf_rem ? 2 : 1), 16);
  L.off_tile_y = off; off += kTileStages * kTT * 8;
  L.off_tile_a = off; off += kTileStages * kTT * 4;
  L.off_tile_d = off; off += kTileStages * kTT * 4 + 64;  // + read-ahead pad of the running-sum loop
  L.ahist_size = L.ycl_size = 0;
  L.off_ahist = L.off_ycl = L.off_e = L.off_etile = L.off_snap = 0;
  if (spec) {
    L.off_etile = off; off += kTileStages * 2 * kTT * 4 + 64;
    L.off_snap = off; off = align_up(off + c.dc_length * 8, 16);
  } else {
    L.ahist_size = next_pow2(kTT + c.win_length);
    L.off_ahist = off; off = align_up(off + L.ahist_size * 4, 16);
    L.ycl_size = next_pow2(kTT + c.dc_length);
    L.off_ycl = off; off = align_up(off + L.ycl_size * 8, 16);
    L.off_e = off; off += 2 * (kTT + 16) * 4;
  }
  L.dstage_samples = head_stage_samples(c);
  L.off_dstage = off; off = align_up(off + L.dstage_samples * 8, 16);
  L.rn16_pad = align_up(c.len_rn16, 16);
  L.win_stride = L.rn16_pad + align_up(c.len_epc, 16);
  L.smem_bytes = off;
}

// number of SM identifiers (%smid < %nsmid; may exceed the SM count)
__global__ void query_nsmid_kernel(unsigned* out)
{
  unsigned n;
  asm("mov.u32 %0, %%nsmid;" : "=r"(n));
  *out = n;
}

// rx_pack_kernel serves the reference configuration (block-sum matched filter with 5 blocks of 5, rings inside a tile);
// its y history must hold a whole EPC window plus the tiles warps A / B / C may be apart, and at most kPTrig windows can
// open within one tile
bool pack_ok(const RxConfig& c)
{
  return c.decim == 5 && c.mf_rem == 0 && c.mf_q == 5 && fast_path_ok(c) && c.len_rn16 >= kT2 / 2 &&
         c.len_epc + c.dc_length + 8 * kT2 <= kYW && ((c.win_length | c.dc_length) & 3) == 0 && c.dc_length <= 124 && c.win_length <= kT2;
}

// shared-memory carve-up of rx_pack_kernel for G segments per CTA
void make_layout_pack(const RxConfig& c, int G, int raw_bytes, PackArgs& L)
{
  L.G = G;
  L.pas = pack_ring_slots(G);
  L.pds = L.pas + 1;
  L.raw_stage_samples = raw_stage_samples(c, raw_bytes);
  L.dstage_samples = chunk_stage_samples(c);   // one per decoder warp
  int o = 0;
  // the two raw stages; warp A1 later uses the region as its decoder stage
  L.o_raw = o; o = align_up(o + std::max(2 * L.raw_stage_samples * raw_bytes, L.dstage_samples * 8), 16);
  L.o_tail_y = o; o = align_up(o + 2 * c.dc_length * 8, 16);
  L.o_ring_a = o; o += L.pas * kT2 * 4;
  L.seg_bytes = align_up(o, 16);
  int off = 0;
  L.off_dA = off; off += L.pas * G * kPChainBuf * 4;
  L.off_dD = off; off += L.pds * 2 * G * kPChainBuf * 4;
  L.off_dstage = align_up(off, 16); off = L.off_dstage + pack_decoders(G) * L.dstage_samples * 8;
  L.off_seg = align_up(off, 16);
  L.smem_bytes = L.off_seg + G * L.seg_bytes;
  if (L.smem_bytes < kPackMinSmem) L.smem_bytes = kPackMinSmem;   // one CTA per SM: the y history is indexed by the SM
}

int pack_segments_per_cta(const rfid_b200_ctx* ctx, int nseg);

typedef void (*fused_fn)(const FusedArgs);
template <class RAW>
fused_fn pick_kernel_fmt(const RxConfig& c)
{
  if (c.decim != 5) return nullptr;
  if (fast_path_ok(c)) {
    if (c.mf_rem == 0 && c.mf_q == 5) return rx_fused_split_kernel<5, 5, RAW>;  // the reference configuration: 25 taps
    return rx_fused_split_kernel<5, 0, RAW>;
  }
  return rx_fused_kernel<5, 0, RAW>;  // long rings (raw rates above 5 MS/s) and any tap count
}
// the same choice for both capture formats
fused_fn pick_kernel(const RxConfig& c, bool sc16 = false)
{
  return sc16 ? pick_kernel_fmt<RawSc16>(c) : pick_kernel_fmt<RawFc32>(c);
}
typedef void (*pack_fn)(const PackArgs);
pack_fn pack_kernel(int pas, bool sc16)
{
  if (sc16) return pas == kPASMax ? rx_pack_kernel<5, 5, kPASMax, RawSc16> : rx_pack_kernel<5, 5, kPASMax - 1, RawSc16>;
  return pas == kPASMax ? rx_pack_kernel<5, 5, kPASMax, RawFc32> : rx_pack_kernel<5, 5, kPASMax - 1, RawFc32>;
}

int grow(rfid_b200_ctx* ctx, DevBuf& b, size_t need)
{
  if (b.bytes >= need) return RFID_B200_OK;
  if (b.p) cudaFree(b.p);
  b.p = nullptr; b.bytes = 0;
  size_t want = need + need / 4 + 256;
  cudaError_t e = cudaMalloc(&b.p, want);
  if (e != cudaSuccess) { ctx->last_error = "cudaMalloc failed"; cudaGetLastError(); return RFID_B200_ENOMEM; }
  b.bytes = want;
  return RFID_B200_OK;
}

// grid of the kernels that run one warp per record slot
unsigned slot_grid(long long slots) { return (unsigned)((slots + kSlotWarps - 1) / kSlotWarps); }

// Segments per CTA of rx_pack_kernel: as few CTAs as fill the device once (one CTA per SM, every SM busy for the
// whole launch); larger batches run kPMaxSeg per CTA in several waves.  With its decoder warps one pool over the
// CTA's windows (rx_pack.cuh) a CTA of kPMaxSeg segments no longer decodes two EPC windows one after the other at its
// end, and it does more work per SM than one of kPMaxSeg - 1 (H100 SXM, 700 W, two runs each: cfg3 6.20-6.21 ms
// against 6.34-6.36 ms at kPMaxSeg - 1, cfg4 10.00-10.01 ms against 10.37-10.39 ms).
int pack_segments_per_cta(const rfid_b200_ctx* ctx, int nseg)
{
  if (ctx->pack_g_override > 0) return ctx->pack_g_override;
  const int sms = ctx->sm_count > 0 ? ctx->sm_count : 132;
  int g = (nseg + sms - 1) / sms;
  if (g < 1) g = 1;
  if (g > kPMaxSeg) g = kPMaxSeg;
  return g;
}

void drain_timing(rfid_b200_ctx* ctx)
{
  for (auto& pr : ctx->pending) {
    float ms = 0.f;
    if (cudaEventSynchronize(pr.second) == cudaSuccess && cudaEventElapsedTime(&ms, pr.first, pr.second) == cudaSuccess) {
      ctx->kernel_ms += ms;
      ctx->kernel_launches++;
    }
    ctx->ev_pool.push_back(pr.first);
    ctx->ev_pool.push_back(pr.second);
  }
  ctx->pending.clear();
}

}  // namespace

extern "C" {

int rfid_b200_abi_version(void) { return RFID_B200_ABI_VERSION; }

const char* rfid_b200_strerror(int code)
{
  int k = -code;
  if (k < 0 || k > 5) return "unknown error";
  return kErrNames[k];
}

const char* rfid_b200_last_cuda_error(const rfid_b200_ctx* ctx) { return ctx ? ctx->last_error.c_str() : ""; }

void rfid_b200_default_params(rfid_b200_params* p)
{
  if (!p) return;
  p->adc_rate = 2000000;  // apps/reader.py:53
  p->decim = 5;           // apps/reader.py:54
  p->ntaps = 25;          // apps/reader.py:65
  p->fixed_q = 0;         // global_vars.h:72
  p->max_queries = 1000;  // global_vars.h:76
  p->max_tags = 100;      // global_vars.h:100
  p->device = 0;
  p->reserved = 0;
}

int rfid_b200_create(const rfid_b200_params* p, rfid_b200_ctx** out)
{
  if (!p || !out) return RFID_B200_EINVAL;
  *out = nullptr;
  RxConfig cfg;
  int rc = derive_config(*p, cfg);
  if (rc) return rc;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || p->device < 0 || p->device >= ndev) { cudaGetLastError(); return RFID_B200_ENODEV; }
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, p->device) != cudaSuccess || prop.major != 9 || prop.minor != 0) { cudaGetLastError(); return RFID_B200_ENODEV; }
  rfid_b200_ctx* ctx = new (std::nothrow) rfid_b200_ctx();
  if (!ctx) return RFID_B200_ENOMEM;
  ctx->params = *p; ctx->cfg = cfg; ctx->device = p->device;
  make_layout(cfg, (int)sizeof(RawFc32::T), ctx->layout);
  make_layout(cfg, (int)sizeof(RawSc16::T), ctx->layout_sc16);
  cudaError_t e = cudaSetDevice(p->device);
  if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking);
  if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&ctx->copy_stream, cudaStreamNonBlocking);
  for (int k = 0; k < 4 && e == cudaSuccess; k++) e = cudaEventCreateWithFlags(&ctx->ev_slice[k], cudaEventDisableTiming);
  if (e == cudaSuccess) e = cudaMalloc(&ctx->d_gate.p, sizeof(GateState));
  if (e == cudaSuccess) e = cudaMalloc(&ctx->d_one.p, sizeof(rfid_b200_window_result));
  if (e == cudaSuccess) e = cudaMemsetAsync(ctx->d_gate.p, 0, sizeof(GateState), ctx->stream);
  if (e == cudaSuccess) {
    // gate_impl ctor (gate_impl.cc:45) + initialize_reader_state (global_vars.cc:47): NEG_EDGE, first SEEK = RN16
    GateState init;
    memset(&init, 0, sizeof(init));
    init.to_ungate = cfg.len_rn16;
    e = cudaMemcpyAsync(ctx->d_gate.p, &init, offsetof(GateState, win_samples), cudaMemcpyHostToDevice, ctx->stream);
  }
  if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
  ctx->sm_count = prop.multiProcessorCount;
  {
    const char* ev = getenv("RFID_B200_PACK_G");
    ctx->pack_g_override = ev ? atoi(ev) : 0;
    if (ctx->pack_g_override < 0 || ctx->pack_g_override > kPMaxSeg) ctx->pack_g_override = 0;
    const char* kv = getenv("RFID_B200_KERNEL");
    ctx->pack_disabled = kv && strcmp(kv, "split") == 0;
  }
  if (e == cudaSuccess && pack_ok(cfg)) {
    // the y history of rx_pack_kernel: one region per SM identifier
    unsigned nsmid = 0, *d_n = nullptr;
    e = cudaMalloc(&d_n, sizeof(unsigned));
    if (e == cudaSuccess) {
      query_nsmid_kernel<<<1, 1, 0, ctx->stream>>>(d_n);
      e = cudaMemcpyAsync(&nsmid, d_n, sizeof(unsigned), cudaMemcpyDeviceToHost, ctx->stream);
      if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
      cudaFree(d_n);
    }
    if (e == cudaSuccess && nsmid < (unsigned)prop.multiProcessorCount) nsmid = prop.multiProcessorCount;
    if (e == cudaSuccess) e = cudaMalloc(&ctx->d_yhist.p, (size_t)nsmid * kPMaxSeg * kYW * sizeof(float2));
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&ctx->ev_hist, cudaEventDisableTiming);
  }
  if (e == cudaSuccess && pack_ok(cfg)) {
    int smem_max = 0;
    for (int G = 1; G <= kPMaxSeg; G++) {
      PackArgs pl;
      make_layout_pack(cfg, G, (int)sizeof(RawFc32::T), pl);   // (sc16 stages are smaller)
      if (pl.smem_bytes > smem_max) smem_max = pl.smem_bytes;
    }
    for (const void* fk : {(const void*)pack_kernel(kPASMax, false), (const void*)pack_kernel(kPASMax - 1, false),
                           (const void*)pack_kernel(kPASMax, true), (const void*)pack_kernel(kPASMax - 1, true)}) {
      if (e == cudaSuccess) e = cudaFuncSetAttribute(fk, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_max);
      if (e == cudaSuccess)
        e = cudaFuncSetAttribute(fk, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    }
  }
  for (int f = 0; f < 2; f++) {
    fused_fn fn = pick_kernel(cfg, f == 1);
    const int smem = (f == 1 ? ctx->layout_sc16 : ctx->layout).smem_bytes;
    if (e == cudaSuccess && fn) e = cudaFuncSetAttribute((const void*)fn, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e == cudaSuccess && fn)
      e = cudaFuncSetAttribute((const void*)fn, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
  }
  if (e == cudaSuccess)
    e = cudaFuncSetAttribute((const void*)decode_block_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             chunk_stage_samples(cfg) * 8);
  if (e != cudaSuccess) {
    cudaGetLastError();
    rfid_b200_destroy(ctx);
    return RFID_B200_ECUDA;
  }
  *out = ctx;
  return RFID_B200_OK;
}

void rfid_b200_destroy(rfid_b200_ctx* ctx)
{
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  drain_timing(ctx);
  for (cudaEvent_t e : ctx->ev_pool) cudaEventDestroy(e);
  ctx->ev_pool.clear();
  if (ctx->h_blk) cudaFreeHost(ctx->h_blk);
  for (int b = 0; b < 2; b++) {
    if (ctx->h_stage[b]) cudaFreeHost(ctx->h_stage[b]);
    if (ctx->ev_stage[b]) cudaEventDestroy(ctx->ev_stage[b]);
  }
  for (int k = 0; k < 4; k++) if (ctx->ev_slice[k]) cudaEventDestroy(ctx->ev_slice[k]);
  if (ctx->ev_hist) cudaEventDestroy(ctx->ev_hist);
  if (ctx->copy_stream) cudaStreamDestroy(ctx->copy_stream);
  if (ctx->stream) cudaStreamDestroy(ctx->stream);
  delete ctx;   // (frees the device buffers)
}

int rfid_b200_window_length(const rfid_b200_ctx* ctx, int kind)
{
  if (!ctx) return RFID_B200_EINVAL;
  return kind == RFID_B200_RN16 ? ctx->cfg.len_rn16 : ctx->cfg.len_epc;
}

int rfid_b200_fs_dec(const rfid_b200_ctx* ctx) { return ctx ? ctx->cfg.fs_dec : RFID_B200_EINVAL; }

int rfid_b200_set_window_tap(rfid_b200_ctx* ctx, float* d_windows)
{
  if (!ctx) return RFID_B200_EINVAL;
  ctx->window_tap = d_windows;
  return RFID_B200_OK;
}

int rfid_b200_enable_kernel_timing(rfid_b200_ctx* ctx, int on)
{
  if (!ctx) return RFID_B200_EINVAL;
  ctx->timing = on != 0;
  if (ctx->timing) {
    cudaSetDevice(ctx->device);
    while (ctx->ev_pool.size() < 128) {  // enough for 64 launches in flight before the first drain
      cudaEvent_t e;
      if (cudaEventCreate(&e) != cudaSuccess) { cudaGetLastError(); break; }
      ctx->ev_pool.push_back(e);
    }
  }
  return RFID_B200_OK;
}

int rfid_b200_kernel_time(rfid_b200_ctx* ctx, int reset, float* ms_total, int* launches)
{
  if (!ctx) return RFID_B200_EINVAL;
  cudaSetDevice(ctx->device);
  drain_timing(ctx);
  if (ms_total) *ms_total = ctx->kernel_ms;
  if (launches) *launches = ctx->kernel_launches;
  if (reset) { ctx->kernel_ms = 0.f; ctx->kernel_launches = 0; }
  return RFID_B200_OK;
}

int rfid_b200_last_launch_count(const rfid_b200_ctx* ctx) { return ctx ? ctx->last_launches : RFID_B200_EINVAL; }

// sc16 = false: d_iq holds fc32 samples (scale unused); true: sc16 samples, each converted with `scale`
static int decode_capture_impl(rfid_b200_ctx* ctx, const void* d_iq, bool sc16, float scale, size_t n_raw,
                               const rfid_b200_segment* d_segs, int nseg, int max_windows_per_segment,
                               rfid_b200_window_result* d_results, int32_t* d_counts, void* stream, int seg_base);

// an sc16 scale is a finite positive float
static bool scale_ok(float scale) { return std::isfinite(scale) && scale > 0.f; }

int rfid_b200_decode_capture(rfid_b200_ctx* ctx, const float* d_iq, size_t n_raw, const rfid_b200_segment* d_segs, int nseg,
                             int max_windows_per_segment, rfid_b200_window_result* d_results, int32_t* d_counts,
                             void* stream)
{
  return decode_capture_impl(ctx, d_iq, false, 1.f, n_raw, d_segs, nseg, max_windows_per_segment, d_results, d_counts, stream, 0);
}

int rfid_b200_decode_capture_sc16(rfid_b200_ctx* ctx, const int16_t* d_iq, size_t n_raw, float scale,
                                  const rfid_b200_segment* d_segs, int nseg, int max_windows_per_segment,
                                  rfid_b200_window_result* d_results, int32_t* d_counts, void* stream)
{
  if (!scale_ok(scale)) return RFID_B200_EINVAL;
  return decode_capture_impl(ctx, d_iq, true, scale, n_raw, d_segs, nseg, max_windows_per_segment, d_results, d_counts, stream, 0);
}

static int decode_capture_impl(rfid_b200_ctx* ctx, const void* d_iq, bool sc16, float scale, size_t n_raw,
                               const rfid_b200_segment* d_segs, int nseg, int max_windows_per_segment,
                               rfid_b200_window_result* d_results, int32_t* d_counts, void* stream, int seg_base)
{
  if (!ctx || !d_iq || !d_segs || !d_results || !d_counts || nseg < 0 || max_windows_per_segment < 1) return RFID_B200_EINVAL;
  if ((reinterpret_cast<uintptr_t>(d_iq) & 15u) != 0) return RFID_B200_EINVAL;  // TMA bulk source alignment
  ctx->last_launches = 0;
  if (nseg == 0) return RFID_B200_OK;
  fused_fn fn = pick_kernel(ctx->cfg, sc16);
  if (!fn) { ctx->last_error = "capture mode supports decim = 5 only in this build"; return RFID_B200_EINVAL; }
  CK(cudaSetDevice(ctx->device));
  cudaStream_t s = (cudaStream_t)stream;  // NULL = the (legacy) default stream, as documented
  FusedArgs A = sc16 ? ctx->layout_sc16 : ctx->layout;
  const bool use_pack = pack_ok(ctx->cfg) && !ctx->pack_disabled;
  if (!use_pack) {
    // window scratch: one RN16 + one EPC window per segment (grown on demand; cudaMalloc synchronises, so a
    // caller that wants a fully asynchronous call sizes the context once with its largest batch)
    int rc = grow(ctx, ctx->d_win, (size_t)nseg * A.win_stride * sizeof(float2));
    if (rc) return rc;
  }
  A.win_scratch = reinterpret_cast<float2*>(ctx->d_win.p);
  A.iq = d_iq;
  A.scale = scale;
  A.n_raw = n_raw;
  A.segs = d_segs;
  A.nseg = nseg;
  A.seg_base = seg_base;
  A.max_windows = max_windows_per_segment;
  A.results = d_results;
  A.counts = d_counts;
  A.window_tap = reinterpret_cast<float2*>(ctx->window_tap);
  A.cfg = ctx->cfg;
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  if (ctx->timing) {
    for (cudaEvent_t* pe : {&e0, &e1}) {
      if (!ctx->ev_pool.empty()) { *pe = ctx->ev_pool.back(); ctx->ev_pool.pop_back(); }
      else CK(cudaEventCreate(pe));
    }
    CK(cudaEventRecord(e0, s));
  }
  if (use_pack) {
    PackArgs P;
    memset(&P, 0, sizeof(P));
    make_layout_pack(ctx->cfg, pack_segments_per_cta(ctx, nseg), sc16 ? (int)sizeof(RawSc16::T) : (int)sizeof(RawFc32::T), P);
    P.iq = A.iq; P.scale = scale; P.n_raw = A.n_raw; P.segs = A.segs; P.nseg = nseg; P.seg_base = seg_base; P.max_windows = A.max_windows;
    P.results = A.results; P.counts = A.counts; P.window_tap = A.window_tap; P.y_hist = reinterpret_cast<float2*>(ctx->d_yhist.p);
    P.cfg = ctx->cfg;
    // the y history belongs to one launch at a time: a launch on another stream than the previous one waits for it
    if (ctx->hist_used && ctx->hist_stream != s) CK(cudaStreamWaitEvent(s, ctx->ev_hist, 0));
    pack_fn kern = pack_kernel(P.pas, sc16);
    kern<<<(nseg + P.G - 1) / P.G, pack_threads(P.G), P.smem_bytes, s>>>(P);
    CK(cudaEventRecord(ctx->ev_hist, s));
    ctx->hist_stream = s; ctx->hist_used = true;
  } else {
    fn<<<nseg, fast_path_ok(ctx->cfg) ? kSplitThreads : kFusedThreads, A.smem_bytes, s>>>(A);
  }
  CK(cudaGetLastError());
  if (ctx->timing) {
    CK(cudaEventRecord(e1, s));
    ctx->pending.emplace_back(e0, e1);
  }
  ctx->last_launches = 1;
  return RFID_B200_OK;
}

int rfid_b200_decode_capture_host(rfid_b200_ctx* ctx, const float* h_iq, size_t n_raw, const rfid_b200_segment* h_segs,
                                  int nseg, int max_windows_per_segment, rfid_b200_window_result* h_results,
                                  int32_t* h_counts)
{
  if (!ctx || !h_iq || !h_segs || !h_results || !h_counts || nseg < 0 || max_windows_per_segment < 1) return RFID_B200_EINVAL;
  if (nseg == 0) return RFID_B200_OK;
  CK(cudaSetDevice(ctx->device));
  int rc;
  const size_t res_bytes = (size_t)nseg * max_windows_per_segment * sizeof(rfid_b200_window_result);
  if ((rc = grow(ctx, ctx->d_iq, n_raw * 8 + 16))) return rc;
  if ((rc = grow(ctx, ctx->d_segs, (size_t)nseg * sizeof(rfid_b200_segment)))) return rc;
  if ((rc = grow(ctx, ctx->d_res, res_bytes))) return rc;
  if ((rc = grow(ctx, ctx->d_cnt, (size_t)nseg * 4))) return rc;
  cudaStream_t s = ctx->stream;
  CK(cudaMemcpyAsync(ctx->d_segs.p, h_segs, (size_t)nseg * sizeof(rfid_b200_segment), cudaMemcpyHostToDevice, s));
  CK(cudaMemsetAsync(ctx->d_res.p, 0, res_bytes, s));
  // Pinned source: the call is a pipeline over slices of the segment table -- upload of slice k+1 (copy stream) beside the
  // decode of slice k and the download of slice k-1's records (compute stream).  The call as a whole is bound by the
  // host -> device link (8 B per sample); the pipeline takes the decode and the record download off its tail.
  // Pageable source: one plain copy (the driver stages it synchronously anyway).
  cudaPointerAttributes attr;
  const bool pinned = cudaPointerGetAttributes(&attr, h_iq) == cudaSuccess && attr.type == cudaMemoryTypeHost;
  cudaGetLastError();
  const int n_slices = (pinned && nseg >= 64) ? 4 : 1;
  if (n_slices == 1) CK(cudaMemcpyAsync(ctx->d_iq.p, h_iq, n_raw * 8, cudaMemcpyHostToDevice, s));
  int launches = 0;
  for (int k = 0; k < n_slices; k++) {
    const int b = (int)((long long)nseg * k / n_slices), e = (int)((long long)nseg * (k + 1) / n_slices);
    if (e <= b) continue;
    if (n_slices > 1) {
      unsigned long long lo = ~0ull, hi = 0;
      for (int i = b; i < e; i++) {
        const unsigned long long o = h_segs[i].offset, t = o + h_segs[i].length;
        if (o < lo) lo = o;
        if (t > hi) hi = t;
      }
      if (hi > n_raw) hi = n_raw;
      if (lo > hi) lo = hi;
      lo = lo >= 4 ? lo - 4 : 0;  // (the tile loader rounds a segment's first sample down to an even index)
      if (hi > lo) CK(cudaMemcpyAsync((char*)ctx->d_iq.p + lo * 8, (const char*)h_iq + lo * 8, (hi - lo) * 8, cudaMemcpyHostToDevice, ctx->copy_stream));
      CK(cudaEventRecord(ctx->ev_slice[k], ctx->copy_stream));
      CK(cudaStreamWaitEvent(s, ctx->ev_slice[k], 0));
    }
    rc = decode_capture_impl(ctx, ctx->d_iq.p, false, 1.f, n_raw, (const rfid_b200_segment*)ctx->d_segs.p + b, e - b,
                             max_windows_per_segment, (rfid_b200_window_result*)ctx->d_res.p + (size_t)b * max_windows_per_segment,
                             (int32_t*)ctx->d_cnt.p + b, s, b);
    if (rc) return rc;
    launches += ctx->last_launches;
    const size_t rb = (size_t)(e - b) * max_windows_per_segment * sizeof(rfid_b200_window_result);
    CK(cudaMemcpyAsync((char*)h_results + (size_t)b * max_windows_per_segment * sizeof(rfid_b200_window_result),
                       (char*)ctx->d_res.p + (size_t)b * max_windows_per_segment * sizeof(rfid_b200_window_result), rb,
                       cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(h_counts + b, (int32_t*)ctx->d_cnt.p + b, (size_t)(e - b) * 4, cudaMemcpyDeviceToHost, s));
  }
  CK(cudaStreamSynchronize(s));
  ctx->last_launches = launches;
  return RFID_B200_OK;
}

// READER_STATS bookkeeping: tag_decoder_impl.cc:269-288 (RN16 too short), :295 (slot++ per EPC window),
// :329-365 (CRC ok), :366-387 (CRC fail), reader_impl.cc:259,336 (n_queries_sent), gate_impl.cc:101-109 (stop rule).
int rfid_b200_reduce_stats(const rfid_b200_ctx* ctx, const rfid_b200_window_result* recs, const int32_t* counts, int nseg,
                           int max_per_seg, int continuous, rfid_b200_stats* out)
{
  if (!ctx || !recs || !counts || !out || nseg < 0 || max_per_seg < 1) return RFID_B200_EINVAL;
  memset(out, 0, sizeof(*out));
  const int max_slot = 1 << ctx->cfg.fixed_q;
  out->max_slot_number = max_slot;
  std::map<int, int> tag_reads;   // what print_results() reports
  std::map<int, int> seg_reads;   // non-continuous mode: the tag_reads of the segment's own (fresh) reader_state
  int round = 1, slot = 1, nq = 1, total_q = 0;
  bool stopped = false;
  for (int s = 0; s < nseg; s++) {
    // an independent segment = a reference run with freshly constructed blocks: counters AND the unique-tag stop rule
    // (gate_impl.cc:101-104) start over; the global map only accumulates for reporting
    if (!continuous) { round = 1; slot = 1; nq = 1; stopped = false; seg_reads.clear(); }
    std::map<int, int>& rule_reads = continuous ? tag_reads : seg_reads;
    const int n = counts[s] < max_per_seg ? counts[s] : max_per_seg;
    const rfid_b200_window_result* r = recs + (size_t)s * max_per_seg;
    for (int k = 0; k < n && !stopped; k++) {
      bool next_query = false;
      if (r[k].kind == RFID_B200_RN16) {
        if (r[k].crc_ok == -2) {
          slot++;
          if (slot > max_slot) { slot = 1; round++; }
          next_query = true;
        }
      } else {
        slot++;
        if (slot > max_slot) { slot = 1; round++; }
        if (r[k].crc_ok == 1) {
          out->n_epc_correct++;
          tag_reads[r[k].tag_id]++;
          if (!continuous) seg_reads[r[k].tag_id]++;
        }
        next_query = true;
      }
      out->n_windows++;
      if (next_query) {
        nq++;
        if (nq > ctx->cfg.max_queries || (int)rule_reads.size() > ctx->cfg.max_tags) stopped = true;
      }
    }
    if (!continuous) total_q += nq;
  }
  out->n_queries_sent = continuous ? nq : total_q;
  out->cur_inventory_round = round;
  out->cur_slot_number = slot;
  out->terminated = stopped ? 1 : 0;
  out->n_unique_tags = (int)tag_reads.size();
  int k = 0;
  for (auto& kv : tag_reads) {
    if (k >= RFID_B200_MAX_TAGS) break;
    out->tag_id[k] = kv.first;
    out->tag_reads[k] = kv.second;
    k++;
  }
  return RFID_B200_OK;
}

// ------------------------------------------------------------------ capture ingest (SURVEY 8f-2)
}  // extern "C"

namespace {

constexpr size_t kUploadBytes = (size_t)1 << 24;    // 16 MiB per upload slice: 2^21 fc32 or 2^22 sc16 samples, multiples of kIngestChunk
constexpr size_t kLevelHead = (size_t)1 << 21;      // CW level is estimated on the head of the capture

struct SegmenterCfg {
  float level_frac;
  unsigned int gap, lead;
  int min_pulses, commands;
};

int resolve_segmenter(const rfid_b200_ctx* ctx, const rfid_b200_segmenter* sp, SegmenterCfg& o)
{
  rfid_b200_segmenter d;
  rfid_b200_default_segmenter(&d);
  if (sp) d = *sp;
  if (!(d.level_frac > 0.f && d.level_frac < 1.f) || !(d.gap_us > 0.f) || !(d.lead_us >= 0.f) || d.min_pulses < 1 ||
      d.commands_per_segment < 1)
    return RFID_B200_EINVAL;
  o.level_frac = d.level_frac;
  o.gap = (unsigned int)((double)d.gap_us * 1e-6 * ctx->cfg.adc_rate);
  o.lead = (unsigned int)((double)d.lead_us * 1e-6 * ctx->cfg.adc_rate);
  if (o.gap < 1) o.gap = 1;
  if (o.lead >= o.gap) return RFID_B200_EINVAL;  // a lead-in must not reach into the previous command
  o.min_pulses = d.min_pulses;
  o.commands = d.commands_per_segment;
  return RFID_B200_OK;
}

int ingest_alloc(rfid_b200_ctx* ctx, size_t n_raw, const SegmenterCfg& sc, long long& n_chunks, unsigned int& burst_cap)
{
  n_chunks = (long long)((n_raw + kIngestChunk - 1) / kIngestChunk);
  burst_cap = (unsigned int)(n_raw / sc.gap + 4);
  int rc;
  if ((rc = grow(ctx, ctx->d_mask, (size_t)n_chunks * 32 * 4))) return rc;
  if ((rc = grow(ctx, ctx->d_chunk, (size_t)n_chunks * 28 + 64))) return rc;
  if ((rc = grow(ctx, ctx->d_bursts, (size_t)burst_cap * sizeof(IngestBurst)))) return rc;
  return grow(ctx, ctx->d_ing, kLevelBlocks * sizeof(double) + sizeof(IngestTotals));
}

struct IngestPtrs {
  double* partial; IngestTotals* tot;
  unsigned int* mask; long long* chunk_last; long long* prev_low; unsigned long long* falls_before; unsigned int* chunk_falls;
};

IngestPtrs ingest_ptrs(rfid_b200_ctx* ctx, long long n_chunks)
{
  IngestPtrs P;
  P.partial = reinterpret_cast<double*>(ctx->d_ing.p);
  P.tot = reinterpret_cast<IngestTotals*>(P.partial + kLevelBlocks);
  P.mask = reinterpret_cast<unsigned int*>(ctx->d_mask.p);
  P.chunk_last = reinterpret_cast<long long*>(ctx->d_chunk.p);
  P.prev_low = P.chunk_last + n_chunks;
  P.falls_before = reinterpret_cast<unsigned long long*>(P.prev_low + n_chunks);
  P.chunk_falls = reinterpret_cast<unsigned int*>(P.falls_before + n_chunks);
  return P;
}

// the capture in device memory: its samples and their format (RAW of rx_common.cuh)
struct DevCapture {
  const void* iq;
  bool sc16;
  float scale;   // sc16 only
};

int launch_level(rfid_b200_ctx* ctx, const DevCapture& X, size_t n_raw, const SegmenterCfg& sc, const IngestPtrs& P, cudaStream_t s)
{
  const unsigned long long n0 = n_raw < kLevelHead ? n_raw : kLevelHead;
  if (X.sc16)
    ingest_level_partial<RawSc16><<<kLevelBlocks, kLevelThreads, 0, s>>>(static_cast<const uint32_t*>(X.iq), X.scale, n0, P.partial);
  else
    ingest_level_partial<RawFc32><<<kLevelBlocks, kLevelThreads, 0, s>>>(static_cast<const float2*>(X.iq), 1.f, n0, P.partial);
  ingest_level_final<<<1, 32, 0, s>>>(P.partial, n0, sc.level_frac, P.tot);
  CK(cudaGetLastError());
  ctx->last_launches += 2;
  return RFID_B200_OK;
}

int launch_mask(rfid_b200_ctx* ctx, const DevCapture& X, size_t n_raw, long long first_chunk, long long n, const IngestPtrs& P,
                cudaStream_t s)
{
  if (n <= 0) return RFID_B200_OK;
  long long blocks = (n + 7) / 8;
  if (blocks > ctx->sm_count * 8) blocks = ctx->sm_count * 8;
  if (X.sc16)
    ingest_mask<RawSc16><<<(unsigned)blocks, 256, 0, s>>>(static_cast<const uint32_t*>(X.iq), X.scale, n_raw, first_chunk, n,
                                                          P.tot, P.mask, P.chunk_last, P.chunk_falls);
  else
    ingest_mask<RawFc32><<<(unsigned)blocks, 256, 0, s>>>(static_cast<const float2*>(X.iq), 1.f, n_raw, first_chunk, n, P.tot,
                                                          P.mask, P.chunk_last, P.chunk_falls);
  CK(cudaGetLastError());
  ctx->last_launches += 1;
  return RFID_B200_OK;
}

// scan + burst extraction + copy back; synchronises `s`
int finish_bursts(rfid_b200_ctx* ctx, long long n_chunks, unsigned int burst_cap, const SegmenterCfg& sc, const IngestPtrs& P,
                  cudaStream_t s, IngestTotals& tot)
{
  ingest_scan<<<1, 1024, 0, s>>>(n_chunks, P.chunk_last, P.chunk_falls, P.prev_low, P.falls_before, P.tot);
  long long blocks = (n_chunks + 7) / 8;
  if (blocks > ctx->sm_count * 8) blocks = ctx->sm_count * 8;
  ingest_bursts<<<(unsigned)blocks, 256, 0, s>>>(n_chunks, P.mask, P.prev_low, P.falls_before, sc.gap,
                                                 reinterpret_cast<IngestBurst*>(ctx->d_bursts.p), burst_cap, P.tot);
  CK(cudaGetLastError());
  ctx->last_launches += 2;
  CK(cudaMemcpyAsync(&tot, P.tot, sizeof(tot), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  if (tot.n_bursts > burst_cap) { ctx->last_error = "segmenter: burst list overflow"; return RFID_B200_ECAPACITY; }
  ctx->h_bursts.resize(tot.n_bursts);
  if (tot.n_bursts) {
    CK(cudaMemcpyAsync(ctx->h_bursts.data(), ctx->d_bursts.p, (size_t)tot.n_bursts * sizeof(IngestBurst), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
  }
  std::sort(ctx->h_bursts.begin(), ctx->h_bursts.end(), [](const IngestBurst& a, const IngestBurst& b) { return a.pos < b.pos; });
  return RFID_B200_OK;
}

// Pair commands into segments.  Segment j covers commands [j*C, (j+1)*C): it starts `lead` samples before its
// first command (rounded down to a multiple of decim so the matched filter keeps the capture's decimation
// phase; the first segment starts at sample 0 like the reference's continuous run) and runs up to the first
// pulse of the next segment's first command, i.e. consecutive segments overlap by the lead-in.
int build_segments(const rfid_b200_ctx* ctx, const std::vector<IngestBurst>& b, unsigned long long n_falls, size_t n_raw,
                   const SegmenterCfg& sc, rfid_b200_segment* out, int capacity, int* nseg)
{
  std::vector<unsigned long long> cmd;
  for (size_t k = 0; k < b.size(); k++) {
    const unsigned long long next_rank = k + 1 < b.size() ? b[k + 1].rank : n_falls;
    if (next_rank - b[k].rank >= (unsigned long long)sc.min_pulses) cmd.push_back(b[k].pos);
  }
  const size_t C = (size_t)sc.commands;
  const size_t ns = cmd.empty() ? (n_raw ? 1 : 0) : (cmd.size() + C - 1) / C;
  *nseg = (int)ns;
  if ((int)ns > capacity) return RFID_B200_ECAPACITY;
  const unsigned long long D = (unsigned long long)ctx->cfg.decim;
  for (size_t j = 0; j < ns; j++) {
    unsigned long long start = 0;
    if (j > 0) {
      const unsigned long long c0 = cmd[j * C];
      start = c0 > sc.lead ? c0 - sc.lead : 0;
      start -= start % D;
    }
    const unsigned long long end = (j + 1) * C < cmd.size() ? cmd[(j + 1) * C] : (unsigned long long)n_raw;
    if (end - start > 0xffffffffull) return RFID_B200_EINVAL;
    out[j].offset = start;
    out[j].length = (uint32_t)(end - start);
    out[j].reserved = 0;
  }
  return RFID_B200_OK;
}

}  // namespace

extern "C" {

void rfid_b200_default_segmenter(rfid_b200_segmenter* sp)
{
  if (!sp) return;
  memset(sp, 0, sizeof(*sp));
  sp->level_frac = 0.5f;
  sp->gap_us = 400.f;
  sp->lead_us = 300.f;
  sp->min_pulses = kNumPulsesCommand + 1;  // gate_impl.cc:164: num_pulses > NUM_PULSES_COMMAND
  sp->commands_per_segment = 2;            // RN16 window + EPC window
}

}  // extern "C"

static int segment_capture_impl(rfid_b200_ctx* ctx, const DevCapture& X, size_t n_raw, const rfid_b200_segmenter* sp,
                                rfid_b200_segment* h_segs, int capacity, int* nseg, void* stream)
{
  if (!ctx || !X.iq || !h_segs || !nseg || capacity < 0) return RFID_B200_EINVAL;
  *nseg = 0;
  SegmenterCfg sc;
  int rc = resolve_segmenter(ctx, sp, sc);
  if (rc) return rc;
  if (n_raw == 0) return RFID_B200_OK;
  CK(cudaSetDevice(ctx->device));
  long long n_chunks;
  unsigned int burst_cap;
  if ((rc = ingest_alloc(ctx, n_raw, sc, n_chunks, burst_cap))) return rc;
  const IngestPtrs P = ingest_ptrs(ctx, n_chunks);
  cudaStream_t s = (cudaStream_t)stream;
  ctx->last_launches = 0;
  if ((rc = launch_level(ctx, X, n_raw, sc, P, s))) return rc;
  if ((rc = launch_mask(ctx, X, n_raw, 0, n_chunks, P, s))) return rc;
  IngestTotals tot;
  if ((rc = finish_bursts(ctx, n_chunks, burst_cap, sc, P, s, tot))) return rc;
  return build_segments(ctx, ctx->h_bursts, tot.n_falls, n_raw, sc, h_segs, capacity, nseg);
}

// h_iq: n_raw samples of sample_bytes each (8 fc32, 4 sc16)
static int ingest_capture_host_impl(rfid_b200_ctx* ctx, const void* h_iq, bool sc16, float scale, size_t n_raw,
                                    const rfid_b200_segmenter* sp, int max_windows_per_segment, rfid_b200_segment* h_segs,
                                    int seg_capacity, int* nseg, rfid_b200_window_result* h_results, int32_t* h_counts)
{
  if (!ctx || !h_iq || !h_segs || !nseg || !h_results || !h_counts || seg_capacity < 0 || max_windows_per_segment < 1)
    return RFID_B200_EINVAL;
  const size_t sb = sc16 ? sizeof(RawSc16::T) : sizeof(RawFc32::T);   // bytes per sample
  const size_t slice_samples = kUploadBytes / sb;
  *nseg = 0;
  SegmenterCfg sc;
  int rc = resolve_segmenter(ctx, sp, sc);
  if (rc) return rc;
  if (n_raw == 0) return RFID_B200_OK;
  if (!pick_kernel(ctx->cfg, sc16)) { ctx->last_error = "capture mode supports decim = 5 only in this build"; return RFID_B200_EINVAL; }
  CK(cudaSetDevice(ctx->device));
  long long n_chunks;
  unsigned int burst_cap;
  if ((rc = ingest_alloc(ctx, n_raw, sc, n_chunks, burst_cap))) return rc;
  if ((rc = grow(ctx, ctx->d_iq, n_raw * sb + 16))) return rc;
  const IngestPtrs P = ingest_ptrs(ctx, n_chunks);
  cudaStream_t s = ctx->stream;
  const DevCapture X{ctx->d_iq.p, sc16, scale};

  // pageable sources go through two pinned staging slices so the host memcpy of slice k+1 overlaps the DMA of
  // slice k; pinned (registered) sources are DMA'd directly.  The threshold pass runs behind each slice.
  cudaPointerAttributes attr;
  bool pinned = cudaPointerGetAttributes(&attr, h_iq) == cudaSuccess && attr.type == cudaMemoryTypeHost;
  cudaGetLastError();
  if (!pinned) {
    for (int b = 0; b < 2; b++) {
      if (!ctx->h_stage[b]) {
        if (cudaHostAlloc(&ctx->h_stage[b], kUploadBytes, cudaHostAllocDefault) != cudaSuccess) {
          cudaGetLastError();
          return RFID_B200_ENOMEM;
        }
        CK(cudaEventCreateWithFlags(&ctx->ev_stage[b], cudaEventDisableTiming));
      }
    }
  }
  ctx->last_launches = 0;
  int launches = 0;
  size_t slice = 0;
  for (size_t off = 0; off < n_raw; off += slice_samples, slice++) {
    const size_t n = n_raw - off < slice_samples ? n_raw - off : slice_samples;
    const char* src = static_cast<const char*>(h_iq) + off * sb;
    if (!pinned) {
      const int b = (int)(slice & 1);
      if (slice >= 2) CK(cudaEventSynchronize(ctx->ev_stage[b]));
      memcpy(ctx->h_stage[b], src, n * sb);
      CK(cudaMemcpyAsync((char*)ctx->d_iq.p + off * sb, ctx->h_stage[b], n * sb, cudaMemcpyHostToDevice, s));
      CK(cudaEventRecord(ctx->ev_stage[b], s));
    } else {
      CK(cudaMemcpyAsync((char*)ctx->d_iq.p + off * sb, src, n * sb, cudaMemcpyHostToDevice, s));
    }
    // (the first slice holds the level's head: kLevelHead <= 2^21 samples)
    if (off == 0 && (rc = launch_level(ctx, X, n_raw, sc, P, s))) return rc;
    const long long first = (long long)(off / kIngestChunk);
    const long long cnt = (long long)((n + kIngestChunk - 1) / kIngestChunk);
    // the mask kernel treats samples beyond `off + n` as not yet present: pass the uploaded extent (samples) as n_raw
    if ((rc = launch_mask(ctx, X, off + n, first, cnt, P, s))) return rc;
  }
  IngestTotals tot;
  if ((rc = finish_bursts(ctx, n_chunks, burst_cap, sc, P, s, tot))) return rc;
  launches = ctx->last_launches;
  if ((rc = build_segments(ctx, ctx->h_bursts, tot.n_falls, n_raw, sc, h_segs, seg_capacity, nseg))) return rc;
  const int ns = *nseg;
  if (ns == 0) return RFID_B200_OK;
  const size_t res_bytes = (size_t)ns * max_windows_per_segment * sizeof(rfid_b200_window_result);
  if ((rc = grow(ctx, ctx->d_segs, (size_t)ns * sizeof(rfid_b200_segment)))) return rc;
  if ((rc = grow(ctx, ctx->d_res, res_bytes))) return rc;
  if ((rc = grow(ctx, ctx->d_cnt, (size_t)ns * 4))) return rc;
  CK(cudaMemcpyAsync(ctx->d_segs.p, h_segs, (size_t)ns * sizeof(rfid_b200_segment), cudaMemcpyHostToDevice, s));
  CK(cudaMemsetAsync(ctx->d_res.p, 0, res_bytes, s));
  rc = decode_capture_impl(ctx, ctx->d_iq.p, sc16, scale, n_raw, (const rfid_b200_segment*)ctx->d_segs.p, ns,
                           max_windows_per_segment, (rfid_b200_window_result*)ctx->d_res.p, (int32_t*)ctx->d_cnt.p, s, 0);
  if (rc) return rc;
  ctx->last_launches += launches;
  CK(cudaMemcpyAsync(h_results, ctx->d_res.p, res_bytes, cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(h_counts, ctx->d_cnt.p, (size_t)ns * 4, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  return RFID_B200_OK;
}

extern "C" {

int rfid_b200_segment_capture(rfid_b200_ctx* ctx, const float* d_iq, size_t n_raw, const rfid_b200_segmenter* sp,
                              rfid_b200_segment* h_segs, int capacity, int* nseg, void* stream)
{
  return segment_capture_impl(ctx, DevCapture{d_iq, false, 1.f}, n_raw, sp, h_segs, capacity, nseg, stream);
}

int rfid_b200_segment_capture_sc16(rfid_b200_ctx* ctx, const int16_t* d_iq, size_t n_raw, float scale,
                                   const rfid_b200_segmenter* sp, rfid_b200_segment* h_segs, int capacity, int* nseg,
                                   void* stream)
{
  if (nseg) *nseg = 0;
  if (!scale_ok(scale) || (reinterpret_cast<uintptr_t>(d_iq) & 15u) != 0) return RFID_B200_EINVAL;
  return segment_capture_impl(ctx, DevCapture{d_iq, true, scale}, n_raw, sp, h_segs, capacity, nseg, stream);
}

int rfid_b200_ingest_capture_host(rfid_b200_ctx* ctx, const float* h_iq, size_t n_raw, const rfid_b200_segmenter* sp,
                                  int max_windows_per_segment, rfid_b200_segment* h_segs, int seg_capacity, int* nseg,
                                  rfid_b200_window_result* h_results, int32_t* h_counts)
{
  return ingest_capture_host_impl(ctx, h_iq, false, 1.f, n_raw, sp, max_windows_per_segment, h_segs, seg_capacity, nseg,
                                  h_results, h_counts);
}

int rfid_b200_ingest_capture_host_sc16(rfid_b200_ctx* ctx, const int16_t* h_iq, size_t n_raw, float scale,
                                       const rfid_b200_segmenter* sp, int max_windows_per_segment, rfid_b200_segment* h_segs,
                                       int seg_capacity, int* nseg, rfid_b200_window_result* h_results, int32_t* h_counts)
{
  if (nseg) *nseg = 0;
  if (!scale_ok(scale)) return RFID_B200_EINVAL;
  return ingest_capture_host_impl(ctx, h_iq, true, scale, n_raw, sp, max_windows_per_segment, h_segs, seg_capacity, nseg,
                                  h_results, h_counts);
}

// ------------------------------------------------------------------ TX synthesiser + slot simulator (SURVEY 8f-1)
}  // extern "C"

namespace {

// waveform table sizes with the reference's arithmetic: float sample period, float quotients, truncation
// (reader_impl.cc:51-71)
int derive_tx_timing(int dac_rate, TxTiming& T)
{
  if (dac_rate <= 0) return RFID_B200_EINVAL;
  const float sample_d = 1.0 / dac_rate * std::pow(10, 6);
  const float n_data0 = 2 * kPW_D / sample_d, n_data1 = 4 * kPW_D / sample_d, n_pw = kPW_D / sample_d;
  const float n_cw = kCW_D / sample_d, n_delim = kDELIM_D / sample_d, n_trcal = kTRCAL_D / sample_d;
  const float TAG_BIT_D = (float)(1.0 / kReaderFreq * std::pow(10, 6));
  const int RN16_D = (int)((kRN16Bits + kTagPreambleBits) * TAG_BIT_D);
  const int EPC_D = (int)((kEPCBits + kTagPreambleBits) * TAG_BIT_D);
  T.n_data0 = (int)n_data0; T.n_data1 = (int)n_data1; T.n_pw = (int)n_pw; T.n_delim = (int)n_delim;
  T.n_rtcal = (int)(n_data0 + n_data1); T.n_trcal = (int)n_trcal; T.n_cw = (int)n_cw;
  T.n_cwquery = (int)((kT1_D + kT2_D + RN16_D) / sample_d);
  T.n_cwack = (int)((3 * kT1_D + kT2_D + EPC_D) / sample_d);
  T.n_pdown = (int)(kP_DOWN_D / sample_d);
  if (T.n_pw < 1 || T.n_data0 < 2) return RFID_B200_EINVAL;
  return RFID_B200_OK;
}

// step response of the TX/RX chain measured on the recording (falling edge, raw 2 MS/s samples)
const float kEdgeFir2Msps[] = {-0.07f, 0.32f, 0.52f, 0.155f, 0.005f, 0.03f, 0.01f, 0.01f, 0.01f, 0.005f, 0.005f};

int build_sim_args(const rfid_b200_ctx* ctx, const rfid_b200_sim_params& p, SimArgs& A)
{
  memset(&A, 0, sizeof(A));
  if (p.n_tags < 0 || p.n_tags > kSimMaxTags || !(p.segment_us > 0.f) || !(p.lead_us >= 0.f) || p.dac_rate <= 0) return RFID_B200_EINVAL;
  if (ctx->cfg.adc_rate % p.dac_rate != 0) return RFID_B200_EINVAL;
  int rc = derive_tx_timing(p.dac_rate, A.T);
  if (rc) return rc;
  A.p = p;
  A.fixed_q = ctx->cfg.fixed_q;
  A.hold = ctx->cfg.adc_rate / p.dac_rate;
  A.sps = ctx->cfg.adc_rate / 1e6;
  A.dac_us = 1e6 / p.dac_rate;
  A.seg_len = (int)std::lround((double)p.segment_us * A.sps);
  A.lead_dac = (int)std::lround((double)p.lead_us / A.dac_us);
  // edge response stretched to the same duration at other ADC rates (linear interpolation, unit DC gain)
  const int n2 = (int)(sizeof(kEdgeFir2Msps) / sizeof(float));
  if (ctx->cfg.adc_rate == 2000000) {
    A.n_fir = n2;
    for (int i = 0; i < n2; i++) A.fir[i] = kEdgeFir2Msps[i];
  } else {
    int L = (int)std::lround(n2 * A.sps / 2.0);
    if (L < 3) L = 3;
    if (L > kSimMaxFir) L = kSimMaxFir;
    double sum = 0.0;
    for (int i = 0; i < L; i++) {
      const double x = (double)i * (n2 - 1) / (L - 1);
      const int i0 = (int)x;
      const int i1 = i0 + 1 < n2 ? i0 + 1 : i0;
      const double v = kEdgeFir2Msps[i0] + (kEdgeFir2Msps[i1] - kEdgeFir2Msps[i0]) * (x - i0);
      A.fir[i] = (float)v;
      sum += v;
    }
    for (int i = 0; i < L; i++) A.fir[i] = (float)(A.fir[i] / sum);
    A.n_fir = L;
  }
  A.mask_words = (A.seg_len + 31) / 32 + 1;
  if (A.seg_len < 64 || sizeof(SimShared) + 16 + (size_t)A.mask_words * 4 > 200 * 1024) return RFID_B200_EINVAL;
  return RFID_B200_OK;
}

}  // namespace

extern "C" {

int rfid_b200_tx_synth(rfid_b200_ctx* ctx, const rfid_b200_tx_command* h_script, int n_commands, int dac_rate, float* d_out,
                       size_t capacity, size_t* n_samples, void* stream)
{
  if (!ctx || !h_script || n_commands < 0 || !n_samples) return RFID_B200_EINVAL;
  TxTiming T;
  int rc = derive_tx_timing(dac_rate, T);
  if (rc) return rc;
  std::vector<unsigned long long> off((size_t)n_commands + 1, 0ull);
  for (int c = 0; c < n_commands; c++) {
    if (h_script[c].kind < RFID_B200_TX_START || h_script[c].kind > RFID_B200_TX_QUERY_ADJUST) return RFID_B200_EINVAL;
    off[c + 1] = off[c] + (unsigned long long)tx_length(T, h_script[c].kind, h_script[c].arg, ctx->cfg.fixed_q);
  }
  *n_samples = (size_t)off[n_commands];
  ctx->last_launches = 0;
  if (!d_out) return RFID_B200_OK;
  if (capacity < *n_samples) return RFID_B200_ECAPACITY;
  if (n_commands == 0) return RFID_B200_OK;
  CK(cudaSetDevice(ctx->device));
  const size_t sb = (size_t)n_commands * sizeof(rfid_b200_tx_command), ob = (size_t)n_commands * 8;
  if ((rc = grow(ctx, ctx->d_script, sb + ob + 16))) return rc;
  cudaStream_t s = (cudaStream_t)stream;
  unsigned long long* d_off = reinterpret_cast<unsigned long long*>(ctx->d_script.p);
  rfid_b200_tx_command* d_scr = reinterpret_cast<rfid_b200_tx_command*>(d_off + n_commands);
  // pageable sources: cudaMemcpyAsync stages them before returning, so the vectors may go out of scope
  CK(cudaMemcpyAsync(d_off, off.data(), ob, cudaMemcpyHostToDevice, s));
  CK(cudaMemcpyAsync(d_scr, h_script, sb, cudaMemcpyHostToDevice, s));
  tx_synth_kernel<<<n_commands, 256, 0, s>>>(T, ctx->cfg.fixed_q, d_scr, d_off, n_commands, d_out);
  CK(cudaGetLastError());
  ctx->last_launches = 1;
  return RFID_B200_OK;
}

void rfid_b200_default_sim(rfid_b200_sim_params* p)
{
  if (!p) return;
  memset(p, 0, sizeof(*p));
  p->seed = 1234;
  p->n_tags = 1;
  p->closed_loop = 1;
  p->dac_rate = 1000000;  // apps/reader.py:56
  p->segment_us = 8480.f;
  p->lead_us = 400.f;
  p->noise_sigma = 0.0030f;
  p->tag_gain = 0.0227f;
  p->tag_phase = std::atan2(0.192f, -0.981f);
  p->clock_pct = 0.8f;
  p->leak_re = 0.2846f;
  p->leak_im = -0.0349f;
  p->floor_level = 0.004f;
}

int rfid_b200_sim_segment_length(const rfid_b200_ctx* ctx, const rfid_b200_sim_params* p)
{
  if (!ctx || !p) return RFID_B200_EINVAL;
  SimArgs A;
  int rc = build_sim_args(ctx, *p, A);
  return rc ? rc : A.seg_len;
}

int rfid_b200_sim_capture(rfid_b200_ctx* ctx, const rfid_b200_sim_params* p, int64_t first_segment, int nseg, float* d_iq,
                          rfid_b200_segment* d_segs, rfid_b200_sim_truth* d_truth, void* stream)
{
  if (!ctx || !p || !d_iq || !d_segs || nseg < 0 || first_segment < 0) return RFID_B200_EINVAL;
  SimArgs A;
  int rc = build_sim_args(ctx, *p, A);
  if (rc) return rc;
  ctx->last_launches = 0;
  if (nseg == 0) return RFID_B200_OK;
  CK(cudaSetDevice(ctx->device));
  cudaStream_t s = (cudaStream_t)stream;
  const size_t smem = ((sizeof(SimShared) + 15) & ~(size_t)15) + (size_t)A.mask_words * 4;
  CK(cudaFuncSetAttribute((const void*)sim_slot_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  A.first_segment = first_segment; A.nseg = nseg;
  A.iq = reinterpret_cast<float2*>(d_iq); A.segs = d_segs; A.truth = d_truth;
  int launches = 0;
  if (!p->closed_loop) {
    A.phase = 2;
    sim_slot_kernel<<<nseg, kSimThreads, smem, s>>>(A);
    CK(cudaGetLastError());
    launches = 1;
  } else {
    // Query + RN16 replies -> decode the RN16 window with this context's receive chain -> ACK(decoded) + EPC
    if (!pick_kernel(ctx->cfg)) { ctx->last_error = "capture mode supports decim = 5 only in this build"; return RFID_B200_EINVAL; }
    if ((rc = grow(ctx, ctx->d_sim_res, (size_t)nseg * sizeof(rfid_b200_window_result)))) return rc;
    if ((rc = grow(ctx, ctx->d_sim_cnt, (size_t)nseg * 4))) return rc;
    A.phase = 0;
    sim_slot_kernel<<<nseg, kSimThreads, smem, s>>>(A);
    CK(cudaGetLastError());
    CK(cudaMemsetAsync(ctx->d_sim_res.p, 0, (size_t)nseg * sizeof(rfid_b200_window_result), s));
    rc = rfid_b200_decode_capture(ctx, d_iq, (size_t)nseg * A.seg_len, d_segs, nseg, 1, (rfid_b200_window_result*)ctx->d_sim_res.p,
                                  (int32_t*)ctx->d_sim_cnt.p, s);
    if (rc) return rc;
    A.phase = 1;
    A.rn16_records = (const rfid_b200_window_result*)ctx->d_sim_res.p;
    A.rn16_counts = (const int32_t*)ctx->d_sim_cnt.p;
    sim_slot_kernel<<<nseg, kSimThreads, smem, s>>>(A);
    CK(cudaGetLastError());
    launches = 3;
  }
  ctx->last_launches = launches;
  return RFID_B200_OK;
}

// ------------------------------------------------------------------ capture mode: the reader's commands
void rfid_b200_default_cmd_params(rfid_b200_cmd_params* cp)
{
  if (!cp) return;
  memset(cp, 0, sizeof(*cp));
  cp->level_frac = 0.5f;   // the segmenter's
  cp->gap_us = 400.f;
  cp->level_abs = 0.f;
}

// the kernel's settings from the caller's (NULL = defaults); RFID_B200_EINVAL when they are out of range
static int resolve_cmd_params(const rfid_b200_ctx* ctx, const rfid_b200_cmd_params* cp, CmdArgs& A)
{
  rfid_b200_cmd_params d;
  rfid_b200_default_cmd_params(&d);
  if (cp) d = *cp;
  if (!(d.level_frac > 0.f && d.level_frac < 1.f) || !(d.level_abs >= 0.f) || !std::isfinite(d.level_abs) || !(d.gap_us > 0.f))
    return RFID_B200_EINVAL;
  A.frac2 = d.level_frac * d.level_frac;
  A.use_abs = d.level_abs > 0.f;
  A.abs2 = d.level_abs * d.level_abs;
  const double gap = (double)d.gap_us * 1e-6 * ctx->cfg.adc_rate;   // (a gap beyond any segment length acts as INT32_MAX)
  A.gap = gap >= 2147483647.0 ? 2147483647 : (int)gap;
  return RFID_B200_OK;
}

static int decode_commands_impl(rfid_b200_ctx* ctx, const void* d_iq, bool sc16, float scale, size_t n_raw,
                                const rfid_b200_segment* d_segs, int nseg, const rfid_b200_cmd_params* cp, int max_cmds,
                                rfid_b200_command* d_cmds, int32_t* d_counts, void* stream)
{
  if (!ctx || !d_iq || !d_segs || !d_counts || nseg < 0 || max_cmds < 0 || (max_cmds > 0 && !d_cmds)) return RFID_B200_EINVAL;
  if ((reinterpret_cast<uintptr_t>(d_iq) & (sc16 ? 15u : 7u)) != 0) return RFID_B200_EINVAL;
  CmdArgs A;
  int rc = resolve_cmd_params(ctx, cp, A);
  if (rc) return rc;
  if (nseg == 0) return RFID_B200_OK;
  CK(cudaSetDevice(ctx->device));
  A.iq = d_iq; A.scale = scale; A.n_raw = n_raw; A.segs = d_segs; A.nseg = nseg; A.max_cmds = max_cmds;
  A.cmds = d_cmds; A.counts = d_counts;
  cudaStream_t s = (cudaStream_t)stream;
  if (sc16) rx_cmd_kernel<RawSc16><<<nseg, kCmdThreads, 0, s>>>(A);
  else rx_cmd_kernel<RawFc32><<<nseg, kCmdThreads, 0, s>>>(A);
  CK(cudaGetLastError());
  return RFID_B200_OK;
}

int rfid_b200_decode_commands(rfid_b200_ctx* ctx, const float* d_iq, size_t n_raw, const rfid_b200_segment* d_segs, int nseg,
                              const rfid_b200_cmd_params* cp, int max_commands_per_segment, rfid_b200_command* d_cmds,
                              int32_t* d_counts, void* stream)
{
  return decode_commands_impl(ctx, d_iq, false, 1.f, n_raw, d_segs, nseg, cp, max_commands_per_segment, d_cmds, d_counts, stream);
}

int rfid_b200_decode_commands_sc16(rfid_b200_ctx* ctx, const int16_t* d_iq, size_t n_raw, float scale,
                                   const rfid_b200_segment* d_segs, int nseg, const rfid_b200_cmd_params* cp,
                                   int max_commands_per_segment, rfid_b200_command* d_cmds, int32_t* d_counts, void* stream)
{
  if (!scale_ok(scale)) return RFID_B200_EINVAL;
  return decode_commands_impl(ctx, d_iq, true, scale, n_raw, d_segs, nseg, cp, max_commands_per_segment, d_cmds, d_counts, stream);
}

int rfid_b200_decode_commands_host(rfid_b200_ctx* ctx, const float* h_iq, size_t n_raw, const rfid_b200_segment* h_segs, int nseg,
                                   const rfid_b200_cmd_params* cp, int max_commands_per_segment, rfid_b200_command* h_cmds,
                                   int32_t* h_counts)
{
  if (!ctx || !h_iq || !h_segs || !h_counts || nseg < 0 || max_commands_per_segment < 0 ||
      (max_commands_per_segment > 0 && !h_cmds))
    return RFID_B200_EINVAL;
  CmdArgs A;
  int rc = resolve_cmd_params(ctx, cp, A);
  if (rc) return rc;
  for (int i = 0; i < nseg; i++)
    if (h_segs[i].length > 0x7fffffffu) return RFID_B200_EINVAL;
  if (nseg == 0) return RFID_B200_OK;
  CK(cudaSetDevice(ctx->device));
  const size_t cmd_bytes = (size_t)nseg * max_commands_per_segment * sizeof(rfid_b200_command);
  if ((rc = grow(ctx, ctx->d_iq, n_raw * 8 + 16))) return rc;
  if ((rc = grow(ctx, ctx->d_segs, (size_t)nseg * sizeof(rfid_b200_segment)))) return rc;
  if ((rc = grow(ctx, ctx->d_cmd, cmd_bytes))) return rc;
  if ((rc = grow(ctx, ctx->d_cnt, (size_t)nseg * 4))) return rc;
  cudaStream_t s = ctx->stream;
  CK(cudaMemcpyAsync(ctx->d_iq.p, h_iq, n_raw * 8, cudaMemcpyHostToDevice, s));
  CK(cudaMemcpyAsync(ctx->d_segs.p, h_segs, (size_t)nseg * sizeof(rfid_b200_segment), cudaMemcpyHostToDevice, s));
  if (cmd_bytes) CK(cudaMemsetAsync(ctx->d_cmd.p, 0, cmd_bytes, s));
  rc = decode_commands_impl(ctx, ctx->d_iq.p, false, 1.f, n_raw, (const rfid_b200_segment*)ctx->d_segs.p, nseg, cp,
                            max_commands_per_segment, (rfid_b200_command*)ctx->d_cmd.p, (int32_t*)ctx->d_cnt.p, s);
  if (rc) return rc;
  if (cmd_bytes) CK(cudaMemcpyAsync(h_cmds, ctx->d_cmd.p, cmd_bytes, cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(h_counts, ctx->d_cnt.p, (size_t)nseg * 4, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  return RFID_B200_OK;
}

// ------------------------------------------------------------------ capture mode: reply quality and slot outcome
void rfid_b200_default_quality_params(rfid_b200_quality_params* qp)
{
  if (!qp) return;
  memset(qp, 0, sizeof(*qp));
  qp->empty_db = 9.5f;       // DESIGN.md 4.6: calibrated on the simulator and the recording
  qp->single_snr_db = 8.8f;
}

int rfid_b200_window_quality(rfid_b200_ctx* ctx, const float* d_windows, const rfid_b200_window_result* d_results,
                             const int32_t* d_counts, int nseg, int max_windows, const rfid_b200_quality_params* qp,
                             rfid_b200_quality* d_quality, void* stream)
{
  if (!ctx || !d_windows || !d_results || !d_counts || !d_quality || nseg < 0 || max_windows < 0) return RFID_B200_EINVAL;
  rfid_b200_quality_params d;
  rfid_b200_default_quality_params(&d);
  if (qp) d = *qp;
  if (!std::isfinite(d.empty_db) || !std::isfinite(d.single_snr_db)) return RFID_B200_EINVAL;
  ctx->last_launches = 0;
  const long long slots = (long long)nseg * max_windows;
  if (slots == 0) return RFID_B200_OK;
  CK(cudaSetDevice(ctx->device));
  QualityArgs A;
  A.windows = reinterpret_cast<const float2*>(d_windows);
  A.results = d_results; A.counts = d_counts; A.quality = d_quality;
  A.nseg = nseg; A.max_windows = max_windows;
  A.empty_ratio = std::pow(10.0, (double)d.empty_db / 10.0);
  A.single_ratio = std::pow(10.0, (double)d.single_snr_db / 10.0);
  A.cfg = ctx->cfg;
  rx_quality_kernel<<<slot_grid(slots), 32 * kSlotWarps, 0, (cudaStream_t)stream>>>(A);
  CK(cudaGetLastError());
  ctx->last_launches = 1;
  return RFID_B200_OK;
}

// ------------------------------------------------------------------ capture mode: EPC replies that fail their CRC
void rfid_b200_default_recover_params(rfid_b200_recover_params* rp)
{
  if (!rp) return;
  memset(rp, 0, sizeof(*rp));
  rp->positions = 12;
  rp->max_flips = 4;
  rp->min_snr_db = 7.0f;   // DESIGN.md 4.7: above the EPC windows of empty slots and the replies that recover wrongly
}

int rfid_b200_recover_epc(rfid_b200_ctx* ctx, const float* d_windows, const rfid_b200_window_result* d_results,
                          const int32_t* d_counts, const rfid_b200_quality* d_quality, int nseg, int max_windows,
                          const rfid_b200_recover_params* rp, rfid_b200_epc_fix* d_fix, void* stream)
{
  if (!ctx || !d_windows || !d_results || !d_counts || !d_quality || !d_fix || nseg < 0 || max_windows < 0)
    return RFID_B200_EINVAL;
  rfid_b200_recover_params d;
  rfid_b200_default_recover_params(&d);
  if (rp) d = *rp;
  if (d.positions < 1 || d.positions > kRecoverMaxPositions || d.max_flips < 1 || d.max_flips > d.positions ||
      !std::isfinite(d.min_snr_db))
    return RFID_B200_EINVAL;
  long long n_candidates = 0, binom = 1;
  for (int k = 1; k <= d.max_flips; k++) {   // binomial(P, k), exact: binomial(P, k - 1) * (P - k + 1) is divisible by k
    binom = binom * (d.positions - k + 1) / k;
    n_candidates += binom;
  }
  if (n_candidates > kRecoverMaxCandidates) return RFID_B200_EINVAL;
  ctx->last_launches = 0;
  const long long slots = (long long)nseg * max_windows;
  if (slots == 0) return RFID_B200_OK;
  CK(cudaSetDevice(ctx->device));
  RecoverArgs A;
  A.windows = reinterpret_cast<const float2*>(d_windows);
  A.results = d_results; A.counts = d_counts; A.quality = d_quality; A.fix = d_fix;
  A.nseg = nseg; A.max_windows = max_windows;
  A.positions = d.positions; A.max_flips = d.max_flips; A.n_candidates = (int)n_candidates;
  A.min_snr_ratio = std::pow(10.0, (double)d.min_snr_db / 10.0);
  A.cfg = ctx->cfg;
  rx_recover_kernel<<<slot_grid(slots), 32 * kSlotWarps, 0, (cudaStream_t)stream>>>(A);
  CK(cudaGetLastError());
  ctx->last_launches = 1;
  return RFID_B200_OK;
}

// ------------------------------------------------------------------ capture mode: the tag inventory report
void rfid_b200_default_report_params(rfid_b200_report_params* rp)
{
  if (!rp) return;
  memset(rp, 0, sizeof(*rp));
  rp->check_length = 1;
}

int rfid_b200_tag_report(rfid_b200_ctx* ctx, const rfid_b200_segment* d_segs, const rfid_b200_window_result* d_results,
                         const int32_t* d_counts, int nseg, int max_windows, const rfid_b200_quality* d_quality,
                         const rfid_b200_epc_fix* d_fix, const rfid_b200_report_params* rp, int max_tags,
                         rfid_b200_tag* d_tags, rfid_b200_tag_summary* d_summary, int32_t* d_read_tag, void* stream)
{
  if (!ctx || !d_segs || !d_results || !d_counts || !d_summary || (!d_tags && max_tags > 0) || nseg < 0 ||
      max_windows < 0 || max_tags < 0)
    return RFID_B200_EINVAL;
  const long long slots = (long long)nseg * max_windows;
  if (slots >= (1ll << 31)) return RFID_B200_EINVAL;
  rfid_b200_report_params d;
  rfid_b200_default_report_params(&d);
  if (rp) d = *rp;
  if (d.check_length != 0 && d.check_length != 1) return RFID_B200_EINVAL;
  ctx->last_launches = 0;
  CK(cudaSetDevice(ctx->device));
  cudaStream_t st = (cudaStream_t)stream;
  CK(cudaMemsetAsync(d_summary, 0, sizeof(rfid_b200_tag_summary), st));
  if (slots == 0) return RFID_B200_OK;
  // scratch: aggregates [slots] | hash table [pow2 >= 2 slots] | rep [slots] | block counts; the first two start zeroed
  const int n_blocks = (int)((slots + kReportBlockSlots - 1) / kReportBlockSlots);
  unsigned long long buckets = 64;
  while (buckets < 2ull * (unsigned long long)slots) buckets <<= 1;
  const size_t agg_bytes = (size_t)slots * sizeof(ReportAgg), table_bytes = (size_t)buckets * 4;
  const size_t rep_bytes = (size_t)slots * 4, need = agg_bytes + table_bytes + rep_bytes + (size_t)n_blocks * 4;
  int rc;
  if ((rc = grow(ctx, ctx->d_report, need))) return rc;
  char* base = static_cast<char*>(ctx->d_report.p);
  CK(cudaMemsetAsync(base, 0, agg_bytes + table_bytes, st));
  ReportArgs A;
  A.segs = d_segs; A.results = d_results; A.counts = d_counts; A.quality = d_quality; A.fix = d_fix;
  A.tags = d_tags; A.summary = d_summary; A.read_tag = d_read_tag;
  A.agg = reinterpret_cast<ReportAgg*>(base);
  A.table = reinterpret_cast<unsigned*>(base + agg_bytes);
  A.rep = reinterpret_cast<int32_t*>(base + agg_bytes + table_bytes);
  A.block_count = reinterpret_cast<int32_t*>(base + agg_bytes + table_bytes + rep_bytes);
  A.max_windows = max_windows; A.n_slots = (int)slots; A.n_blocks = n_blocks; A.max_tags = max_tags;
  A.check_length = d.check_length; A.decim = ctx->params.decim;
  A.table_mask = (unsigned)(buckets - 1);
  rx_report_insert_kernel<<<n_blocks, 32 * kReportWarps, 0, st>>>(A);
  rx_report_count_kernel<<<n_blocks, kReportThreads, 0, st>>>(A);
  rx_report_scan_kernel<<<1, kReportScanThreads, 0, st>>>(A);
  rx_report_write_kernel<<<n_blocks, kReportThreads, 0, st>>>(A, false);
  int launches = 4;
  if (d_read_tag) {
    rx_report_write_kernel<<<n_blocks, kReportThreads, 0, st>>>(A, true);
    launches++;
  }
  CK(cudaGetLastError());
  ctx->last_launches = launches;
  return RFID_B200_OK;
}

// ------------------------------------------------------------------ capture mode: EPC replies from tags you already know
void rfid_b200_default_match_params(rfid_b200_match_params* mp)
{
  if (!mp) return;
  memset(mp, 0, sizeof(*mp));
  mp->max_cost = 12.0f;    // DESIGN.md 4.9: below every noise window at K = 65,536, above the weak replies' costs
  mp->min_margin = 4.0f;
}

int rfid_b200_match_epc(rfid_b200_ctx* ctx, const float* d_windows, const rfid_b200_window_result* d_results,
                        const int32_t* d_counts, const rfid_b200_epc_fix* d_fix, int nseg, int max_windows,
                        const uint8_t* d_dict, const int32_t* d_n_dict, int max_dict, const rfid_b200_match_params* mp,
                        rfid_b200_epc_match* d_match, rfid_b200_match_count* d_count, void* stream)
{
  if (!ctx || !d_windows || !d_results || !d_counts || !d_match || (!d_dict && max_dict > 0) || nseg < 0 ||
      max_windows < 0 || max_dict < 0 || max_dict > kMatchMaxDict || ((uintptr_t)d_dict & 15u))
    return RFID_B200_EINVAL;
  const long long slots = (long long)nseg * max_windows;
  if (slots >= (1ll << 31)) return RFID_B200_EINVAL;
  rfid_b200_match_params d;
  rfid_b200_default_match_params(&d);
  if (mp) d = *mp;
  if (!std::isfinite(d.max_cost) || !std::isfinite(d.min_margin) || d.max_cost < 0.0f || d.min_margin < 0.0f)
    return RFID_B200_EINVAL;
  ctx->last_launches = 0;
  CK(cudaSetDevice(ctx->device));
  cudaStream_t st = (cudaStream_t)stream;
  MatchArgs A;
  A.windows = reinterpret_cast<const float2*>(d_windows);
  A.results = d_results; A.counts = d_counts; A.fix = d_fix;
  A.dict = reinterpret_cast<const uint4*>(d_dict); A.n_dict = d_n_dict;
  A.match = d_match; A.match_count = d_count;
  A.nseg = nseg; A.max_windows = max_windows; A.max_dict = max_dict;
  A.max_cost16 = (double)d.max_cost * 16.0;
  A.min_margin16 = (double)d.min_margin * 16.0;
  A.cfg = ctx->cfg;
  int launches = 0;
  if (d_count && max_dict > 0) {
    rx_match_init_kernel<<<(unsigned)((max_dict + 255) / 256), 256, 0, st>>>(A);
    launches++;
  }
  if (slots > 0) {
    // scratch: row count | rows [slots] (every attempted window is a row)
    const size_t need = 256 + (size_t)slots * sizeof(MatchRow);
    int rc;
    if ((rc = grow(ctx, ctx->d_match, need))) return rc;
    char* base = static_cast<char*>(ctx->d_match.p);
    A.n_rows = reinterpret_cast<int32_t*>(base);
    A.rows = reinterpret_cast<MatchRow*>(base + 256);
    CK(cudaMemsetAsync(A.n_rows, 0, sizeof(int32_t), st));
    rx_match_prepare_kernel<<<slot_grid(slots), 32 * kSlotWarps, 0, st>>>(A);
    rx_match_score_kernel<<<(unsigned)((slots + kMatchRows - 1) / kMatchRows), 32 * kMatchWarps, 0, st>>>(A);
    launches += 2;
  }
  CK(cudaGetLastError());
  ctx->last_launches = launches;
  return RFID_B200_OK;
}

// ------------------------------------------------------------------ block mode
int rfid_b200_gate_work(rfid_b200_ctx* ctx, int seek, const float* in, int n_in, float* out, int out_capacity,
                        int* consumed, int* written, int* closed, float* magn2_out)
{
  if (!ctx || !in || !out || !consumed || !written || n_in < 0 || seek < 0 || seek > 2) return RFID_B200_EINVAL;
  if (out_capacity < n_in) return RFID_B200_ECAPACITY;  // the reference may write up to ninput items (gate_impl.cc:95,174,187)
  *consumed = 0; *written = 0;
  if (closed) *closed = 0;
  if (n_in == 0 && seek == 0) return RFID_B200_OK;
  CK(cudaSetDevice(ctx->device));
  int rc;
  const size_t ns = (size_t)(n_in > 0 ? n_in : 1);
  // one device block [GateCallOut (64 B) | out: ns complex | |out|^2: ns floats] and its pinned host mirror: the kernel's
  // whole result comes back with ONE copy and ONE synchronisation per work call (it was two of each)
  const size_t off_out = 64, off_m2 = off_out + ns * 8, blk = off_m2 + ns * 4;
  if ((rc = grow(ctx, ctx->d_in, ns * 8))) return rc;
  if ((rc = grow(ctx, ctx->d_blk, blk))) return rc;
  if (ctx->h_blk_bytes < blk) {
    if (ctx->h_blk) cudaFreeHost(ctx->h_blk);
    ctx->h_blk = nullptr; ctx->h_blk_bytes = 0;
    const size_t want = blk + blk / 4 + 256;
    if (cudaHostAlloc(&ctx->h_blk, want, cudaHostAllocDefault) != cudaSuccess) { cudaGetLastError(); return RFID_B200_ENOMEM; }
    ctx->h_blk_bytes = want;
  }
  cudaStream_t s = ctx->stream;
  char* db = (char*)ctx->d_blk.p;
  if (n_in) CK(cudaMemcpyAsync(ctx->d_in.p, in, (size_t)n_in * 8, cudaMemcpyHostToDevice, s));
  gate_block_kernel<<<1, 32, 0, s>>>(ctx->cfg, (GateState*)ctx->d_gate.p, seek, (const float2*)ctx->d_in.p, n_in, (float2*)(db + off_out),
                                     (float*)(db + off_m2), (GateCallOut*)db);
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(ctx->h_blk, db, blk, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  GateCallOut r;
  memcpy(&r, ctx->h_blk, sizeof(r));
  if (r.written > 0) {
    memcpy(out, (char*)ctx->h_blk + off_out, (size_t)r.written * 8);
    if (magn2_out) memcpy(magn2_out, (char*)ctx->h_blk + off_m2, (size_t)r.written * 4);
  }
  *consumed = r.consumed; *written = r.written;
  if (closed) *closed = r.closed;
  ctx->last_launches = 1;
  return RFID_B200_OK;
}

int rfid_b200_decoder_work(rfid_b200_ctx* ctx, int kind, const float* win, int n, rfid_b200_window_result* res,
                           float* bits_out)
{
  if (!ctx || !win || !res || (kind != RFID_B200_RN16 && kind != RFID_B200_EPC)) return RFID_B200_EINVAL;
  const int need = kind == RFID_B200_RN16 ? ctx->cfg.len_rn16 : ctx->cfg.len_epc;
  if (n < need) return RFID_B200_EINVAL;  // the reference only fires on a complete window (tag_decoder_impl.cc:223,291)
  CK(cudaSetDevice(ctx->device));
  int rc;
  if ((rc = grow(ctx, ctx->d_in, (size_t)need * 8))) return rc;
  cudaStream_t s = ctx->stream;
  CK(cudaMemcpyAsync(ctx->d_in.p, win, (size_t)need * 8, cudaMemcpyHostToDevice, s));
  const int stage = chunk_stage_samples(ctx->cfg);
  decode_block_kernel<<<1, 32, (size_t)stage * 8, s>>>(ctx->cfg, kind, (const float2*)ctx->d_in.p, need, stage, (rfid_b200_window_result*)ctx->d_one.p);
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(res, ctx->d_one.p, sizeof(*res), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  if (bits_out) {
    const int nb = kind == RFID_B200_RN16 ? 16 : 128;
    for (int i = 0; i < nb; i++) bits_out[i] = (res->bits[i >> 3] >> (7 - (i & 7))) & 1 ? 1.0f : 0.0f;
  }
  ctx->last_launches = 1;
  return RFID_B200_OK;
}

int rfid_b200_mf_work(rfid_b200_ctx* ctx, const float* in, int n_in, float* out, int out_capacity, int* written)
{
  if (!ctx || !in || !out || !written || n_in < 0) return RFID_B200_EINVAL;
  *written = 0;
  CK(cudaSetDevice(ctx->device));
  const int D = ctx->cfg.decim, K = ctx->cfg.ntaps;
  const long long abs_end = ctx->mf_abs0 + ctx->mf_have + n_in;       // one past the newest sample
  const long long last_n = abs_end / D - 1;  // floor(total/decim) outputs exist so far (fixed-rate decimator)
  const long long n_out = last_n - ctx->mf_next_n + 1 > 0 ? last_n - ctx->mf_next_n + 1 : 0;
  if (n_out > out_capacity) return RFID_B200_ECAPACITY;
  int rc;
  const size_t total = (size_t)(ctx->mf_have + n_in);
  // staging buffer = carried history + new chunk
  if ((rc = grow(ctx, ctx->d_out, (total + 1) * 8))) return rc;
  cudaStream_t s = ctx->stream;
  if (ctx->mf_have) CK(cudaMemcpyAsync(ctx->d_out.p, ctx->d_mf.p, (size_t)ctx->mf_have * 8, cudaMemcpyDeviceToDevice, s));
  if (n_in) CK(cudaMemcpyAsync((char*)ctx->d_out.p + (size_t)ctx->mf_have * 8, in, (size_t)n_in * 8, cudaMemcpyHostToDevice, s));
  if (n_out > 0) {
    if ((rc = grow(ctx, ctx->d_m2, (size_t)n_out * 8))) return rc;
    const int threads = 128;
    mf_block_kernel<<<(unsigned)((n_out + threads - 1) / threads), threads, 0, s>>>(
        ctx->cfg, (const float2*)ctx->d_out.p, ctx->mf_abs0, ctx->mf_next_n, (int)n_out, (float2*)ctx->d_m2.p);
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(out, ctx->d_m2.p, (size_t)n_out * 8, cudaMemcpyDeviceToHost, s));
  }
  // keep what the next output still needs: samples from D*next_n - (K-1) on
  const long long next_n = ctx->mf_next_n + n_out;
  long long keep_from = (long long)D * next_n - (K - 1);
  if (keep_from < ctx->mf_abs0) keep_from = ctx->mf_abs0;
  if (keep_from > abs_end) keep_from = abs_end;
  const long long keep = abs_end - keep_from;
  if ((rc = grow(ctx, ctx->d_mf, (size_t)(keep + 1) * 8))) return rc;
  if (keep) CK(cudaMemcpyAsync(ctx->d_mf.p, (char*)ctx->d_out.p + (size_t)(keep_from - ctx->mf_abs0) * 8, (size_t)keep * 8,
                               cudaMemcpyDeviceToDevice, s));
  CK(cudaStreamSynchronize(s));
  ctx->mf_abs0 = keep_from; ctx->mf_have = keep; ctx->mf_next_n = next_n;
  *written = (int)n_out;
  ctx->last_launches = n_out > 0 ? 1 : 0;
  return RFID_B200_OK;
}

}  // extern "C"
