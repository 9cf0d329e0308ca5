// rx_recover.cuh -- recovery of EPC windows that fail their CRC (rfid_b200_recover_epc; the rule is stated in
// include/rfid_b200.h).  One warp per record slot.  An attempted window's 128 projections are the quality kernel's
// (epc_projection); the warp picks the P least reliable decisions by P rounds of a warp argmin, then tries every flip
// set of at most W of them, the candidates split across lanes by rank.  A candidate is tested through its syndrome, which
// is affine in the bits, so each costs |F| XORs; tests/recover_model.py restates the rule bit for bit.
#pragma once

#include "rx_quality.cuh"

namespace rfid_b200 {

constexpr int kRecoverMaxPositions = 32;         // P: one candidate position per lane
constexpr long long kRecoverMaxCandidates = 65536;

struct RecoverArgs {
  const float2* windows;                         // window tap: slot s * max_windows + k at stride cfg.len_epc
  const rfid_b200_window_result* results;
  const int32_t* counts;
  const rfid_b200_quality* quality;
  rfid_b200_epc_fix* fix;
  int nseg, max_windows;
  int positions, max_flips, n_candidates;        // P, W, sum over k = 1..W of binomial(P, k)
  double min_snr_ratio;                          // linear
  RxConfig cfg;
};

// The syndrome of a 128-bit EPC window (bit j = message bit j, MSB first): bits 0..15 the CRC-16 of bytes 0..13 xor
// bytes 14..15, bits 16..20 PC bits 0..4 xor 00110 (PC bit 0 at bit 20).  A window passes iff its syndrome is 0.  It is
// affine in the bits: syndrome(x) = zero + xor of col[j] over the set bits j of x, where col[j] is the CRC of the message
// holding bit j alone with zero init and no final complement (j < 112), or the received CRC bit (j >= 112), plus PC bit j
// (j < 5), and zero the syndrome of the all-zero window.
struct EpcSyndrome {
  uint32_t col[128];
  uint32_t zero;
};

constexpr uint32_t epc_crc_bits(uint32_t crc, int one_at)   // 112 message bits, all zero but bit one_at (-1: none)
{
  for (int m = 0; m < 112; m++) {
    const uint32_t fb = ((crc >> 15) & 1u) ^ (m == one_at ? 1u : 0u);
    crc = (crc << 1) & 0xFFFFu;
    if (fb) crc ^= 0x1021u;
  }
  return crc;
}

constexpr EpcSyndrome make_epc_syndrome()
{
  EpcSyndrome t{};
  for (int j = 0; j < 128; j++) {
    uint32_t s = j < 112 ? epc_crc_bits(0u, j) : 1u << (127 - j);
    if (j < 5) s |= 1u << (20 - j);
    t.col[j] = s;
  }
  t.zero = ((~epc_crc_bits(0xFFFFu, -1)) & 0xFFFFu) | (0x06u << 16);   // PC length field 00000 xor 00110
  return t;
}

__constant__ EpcSyndrome kEpcSyndrome = make_epc_syndrome();

__device__ __forceinline__ uint32_t recover_binom(int n, int k)
{
  if (k < 0 || k > n) return 0u;
  unsigned long long r = 1;
  for (int i = 0; i < k; i++) r = r * (unsigned long long)(n - i) / (unsigned long long)(i + 1);
  return (uint32_t)r;
}

// the k-subset of {0..P-1} of colex rank r (= the r-th smallest integer with k bits set)
__device__ __forceinline__ unsigned long long recover_unrank(uint32_t r, int k, int P)
{
  unsigned long long m = 0;
  int c = P - 1;
  for (int i = k; i >= 1; i--) {
    while (recover_binom(c, i) > r) c--;
    m |= 1ull << c;
    r -= recover_binom(c, i);
    c--;
  }
  return m;
}

__device__ __forceinline__ void recover_store(rfid_b200_epc_fix* out, int status, int n_flips, int n_pass, float cost,
                                              const uint32_t mem[4])
{
  int4* o = reinterpret_cast<int4*>(out);
  o[0] = make_int4(status, n_flips, n_pass, __float_as_int(cost));
  o[1] = make_int4((int)mem[0], (int)mem[1], (int)mem[2], (int)mem[3]);
}

__global__ void __launch_bounds__(32 * kSlotWarps) rx_recover_kernel(const RecoverArgs A)
{
  __shared__ uint32_t s_col[kSlotWarps][kRecoverMaxPositions];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  TapWindow t;
  if (!tap_window(A, t)) return;
  const rfid_b200_window_result& rec = *t.rec;
  const float nan = __int_as_float(0x7fc00000);
  uint32_t mem[4];   // the record's 16 bytes as 4 little-endian words
  {
    const uint4 b = *reinterpret_cast<const uint4*>(rec.bits);
    mem[0] = b.x; mem[1] = b.y; mem[2] = b.z; mem[3] = b.w;
  }
  rfid_b200_epc_fix* out = A.fix + t.slot;
  if (rec.kind != RFID_B200_EPC || rec.crc_ok == 1) {
    if (lane == 0) recover_store(out, rec.kind != RFID_B200_EPC ? RFID_B200_FIX_NOT_EPC : RFID_B200_FIX_CRC_OK, 0, 0, nan, mem);
    return;
  }
  const rfid_b200_quality q = A.quality[t.slot];
  if (!(q.n_decisions == 128 && (double)q.snr >= A.min_snr_ratio)) {
    if (lane == 0) recover_store(out, RFID_B200_FIX_SKIPPED, 0, 0, nan, mem);
    return;
  }
  // bits and projections: lane l holds decisions j = 32 q + l, q = 0..3
  uint32_t word[4];   // bit j at word[j >> 5], bit j & 31
#pragma unroll
  for (int i = 0; i < 4; i++) word[i] = __brev(__byte_perm(mem[i], 0, 0x0123));
  float rho[4];
  uint32_t syn = 0u;
#pragma unroll
  for (int i = 0; i < 4; i++) {
    const int j = i * 32 + lane;
    rho[i] = fabsf(epc_projection(t, j));
    if ((word[i] >> lane) & 1u) syn ^= kEpcSyndrome.col[j];
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) syn ^= __shfl_xor_sync(0xffffffffu, syn, off);
  syn ^= kEpcSyndrome.zero;
  // the P least reliable decisions, (rho, j) ascending: rank i goes to lane i.  rho >= 0, so its bits order like it.
  const int P = A.positions;
  unsigned taken = 0u;
  int my_pos = -1;
  for (int i = 0; i < P; i++) {
    unsigned long long best = ~0ull;
#pragma unroll
    for (int t = 0; t < 4; t++) {
      const unsigned long long key = ((unsigned long long)__float_as_uint(rho[t]) << 8) | (unsigned)(t * 32 + lane);
      if (!((taken >> t) & 1u) && key < best) best = key;
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      const unsigned long long o = __shfl_xor_sync(0xffffffffu, best, off);
      best = o < best ? o : best;
    }
    const int j = (int)(best & 0xFFu);
    if ((j & 31) == lane) taken |= 1u << (j >> 5);
    if (lane == i) my_pos = j;
  }
  s_col[warp][lane] = my_pos < 0 ? 0u : kEpcSyndrome.col[my_pos] ^ (my_pos < 127 ? kEpcSyndrome.col[my_pos + 1] : 0u);
  __syncwarp();
  // candidates: ranks [lo, hi) of the order (|F|, colex) to this lane
  const uint32_t C = (uint32_t)A.n_candidates;
  uint32_t r = (uint32_t)(((unsigned long long)lane * C) >> 5);
  const uint32_t cnt = (uint32_t)(((unsigned long long)(lane + 1) * C) >> 5) - r;
  int size = 1;
  while (size < A.max_flips && r >= recover_binom(P, size)) r -= recover_binom(P, size++);
  unsigned long long m = recover_unrank(r, size, P);
  int n_pass_lane = 0;
  unsigned long long pass_mask = 0ull;
  for (uint32_t e = 0; e < cnt; e++) {
    uint32_t s = syn;
    for (unsigned long long b = m; b; b &= b - 1) s ^= s_col[warp][__ffsll((long long)b) - 1];
    if (s == 0u) {
      if (n_pass_lane == 0) pass_mask = m;
      n_pass_lane++;
    }
    const unsigned long long u = m & (~m + 1ull), v = m + u;   // Gosper: the next integer with as many bits set
    m = v | (((v ^ m) / u) >> 2);
    if (m >> P) m = (1ull << ++size) - 1ull;
  }
  int n_pass = n_pass_lane;
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) n_pass += __shfl_xor_sync(0xffffffffu, n_pass, off);
  if (n_pass != 1) {
    if (lane == 0) recover_store(out, n_pass == 0 ? RFID_B200_FIX_FAILED : RFID_B200_FIX_AMBIGUOUS, 0, n_pass, nan, mem);
    return;
  }
  const int src = __ffs(__ballot_sync(0xffffffffu, n_pass_lane != 0)) - 1;
  const unsigned long long F = __shfl_sync(0xffffffffu, pass_mask, src);
  uint32_t sflip[4] = {0u, 0u, 0u, 0u};   // flipped signs, bit j at sflip[j >> 5], bit j & 31
  for (int i = 0; i < P; i++) {
    const int pj = __shfl_sync(0xffffffffu, my_pos, i);
    const uint32_t bit = ((F >> i) & 1ull) ? 1u << (pj & 31) : 0u;
#pragma unroll
    for (int t = 0; t < 4; t++) sflip[t] |= (pj >> 5) == t ? bit : 0u;
  }
  // cost: the flipped reliabilities (ascending j) over the mean reliability (the quality rule's S1 / 128)
  double a1 = 0.0, flipped = 0.0;
#pragma unroll
  for (int i = 0; i < 4; i++) {
    a1 = __dadd_rn(a1, (double)rho[i]);
    for (uint32_t b = sflip[i]; b; b &= b - 1) {   // (sflip is the same in every lane)
      const int l = __ffs((int)b) - 1;
      flipped = __dadd_rn(flipped, (double)__shfl_sync(0xffffffffu, rho[i], l));
    }
  }
  const double mean = __ddiv_rn(quality_lane_sum(a1), 128.0);
  const float cost = quality_canonical(__ddiv_rn(flipped, mean));
  uint32_t carry = 0u;
#pragma unroll
  for (int i = 0; i < 4; i++) {   // flipping sign j flips bits j and j + 1
    const uint32_t bflip = sflip[i] ^ (sflip[i] << 1) ^ carry;
    carry = sflip[i] >> 31;
    mem[i] ^= __byte_perm(__brev(bflip), 0, 0x0123);
  }
  if (lane == 0) recover_store(out, RFID_B200_FIX_RECOVERED, __popcll(F), 1, cost, mem);
}

}  // namespace rfid_b200
