// rx_match.cuh -- attribution of failing EPC windows to a dictionary of known frames (rfid_b200_match_epc; the rule is
// stated in include/rfid_b200.h).  Three kernels:
//   - init: the per-entry counts (optional);
//   - prepare: one warp per record slot assigns the statuses of windows that are not attempted and, for attempted ones,
//     computes the quality rule's projections (epc_projection), the integer reliabilities q_j and appends a compact row
//     {int8 u[128], signs, A, slot} through an atomic counter;
//   - score: D = A + u . c^T as an int8 tensor-core GEMM (mma.sync m16n8k32 s8.s8.s32) with a fused top-2 epilogue.  A
//     CTA owns 128 rows (32 per warp) and sweeps every 128-entry column tile of the dictionary; the frames of the next
//     tile arrive by cp.async while the current one is scored, and each tile is expanded once per CTA into the B
//     fragments of its codeword signs.
// Every result is an integer, a min or a max, so the output does not depend on the rows' order.  tests/match_model.py
// restates the rule bit for bit.
#pragma once

#include "rx_quality.cuh"

namespace rfid_b200 {

constexpr int kMatchWarps = 4;                      // score: warps per CTA
constexpr int kMatchWarpRows = 32;                  // rows per warp (two m16 tiles)
constexpr int kMatchRows = kMatchWarps * kMatchWarpRows;
constexpr int kMatchCols = 32 * kMatchWarps;        // dictionary entries per column tile, one per thread
constexpr int kMatchMaxDict = 1 << 24;

// One attempted window: u_j = q_j (1 - 2 s_j), the sign bits s (bit j at s[j >> 5], bit j & 31), A = sum q_j s_j.
struct MatchRow {
  int8_t u[128];
  uint32_t s[4];
  int32_t A, slot, reserved[2];
};
static_assert(sizeof(MatchRow) == 160, "MatchRow is 160 bytes");

struct MatchArgs {
  const float2* windows;                            // window tap: slot s * max_windows + k at stride cfg.len_epc
  const rfid_b200_window_result* results;
  const int32_t* counts;
  const rfid_b200_epc_fix* fix;                     // may be null
  const uint4* dict;                                // [max_dict] 16-byte frames
  const int32_t* n_dict;                            // may be null: max_dict
  rfid_b200_epc_match* match;
  rfid_b200_match_count* match_count;               // may be null
  MatchRow* rows;
  int32_t* n_rows;
  int nseg, max_windows, max_dict;
  double max_cost16, min_margin16;                  // thresholds in reliability steps (16 per mean reliability)
  RxConfig cfg;
};

__device__ __forceinline__ void match_store(rfid_b200_epc_match* out, int status, int entry, int cost, int runner_up,
                                            int n_diff)
{
  int4* o = reinterpret_cast<int4*>(out);
  o[0] = make_int4(status, entry, cost, runner_up);
  o[1] = make_int4(n_diff, 0, 0, 0);
}

__device__ __forceinline__ int match_dict_size(const MatchArgs& A)
{
  return A.n_dict ? min(max(*A.n_dict, 0), A.max_dict) : A.max_dict;
}

// The codeword signs of a frame (its 16 bytes as 4 little-endian words): c_j = c_(j-1) xor bit_j, c_(-1) = 1; bit j at
// c[j >> 5], bit j & 31.
__device__ __forceinline__ void match_codeword(const uint4 f, uint32_t c[4])
{
  const uint32_t mem[4] = {f.x, f.y, f.z, f.w};
  uint32_t carry = 0xFFFFFFFFu;
#pragma unroll
  for (int i = 0; i < 4; i++) {
    uint32_t x = __brev(__byte_perm(mem[i], 0, 0x0123));   // bit j of the message at bit j & 31
    x ^= x << 1;
    x ^= x << 2;
    x ^= x << 4;
    x ^= x << 8;
    x ^= x << 16;
    c[i] = x ^ carry;
    carry = (uint32_t)((int32_t)c[i] >> 31);
  }
}

// four sign bits (the low nibble of x) as four int8 0 / 1, the lowest bit in the lowest byte
__device__ __forceinline__ uint32_t match_nibble_bytes(uint32_t x) { return ((x & 0xFu) * 0x00204081u) & 0x01010101u; }

__global__ void rx_match_init_kernel(const MatchArgs A)
{
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e < A.max_dict) reinterpret_cast<int4*>(A.match_count)[e] = make_int4(0, -1, -1, 0);
}

__global__ void __launch_bounds__(32 * kSlotWarps) rx_match_prepare_kernel(const MatchArgs A)
{
  const int lane = threadIdx.x & 31;
  TapWindow t;
  if (!tap_window(A, t)) return;
  const long long slot = t.slot;
  const rfid_b200_window_result& rec = *t.rec;
  rfid_b200_epc_match* out = A.match + slot;
  if (rec.kind != RFID_B200_EPC || rec.crc_ok == 1 || (A.fix && A.fix[slot].status == RFID_B200_FIX_RECOVERED)) {
    if (lane == 0)
      match_store(out, rec.kind != RFID_B200_EPC ? RFID_B200_MATCH_NOT_EPC : RFID_B200_MATCH_ALREADY_READ, -1, -1, -1, -1);
    return;
  }
  if (rec.crc_ok != 0) {   // the decoder made no EPC decisions
    if (lane == 0) match_store(out, RFID_B200_MATCH_SKIPPED, -1, -1, -1, -1);
    return;
  }
  float r[4];
  double a1 = 0.0;
#pragma unroll
  for (int i = 0; i < 4; i++) {   // lane l holds decisions j = 32 i + l
    r[i] = epc_projection(t, i * 32 + lane);
    a1 = __dadd_rn(a1, (double)fabsf(r[i]));
  }
  const double s1 = quality_lane_sum(a1);
  if (!(s1 > 0.0 && s1 <= 1.7976931348623157e308)) {   // zero, infinite or NaN
    if (lane == 0) match_store(out, RFID_B200_MATCH_SKIPPED, -1, -1, -1, -1);
    return;
  }
  const double m = __ddiv_rn(s1, 128.0);
  int q_sum = 0;
  int8_t u[4];
  uint32_t sw[4];
#pragma unroll
  for (int i = 0; i < 4; i++) {
    const int q = (int)fmin(127.0, rint(__ddiv_rn(__dmul_rn((double)fabsf(r[i]), 16.0), m)));
    const bool pos = r[i] > 0.0f;
    u[i] = (int8_t)(pos ? -q : q);
    q_sum += pos ? q : 0;
    sw[i] = __ballot_sync(0xffffffffu, pos);
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) q_sum += __shfl_xor_sync(0xffffffffu, q_sum, off);
  int row = 0;
  if (lane == 0) row = atomicAdd(A.n_rows, 1);
  row = __shfl_sync(0xffffffffu, row, 0);
  MatchRow* dst = A.rows + row;
#pragma unroll
  for (int i = 0; i < 4; i++) dst->u[i * 32 + lane] = u[i];
  if (lane == 0) {
    *reinterpret_cast<uint4*>(dst->s) = make_uint4(sw[0], sw[1], sw[2], sw[3]);
    *reinterpret_cast<int4*>(&dst->A) = make_int4(q_sum, (int)slot, 0, 0);
  }
}

__device__ __forceinline__ void match_mma(int (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1)
{
  asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.s8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
               : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// top-2 of a row over columns seen in ascending order: (d1, k1) the smallest and its lowest column, d2 the second
// smallest value of the multiset
__device__ __forceinline__ void match_top2(int& d1, int& k1, int& d2, int d, int col)
{
  d2 = min(d2, max(d, d1));
  if (d < d1) k1 = col;
  d1 = min(d1, d);
}

// merge with the state of lane `lane ^ off` (columns of either lane in any order: ties go to the lower column)
__device__ __forceinline__ void match_merge(int& d1, int& k1, int& d2, int off)
{
  const int o1 = __shfl_xor_sync(0xffffffffu, d1, off), ok = __shfl_xor_sync(0xffffffffu, k1, off);
  const int o2 = __shfl_xor_sync(0xffffffffu, d2, off);
  d2 = min(max(d1, o1), min(d2, o2));
  if (o1 < d1 || (o1 == d1 && ok < k1)) k1 = ok;
  d1 = min(d1, o1);
}

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem, bool valid)
{
  const unsigned s = (unsigned)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(s), "l"(gmem), "r"(valid ? 16 : 0));
}

// score one column tile from its fragments: the full-tile path skips the column bound
template <bool TAIL>
__device__ __forceinline__ void match_tile(const uint4 (*frag)[32][2], int col0, int K, const uint32_t (&a)[2][4][4],
                                           const int (&arow)[4], int (&d1)[4], int (&k1)[4], int (&d2)[4])
{
  const int lane = threadIdx.x & 31, t = lane & 3;
#pragma unroll 2
  for (int b = 0; b < kMatchCols / 8; b++) {
    const int n0 = col0 + b * 8;
    if (TAIL && n0 >= K) break;
    const uint4 f0 = frag[b][lane][0], f1 = frag[b][lane][1];
    const int c0 = n0 + 2 * t, c1 = c0 + 1;
#pragma unroll
    for (int mt = 0; mt < 2; mt++) {
      int acc[4] = {0, 0, 0, 0};
      match_mma(acc, a[mt][0], f0.x, f0.y);
      match_mma(acc, a[mt][1], f0.z, f0.w);
      match_mma(acc, a[mt][2], f1.x, f1.y);
      match_mma(acc, a[mt][3], f1.z, f1.w);
      const int INF = 0x7FFFFFFF;
      // acc[0], acc[1]: row g at columns c0, c1; acc[2], acc[3]: row g + 8
      match_top2(d1[2 * mt], k1[2 * mt], d2[2 * mt], (!TAIL || c0 < K) ? arow[2 * mt] + acc[0] : INF, c0);
      match_top2(d1[2 * mt], k1[2 * mt], d2[2 * mt], (!TAIL || c1 < K) ? arow[2 * mt] + acc[1] : INF, c1);
      match_top2(d1[2 * mt + 1], k1[2 * mt + 1], d2[2 * mt + 1], (!TAIL || c0 < K) ? arow[2 * mt + 1] + acc[2] : INF, c0);
      match_top2(d1[2 * mt + 1], k1[2 * mt + 1], d2[2 * mt + 1], (!TAIL || c1 < K) ? arow[2 * mt + 1] + acc[3] : INF, c1);
    }
  }
}

__global__ void __launch_bounds__(32 * kMatchWarps) rx_match_score_kernel(const MatchArgs A)
{
  __shared__ __align__(16) uint4 s_frame[2][kMatchCols];
  __shared__ __align__(16) uint4 s_frag[2][kMatchCols / 8][32][2];   // [buffer][n8 block][lane][b registers 0..3, 4..7]
  const int n_rows = *A.n_rows;
  const int row0 = blockIdx.x * kMatchRows;
  if (row0 >= n_rows) return;
  const int K = match_dict_size(A);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, t = lane & 3;
  // A fragments of the warp's two m16 tiles (rows beyond n_rows are zero and never written), and A of rows g, g + 8
  uint32_t a[2][4][4];
  int arow[4];
#pragma unroll
  for (int mt = 0; mt < 2; mt++) {
#pragma unroll
    for (int hi = 0; hi < 2; hi++) {
      const int row = row0 + warp * kMatchWarpRows + mt * 16 + g + 8 * hi;
      const bool ok = row < n_rows;
      const MatchRow* src = A.rows + (ok ? row : 0);
#pragma unroll
      for (int ks = 0; ks < 4; ks++) {
        a[mt][ks][hi] = ok ? *reinterpret_cast<const uint32_t*>(src->u + 32 * ks + 4 * t) : 0u;
        a[mt][ks][2 + hi] = ok ? *reinterpret_cast<const uint32_t*>(src->u + 32 * ks + 16 + 4 * t) : 0u;
      }
      arow[2 * mt + hi] = ok ? src->A : 0;
    }
  }
  int d1[4], k1[4], d2[4];
#pragma unroll
  for (int i = 0; i < 4; i++) { d1[i] = d2[i] = 0x7FFFFFFF; k1[i] = 0x7FFFFFFF; }
  const int n_tiles = (K + kMatchCols - 1) / kMatchCols;
  if (n_tiles > 0) {
    cp_async16(&s_frame[0][tid], A.dict + min(tid, K - 1), tid < K);
    asm volatile("cp.async.commit_group;\n" ::);
  }
  for (int tile = 0; tile < n_tiles; tile++) {
    const int buf = tile & 1;
    if (tile + 1 < n_tiles) {   // this thread's frame of the next tile; its slot was last read by this thread
      const int e = (tile + 1) * kMatchCols + tid;
      cp_async16(&s_frame[buf ^ 1][tid], A.dict + min(e, K - 1), e < K);
      asm volatile("cp.async.commit_group;\n" ::);
      asm volatile("cp.async.wait_group 1;\n" ::);
    } else {
      asm volatile("cp.async.wait_group 0;\n" ::);
    }
    {   // expand this thread's entry into the B fragments of lanes 4 g .. 4 g + 3 of its n8 block (fragment buffer `buf`
        // was last read while scoring tile - 2, before the previous iteration's barrier)
      uint32_t c[4];
      match_codeword(s_frame[buf][tid], c);
      const int b = tid >> 3, eg = tid & 7;
#pragma unroll
      for (int tt = 0; tt < 4; tt++) {
        uint32_t r[8];
#pragma unroll
        for (int ks = 0; ks < 4; ks++) {
          r[2 * ks] = match_nibble_bytes(c[ks] >> (4 * tt));
          r[2 * ks + 1] = match_nibble_bytes(c[ks] >> (16 + 4 * tt));
        }
        s_frag[buf][b][eg * 4 + tt][0] = make_uint4(r[0], r[1], r[2], r[3]);
        s_frag[buf][b][eg * 4 + tt][1] = make_uint4(r[4], r[5], r[6], r[7]);
      }
    }
    __syncthreads();
    const int col0 = tile * kMatchCols;
    if (col0 + kMatchCols <= K) match_tile<false>(s_frag[buf], col0, K, a, arow, d1, k1, d2);
    else match_tile<true>(s_frag[buf], col0, K, a, arow, d1, k1, d2);
  }
  // merge the four lanes of each row group; then lane t writes row (mt, hi) = (t >> 1, t & 1)
#pragma unroll
  for (int i = 0; i < 4; i++) {
    match_merge(d1[i], k1[i], d2[i], 1);
    match_merge(d1[i], k1[i], d2[i], 2);
  }
  const int mine = t;   // index into d1 / k1 / d2: 2 * mt + hi
  int D1 = d1[0], K1 = k1[0], D2 = d2[0];
#pragma unroll
  for (int i = 1; i < 4; i++)
    if (mine == i) { D1 = d1[i]; K1 = k1[i]; D2 = d2[i]; }
  const int row = row0 + warp * kMatchWarpRows + (mine >> 1) * 16 + g + 8 * (mine & 1);
  if (row >= n_rows) return;
  const MatchRow& src = A.rows[row];
  const int slot = src.slot;
  rfid_b200_epc_match* out = A.match + slot;
  if (K == 0) {
    match_store(out, RFID_B200_MATCH_NO_MATCH, -1, 0x7FFFFFFF, 0x7FFFFFFF, -1);
    return;
  }
  uint32_t c[4];
  match_codeword(A.dict[K1], c);
  const uint4 s = *reinterpret_cast<const uint4*>(src.s);
  const int n_diff = __popc(s.x ^ c[0]) + __popc(s.y ^ c[1]) + __popc(s.z ^ c[2]) + __popc(s.w ^ c[3]);
  int status = RFID_B200_MATCH_NO_MATCH;
  if ((double)D1 <= A.max_cost16)
    status = (double)((long long)D2 - D1) >= A.min_margin16 ? RFID_B200_MATCH_MATCHED : RFID_B200_MATCH_AMBIGUOUS;
  match_store(out, status, K1, D1, D2, n_diff);
  if (status == RFID_B200_MATCH_MATCHED && A.match_count) {
    rfid_b200_match_count* mc = A.match_count + K1;
    atomicAdd(&mc->matched, 1);
    atomicMin(reinterpret_cast<unsigned*>(&mc->first_slot), (unsigned)slot);   // -1 (none) is the largest unsigned
    atomicMax(&mc->last_slot, slot);
  }
}

}  // namespace rfid_b200
