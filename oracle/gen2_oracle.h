/* TEST INFRASTRUCTURE -- CPU restatement (plain C) of the reference's Gen2 RX
 * decode path: matched filter -> gate -> tag_decoder -> READER_STATS.
 *
 * PARITY PINNED: this restatement is checked bit-for-bit (records, scores,
 * channel estimates, stats) against oracle/_ref -- the reference's own C++
 * blocks compiled unchanged -- on misc/data/file_source_test and on synthetic
 * captures (tests/test_oracle.py), and against the reference's only golden
 * vectors (README.md:46-53 and the RN16s in misc/data/file_sink).  The one
 * stage that is "parity unpinned" at the bit level is the matched filter, whose
 * arithmetic lives in GNU Radio/VOLK outside /root/reference (see
 * mf_canonical.h).
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline/--impl
 * reference legs may link or call this.  The product never does.
 *
 * Citations are to /root/reference/gr-rfid/.
 */
#ifndef GEN2_ORACLE_H
#define GEN2_ORACLE_H

#include <stddef.h>
#include <stdint.h>

#include "../include/rfid_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

#define GEN2_ORACLE_API __attribute__((visibility("default")))

/* Derived constants, computed with the reference's own expressions
 * (gate_impl.cc:48-53,115,121; tag_decoder_impl.cc:60; global_vars.h:90-143). */
typedef struct gen2_oracle_cfg {
  int fs_dec;        /* sample rate after decimation */
  int n_T1;          /* T1_D  * fs/1e6 (int)            gate_impl.cc:48 */
  int n_PW;          /* PW_D  * fs/1e6 (int)            gate_impl.cc:49 */
  int n_tag_bit_i;   /* TAG_BIT_D * fs/1e6 (int, gate)  gate_impl.cc:50 */
  float n_tag_bit_f; /* same as float (decoder)         tag_decoder_impl.cc:60 */
  int win_length;    /* WIN_SIZE_D * fs/1e6             gate_impl.cc:52 */
  int dc_length;     /* DC_SIZE_D * fs/1e6              gate_impl.cc:53 */
  int len_rn16;      /* (17+6)*n + 2n                   gate_impl.cc:121 */
  int len_epc;       /* (129+6)*n + 2n                  gate_impl.cc:115 */
  int fixed_q, max_queries, max_tags;
  int adc_rate, decim, ntaps;
  int defined;       /* 1: every read of tag_decoder_impl.cc stays inside its window and an RN16 window holds its 32
                      * half-bits, for every sync index; 0: the reference has no defined output to restate */
} gen2_oracle_cfg;

GEN2_ORACLE_API void gen2_oracle_make_cfg(const rfid_b200_params* p, gen2_oracle_cfg* c);

/* gate_impl::general_work as a pure function of one decimated stream
 * (gate_impl.cc:85-200 + the alternation rule of SURVEY.md 3.5).
 * open_idx[k], dc[2k..2k+1] for each COMPLETED window k (capacity max_windows);
 * win_out (may be NULL): window k's ungated samples at win_out + 2*k*len_epc.
 * avg_out (may be NULL): avg_ampl after every sample.  Returns windows found. */
GEN2_ORACLE_API int gen2_oracle_gate(const gen2_oracle_cfg* c, const float* y, size_t ny, int max_windows,
                                     int32_t* open_idx, float* dc, float* win_out, float* avg_out);

/* tag_decoder_impl::general_work on one window (tag_decoder_impl.cc:196-397).
 * Fills sync_index, score, h, T, bits, crc_ok, tag_id, kind, length. */
GEN2_ORACLE_API void gen2_oracle_decode_window(const gen2_oracle_cfg* c, int kind, const float* win, int n,
                                               rfid_b200_window_result* r);

/* whole chain on a decimated stream; returns number of windows */
GEN2_ORACLE_API int gen2_oracle_decode_decimated(const gen2_oracle_cfg* c, const float* y, size_t ny, int segment,
                                                 rfid_b200_window_result* recs, int max_recs);

/* whole chain on raw segments (canonical MF with zero history per segment) */
GEN2_ORACLE_API int gen2_oracle_decode_segments(const gen2_oracle_cfg* c, const float* iq_raw,
                                                const rfid_b200_segment* segs, int nseg,
                                                rfid_b200_window_result* recs, int max_per_seg, int32_t* counts,
                                                double* seconds);

GEN2_ORACLE_API size_t gen2_oracle_mf(const float* x, size_t n_in, int ntaps, int decim, float* y);
GEN2_ORACLE_API size_t gen2_oracle_mf_variant(const float* x, size_t n_in, int ntaps, int decim, float* y, int variant);

/* READER_STATS bookkeeping (tag_decoder_impl.cc:269-288,295,329-387; reader_impl.cc:251-344;
 * stop rule gate_impl.cc:101-109) replayed over records in stream order. */
GEN2_ORACLE_API void gen2_oracle_reduce_stats(const gen2_oracle_cfg* c, const rfid_b200_window_result* recs,
                                              const int32_t* counts, int nseg, int max_per_seg, int continuous,
                                              rfid_b200_stats* out);

/* check_crc (tag_decoder_impl.cc:401-445): bits = 16 bytes MSB first; returns 1 / 0 */
GEN2_ORACLE_API int gen2_oracle_crc16_ok(const uint8_t bits[16]);
/* CRC-16 the tag appends (same polynomial, used by the synthetic tag model) */
GEN2_ORACLE_API uint16_t gen2_oracle_crc16(const uint8_t* data, int nbytes);
/* reader_impl::crc_append (reader_impl.cc:383-443): 17 query bits -> 5 CRC bits (MSB first) */
GEN2_ORACLE_API void gen2_oracle_crc5(const uint8_t q[17], uint8_t crc_out[5]);
/* reader_impl::gen_query_bits (reader_impl.cc:131-146): 22 bits for a given Q */
GEN2_ORACLE_API void gen2_oracle_query_bits(int fixed_q, uint8_t out[22]);

/* cabsf as the reference's libm evaluates it (gate_impl.cc:130) */
GEN2_ORACLE_API float gen2_oracle_cabsf(float re, float im);

#ifdef __cplusplus
}
#endif
#endif
