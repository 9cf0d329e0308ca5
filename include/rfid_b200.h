/* rfid_b200.h -- C-ABI of the H100-native Gen2 receive/decode chain.
 *
 * This is the drop-in boundary: a plain-C shared library (librfid_b200.so) whose
 * entry points are what the reference's three GNU Radio blocks would bind if
 * their work() loops were replaced by GPU calls.  Nothing like it exists in the
 * reference (it has no FFI); each entry point cites the reference interface it
 * replaces (paths relative to /root/reference/gr-rfid).
 *
 *   reference                                   | replaced by
 *   --------------------------------------------+--------------------------------------
 *   filter.fir_filter_ccc(5,[1]*25)             | rfid_b200_mf_work      (block mode)
 *     apps/reader.py:65,75 (GNU Radio, external)|   + fused into rfid_b200_decode_capture
 *   gate_impl::general_work  lib/gate_impl.cc:85| rfid_b200_gate_work    (block mode)
 *   tag_decoder_impl::general_work              | rfid_b200_decoder_work (block mode)
 *     lib/tag_decoder_impl.cc:196               |
 *   whole RX chain on a recorded capture        | rfid_b200_decode_capture (capture mode)
 *   READER_STATS bookkeeping                    | rfid_b200_reduce_stats
 *     lib/tag_decoder_impl.cc:269-288,329-387   |
 *
 * Conventions: every function returns 0 on success or a negative RFID_B200_E*
 * code (rfid_b200_strerror() names it); no exception crosses the boundary; no
 * torch/C++ types appear in a signature.  Complex samples are interleaved
 * float32 I,Q (GNU Radio gr_complex / the on-disk format of
 * misc/data/file_source_test, apps/reader.py:102).  There is NO CPU fallback:
 * rfid_b200_create() fails with RFID_B200_ENODEV when no sm_90 device is
 * usable.
 */
#ifndef RFID_B200_H
#define RFID_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RFID_B200_API __attribute__((visibility("default")))

#define RFID_B200_ABI_VERSION 1

/* error codes */
enum {
  RFID_B200_OK = 0,
  RFID_B200_EINVAL = -1,   /* bad argument */
  RFID_B200_ENODEV = -2,   /* no usable sm_90 CUDA device */
  RFID_B200_ENOMEM = -3,   /* host or device allocation failed */
  RFID_B200_ECUDA = -4,    /* CUDA runtime error (see rfid_b200_last_cuda_error) */
  RFID_B200_ECAPACITY = -5 /* caller-provided output buffer too small */
};

/* window kinds (reference: DECODER_DECODE_RN16 / DECODER_DECODE_EPC, include/rfid/global_vars.h:34) */
enum { RFID_B200_RN16 = 0, RFID_B200_EPC = 1 };

/* Configuration.  Defaults reproduce apps/reader.py:52-65 + include/rfid/global_vars.h:72-143. */
typedef struct rfid_b200_params {
  int32_t adc_rate;    /* raw complex sample rate, Hz            (reader.py:53  -> 2000000) */
  int32_t decim;       /* matched-filter decimation              (reader.py:54  -> 5)       */
  int32_t ntaps;       /* boxcar length = half an FM0 symbol     (reader.py:65  -> 25)      */
  int32_t fixed_q;     /* slots per round = 2^fixed_q            (global_vars.h:72 -> 0)    */
  int32_t max_queries; /* stop after this many Query/QueryRep    (global_vars.h:76 -> 1000) */
  int32_t max_tags;    /* stop after more than this many unique tags (global_vars.h:100 -> 100) */
  int32_t device;      /* CUDA device ordinal */
  int32_t reserved;
} rfid_b200_params;

/* One capture segment: a contiguous range of RAW samples that is decoded as an
 * independent stream with freshly constructed gate state (SURVEY.md section 8e). */
typedef struct rfid_b200_segment {
  uint64_t offset; /* first raw complex sample */
  uint32_t length; /* number of raw complex samples */
  uint32_t reserved;
} rfid_b200_segment;

/* One decoded window (64 bytes).  Everything the reference's tag_decoder
 * derives from one ungated window, including the quantities it keeps private
 * (score = local `max` in tag_sync, tag_decoder_impl.cc:81,94-98). */
typedef struct rfid_b200_window_result {
  int32_t segment;    /* index into the segment table */
  int32_t window;     /* ordinal inside the segment: even = RN16, odd = EPC (SURVEY.md 3.5) */
  int32_t open_index; /* decimated index (segment relative) of the first ungated sample, gate_impl.cc:164-175 */
  int32_t length;     /* n_samples_to_ungate, gate_impl.cc:115,121 */
  int32_t kind;       /* RFID_B200_RN16 / RFID_B200_EPC */
  int32_t sync_index; /* argmax offset of the preamble correlation, tag_decoder_impl.cc:85-100 */
  float score;        /* |c(sync_index)|^2, tag_decoder_impl.cc:94 */
  float h_re, h_im;   /* channel estimate h_est, tag_decoder_impl.cc:103 */
  float T;            /* EPC half-symbol period T_global, tag_decoder_impl.cc:166-169; 0 for RN16 */
  int32_t crc_ok;     /* EPC: 1 pass / 0 fail (check_crc, tag_decoder_impl.cc:401-445); RN16: -1 */
  int32_t tag_id;     /* EPC: bits[104..111] as an integer, tag_decoder_impl.cc:348-352; RN16: the 16-bit RN16 */
  uint8_t bits[16];   /* decoded bits, MSB first; RN16 uses bits[0..1], EPC all 16 bytes */
} rfid_b200_window_result;

/* READER_STATS as a plain struct (include/rfid/global_vars.h:36-53). */
#define RFID_B200_MAX_TAGS 256
typedef struct rfid_b200_stats {
  int32_t n_queries_sent;
  int32_t cur_inventory_round;
  int32_t cur_slot_number;
  int32_t max_slot_number;
  int32_t n_epc_correct;
  int32_t n_windows;      /* windows that entered the statistics */
  int32_t terminated;     /* 1 once the reference's stop rule fired, gate_impl.cc:101-109 */
  int32_t n_unique_tags;
  int32_t tag_id[RFID_B200_MAX_TAGS];    /* ascending (std::map order) */
  int32_t tag_reads[RFID_B200_MAX_TAGS];
} rfid_b200_stats;

typedef struct rfid_b200_ctx rfid_b200_ctx;

RFID_B200_API int rfid_b200_abi_version(void);
RFID_B200_API const char* rfid_b200_strerror(int code);
RFID_B200_API const char* rfid_b200_last_cuda_error(const rfid_b200_ctx* ctx);
RFID_B200_API void rfid_b200_default_params(rfid_b200_params* p);

/* Context: one per block instance (block mode) or per decode stream (capture mode).
 * Replaces the constructors gate_impl.cc:41-70 / tag_decoder_impl.cc:50-62 and the
 * process-global reader_state (global_vars.cc:34-54).
 *
 * Fails with RFID_B200_EINVAL, before looking for a device, when the configuration
 * is not well defined: the reference decoder takes its read indices from the float
 * samples-per-tag-bit but the gate sizes its windows from the truncated integer, so
 * at most rates whose tag bit is not a whole number of decimated samples the EPC
 * symbol-period search reads past the end of its window (undefined behaviour in the
 * reference) or an RN16 window ends before its 32 half-bits.  Well defined are the
 * rates where, for every sync index, all of the decoder's reads stay inside the
 * window.  With decimation 5 these are 314 of the 7001 rates on the 1 kHz grid from
 * 1 to 8 MS/s: every multiple of 200 kHz but 5.8 MS/s (where the gate's double
 * product 25 * 1.16 truncates to 28 samples per tag bit and the decoder's float
 * is 29), and some rates in between. */
RFID_B200_API int rfid_b200_create(const rfid_b200_params* p, rfid_b200_ctx** out);
RFID_B200_API void rfid_b200_destroy(rfid_b200_ctx* ctx);

/* Derived sample counts (gate_impl.cc:48-53,115,121; tag_decoder_impl.cc:60). */
RFID_B200_API int rfid_b200_window_length(const rfid_b200_ctx* ctx, int kind);
RFID_B200_API int rfid_b200_fs_dec(const rfid_b200_ctx* ctx);

/* ---------------- capture mode (throughput path) ----------------
 * Decode nseg independent segments of a raw capture that is ALREADY RESIDENT in
 * device memory: matched filter + decimation, gate, tag_decoder, all on the GPU,
 * asynchronously on `stream` (a cudaStream_t passed as void*; NULL = default).
 * d_iq: device pointer, interleaved float32 I,Q.  d_segs: device pointer to nseg
 * segment descriptors.  d_results: device buffer of nseg*max_windows_per_segment
 * records; record k of segment s lands at d_results[s*max_windows_per_segment+k].
 * d_counts: device int32[nseg], number of windows found per segment.
 * Windows beyond max_windows_per_segment are counted but not stored. */
RFID_B200_API int rfid_b200_decode_capture(rfid_b200_ctx* ctx, const float* d_iq, size_t n_raw,
                                           const rfid_b200_segment* d_segs, int nseg,
                                           int max_windows_per_segment,
                                           rfid_b200_window_result* d_results, int32_t* d_counts,
                                           void* stream);

/* Complex int16 captures (the radio's own wire format; UHD's `sc16` CPU format:
 * n_raw complex samples, sample k = (d_iq[2k], d_iq[2k+1]) = (I, Q), 4 bytes each).
 * Every sample is decoded as ((float)I * scale, (float)Q * scale), each component one
 * round-to-nearest float multiply, so records, segment tables and window-tap contents
 * equal, bit for bit, those of the fc32 entry point on that conversion of the capture.
 * scale must be finite and > 0 (the usual choice is 1/32767, the factor UHD's host
 * converters apply when they widen sc16 to fc32; any value works, what matters is that
 * the same float is used wherever the two are compared).  Returns RFID_B200_EINVAL for
 * any other scale, and for a device pointer that is not 16-byte aligned.  Segment
 * offsets and lengths have no further alignment requirement.  The capture kernels and
 * their choice are those of rfid_b200_decode_capture; their raw stages carry 4 bytes
 * per sample instead of 8. */
RFID_B200_API int rfid_b200_decode_capture_sc16(rfid_b200_ctx* ctx, const int16_t* d_iq, size_t n_raw, float scale,
                                                const rfid_b200_segment* d_segs, int nseg,
                                                int max_windows_per_segment,
                                                rfid_b200_window_result* d_results, int32_t* d_counts,
                                                void* stream);

/* Same, but every pointer is a HOST pointer: copies in, decodes, copies the
 * records out, synchronises.  This is the end-to-end call a reference user makes
 * on a recorded file (apps/reader.py:102-112 in DEBUG mode). */
RFID_B200_API int rfid_b200_decode_capture_host(rfid_b200_ctx* ctx, const float* h_iq, size_t n_raw,
                                                const rfid_b200_segment* h_segs, int nseg,
                                                int max_windows_per_segment,
                                                rfid_b200_window_result* h_results, int32_t* h_counts);

/* Kernel launches issued by the last decode_capture call on this context. */
RFID_B200_API int rfid_b200_last_launch_count(const rfid_b200_ctx* ctx);
/* Device time (ms, CUDA events on the launch stream) of the dominant kernel
 * (fused matched-filter+gate) accumulated since the last reset; and its launches. */
RFID_B200_API int rfid_b200_kernel_time(rfid_b200_ctx* ctx, int reset, float* ms_total, int* launches);
RFID_B200_API int rfid_b200_enable_kernel_timing(rfid_b200_ctx* ctx, int on);

/* Optional debug taps for capture mode (device pointers, may be NULL):
 * d_windows receives the ungated, DC-removed samples of every stored window
 * (gate output, gate_impl.cc:173,187) at a stride of rfid_b200_window_length(EPC)
 * complex samples per record slot. */
RFID_B200_API int rfid_b200_set_window_tap(rfid_b200_ctx* ctx, float* d_windows);

/* Host-side reduction of window records into READER_STATS, replaying the
 * bookkeeping of tag_decoder_impl.cc:269-288,295,329-387 and the stop rule of
 * gate_impl.cc:101-109 in stream order.  `continuous` != 0: all records belong to
 * one continuous reader session (counters carry across segments);
 * 0: every segment is its own session and the per-session stats are summed. */
RFID_B200_API int rfid_b200_reduce_stats(const rfid_b200_ctx* ctx, const rfid_b200_window_result* h_results,
                                         const int32_t* h_counts, int nseg, int max_windows_per_segment,
                                         int continuous, rfid_b200_stats* out);

/* ---------------- capture ingest (SURVEY.md section 8f, rank 2) ----------------
 * The reference decodes a recorded file (apps/reader.py:101-112, format: raw interleaved
 * float32 I,Q, misc/code/plot_signal.m:5-9) through ONE sequential gate.  Capture mode wants
 * independent segments, so a recording is first cut where nothing happens: reader commands are
 * bursts of low pulses (PW = 12 us, reader_impl.cc:55-71) separated by CW; every burst with more
 * than NUM_PULSES_COMMAND pulses arms exactly one gate window (gate_impl.cc:150-180) and the
 * window kinds alternate RN16/EPC, so a segment = `commands_per_segment` consecutive commands
 * plus the CW after each, starting `lead_us` of CW before the first.  Segment offsets are
 * multiples of `decim` (the matched filter keeps the capture's decimation phase); segment 0
 * starts at sample 0.  Decoding the segments reproduces the continuous reference run bit for
 * bit in every decision (open index, sync index, T, bits, CRC); correlation scores agree to the
 * drift of the reference's float running means (SURVEY.md 8e). */
typedef struct rfid_b200_segmenter {
  float level_frac;             /* low when |x| < level_frac * (mean |x| of the first 2^21 samples); 0.5 */
  float gap_us;                 /* CW longer than this separates two commands; 400 (> TRcal = 200 us) */
  float lead_us;                /* CW kept in front of a segment's first command; 300 (< gap_us) */
  int32_t min_pulses;           /* bursts with fewer low pulses are not commands; 6 (gate_impl.cc:164) */
  int32_t commands_per_segment; /* 2: one RN16 window + one EPC window */
  int32_t reserved[3];
} rfid_b200_segmenter;

RFID_B200_API void rfid_b200_default_segmenter(rfid_b200_segmenter* sp);

/* Segment table of a capture that is already in device memory.  sp may be NULL (defaults).
 * h_segs: HOST array of `capacity` entries; *nseg receives the number of segments (also when
 * RFID_B200_ECAPACITY is returned).  Runs on `stream` and synchronises it. */
RFID_B200_API int rfid_b200_segment_capture(rfid_b200_ctx* ctx, const float* d_iq, size_t n_raw,
                                            const rfid_b200_segmenter* sp, rfid_b200_segment* h_segs,
                                            int capacity, int* nseg, void* stream);
/* The same on a complex int16 capture (format, scale and argument checks as
 * rfid_b200_decode_capture_sc16): the CW level and the low-sample mask are computed on
 * the converted samples, so the table equals that of the fc32 conversion. */
RFID_B200_API int rfid_b200_segment_capture_sc16(rfid_b200_ctx* ctx, const int16_t* d_iq, size_t n_raw, float scale,
                                                 const rfid_b200_segmenter* sp, rfid_b200_segment* h_segs,
                                                 int capacity, int* nseg, void* stream);

/* File-to-records ingest, HOST pointers: uploads the capture in 16 MiB slices (pageable memory
 * through two pinned staging buffers, registered/pinned memory directly) with the threshold
 * pass of the segmenter running behind each slice, builds the segment table, decodes it and
 * copies table, records and counts back.  h_results holds seg_capacity*max_windows_per_segment
 * records, h_counts seg_capacity ints. */
RFID_B200_API int rfid_b200_ingest_capture_host(rfid_b200_ctx* ctx, const float* h_iq, size_t n_raw,
                                                const rfid_b200_segmenter* sp, int max_windows_per_segment,
                                                rfid_b200_segment* h_segs, int seg_capacity, int* nseg,
                                                rfid_b200_window_result* h_results, int32_t* h_counts);
/* The same for a recorded complex int16 file (e.g. `rx_samples_to_file --type short`,
 * `uhd_rx_cfile --output-shorts`): n_raw complex samples at h_iq, format and scale as
 * rfid_b200_decode_capture_sc16.  The 16 MiB upload slices carry twice the samples. */
RFID_B200_API int rfid_b200_ingest_capture_host_sc16(rfid_b200_ctx* ctx, const int16_t* h_iq, size_t n_raw, float scale,
                                                     const rfid_b200_segmenter* sp, int max_windows_per_segment,
                                                     rfid_b200_segment* h_segs, int seg_capacity, int* nseg,
                                                     rfid_b200_window_result* h_results, int32_t* h_counts);

/* ---------------- reader TX synthesiser + closed-loop slot simulator (SURVEY.md section 8f, rank 1) ----------------
 * The reader block's PIE command waveforms (reader_impl.cc:51-125 tables, :237-372 what every
 * Gen2-logic state emits, :383-443 CRC-5) generated on the GPU, sample for sample identical to
 * what reader_impl::general_work writes to its output port (float 0.0/1.0 at the DAC rate). */
enum {
  RFID_B200_TX_START = 0,        /* START: carrier before the first Query          (reader_impl.cc:237-243) */
  RFID_B200_TX_QUERY = 1,        /* SEND_QUERY: preamble + Query + carrier         (:265-285) */
  RFID_B200_TX_QUERY_REP = 2,    /* SEND_QUERY_REP                                 (:330-344) */
  RFID_B200_TX_ACK = 3,          /* SEND_ACK: frame-sync + 01 + RN16 (arg)         (:290-320) */
  RFID_B200_TX_CW = 4,           /* SEND_CW: carrier during the EPC reply          (:322-328) */
  RFID_B200_TX_NAK = 5,          /* SEND_NAK_Q / SEND_NAK_QR                       (:245-263) */
  RFID_B200_TX_POWER_DOWN = 6,   /* POWER_DOWN                                     (:228-235) */
  RFID_B200_TX_QUERY_ADJUST = 7  /* SEND_QUERY_ADJUST                              (:346-366) */
};
typedef struct rfid_b200_tx_command {
  int32_t kind; /* RFID_B200_TX_* */
  int32_t arg;  /* ACK: the 16-bit RN16 to echo */
} rfid_b200_tx_command;

/* Waveform of a script of emissions, written to d_out (device, `capacity` floats).  *n_samples
 * receives the total length (also on RFID_B200_ECAPACITY); d_out may be NULL to query it. */
RFID_B200_API int rfid_b200_tx_synth(rfid_b200_ctx* ctx, const rfid_b200_tx_command* h_script, int n_commands,
                                     int dac_rate, float* d_out, size_t capacity, size_t* n_samples, void* stream);

/* Inventory-slot simulator: one segment = one slot = carrier, Query (slot 0 of a round) or QueryRep,
 * RN16 replies of the tags that picked this slot, ACK, EPC reply, carrier.  Signal model (SURVEY.md 8d,
 * calibrated on misc/data/file_source_test): rx = (L + sum_k g_k b_k[n]) * env[n] + w[n], env = the
 * reader waveform above held to the ADC rate and shaped by the measured TX/RX edge response, b_k = FM0
 * half-symbol levels (TAG_PREAMBLE, data, dummy 1) at BLF 40 kHz starting T1 after the command.
 * closed_loop != 0: the first part of every slot is generated and decoded by this context's receive
 * chain, the ACK echoes the RN16 that was decoded, and only a tag whose RN16 matches sends its EPC
 * (collided or empty slots therefore end in silence, as with a real reader); closed_loop == 0: the ACK
 * echoes the strongest tag's RN16.  All randomness is counter-based: segment i of the global numbering is
 * the same whichever rank generates it. */
typedef struct rfid_b200_sim_params {
  uint64_t seed;
  int32_t n_tags;      /* tags in the field (0..16); each draws a slot per inventory round */
  int32_t closed_loop;
  int32_t dac_rate;    /* reader TX rate (apps/reader.py:56 -> 1000000); adc_rate must be a multiple */
  float segment_us;    /* slot length (8480 = the recording's round period) */
  float lead_us;       /* carrier before the first command (400) */
  float noise_sigma;   /* per component (0.0030) */
  float tag_gain;      /* |g| (0.0227) */
  float tag_phase;     /* arg g, rad */
  float clock_pct;     /* tag clock tolerance, percent (0.8) */
  float leak_re, leak_im; /* carrier leakage (0.2846, -0.0349) */
  float floor_level;   /* envelope inside a low pulse (0.004) */
  int32_t reserved[2];
} rfid_b200_sim_params;

typedef struct rfid_b200_sim_truth {
  int32_t is_query;       /* 1: the slot starts with a Query, 0: QueryRep */
  int32_t n_replies;      /* tags that answered with an RN16 */
  int32_t strongest_rn16; /* RN16 of the strongest of them, -1: empty slot */
  int32_t acked_rn16;     /* RN16 in the ACK (closed loop: what the receive chain decoded), -1: no ACK sent */
  int32_t replier;        /* tag that sent its EPC, -1: none */
  int32_t reserved[3];
  uint8_t epc[16];        /* PC + EPC + CRC-16 it sent (zeros if none) */
} rfid_b200_sim_truth;

RFID_B200_API void rfid_b200_default_sim(rfid_b200_sim_params* p);
/* raw samples per segment for these settings (negative: error) */
RFID_B200_API int rfid_b200_sim_segment_length(const rfid_b200_ctx* ctx, const rfid_b200_sim_params* p);
/* Generate segments [first_segment, first_segment + nseg) into d_iq (device, nseg * segment_length
 * complex64), with their segment table (device, offsets relative to d_iq) and ground truth (device, may
 * be NULL).  Asynchronous on `stream` except for buffer growth. */
RFID_B200_API int rfid_b200_sim_capture(rfid_b200_ctx* ctx, const rfid_b200_sim_params* p, int64_t first_segment,
                                        int nseg, float* d_iq, rfid_b200_segment* d_segs,
                                        rfid_b200_sim_truth* d_truth, void* stream);

/* ---------------- capture mode: the reader's commands ----------------
 * In a monostatic capture the reader's TX leaks into the RX at full carrier level, so every segment holds the reader's
 * PIE commands (reader_impl.cc:51-125,251-372) besides the tag's replies.  rfid_b200_decode_commands reads them back, per
 * segment and independently of every other segment and of the capture outside it (so the result does not depend on how a
 * capture is sharded):
 *   - p[i] = re*re + im*im of the (converted) sample, in float with each operation rounded;
 *   - thr2 = (level_frac*level_frac) * P, P = max p over the segment (NaN samples ignored); level_abs > 0 gives
 *     thr2 = level_abs*level_abs instead, for captures with outliers above 1/level_frac of the carrier amplitude.
 *     Sample i is low iff p[i] < thr2;
 *   - a fall is a low sample whose predecessor inside the segment is high (a low first sample is a fall);
 *   - a burst starts at a fall that has no low sample before it in the segment, or whose previous low sample prev
 *     satisfies fall - prev - 1 >= gap, gap = (int)(gap_us * 1e-6 * adc_rate) raw samples (the segmenter's test);
 *   - bursts of fewer than 4 falls are not reported.  Of the others, with d_k the fall-to-fall intervals: tari = d_0,
 *     rtcal = d_1; d_2 > rtcal means a preamble (trcal = d_2, data from d_3), otherwise a frame-sync (trcal = 0, data
 *     from d_2); every data interval is one bit, 1 iff 2*d > rtcal (every PIE symbol ends with its pulse);
 *   - start = the burst's first fall, end = the sample after its last low sample (or the segment length): raw samples
 *     relative to the segment;
 *   - kind (sync, bits, prefix -> arg, crc_ok):
 *       RFID_B200_TX_QUERY         preamble   22  1000      Q (bits 13-16), CRC-5 of bits 0-16 = bits 17-21 ? 1 : 0
 *       RFID_B200_TX_QUERY_REP     frame-sync  4  00        session (bits 2-3), -1
 *       RFID_B200_TX_ACK           frame-sync 18  01        RN16 (bits 2-17), -1
 *       RFID_B200_TX_QUERY_ADJUST  frame-sync  9  1001      session (bits 4-5), -1
 *       RFID_B200_TX_NAK           frame-sync  8  11000000  -1, -1
 *     anything else is RFID_B200_CMD_OTHER (arg and crc_ok -1) with its bits stored.
 * Inside a command the longest high stretch is TRcal - PW (188 us); between the commands of an inventory lies a tag
 * reply.  The reference's NAK is followed by only CW_D = 250 us of carrier (reader_impl.cc:233-249), so at the default
 * gap of 400 us a NAK and the command after it form one burst, reported as OTHER; a gap_us between about 190 and 249
 * separates them. */
#define RFID_B200_CMD_OTHER (-1)

typedef struct rfid_b200_cmd_params {
  float level_frac;    /* in (0, 1); 0.5 */
  float level_abs;     /* >= 0, finite; 0 = use level_frac */
  float gap_us;        /* > 0; 400 */
  int32_t reserved[5];
} rfid_b200_cmd_params;

typedef struct rfid_b200_command { /* 64 bytes */
  int32_t segment, index;         /* segment-table index; ordinal inside the segment */
  int32_t start, end;             /* raw samples, segment relative (rule above) */
  int32_t kind, n_bits;           /* RFID_B200_TX_* / RFID_B200_CMD_OTHER; all data bits (> 128: the first 128 stored) */
  int32_t tari, rtcal, trcal;     /* raw samples; trcal 0 = frame-sync */
  int32_t crc_ok, arg, reserved;
  uint8_t bits[16];               /* data bits, MSB first */
} rfid_b200_command;

RFID_B200_API void rfid_b200_default_cmd_params(rfid_b200_cmd_params* cp);

/* Commands of nseg segments of a capture resident in device memory (fc32; d_iq 8-byte aligned), asynchronously on
 * `stream`, conventions of rfid_b200_decode_capture: command k of segment s goes to d_cmds[s*max_commands_per_segment+k],
 * d_counts[s] receives the number of commands found (those beyond max_commands_per_segment are counted, not stored;
 * max_commands_per_segment may be 0, and d_cmds NULL with it).  A segment is cut at the end of the capture.  A segment
 * longer than INT32_MAX samples gets d_counts[s] = RFID_B200_EINVAL and no records.  cp NULL = defaults.  Returns
 * RFID_B200_EINVAL for level_frac outside (0, 1), a negative or non-finite level_abs, gap_us <= 0 and negative counts.
 * One CTA per segment reads the segment twice (peak, then masks). */
RFID_B200_API int rfid_b200_decode_commands(rfid_b200_ctx* ctx, const float* d_iq, size_t n_raw,
                                            const rfid_b200_segment* d_segs, int nseg, const rfid_b200_cmd_params* cp,
                                            int max_commands_per_segment, rfid_b200_command* d_cmds, int32_t* d_counts,
                                            void* stream);
/* The same on a complex int16 capture (format, scale and argument checks as rfid_b200_decode_capture_sc16): the records
 * equal those of the fc32 conversion. */
RFID_B200_API int rfid_b200_decode_commands_sc16(rfid_b200_ctx* ctx, const int16_t* d_iq, size_t n_raw, float scale,
                                                 const rfid_b200_segment* d_segs, int nseg, const rfid_b200_cmd_params* cp,
                                                 int max_commands_per_segment, rfid_b200_command* d_cmds,
                                                 int32_t* d_counts, void* stream);
/* HOST pointers (fc32): copies in, decodes, copies the records out, synchronises.  A segment longer than INT32_MAX
 * samples is RFID_B200_EINVAL. */
RFID_B200_API int rfid_b200_decode_commands_host(rfid_b200_ctx* ctx, const float* h_iq, size_t n_raw,
                                                 const rfid_b200_segment* h_segs, int nseg, const rfid_b200_cmd_params* cp,
                                                 int max_commands_per_segment, rfid_b200_command* h_cmds,
                                                 int32_t* h_counts);

/* ---------------- capture mode: reply quality and slot outcome ----------------
 * The decoder says which bits a window holds, never whether a tag answered.  rfid_b200_window_quality measures the
 * reply of every stored window and classifies its slot as empty, one reply or a collision.  It works per stored window
 * on the window's DC-removed samples w[0, n), n = min(length, window_length(EPC)) -- what the window tap
 * (rfid_b200_set_window_tap) holds and the decoder read -- and on the record's sync_index, h, T and length:
 *   - projections r_j = c_proj(s_a, s_b, h) = Re((s_a - s_b) * conj(h)) in float with every operation rounded, the
 *     floats whose signs the decoder turned into bits, at the decoder's own positions (a sample outside [0, n) is 0):
 *       RN16, k = 16: s_a, s_b = w[roundf(jm_2j)], w[roundf(jm_2j+1)], jm_0 = index, jm_m+1 = jm_m + n_tag_bit/2;
 *       EPC, k = 128: a = (int)(j*(2T) + index), b = (int)(j*2*T + T + index);
 *     index = (int)(sync_index + 6*n_tag_bit + n_tag_bit/2).  An RN16 window with a half-bit jm_0..31 >= n (the
 *     decoder's crc_ok = -2) gets energy = snr = NaN, n_decisions = 0 and outcome EMPTY;
 *   - snr = m*m / (S2/k - m*m), m = S1/k, S1 = sum |r_j|, S2 = sum r_j*r_j in double (r*r of a float is exact); a zero
 *     denominator gives +inf;
 *   - energy = (Er / (r1 - sync_index)) / (En / m): Er = sum |w|^2 over the reply [sync_index, r1), En over the noise
 *     reference, m its sample count, |w|^2 = re*re + im*im in double (both squares exact).  With n_i = n_tag_bit_i:
 *     e = the decoder's position two half-bits after its last decision sample, + n_i/5 (integer division): RN16
 *     roundf(jm_33) + n_i/5, EPC (int)(128*2*T + T + index) + n_i/5 (the last decision sample lies in the first half of
 *     the dummy 1 a tag appends to every reply; e is past its second half and the matched filter's response to it).
 *     The reply begins about half a bit before sync_index, so the reference is the head [0, h) with
 *     h = min(max(sync_index - 2*n_i/5, 0), n), then the tail [t, n) with t = min(e, n); when h + n - t < n_i,
 *     t = max(n - (n_i - h), h) (the tail moved back into the reply's end).  r1 = min(e, t).  At every sync index the
 *     preamble search can return and every well-defined rate with decimation 5, an RN16 reference holds at least n_i
 *     samples before or after the reply, so a late reply is measured like an early one; an EPC reply of a slow tag
 *     clock (T near its maximum) can reach the end of its window, and then part of the reference lies in it and the
 *     energy reads low.  A record with sync_index < 0, r1 <= sync_index or m = 0 gets energy NaN;
 *   - every sum has one order: term i to lane i % 32 (i ascending within a lane, from 0.0), then the 32 lane sums in
 *     ascending lane order; all arithmetic in double with round-to-nearest, snr and energy rounded once to float (one
 *     NaN pattern, 0x7fc00000).  They are linear ratios; convert to dB for display;
 *   - outcome: EMPTY unless energy >= empty_ratio (so also for NaN); then an RN16 window is SINGLE if snr >=
 *     single_ratio, else COLLISION; an EPC window is SINGLE (a collision is a property of the RN16 slot).  The
 *     thresholds are pow(10, dB / 10) in double of the float parameters, compared with the stored floats.
 * Defaults (calibrated on the simulators and on the reference's recording, its replies also moved up to 9 samples
 * later in their windows; DESIGN.md 4.6): empty_db 9.5 lies between the loudest empty slot of the closed-loop
 * simulator (9.0 dB) and the recording's weakest reply (9.8 dB); single_snr_db 8.8 lies below the simulators' weakest
 * single reply (9.0 dB) and above all but a few of their collided slots. */
enum { RFID_B200_SLOT_EMPTY = 0, RFID_B200_SLOT_SINGLE = 1, RFID_B200_SLOT_COLLISION = 2 };

typedef struct rfid_b200_quality_params {
  float empty_db;      /* finite; 9.5 */
  float single_snr_db; /* finite; 8.8 */
  int32_t reserved[6];
} rfid_b200_quality_params;

/* One window's quality (16 bytes), at the index of its window record.  (Named without "window_" because that is the
 * entry point's name.) */
typedef struct rfid_b200_quality {
  float energy, snr;   /* linear ratios (rule above) */
  int32_t outcome;     /* RFID_B200_SLOT_* */
  int32_t n_decisions; /* 16 (RN16), 128 (EPC), 0 (no RN16 decision) */
} rfid_b200_quality;

RFID_B200_API void rfid_b200_default_quality_params(rfid_b200_quality_params* qp);

/* Quality records of the stored windows of a decode_capture call (device pointers, asynchronous on `stream`):
 * d_windows = the window tap the call wrote (set before it with rfid_b200_set_window_tap, nseg * max_windows *
 * window_length(EPC) complex samples), d_results / d_counts its records and counts.  Record k of segment s goes to
 * d_quality[s * max_windows + k] for k < min(d_counts[s], max_windows); nothing else is written.  qp NULL = defaults.
 * Returns RFID_B200_EINVAL for a NULL pointer, non-finite thresholds and negative counts.  One warp per record slot
 * reads its window once. */
RFID_B200_API int rfid_b200_window_quality(rfid_b200_ctx* ctx, const float* d_windows,
                                           const rfid_b200_window_result* d_results, const int32_t* d_counts, int nseg,
                                           int max_windows, const rfid_b200_quality_params* qp,
                                           rfid_b200_quality* d_quality, void* stream);

/* ---------------- capture mode: EPC replies that fail their CRC ----------------
 * One wrong sign among an EPC window's 128 decisions loses the read.  rfid_b200_recover_epc flips the least reliable
 * decisions of a failing EPC window and keeps the result when exactly one flip set makes the window pass.  Per stored
 * window slot (s, k), k < min(count, max_windows), of a decode_capture call, from that call's window tap, records and
 * rfid_b200_window_quality records:
 *   1. an RN16 window: status NOT_EPC, the record's bits;
 *   2. an EPC window with crc_ok == 1: status CRC_OK, the record's bits (the tap is not read);
 *   3. a failing EPC window is SKIPPED unless its quality record has n_decisions == 128 and snr >= min_snr_ratio
 *      (NaN: SKIPPED), min_snr_ratio = pow(10, min_snr_db / 10) in double of the float parameter, compared with the
 *      stored float (the convention of the quality thresholds);
 *   4. otherwise a recovery is attempted:
 *      - the projections r_j, j = 0..127, exactly as the quality rule computes them (c_proj at win_epc_pos_a/b, a
 *        sample outside [0, n) taken as 0).  Their signs s_j = r_j > 0 are the record's bits through
 *        bit_j = s_j xor s_(j-1), s_(-1) = 1;
 *      - reliability p_j = |r_j| (float); the P = `positions` least reliable positions, ordered by (p_j, j) ascending;
 *      - candidates: every subset F of those P positions with 1 <= |F| <= W = `max_flips`.  Flipping s_j flips bits j
 *        and j + 1 (for j = 127 bit 127 only);
 *      - a candidate passes iff its bits pass the decoder's CRC-16 (bytes 0..13 against bytes 14..15) and its PC bits
 *        0..4 (the EPC length field, MSB first) are 00110: 6 words, the 96-bit EPC a 128-bit window holds;
 *      - n_pass = the number of passing candidates.  RECOVERED iff n_pass == 1: the record gets the corrected bits,
 *        n_flips = |F| and cost = (sum of p_j over F in double, ascending j) / (S1 / 128), rounded once to float, with
 *        S1 = sum of |r_j| in double in the quality rule's order.  AMBIGUOUS iff n_pass >= 2, FAILED iff n_pass == 0.
 * Every status but RECOVERED stores the record's bits, n_flips = 0 and cost = NaN (0x7fc00000); n_pass is 0 unless a
 * recovery was attempted.  The result does not depend on the order the candidates are tried in.
 * False accepts: a window whose true error set is not a candidate passes each candidate with probability about 2^-21
 * (16 CRC bits and 5 length bits) when its bits are random, so it is RECOVERED wrongly with probability at most
 * C * 2^-21, C = sum over k = 1..W of binomial(P, k); at the defaults P = 12, W = 4, C = 793: 3.8e-4.  A real reply's
 * length field is usually decoded right, and a candidate that flips no sign in 0..4 leaves it right, so for such a
 * window only the 16 CRC bits test the candidate: at most C * 2^-16, 1.2 % at the defaults.  The SNR gate keeps the
 * attempts to windows whose few errors are likely candidates.
 * Default min_snr_db 7.0 (DESIGN.md 4.7): the EPC windows of empty slots reach about 4.2 dB (pure noise: about
 * 2.4 dB); below 7 dB the simulated weak tag's failing replies gave wrong unique passes, above it none. */
enum {
  RFID_B200_FIX_CRC_OK = 0,
  RFID_B200_FIX_RECOVERED = 1,
  RFID_B200_FIX_AMBIGUOUS = 2,
  RFID_B200_FIX_FAILED = 3,
  RFID_B200_FIX_SKIPPED = 4,
  RFID_B200_FIX_NOT_EPC = 5
};

typedef struct rfid_b200_recover_params {
  int32_t positions;   /* P: 1..32; 12 */
  int32_t max_flips;   /* W: 1..P; 4 */
  float min_snr_db;    /* finite; 7.0 */
  int32_t reserved[5];
} rfid_b200_recover_params;

/* One window's recovery (32 bytes), at the index of its window record. */
typedef struct rfid_b200_epc_fix {
  int32_t status;   /* RFID_B200_FIX_* */
  int32_t n_flips;  /* |F| of a RECOVERED window, else 0 */
  int32_t n_pass;   /* passing candidates of an attempted window, else 0 */
  float cost;       /* RECOVERED: flipped reliability over the mean reliability; else NaN */
  uint8_t bits[16]; /* corrected (RECOVERED) or the record's bits */
} rfid_b200_epc_fix;

RFID_B200_API void rfid_b200_default_recover_params(rfid_b200_recover_params* rp);

/* Recovery records of the stored windows of a decode_capture call (device pointers, asynchronous on `stream`):
 * d_windows / d_results / d_counts as for rfid_b200_window_quality, d_quality its output for the same windows.  Record k
 * of segment s goes to d_fix[s * max_windows + k] for k < min(d_counts[s], max_windows); nothing else is written.
 * rp NULL = defaults.  Returns RFID_B200_EINVAL for a NULL pointer, negative counts, P outside 1..32, W outside 1..P,
 * a non-finite min_snr_db, or more than 65536 candidates.  One warp per record slot; only attempted windows read the
 * tap. */
RFID_B200_API int rfid_b200_recover_epc(rfid_b200_ctx* ctx, const float* d_windows,
                                        const rfid_b200_window_result* d_results, const int32_t* d_counts,
                                        const rfid_b200_quality* d_quality, int nseg, int max_windows,
                                        const rfid_b200_recover_params* rp, rfid_b200_epc_fix* d_fix, void* stream);

/* ---------------- capture mode: the tag inventory report ----------------
 * Which tags were read, how often, when and how strongly: one entry per full PC + EPC (the records' READER_STATS,
 * rfid_b200_reduce_stats, keys a tag by the 8 bits 104..111 as the reference does).  Built on the device from the records
 * and counts of a decode_capture call and, optionally, its quality and recovery records.  Only stored slots are read:
 * slot i = s * max_windows + k with k < min(max(count[s], 0), max_windows).
 *   - candidate: an EPC record with crc_ok == 1 (key = the record's bits), or else, with d_fix given, a slot whose fix has
 *     status RFID_B200_FIX_RECOVERED (key = the fix's bits; such a read is `recovered`);
 *   - a candidate is rejected for its length when check_length is 1 and PC bits 0..4 are not 00110 ((key[0] >> 3) != 6:
 *     a 128-bit window holds exactly the 6-word EPC), else for an empty slot when d_quality is given and the slot's outcome
 *     is RFID_B200_SLOT_EMPTY.  Every other candidate is a read;
 *   - the key is all 16 bytes (PC + EPC + CRC-16).  Tags are numbered 0, 1, ... in the order of their first read by
 *     ascending slot index (with a table in capture order: first seen first), whatever the launch geometry;
 *   - per tag: reads, recovered; first_slot, last_slot = smallest and largest slot of its reads; peak_slot = the read with
 *     the largest p = (float)((double)h_re*h_re + (double)h_im*h_im) (both squares exact, the sum rounded in double, then
 *     to float), the lowest slot on ties, a NaN p below every number; peak_power = its p (0x7fc00000 when every p of the
 *     tag is NaN); last_h = h of the last read, whose argument is the tag's latest carrier phase; first_time, last_time =
 *     the raw-sample time of the first and last read: segs[s].offset + decim * (open_index + sync_index) in int64 (two's
 *     complement wrap-around), s the slot's table position (the record's segment field is not read): where the reply
 *     starts, in samples of the capture the table indexes.  Every field is an order-independent aggregate, so the report
 *     does not depend on the order the device runs in;
 *   - summary: n_tags counts every tag, also those at index >= max_tags, which are not stored; reads, recovered;
 *     rejected_length, rejected_empty (a candidate is counted once, under the first test it fails);
 *   - d_read_tag (may be NULL): per stored slot, the tag index of a read (also >= max_tags), -1 for a slot that is not a
 *     candidate, -2 for a rejected candidate.  Slots that are not stored are not written.
 * h is in the matched filter's boxcar-sum units (ntaps samples), so 10*log10(peak_power / ntaps^2) is the reply's power
 * in dB relative to a full-scale sample. */
typedef struct rfid_b200_report_params {
  int32_t check_length; /* 0 or 1; 1 */
  int32_t reserved[7];
} rfid_b200_report_params;

typedef struct rfid_b200_tag { /* 64 bytes */
  uint8_t epc[16];                /* PC + EPC + CRC-16: the key */
  int32_t reads, recovered;       /* reads; those whose bits came from a RECOVERED fix */
  int32_t first_slot, last_slot;  /* slot indices s * max_windows + k */
  int32_t peak_slot;              /* read with the largest p (rule above) */
  float peak_power;               /* its p, boxcar-sum units squared */
  float last_h_re, last_h_im;     /* channel estimate of the last read */
  int64_t first_time, last_time;  /* raw samples (rule above) */
} rfid_b200_tag;

typedef struct rfid_b200_tag_summary { /* 32 bytes */
  int32_t n_tags;                 /* all tags, also beyond max_tags */
  int32_t reads, recovered;
  int32_t rejected_length, rejected_empty;
  int32_t reserved[3];
} rfid_b200_tag_summary;

RFID_B200_API void rfid_b200_default_report_params(rfid_b200_report_params* rp);

/* The report of the stored slots of a decode_capture call (device pointers, asynchronous on `stream` except when the
 * context's scratch has to grow, which synchronises): d_segs the segment table it decoded, d_results / d_counts its
 * records and counts, d_quality its rfid_b200_window_quality records (NULL: no EMPTY rejection), d_fix its
 * rfid_b200_recover_epc records (NULL: no recovered reads); rp NULL = defaults.  Tag j < max_tags goes to d_tags[j]; the
 * summary to *d_summary.  Returns RFID_B200_EINVAL for a NULL ctx, segs, results, counts or summary, d_tags NULL with
 * max_tags > 0, a negative nseg, max_windows or max_tags, nseg * max_windows >= 2^31, and check_length not 0 or 1.  A
 * thread per slot inserts the keys into an open-addressing table (warp-aggregated), then a scan over the slots numbers
 * the tags. */
RFID_B200_API int rfid_b200_tag_report(rfid_b200_ctx* ctx, const rfid_b200_segment* d_segs,
                                       const rfid_b200_window_result* d_results, const int32_t* d_counts, int nseg,
                                       int max_windows, const rfid_b200_quality* d_quality,
                                       const rfid_b200_epc_fix* d_fix, const rfid_b200_report_params* rp, int max_tags,
                                       rfid_b200_tag* d_tags, rfid_b200_tag_summary* d_summary, int32_t* d_read_tag,
                                       void* stream);

/* ---------------- capture mode: EPC replies from tags you already know ----------------
 * A failing EPC window need not be decoded from scratch when the tag population is known (tags read earlier, or a
 * manifest): it only has to be attributed to one of K known frames, maximum-likelihood decoding over a small codebook,
 * which works far below the point where flipping a few signs (rfid_b200_recover_epc) does.  rfid_b200_match_epc scores
 * every failing EPC window of a decode_capture call against a dictionary d_dict[k], k < K, of 16-byte PC + EPC + CRC
 * frames (an entry need not pass its CRC); K = min(max(*d_n_dict, 0), max_dict), or max_dict when d_n_dict is NULL.
 * Per stored slot i = s * max_windows + k, k < min(max(count[s], 0), max_windows):
 *   1. an RN16 window (kind != EPC): NOT_EPC;
 *   2. an EPC window with crc_ok == 1, or, with d_fix given, whose fix has status RFID_B200_FIX_RECOVERED: ALREADY_READ;
 *   3. otherwise the window is attempted.  It is SKIPPED when crc_ok != 0 (the decoder made no EPC decisions), or when
 *      S1 = sum of |r_j| (double, the quality rule's lane order) is 0 or not finite, with r_j, j = 0..127, the
 *      projections exactly as the quality rule computes them.  Else, with m = S1 / 128 (double):
 *      - reliability q_j = min(127, rint(|r_j| * 16 / m)) in double (16 steps per mean reliability, capped near 8x it);
 *      - signs s_j = (r_j > 0); entry k's signs c_kj = c_k,j-1 xor bit_kj (frame bit j, MSB first), c_k,-1 = 1: the
 *        signs the decoder's FM0 rule turns into that frame;
 *      - cost D_k = sum over j of q_j * [s_j != c_kj], an exact integer (= A + sum u_j c_kj, A = sum q_j s_j,
 *        u_j = q_j (1 - 2 s_j): the int8 product the kernel computes);
 *      - k* = argmin D_k, ties to the lowest k; D1 = D_k*; D2 = the second smallest value of the multiset {D_k} (a
 *        duplicate entry gives D2 = D1), INT32_MAX when K = 1;
 *      - MATCHED iff D1 <= max_cost16 and D2 - D1 >= min_margin16; AMBIGUOUS iff only the first holds; else NO_MATCH.
 *        The thresholds are (double)max_cost * 16 and (double)min_margin * 16 of the float parameters, compared with
 *        the integers converted to double (the convention of the quality thresholds);
 *      - K = 0: NO_MATCH, entry -1, cost = runner_up = INT32_MAX, n_diff -1.
 *   Record: status, entry = k* (-1 unless a cost was computed), cost = D1, runner_up = D2, n_diff = the number of j with
 *   s_j != c_k*j; a window that is not attempted, or SKIPPED, has entry = cost = runner_up = n_diff = -1.
 *   Per entry k < max_dict (d_count, may be NULL; every entry is initialised by the call): matched = the MATCHED windows
 *   naming k, first_slot / last_slot = their smallest and largest slot, -1 when there are none.
 * Every result is an integer, a min or a max, so the bytes do not depend on launch geometry or order.  Costs are in
 * sixteenths of the window's mean reliability (D / 16 "mean reliabilities").
 * False attribution -- a match is an attribution under a closed-population assumption, not a CRC-verified read, which
 * is why rfid_b200_tag_report does not count it:
 *   - pure noise: the best of K random frames comes closer as K grows.  The smallest D1 / 16 measured (DESIGN.md 4.9)
 *     was 31.1 / 27.1 / 20.8 at K = 16 / 1,024 / 65,536 over 10^5 Gaussian windows, and 39.1 / 30.4 / 27.6 over the
 *     EPC windows of 612 empty simulated slots: none comes within 8 units of max_cost 12 at K = 65,536.  Larger
 *     dictionaries lower this floor further; keep K no larger than the population can be;
 *   - a tag outside the dictionary: two valid frames with the same PC length field can be as little as 4 sign positions
 *     apart (e.g. frames that differ in bits 110, 111, 114, 115, 121, 122, 126, 127).  A reply from an unlisted tag that
 *     close to a listed one is MATCHED to it at any useful max_cost.  With the replying tag held out and one CRC-valid
 *     decoy at sign distance w from it in a 1,024-entry dictionary, the simulated weak replies were MATCHED to the decoy
 *     in over 99 % of trials for w <= 7, in 40-45 % at w = 12 and under 1 % at w = 16 (62-64 % over w = 4..16,
 *     DESIGN.md 4.9).  Against 1,024 random frames with the tag held out, none was MATCHED.
 * Defaults (DESIGN.md 4.9): max_cost 12, min_margin 4. */
enum {
  RFID_B200_MATCH_ALREADY_READ = 0,
  RFID_B200_MATCH_MATCHED = 1,
  RFID_B200_MATCH_AMBIGUOUS = 2,
  RFID_B200_MATCH_NO_MATCH = 3,
  RFID_B200_MATCH_SKIPPED = 4,
  RFID_B200_MATCH_NOT_EPC = 5
};

typedef struct rfid_b200_match_params {
  float max_cost;      /* finite, >= 0, mean reliabilities; 12 */
  float min_margin;    /* finite, >= 0, mean reliabilities; 4 */
  int32_t reserved[6];
} rfid_b200_match_params;

/* One window's attribution (32 bytes), at the index of its window record. */
typedef struct rfid_b200_epc_match {
  int32_t status;      /* RFID_B200_MATCH_* */
  int32_t entry;       /* k*, or -1 */
  int32_t cost;        /* D1, sixteenths of the mean reliability */
  int32_t runner_up;   /* D2 */
  int32_t n_diff;      /* sign disagreements with entry k* */
  int32_t reserved[3];
} rfid_b200_epc_match;

/* One dictionary entry's MATCHED windows (16 bytes). */
typedef struct rfid_b200_match_count {
  int32_t matched;
  int32_t first_slot, last_slot;   /* -1 when nothing matched */
  int32_t reserved;
} rfid_b200_match_count;

RFID_B200_API void rfid_b200_default_match_params(rfid_b200_match_params* mp);

/* Attribution records of the stored windows of a decode_capture call (device pointers, asynchronous on `stream` except
 * when the context's scratch has to grow, which synchronises): d_windows / d_results / d_counts as for
 * rfid_b200_window_quality, d_fix its rfid_b200_recover_epc records (may be NULL), d_dict max_dict frames of 16 bytes
 * (16-byte aligned), d_n_dict (may be NULL) the live count on the device.  Record k of segment s goes to
 * d_match[s * max_windows + k] for k < min(d_counts[s], max_windows); nothing else is written; d_count (may be NULL)
 * gets max_dict entries.  mp NULL = defaults.  Returns RFID_B200_EINVAL for a NULL ctx, windows, results, counts or
 * match, d_dict NULL with max_dict > 0 or not 16-byte aligned, negative nseg, max_windows or max_dict, nseg *
 * max_windows >= 2^31, max_dict > 2^24, and a non-finite or negative max_cost or min_margin.  One warp per slot prepares the attempted windows; the
 * scores are an int8 tensor-core product with a fused top-2. */
RFID_B200_API int rfid_b200_match_epc(rfid_b200_ctx* ctx, const float* d_windows, const rfid_b200_window_result* d_results,
                                      const int32_t* d_counts, const rfid_b200_epc_fix* d_fix, int nseg, int max_windows,
                                      const uint8_t* d_dict, const int32_t* d_n_dict, int max_dict,
                                      const rfid_b200_match_params* mp, rfid_b200_epc_match* d_match,
                                      rfid_b200_match_count* d_count, void* stream);

/* ---------------- block mode (GNU Radio drop-in) ----------------
 * Called from the thin host blocks' general_work(); HOST pointers, owned by the
 * scheduler, touched only during the call.  State lives in the context (device
 * memory) between calls. */

/* gate_impl::general_work (gate_impl.cc:85-200).  seek: 0 = none, 1 = the Gen2
 * logic asked for an RN16 window, 2 = for an EPC window since the previous call
 * (reader_state->gate_status SEEK flags, gate_impl.cc:112-123).  Returns through
 * *consumed / *written the values the reference passes to consume_each() and
 * returns; *closed = 1 when a window completed inside this call.  magn2_out
 * (may be NULL) receives |out|^2 per written sample (reader_state->magn_squared_samples). */
RFID_B200_API int rfid_b200_gate_work(rfid_b200_ctx* ctx, int seek, const float* in, int n_in, float* out,
                                      int out_capacity, int* consumed, int* written, int* closed,
                                      float* magn2_out);

/* tag_decoder_impl::general_work on one complete window (tag_decoder_impl.cc:223-393):
 * win = n complex samples (n >= window length of `kind`), result in *res.
 * bits_out (may be NULL): 16 (RN16) or 128 (EPC) floats in {0.,1.} exactly as the
 * reference writes them to stream port 0 (tag_decoder_impl.cc:261-266). */
RFID_B200_API int rfid_b200_decoder_work(rfid_b200_ctx* ctx, int kind, const float* win, int n,
                                         rfid_b200_window_result* res, float* bits_out);

/* fir_filter_ccc(decim,[1]*ntaps) replacement (apps/reader.py:75): canonical
 * boxcar + decimation with ntaps-1 samples of history kept in the context.
 * Writes floor((n_in + carry)/decim) outputs. */
RFID_B200_API int rfid_b200_mf_work(rfid_b200_ctx* ctx, const float* in, int n_in, float* out, int out_capacity,
                                    int* written);

#ifdef __cplusplus
}
#endif
#endif /* RFID_B200_H */
