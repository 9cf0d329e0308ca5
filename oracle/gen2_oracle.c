/* TEST INFRASTRUCTURE -- see gen2_oracle.h.  CPU restatement of the reference's
 * Gen2 RX decode path in plain C.  Every float operation below is written as a
 * separately rounded IEEE binary32 operation (build with -ffp-contract=off, no
 * fast-math; plain x86-64 has no FMA), mirroring what g++ emits for the
 * reference's std::complex<float> expressions.  Citations: /root/reference/gr-rfid/.
 */
#include "gen2_oracle.h"

#include <complex.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>

#include "mf_canonical.h"

/* ---- constants: include/rfid/global_vars.h:72-143 ---- */
enum {
  O_T1_D = 240, O_PW_D = 12, O_NUM_PULSES_COMMAND = 5, O_TAG_PREAMBLE_BITS = 6, O_RN16_BITS = 17,
  O_EPC_BITS = 129, O_WIN_SIZE_D = 250, O_DC_SIZE_D = 120, O_T_READER_FREQ = 40000
};
static const int O_TAG_PREAMBLE[12] = {1, 1, 0, 1, 0, 0, 1, 0, 0, 0, 1, 1}; /* global_vars.h:136 */
static const float O_THRESH_FRACTION = 0.75f;                               /* global_vars.h:139 */

/* Does tag_decoder_impl.cc stay inside its windows?  The decoder's indices come from the float n_samples_TAG_BIT, the
 * window lengths from its truncation (gate_impl.cc:115,121).  For each sync index tag_sync can return (i < 1.5 n, :85),
 * the largest index of every read is formed with the expressions below (the same ones o_tag_sync and
 * gen2_oracle_decode_window evaluate) and compared with the window it reads. */
static int o_defined(const gen2_oracle_cfg* c)
{
  const float n = c->n_tag_bit_f;
  if (c->n_tag_bit_i < 1) return 0;
  for (int i = 0; i < 1.5 * n; i++) {
    int reach = 0;
    for (int j = 0; j < 2 * O_TAG_PREAMBLE_BITS; j++) { /* :92; h_est's taps (:103) are among these */
      int k = (int)(i + j * n / 2);
      if (k > reach) reach = k;
    }
    if (reach >= c->len_rn16) return 0;
    int index = (int)(i + O_TAG_PREAMBLE_BITS * n + n / 2); /* :107 */
    int half_bits = 0;                                      /* :237-253 */
    for (float j = (float)index; j < c->len_rn16; j += n / 2) {
      if ((int)round(j) >= c->len_rn16) return 0;
      half_bits++;
      if (half_bits == 2 * (O_RN16_BITS - 1)) break;
    }
    if (half_bits != 2 * (O_RN16_BITS - 1)) return 0;
    float min_val = (float)(n / 2.0 - n / 2.0 / 100), max_val = (float)(n / 2.0 + n / 2.0 / 100); /* :151-152 */
    reach = 0;
    for (int t = 0; t < 20; t++) {
      float step = min_val + t * (max_val - min_val) / (20 - 1); /* :161 and T, :166 */
      for (int q = 0; q < 256; q++) {
        int p = (int)(q * step + index);
        if (p > reach) reach = p;
      }
      for (int q = 0; q < 128; q++) { /* :173 */
        int a = (int)(q * (2 * step) + index), b = (int)(q * 2 * step + step + index);
        if (a > reach) reach = a;
        if (b > reach) reach = b;
      }
    }
    if (reach >= c->len_epc) return 0;
  }
  return 1;
}

void gen2_oracle_make_cfg(const rfid_b200_params* p, gen2_oracle_cfg* c)
{
  memset(c, 0, sizeof(*c));
  c->adc_rate = p->adc_rate;
  c->decim = p->decim;
  c->ntaps = p->ntaps;
  int sample_rate = p->adc_rate / p->decim; /* apps/reader.py:76: int(adc_rate/decim) */
  c->fs_dec = sample_rate;
  /* global_vars.h:110-111: const float TAG_BIT_D = 1.0/T_READER_FREQ * pow(10,6) */
  const float TAG_BIT_D = (float)(1.0 / O_T_READER_FREQ * pow(10, 6));
  /* gate_impl.cc:48-53: int = int * (int / double) ... */
  c->n_T1 = (int)(O_T1_D * (sample_rate / pow(10, 6)));
  c->n_PW = (int)(O_PW_D * (sample_rate / pow(10, 6)));
  c->n_tag_bit_i = (int)(TAG_BIT_D * (sample_rate / pow(10, 6)));
  c->win_length = (int)(O_WIN_SIZE_D * (sample_rate / pow(10, 6)));
  c->dc_length = (int)(O_DC_SIZE_D * (sample_rate / pow(10, 6)));
  /* tag_decoder_impl.cc:60: float = float * int / double */
  c->n_tag_bit_f = (float)(TAG_BIT_D * sample_rate / pow(10, 6));
  /* gate_impl.cc:115,121 */
  c->len_epc = (O_EPC_BITS + O_TAG_PREAMBLE_BITS) * c->n_tag_bit_i + 2 * c->n_tag_bit_i;
  c->len_rn16 = (O_RN16_BITS + O_TAG_PREAMBLE_BITS) * c->n_tag_bit_i + 2 * c->n_tag_bit_i;
  c->fixed_q = p->fixed_q;
  c->max_queries = p->max_queries;
  c->max_tags = p->max_tags;
  c->defined = o_defined(c);
}

size_t gen2_oracle_mf(const float* x, size_t n_in, int ntaps, int decim, float* y)
{
  return oracle_mf_boxcar(x, n_in, ntaps, decim, y);
}

size_t gen2_oracle_mf_variant(const float* x, size_t n_in, int ntaps, int decim, float* y, int variant)
{
  /* variant 0: canonical; 1: sequential ascending float32; 2: float64 accumulation; 3: canonical order, every block
   * sum formed once (what the CPU reference arm times) */
  if (variant == 0) return oracle_mf_boxcar(x, n_in, ntaps, decim, y);
  if (variant == 3) {
    float* scratch = (float*)malloc(sizeof(float) * 2 * (n_in / (size_t)decim + (size_t)(ntaps / decim) + 2));
    if (!scratch) return 0;
    size_t n = oracle_mf_boxcar_blocked(x, n_in, ntaps, decim, y, scratch);
    free(scratch);
    return n;
  }
  return oracle_mf_boxcar_sequential(x, n_in, ntaps, decim, y, variant == 2);
}

/* std::abs(std::complex<float>) -> cabsf (gate_impl.cc:130) */
float gen2_oracle_cabsf(float re, float im)
{
  return cabsf(CMPLXF(re, im));
}

/* ------------------------------------------------------------------ gate */
int gen2_oracle_gate(const gen2_oracle_cfg* c, const float* y, size_t ny, int max_windows, int32_t* open_idx,
                     float* dc_out, float* win_out, float* avg_out)
{
  /* members, gate_impl.cc:45 + gate_impl.h:34-44 */
  int n_samples = 0, win_index = 0, dc_index = 0;
  float avg_ampl = 0.0f, num_pulses = 0.0f, sample_thresh;
  float dc_re = 0.0f, dc_im = 0.0f;
  enum { NEG_EDGE, POS_EDGE } signal_state = NEG_EDGE;
  const int win_length = c->win_length, dc_length = c->dc_length;
  float* win_samples = (float*)calloc((size_t)win_length, sizeof(float));
  float* dc_samples = (float*)calloc((size_t)dc_length * 2, sizeof(float));
  /* reader_state: first SEEK is for an RN16 window (global_vars.cc:47; reader_impl.cc:262) */
  int gate_open = 0;
  int n_samples_to_ungate = c->len_rn16;
  int nwin = 0, cur_open = 0;
  /* stop rule gate_impl.cc:101-109, n_queries_sent part: 1 Query at start + 1 per EPC window */
  int n_queries_sent = 1;
  float* cur_win = NULL;

  for (size_t i = 0; i < ny; i++) {
    float in_re = y[2 * i], in_im = y[2 * i + 1];
    /* gate_impl.cc:130-133 */
    float sample_ampl = cabsf(CMPLXF(in_re, in_im));
    avg_ampl = avg_ampl + (sample_ampl - win_samples[win_index]) / (float)win_length;
    win_samples[win_index] = sample_ampl;
    win_index = (win_index + 1) % win_length;
    /* gate_impl.cc:136 */
    sample_thresh = avg_ampl * O_THRESH_FRACTION;
    if (avg_out) avg_out[i] = avg_ampl;

    if (!gate_open) {
      /* gate_impl.cc:141-143: dc_est + (in - ring)/complex<float>(dc_length,0); the divisor has a
       * zero imaginary part, for which libgcc's __divsc3 reduces to one division per component */
      float dr = in_re - dc_samples[2 * dc_index], di = in_im - dc_samples[2 * dc_index + 1];
      dc_re = dc_re + dr / (float)dc_length;
      dc_im = dc_im + di / (float)dc_length;
      dc_samples[2 * dc_index] = in_re;
      dc_samples[2 * dc_index + 1] = in_im;
      dc_index = (dc_index + 1) % dc_length;

      n_samples++; /* :145 */
      if (sample_ampl < sample_thresh && signal_state == POS_EDGE) { /* :148-152 */
        n_samples = 0;
        signal_state = NEG_EDGE;
      } else if (sample_ampl > sample_thresh && signal_state == NEG_EDGE) { /* :154-162 */
        signal_state = POS_EDGE;
        if (n_samples > c->n_PW / 2)
          num_pulses++;
        else
          num_pulses = 0;
        n_samples = 0;
      }
      if (n_samples > c->n_T1 && signal_state == POS_EDGE && num_pulses > O_NUM_PULSES_COMMAND) { /* :164 */
        gate_open = 1;
        cur_open = (int)i;
        cur_win = (win_out && nwin < max_windows) ? win_out + (size_t)2 * nwin * c->len_epc : NULL;
        if (cur_win) { cur_win[0] = in_re - dc_re; cur_win[1] = in_im - dc_im; } /* :173 */
        num_pulses = 0;
        n_samples = 1;
      }
    } else {
      n_samples++; /* :184 */
      if (cur_win) { cur_win[2 * (n_samples - 1)] = in_re - dc_re; cur_win[2 * (n_samples - 1) + 1] = in_im - dc_im; }
      if (n_samples >= n_samples_to_ungate) { /* :189-194 */
        gate_open = 0;
        if (nwin < max_windows) {
          open_idx[nwin] = cur_open;
          if (dc_out) { dc_out[2 * nwin] = dc_re; dc_out[2 * nwin + 1] = dc_im; }
        }
        int was_epc = nwin & 1;
        nwin++;
        /* the decoder and the Gen2 logic run now; the reader answers with ACK after an RN16
         * (-> GATE_SEEK_EPC, reader_impl.cc:296) or Query/QueryRep after an EPC (-> GATE_SEEK_RN16,
         * reader_impl.cc:262,335), and the next gate call applies it (gate_impl.cc:112-123) */
        n_samples_to_ungate = was_epc ? c->len_rn16 : c->len_epc;
        n_samples = 0;
        if (was_epc) {
          n_queries_sent++;
          if (n_queries_sent > c->max_queries) break; /* gate_impl.cc:101-109,125 */
        }
      }
    }
  }
  free(win_samples);
  free(dc_samples);
  return nwin;
}

/* ------------------------------------------------------------------ decoder */
/* tag_decoder_impl::tag_sync, tag_decoder_impl.cc:78-109 */
static int o_tag_sync(const gen2_oracle_cfg* c, const float* in, int* raw_index, float* score, float* h_re, float* h_im)
{
  const float n = c->n_tag_bit_f;
  int max_index = 0;
  float max = 0.0f, corr;
  for (int i = 0; i < 1.5 * n; i++) { /* :85 */
    float c2r = 0.0f, c2i = 0.0f;
    for (int j = 0; j < 2 * O_TAG_PREAMBLE_BITS; j++) {
      int k = (int)(i + j * n / 2); /* :92, float arithmetic */
      float sr = in[2 * k], si = in[2 * k + 1];
      float cr = (float)O_TAG_PREAMBLE[j], ci = 0.0f;
      /* complex multiply as g++ inlines it: (ac - bd, ad + bc) */
      float pr = sr * cr - si * ci;
      float pi = sr * ci + si * cr;
      c2r = c2r + pr;
      c2i = c2i + pi;
    }
    corr = c2r * c2r + c2i * c2i; /* std::norm, :94 */
    if (corr > max) {
      max = corr;
      max_index = i;
    }
  }
  /* :103, six preamble-high taps, left-to-right sum, then / complex<float>(6,0) */
  int t1 = (int)(max_index + n / 2), t3 = (int)(max_index + 3 * n / 2), t6 = (int)(max_index + 6 * n / 2);
  int t10 = (int)(max_index + 10 * n / 2), t11 = (int)(max_index + 11 * n / 2);
  float sr = in[2 * max_index], si = in[2 * max_index + 1];
  sr = sr + in[2 * t1];  si = si + in[2 * t1 + 1];
  sr = sr + in[2 * t3];  si = si + in[2 * t3 + 1];
  sr = sr + in[2 * t6];  si = si + in[2 * t6 + 1];
  sr = sr + in[2 * t10]; si = si + in[2 * t10 + 1];
  sr = sr + in[2 * t11]; si = si + in[2 * t11 + 1];
  *h_re = sr / 6.0f;
  *h_im = si / 6.0f;
  *raw_index = max_index;
  *score = max;
  /* :107 */
  max_index = (int)(max_index + O_TAG_PREAMBLE_BITS * n + n / 2);
  return max_index;
}

/* the differential FM0 decision shared by tag_detection_RN16/EPC (:121-140, :171-191) */
static inline int o_decide(float result, int* prev)
{
  int bit;
  if (result > 0) {
    bit = (*prev == 1) ? 0 : 1;
    *prev = 1;
  } else {
    bit = (*prev == -1) ? 0 : 1;
    *prev = -1;
  }
  return bit;
}

static inline float o_proj(float ar, float ai, float br, float bi, float h_re, float h_im)
{
  /* std::real((a - b) * std::conj(h)) : (x+iy)(c+id), c = h_re, d = -h_im ; real = x*c - y*d */
  float x = ar - br, y = ai - bi;
  float cc = h_re, d = -h_im;
  return x * cc - y * d;
}

static inline void o_setbit(uint8_t* bits, int i, int v)
{
  if (v) bits[i >> 3] |= (uint8_t)(0x80 >> (i & 7));
}

uint16_t gen2_oracle_crc16(const uint8_t* data, int nbytes)
{
  /* tag_decoder_impl.cc:424-440 */
  uint16_t crc_16 = 0xFFFF;
  for (int i = 0; i < nbytes; i++) {
    crc_16 ^= (uint16_t)(data[i] << 8);
    for (int j = 0; j < 8; j++) {
      if (crc_16 & 0x8000) {
        crc_16 <<= 1;
        crc_16 ^= 0x1021;
      } else
        crc_16 <<= 1;
    }
  }
  return (uint16_t)~crc_16;
}

int gen2_oracle_crc16_ok(const uint8_t bits[16])
{
  uint16_t rcvd = (uint16_t)((bits[14] << 8) + bits[15]); /* :422 */
  return rcvd == gen2_oracle_crc16(bits, 14) ? 1 : 0;
}

void gen2_oracle_decode_window(const gen2_oracle_cfg* c, int kind, const float* in, int ninput,
                               rfid_b200_window_result* r)
{
  const float n = c->n_tag_bit_f;
  int raw_index;
  float score, h_re, h_im;
  int index = o_tag_sync(c, in, &raw_index, &score, &h_re, &h_im);
  r->kind = kind;
  r->length = kind == RFID_B200_RN16 ? c->len_rn16 : c->len_epc;
  r->sync_index = raw_index;
  r->score = score;
  r->h_re = h_re;
  r->h_im = h_im;
  memset(r->bits, 0, 16);

  if (kind == RFID_B200_RN16) {
    /* tag_decoder_impl.cc:237-256 */
    float sr[64], si[64];
    int number_of_half_bits = 0;
    for (float j = (float)index; j < ninput; j += n / 2) {
      number_of_half_bits++;
      int k = (int)round(j);
      sr[number_of_half_bits - 1] = in[2 * k];
      si[number_of_half_bits - 1] = in[2 * k + 1];
      if (number_of_half_bits == 2 * (O_RN16_BITS - 1)) break;
    }
    r->T = 0.0f;
    r->crc_ok = -1;
    if (number_of_half_bits == 2 * (O_RN16_BITS - 1)) {
      int prev = 1; /* :121 */
      for (int j = 0; j < number_of_half_bits / 2; j++) {
        float res = o_proj(sr[2 * j], si[2 * j], sr[2 * j + 1], si[2 * j + 1], h_re, h_im);
        o_setbit(r->bits, j, o_decide(res, &prev));
      }
      r->tag_id = (r->bits[0] << 8) | r->bits[1];
    } else {
      r->crc_ok = -2; /* RN16 window too short: the branch at tag_decoder_impl.cc:269-288 */
      r->tag_id = -1;
    }
    return;
  }

  /* tag_detection_EPC, tag_decoder_impl.cc:145-193.  magn_squared_samples[p] is
   * std::norm(in[p]) of the ungated sample (gate_impl.cc:172,186) */
  const int number_steps = 20;
  float min_val = (float)(n / 2.0 - n / 2.0 / 100), max_val = (float)(n / 2.0 + n / 2.0 / 100); /* :151-152 */
  float energy[20];
  for (int t = 0; t < number_steps; t++) {
    energy[t] = 0.0f;
    for (int i = 0; i < 256; i++) {
      int p = (int)(i * (min_val + t * (max_val - min_val) / (number_steps - 1)) + index); /* :161 */
      float xr = in[2 * p], xi = in[2 * p + 1];
      energy[t] += xr * xr + xi * xi;
    }
  }
  int index_T = 0; /* std::max_element: first largest, :165 */
  for (int t = 1; t < number_steps; t++)
    if (energy[t] > energy[index_T]) index_T = t;
  float T = min_val + index_T * (max_val - min_val) / (number_steps - 1); /* :166 */
  r->T = T;
  int prev = 1;
  for (int j = 0; j < 128; j++) {
    int a = (int)(j * (2 * T) + index);    /* :173 */
    int b = (int)(j * 2 * T + T + index);
    float res = o_proj(in[2 * a], in[2 * a + 1], in[2 * b], in[2 * b + 1], h_re, h_im);
    o_setbit(r->bits, j, o_decide(res, &prev));
  }
  r->crc_ok = gen2_oracle_crc16_ok(r->bits); /* :327 */
  r->tag_id = r->bits[13];                   /* bits[104..111], :348-352 */
}

int gen2_oracle_decode_decimated(const gen2_oracle_cfg* c, const float* y, size_t ny, int segment,
                                 rfid_b200_window_result* recs, int max_recs)
{
  int cap = (int)(ny / (size_t)c->len_rn16) + 2;
  int32_t* open_idx = (int32_t*)malloc(sizeof(int32_t) * (size_t)cap);
  float* dc = (float*)malloc(sizeof(float) * 2 * (size_t)cap);
  int nwin = gen2_oracle_gate(c, y, ny, cap, open_idx, dc, NULL, NULL);
  float* win = (float*)malloc(sizeof(float) * 2 * (size_t)c->len_epc);
  for (int k = 0; k < nwin && k < max_recs; k++) {
    int kind = (k & 1) ? RFID_B200_EPC : RFID_B200_RN16;
    int len = kind == RFID_B200_RN16 ? c->len_rn16 : c->len_epc;
    for (int s = 0; s < len; s++) { /* out = in - dc_est, gate_impl.cc:173,187 */
      win[2 * s] = y[2 * ((size_t)open_idx[k] + s)] - dc[2 * k];
      win[2 * s + 1] = y[2 * ((size_t)open_idx[k] + s) + 1] - dc[2 * k + 1];
    }
    rfid_b200_window_result* r = &recs[k];
    memset(r, 0, sizeof(*r));
    gen2_oracle_decode_window(c, kind, win, len, r);
    r->segment = segment;
    r->window = k;
    r->open_index = open_idx[k];
  }
  free(open_idx);
  free(dc);
  free(win);
  return nwin;
}

int gen2_oracle_decode_segments(const gen2_oracle_cfg* c, const float* iq_raw, const rfid_b200_segment* segs, int nseg,
                                rfid_b200_window_result* recs, int max_per_seg, int32_t* counts, double* seconds)
{
  struct timespec t0, t1;
  clock_gettime(CLOCK_MONOTONIC, &t0);
  size_t cap = 0;
  for (int s = 0; s < nseg; s++)
    if (segs[s].length > cap) cap = segs[s].length;
  float* y = (float*)malloc(sizeof(float) * 2 * (cap / (size_t)c->decim + 1));
  rfid_b200_window_result dummy[4];
  for (int s = 0; s < nseg; s++) {
    size_t ny = oracle_mf_boxcar(iq_raw + 2 * segs[s].offset, segs[s].length, c->ntaps, c->decim, y);
    int n = gen2_oracle_decode_decimated(c, y, ny, s, recs ? recs + (size_t)s * max_per_seg : dummy,
                                         recs ? max_per_seg : 4);
    if (counts) counts[s] = n;
  }
  free(y);
  clock_gettime(CLOCK_MONOTONIC, &t1);
  if (seconds) *seconds = (double)(t1.tv_sec - t0.tv_sec) + 1e-9 * (double)(t1.tv_nsec - t0.tv_nsec);
  return 0;
}

/* ------------------------------------------------------------------ stats */
static void o_tag_read(rfid_b200_stats* st, int id)
{
  /* std::map<int,int> tag_reads kept sorted (tag_decoder_impl.cc:355-364) */
  int n = st->n_unique_tags < RFID_B200_MAX_TAGS ? st->n_unique_tags : RFID_B200_MAX_TAGS;
  int k = 0;
  while (k < n && st->tag_id[k] < id) k++;
  if (k < n && st->tag_id[k] == id) {
    st->tag_reads[k]++;
    return;
  }
  if (st->n_unique_tags < RFID_B200_MAX_TAGS) {
    for (int m = n; m > k; m--) {
      st->tag_id[m] = st->tag_id[m - 1];
      st->tag_reads[m] = st->tag_reads[m - 1];
    }
    st->tag_id[k] = id;
    st->tag_reads[k] = 1;
  }
  st->n_unique_tags++;
}

/* one reader session: START -> Query, then RN16/EPC windows alternate */
static void o_session(const gen2_oracle_cfg* c, const rfid_b200_window_result* recs, int n, rfid_b200_stats* st,
                      int* cur_round, int* cur_slot, int* n_queries, int* terminated)
{
  const int max_slot = 1 << c->fixed_q; /* global_vars.cc:48 */
  for (int k = 0; k < n && !*terminated; k++) {
    const rfid_b200_window_result* r = &recs[k];
    int next_query = 0;
    if (r->kind == RFID_B200_RN16) {
      if (r->crc_ok == -2) { /* tag_decoder_impl.cc:269-288 */
        (*cur_slot)++;
        if (*cur_slot > max_slot) { *cur_slot = 1; (*cur_round)++; }
        next_query = 1;
      }
    } else {
      (*cur_slot)++; /* :295 */
      if (*cur_slot > max_slot) { *cur_slot = 1; (*cur_round)++; } /* :331-337 / :369-373 */
      if (r->crc_ok == 1) {
        st->n_epc_correct++; /* :346 */
        o_tag_read(st, r->tag_id);
      }
      next_query = 1;
    }
    st->n_windows++;
    if (next_query) {
      (*n_queries)++; /* reader_impl.cc:259,336 */
      /* gate_impl.cc:101-104, evaluated at the top of the next gate call */
      if (*n_queries > c->max_queries || st->n_unique_tags > c->max_tags) *terminated = 1;
    }
  }
}

void gen2_oracle_reduce_stats(const gen2_oracle_cfg* c, const rfid_b200_window_result* recs, const int32_t* counts,
                              int nseg, int max_per_seg, int continuous, rfid_b200_stats* out)
{
  memset(out, 0, sizeof(*out));
  out->max_slot_number = 1 << c->fixed_q;
  int cur_round = 1, cur_slot = 1, n_queries = 1, terminated = 0; /* global_vars.cc:50-51; reader_impl.cc:259 */
  int total_queries = 0;
  for (int s = 0; s < nseg; s++) {
    int n = counts[s] < max_per_seg ? counts[s] : max_per_seg;
    if (!continuous) {
      /* an independent segment is a run of the reference with freshly constructed blocks and reader_state
       * (SURVEY.md 8e): its stop rule sees only its own tag_reads; the global map is for reporting */
      static rfid_b200_stats seg; /* (large struct: keep it off the stack; this library is single-threaded test code) */
      memset(&seg, 0, sizeof(seg));
      cur_round = 1; cur_slot = 1; n_queries = 1; terminated = 0;
      o_session(c, recs + (size_t)s * max_per_seg, n, &seg, &cur_round, &cur_slot, &n_queries, &terminated);
      out->n_epc_correct += seg.n_epc_correct;
      out->n_windows += seg.n_windows;
      int nt = seg.n_unique_tags < RFID_B200_MAX_TAGS ? seg.n_unique_tags : RFID_B200_MAX_TAGS;
      for (int k = 0; k < nt; k++)
        for (int j = 0; j < seg.tag_reads[k]; j++) o_tag_read(out, seg.tag_id[k]);
      total_queries += n_queries;
    } else {
      o_session(c, recs + (size_t)s * max_per_seg, n, out, &cur_round, &cur_slot, &n_queries, &terminated);
    }
  }
  out->n_queries_sent = continuous ? n_queries : total_queries;
  out->cur_inventory_round = cur_round;
  out->cur_slot_number = cur_slot;
  out->terminated = terminated;
}

/* ------------------------------------------------------------------ TX-side CRC-5 */
void gen2_oracle_crc5(const uint8_t q[17], uint8_t crc_out[5])
{
  /* reader_impl.cc:383-443: 5-bit LFSR (x^5+x^3+1), preset 01001 held LSB first */
  int crc[5] = {1, 0, 0, 1, 0};
  for (int i = 0; i < 17; i++) {
    int tmp[5] = {0, 0, 0, 0, 0};
    tmp[4] = crc[3];
    int fb = (crc[4] == 1) != (q[i] == 1); /* the four branches collapse to one feedback bit */
    tmp[0] = fb;
    tmp[1] = crc[0];
    tmp[2] = crc[1];
    tmp[3] = fb ? !crc[2] : crc[2];
    memcpy(crc, tmp, sizeof(crc));
  }
  for (int i = 4; i >= 0; i--) crc_out[4 - i] = (uint8_t)crc[i];
}

void gen2_oracle_query_bits(int fixed_q, uint8_t out[22])
{
  /* reader_impl.cc:131-146 with global_vars.h:113-119: code 1000, DR 0, M 00, TRext 0, Sel 00,
   * Session 00, Target 0, Q (4 bits, MSB first) */
  static const uint8_t head[13] = {1, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
  memcpy(out, head, 13);
  for (int b = 0; b < 4; b++) out[13 + b] = (uint8_t)((fixed_q >> (3 - b)) & 1);
  gen2_oracle_crc5(out, out + 17);
}
