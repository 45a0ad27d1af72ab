/*
 * acars_b200 — C ABI of the H100-native acarsdec hot path
 * (u8 IQ -> per-channel mix+boxcar+decimate -> |.| -> demodMSK -> ACARS frame sync -> block FEC).
 *
 * Two layers, both plain C:
 *
 *  1. The context API below (acb_*): N independent IQ streams x C channels per GPU, the
 *     superset needed beyond MAXNBCHANNELS=16 (acarsdec.h:30).  Every entry point cites the
 *     reference interface it replaces.
 *  2. The reference's own symbols (initMsk/demodMSK/initAcars/decodeAcars/deinitAcars and the
 *     initRtl/runRtlSample/runRtlCancel/runRtlClose front-end trio) exported by
 *     libacarsdec_compat.so, declared in include/acarsdec_compat.h, implemented as a thin shim
 *     over this API so that acarsdec.c links against it unchanged.
 *
 * There is no CPU fallback: every processing call fails with ACB_ERR_CUDA when no sm_90
 * device / kernel image is available.
 */
#ifndef ACARS_B200_H
#define ACARS_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ACB_INTRATE 12500   /* acarsdec.h:31  INTRATE */
#define ACB_OUTBLK 1024     /* rtl.c:49       RTLOUTBUFSZ: output samples per IQ block */
#define ACB_TXTMAX 250      /* acarsdec.h:55  msgblk_t.txt */
#define ACB_MAXK 2048       /* rtl.c:39 caps rtlMult at 320; wideband configs go beyond */
#define ACB_MAXSTREAMS 65535 /* streams per context: they are grid.y of the channelizer launches (CUDA's limit) */

enum {
	ACB_OK = 0,
	ACB_ERR_ARG = -1,       /* bad argument */
	ACB_ERR_CUDA = -2,      /* CUDA runtime error / no device (see acb_last_error) */
	ACB_ERR_NOMEM = -3,
	ACB_ERR_OVERFLOW = -4,  /* device message ring overflowed: frames were lost */
	ACB_ERR_PLAN = -5       /* frequency plan impossible (rtl.c:149-152) */
};

typedef struct acb_ctx acb_ctx_t;

typedef struct {
	int device;             /* CUDA ordinal */
	int K;                  /* rtlMult: input rate = K*12500, taps == decimation (rtl.c:213-214) */
	int nstreams;           /* independent IQ streams served by this context, 1..ACB_MAXSTREAMS (65535): every
	                           channelizer launch puts the streams in grid.y, which CUDA limits to 65535, so
	                           acb_create refuses more with ACB_ERR_ARG */
	int nch;                /* channels per stream */
	int max_blocks;         /* largest nblk a submit call may carry (sizes device staging) */
	int flags;              /* ACB_FLAG_* */
	int taps;               /* FIR length per output: 0 = K (the reference: boxcar x NCO over the whole
	                           decimation period, rtl.c:283-286).  1..K selects the generalised case of
	                           BASELINE configs 3/5: only the first `taps` samples of every K-sample row
	                           are weighted (tables from acb_set_wf, nch x 2*taps floats), same arithmetic.
	                           K < taps <= ACB_MAXTAPS_PER_K*K: an overlapping window (a real channel filter, see
	                           acb_build_lowpass), any input kind.  With H = taps - K, output row m (counted from
	                           acb_create / acb_reset) is
	                             dm[m] = | sum_{i<taps} x[m*K - H + i] * w[i] |
	                           with x the front-end's converted sample ((float)u8 - 127.37f, (float)int16, the float
	                           itself), the same rounded operations in ascending tap order, and the terms whose
	                           sample index is negative omitted.  Row m still completes with sample (m+1)*K - 1, so
	                           pos / block / soh_pos and the emission groups keep their meaning; the filter's extra
	                           group delay of about (taps - K)/(2K) output samples is not compensated.  The context
	                           keeps each stream's last H samples (rounded up to 16 bytes) across submits; acb_reset
	                           clears them.  ACB_FLAG_FAST_CHANNELIZER is accepted and the exact kernel runs;
                           ACB_FLAG_FAST_FILTER (u8, CS16) and ACB_FLAG_FAST_FILTER_REAL (real input) select
                           the polyphase fast form of this filter. */
} acb_config_t;

#define ACB_MAXTAPS_PER_K 16          /* longest overlapping window, in decimation periods */

#define ACB_FLAG_NO_INPUT_STAGING 1   /* caller only uses acb_submit_device / acb_submit_dm_* */
#define ACB_FLAG_CS16_INPUT 4         /* SoapySDR / SDRplay front-ends (soapy.c, sdrplay.c): int16 I,Q samples;
                                         use acb_set_plan_cs16 / acb_submit_cs16_host (or _planar_host) */
#define ACB_FLAG_FAST_CHANNELIZER 8    /* u8 IQ contexts planned with acb_set_plan and CS16 contexts planned with
                                         acb_set_plan_cs16, K = 160 or 192 (real-input contexts planned with
                                         acb_set_plan_air, K = 200, 240, 400, 480 or 800: the same idea on a real row,
                                         k_channelize_rdft): run the channelizer
                                         as a shared 4-point DFT across the row quarters + K/4 MACs per channel
                                         (5x less FP32 work) when every stream's channels sit on the 12.5 kHz raster
                                         around Fc; otherwise the exact kernel runs.  NOT the reference's operation
                                         order: relative to the total in-band signal the envelope is within 1e-6 of the exact DFT
                                         bin and within the reference's own table rounding (1e-5) of the reference; decoded
                                         messages are the same; without this flag the envelope is bit-identical */
#define ACB_FLAG_FAST_FILTER 16        /* taps > K (the overlapping window) on u8 IQ contexts planned with acb_set_plan,
                                         acb_set_plan_at or acb_multi_set_plan and CS16 contexts planned with
                                         acb_set_plan_cs16, K = 160 or 192, every stream's channels on the 12.5 kHz raster
                                         around Fc (as ACB_FLAG_FAST_CHANNELIZER decides it): the polyphase fast form.  The
                                         window is pre-summed once per stream into one K-sample row per output,
                                           z_m[n] = sum_r p[n + H + r*K] * x[m*K + n + r*K],  p = fl(K * h)  (h: acb_build_lowpass)
                                         (ascending tap order, one FMA per term, terms before the stream start omitted), and
                                         each channel's bin of that row is taken as the boxcar fast form takes it:
                                         2*taps/K + ~7 FP32 lane-ops per complex sample instead of 8*C*taps/K.  NOT the
                                         exact form's operation order: per output row, with S = sum |x|*|w|, the envelope is
                                         within 1e-5*S of the exact form's and within 1e-6*S of the float64 definition;
                                         decoded messages are the same.  Anything else (a stream off the raster, a table given
                                         through acb_set_wf, another K, real input) runs the exact kernel, as does taps <= K,
                                         where this flag has no effect.  Real input has its own bit,
                                         ACB_FLAG_FAST_FILTER_REAL. */
#define ACB_FLAG_FAST_FILTER_REAL 32   /* taps > K on real-input contexts (ACB_FLAG_REAL_INPUT) with K = 200, 240, 400, 480 or
                                         800, every stream planned by acb_set_plan_air with every channel on the 12.5 kHz
                                         raster (acb_fast_plan_air returns 1): the polyphase fast form for real input.  The
                                         window is pre-summed into one K-sample real row per output,
                                           z_m[n] = sum_r p[n + H + r*K] * x[m*K + n + r*K],  p = fl(K * h)  (h: acb_build_lowpass)
                                         (ascending tap order, one FMA per term, terms before the stream start omitted), and
                                         each channel's bin of that row is taken exactly as ACB_FLAG_FAST_CHANNELIZER takes it
                                         from a row of input (k_channelize_rdft's operations, |D| in double): taps/K + ~10
                                         FP32 lane-ops per sample for 8 channels instead of 4*C*taps/K.  NOT the exact form's
                                         operation order: per output row, with S = sum |x|*|w|, the envelope is within 1e-5*S
                                         of the exact form's and within 1e-6*S of the float64 definition; decoded messages are
                                         the same.  Anything else (acb_set_wf tables, a stream off the raster, another K) runs
                                         the exact kernel, unchanged, as does taps <= K; on u8 and CS16 contexts this flag has
                                         no effect, and ACB_FLAG_FAST_FILTER alone selects nothing on a real context. */
#define ACB_FLAG_FAST_WIDEBAND 64      /* u8 IQ and CS16 contexts (interleaved and planar) with K % 8 == 0 (K <= ACB_MAXK), any
                                         nch, taps >= K, every stream planned by acb_set_plan, acb_set_plan_at,
                                         acb_multi_set_plan or acb_set_plan_cs16 with acb_fast_plan / acb_fast_plan_cs16
                                         returning 1 (every channel on the 12.5 kHz raster): the fast forms for any shape.
                                         The row's shared work (the fold and 4-point split, and at taps > K the pre-sum) is
                                         done once per row for all channels, and every channel's twiddles come from one
                                         table per context.  At taps = K the envelope is bit-identical to
                                         ACB_FLAG_FAST_CHANNELIZER's definition (the folded form, oracle
                                         orc_channelize_dft8*), at taps > K to ACB_FLAG_FAST_FILTER's (the polyphase form),
                                         with the same tolerances.  Where ACB_FLAG_FAST_CHANNELIZER or ACB_FLAG_FAST_FILTER
                                         also applies (K = 160 or 192) their kernels run; the bits are the same.  Anything
                                         else runs what runs without this flag: taps < K, acb_set_wf tables, a stream off the
                                         raster, K % 8 != 0, real input (no effect; real input has its own bit,
                                         ACB_FLAG_FAST_WIDEBAND_REAL).  ACB_FAST_FOLD8 does not apply. */
#define ACB_FLAG_FAST_WIDEBAND_REAL 128 /* real-input contexts (ACB_FLAG_REAL_INPUT) with K % 8 == 0 (K <= ACB_MAXK), any nch,
                                         taps >= K, every stream planned by acb_set_plan_air with acb_fast_plan_air returning
                                         1 (every channel on the 12.5 kHz raster): the real-input fast forms for any shape.
                                         The row's shared work (the quarter split, and at taps > K the pre-sum) is done once
                                         per row for all channels, and every channel's twiddles come from one table per
                                         context.  At taps = K the envelope is bit-identical to ACB_FLAG_FAST_CHANNELIZER's
                                         real-input definition (oracle orc_channelize_rdft, its lanes-per-row ranges and
                                         pairwise tree included, at any such K), at taps > K to ACB_FLAG_FAST_FILTER_REAL's
                                         (the pre-sum, then the same), with the same tolerances: per output row, with
                                         S = sum |x|*|w|, within 1e-5*S of the exact form's envelope and within 1e-6*S of the
                                         float64 definition; decoded messages are the same.  Where ACB_FLAG_FAST_CHANNELIZER
                                         (taps = K) or ACB_FLAG_FAST_FILTER_REAL (taps > K) also applies (K = 200, 240, 400,
                                         480 or 800) their kernels run; the bits are the same.  Anything else runs what runs
                                         without this flag: taps < K, acb_set_wf tables, a stream off the raster,
                                         K % 8 != 0; on u8 and CS16 contexts this flag has no effect, and
                                         ACB_FLAG_FAST_WIDEBAND alone selects nothing on a real context. */
#define ACB_FLAG_REAL_INPUT 2         /* Airspy front-end (air.c): float32 REAL samples at IF = rate/4,
                                         rate = K*12500; use acb_set_plan_air / acb_submit_real_host */
#define ACB_FLAG_DECODE_STATS 256     /* keep per-chain decode statistics (acb_decode_stats_t, acb_get_decode_stats): why
                                         frames were lost, counted where the reference's -v output prints a line.  The
                                         demodulator and the block FEC run their counting forms (same arithmetic, same
                                         launch rules); messages, envelope and chain states are unchanged.  Any input kind
                                         and channelizer form.  With this flag, ACB_DEMOD_LANES values other than 1, 2, 4 and
                                         8 are ignored and the picked default width runs (the other kernel forms have no
                                         counting form).  Without it acb_get_decode_stats returns ACB_ERR_ARG. */
#define ACB_FLAG_LEVEL_STATS 512      /* keep per-stream input levels and per-chain envelope levels (acb_input_level_t,
                                         acb_chan_level_t, acb_get_level_stats): input power, clipping and peak, channel
                                         power, peak and noise floor, reduced on the device from the input and envelope
                                         each submit already holds.  Any input kind and channelizer form, with or without
                                         ACB_FLAG_DECODE_STATS; messages, envelope, chain states and decode statistics are
                                         unchanged.  Without it acb_get_level_stats returns ACB_ERR_ARG. */
#define ACB_FLAG_FREQ_STATS 1024      /* measure each chain's carrier offset from its planned frequency (acb_chan_freq_t,
                                         acb_get_freq_stats, acb_freq_error): how far off frequency each receiver is tuned,
                                         from the phase rotation of the channel's carrier within each row.  Any input kind
                                         and channelizer form, with or without the other statistics flags; messages,
                                         envelope, chain states, decode and level statistics are unchanged.  Without it
                                         acb_get_freq_stats returns ACB_ERR_ARG. */

/* One decoded block, after parity/CRC repair: msgblk_t (acarsdec.h:48-57) without the queue
 * link, plus where it came from.  `txt` is parity-stripped (acars.c:200). */
typedef struct {
	int stream;
	int chn;
	int len;
	int err;                /* parity errors repaired (acars.c:156) */
	float lvl;              /* 10*log10(MskLvlSum/MskBitCount), acars.c:351 */
	uint64_t block;         /* index of the 1024-sample block in which the frame completed */
	uint64_t pos;           /* channel sample index (12.5 kS/s) at which the frame completed */
	uint64_t soh_pos;       /* channel sample index of the SOH byte (reference: gettimeofday, acars.c:290) */
	unsigned char txt[ACB_TXTMAX];
	unsigned char crc[2];
} acb_msg_t;

/* Per-channel demodulator + framing state: the persistent part of channel_t (acarsdec.h:76-89). */
typedef struct {
	double MskPhi, MskDf, MskLvlSum;
	float MskClk;
	int MskBitCount;
	unsigned MskS, idx;
	int nbits, Acarsstate;
	unsigned outbits;
	int blk_len, blk_err;
	uint64_t pos, soh_pos;
	float inb_re[11], inb_im[11];   /* msk.c:40 ring, FLEN=11 */
	unsigned char blk_crc[2];
	unsigned char blk_txt[ACB_TXTMAX];
} acb_chan_state_t;

/* ---- message formatting (SURVEY §8 f3): for hosts that take acb_msg_t blocks and do not link the reference's output.c ----
 * outputmsg()'s field split (output.c:486-640), label.c's OOOI fields, and the reference's wire formats, byte for byte
 * (tests/test_outfmt.py diffs them against output.c / label.c / netout.c / cJSON.c compiled in place).  Host only.
 * Not rebuilt: MQTT, libacars decoding, log-file rotation. */
#define ACB_REFERENCE_VERSION "3.7"      /* ACARSDEC_VERSION (acarsdec.h:28): the "app" object of the JSON format carries it */
typedef struct {
	char mode, ack, bid, bs, be;          /* ack: '!' for NAK; bs / be: the text's start and end bytes (STX/ETX/ETB) */
	char addr[8], label[3], no[5], fid[7];
	int downlink;                         /* block id '0'..'9' (output.c:31): message number and flight id are present */
	int txt_off, txt_len;                 /* the message text inside acb_msg_t.txt */
	int has_oooi;                         /* label.c's DecodeLabel matched; fields below are 4 characters or empty */
	char da[5], sa[5], eta[5], gout[5], gin[5], woff[5], won[5];
} acb_fields_t;
/* 1 = split done, 0 = not a block blk_thread would deliver (len < 13) */
int acb_msg_fields(const acb_msg_t *m, acb_fields_t *out);
typedef struct {
	int64_t tv_sec, tv_usec;              /* msgblk_t.tv */
	unsigned freq_hz;                     /* channel[chn].Fr: printed by the full format when inmode >= 3, and by JSON */
	int inmode;                           /* acarsdec.c's input mode: >= 3 shows the frequency, 2 (sound file) shows no date */
	int airflt, emptymsg;                 /* -A: downlinks only; -e: messages with text only */
	const char *labels;                   /* -i "H1:Q0:...": labels to keep; NULL keeps all */
	const char *station_id;               /* idstation; NULL or "" for none */
} acb_fmt_opts_t;
enum { ACB_FMT_ONELINE = 1, ACB_FMT_FULL = 2, ACB_FMT_JSON = 4,          /* -o 1 / 2 / 4 (without the JSON line's "\n") */
       ACB_FMT_NET_PP = 11, ACB_FMT_NET_NATIVE = 12, ACB_FMT_NET_JSON = 13 };   /* -N / -n / -j datagrams */
/* Writes the message in `format` to out (NUL-terminated; the formats may contain NUL bytes themselves where the reference
 * prints one).  Returns the length, 0 when a filter of `opt` drops the message, or a negative ACB_ERR_*. */
int acb_format_msg(const acb_msg_t *m, int format, const acb_fmt_opts_t *opt, char *out, size_t cap);
/* The flight table of output.c:349-426 (one entry per aircraft heard on a downlink; entries silent for `mdly_seconds`,
 * acarsdec's -t, default 600, are dropped) and the two outputs that need it.  Feed every block, in emission order, to ONE
 * of the two calls:
 *   acb_flights_route_json  -o 5: one JSON object per flight, the first time flight id, departure and destination are all
 *                           known (output.c:428-456); returns its length, 0 when this block produces none;
 *   acb_flights_monitor     -o 3: the monitor screen as redrawn after this block (output.c:458-484), `nbch` = channels
 *                           of the receiver (<= 16). */
typedef struct acb_flights acb_flights_t;
acb_flights_t *acb_flights_new(int mdly_seconds);
void acb_flights_free(acb_flights_t *t);
int acb_flights_route_json(acb_flights_t *t, const acb_msg_t *m, const acb_fmt_opts_t *opt, char *out, size_t cap);
int acb_flights_monitor(acb_flights_t *t, const acb_msg_t *m, int nbch, const acb_fmt_opts_t *opt, char *out, size_t cap);

/* ---- front-end planning: host-side, bit-identical to the reference's initRtl ---- */

/* rtl.c:245-247 — "131.525" -> Hz on the 12.5 kHz raster */
int acb_round_freq(double mhz);
/* rtl.c:255 — the value initRtl leaves in channel[].Fr (int <- float <- unsigned) */
int acb_stored_fr(unsigned freq_hz);
/* rtl.c:131-168 chooseFc — 0 when the span does not fit */
unsigned acb_choose_fc(const unsigned *freqs_hz, int n, int K);
/* Channel sets wider than one tuner span (rtl.c:149-152 gives up; scan.sh:1-16 walks the band sequentially): the
 * fewest receiver bands that cover them, each with its chooseFc centre.  group_of[i] = band of freqs_hz[i],
 * fc_out[g] = centre of band g; returns the number of bands (<= max_groups) or a negative error. */
int acb_plan_bands(const unsigned *freqs_hz, int n, int K, int *group_of, unsigned *fc_out, int max_groups);
/* rtl.c:283-286 — wf[ind] = cexpf(-j*AMFreq*ind)/K/127.5 as 2K floats (re,im interleaved) */
void acb_build_wf(int fr_stored, unsigned fc_hz, int K, float *wf);
/* air.c:42-64 (filter == 0) — Airspy tuner centre for the span [min,max] */
unsigned acb_air_choose_fc(unsigned min_hz, unsigned max_hz);
/* air.c:263-285 — wf[i] = cexpf(-j*Ph_i)/AIRMULT with the reference's double phase accumulator */
void acb_air_build_wf(int fr_hz, int fc_hz, unsigned rate, float *wf);
/* soapy.c:159-162 (variant ACB_CS16_SOAPY, with soapy.c:242's /32768.0 folded in) and
 * sdrplay.c:133-137 (ACB_CS16_SDRPLAY, with sdrplay.c:225's /4 folded in): effective mixer tables */
#define ACB_CS16_SOAPY 0
#define ACB_CS16_SDRPLAY 1
void acb_cs16_build_wf(int variant, unsigned freq_hz, unsigned fc_hz, int K, float *wf);
/* Planning step of ACB_FLAG_FAST_CHANNELIZER: returns 1 when every channel's mixer offset (float image
 * of the stored Fr minus float image of Fc, as rtl.c:283 computes it) is a whole, even number k of
 * 12.5 kHz steps with 0 < |k| < K/2; then k_out[ch] = k and tw[(ch*(K/4) + n2)*2 + {0,1}] =
 * exp(-j*2*pi*k*n2/K)/K/127.5.  k_out and tw may be NULL.  Returns 0 otherwise (the exact kernel runs). */
int acb_fast_plan(const unsigned *freqs_hz, int nch, int K, unsigned fc_hz, int *k_out, float *tw);
/* The same for CS16 contexts (soapy.c:159-165 / sdrplay.c:133-137: the offset is (float)Fr - (float)Fc); the twiddles
 * carry the variant's power-of-two scale, exp(-j*2*pi*k*n2/K)/K/32768 (soapy.c:242) or /K/4 (sdrplay.c:225). */
int acb_fast_plan_cs16(int variant, const unsigned *freqs_hz, int nch, int K, unsigned fc_hz, int *k_out, float *tw);
/* The same for real-input contexts (air.c:278-285): k = (Fc - Fr + rate/4)/12500 must be whole, 0 < k < K (any parity: the
 * real form splits the row in quarters only), tw = exp(-j*2*pi*k*n2/K)/K; K a multiple of 8. */
int acb_fast_plan_air(const unsigned *freqs_hz, int nch, int K, unsigned fc_hz, int *k_out, float *tw);
/* msk.c:44-48 — 133-tap oversampled half-cosine matched filter */
void acb_build_h(float *h);
/* Channel filter prototype for K < taps <= ACB_MAXTAPS_PER_K*K (no reference counterpart): an ideal low-pass with cutoff
 * ACB_INTRATE/2 (1/(2K) of the input rate) centred at (taps-1)/2, times a Kaiser window with beta = 6.0, normalised to
 * sum 1 in double and stored as float.  Returns ACB_OK, or ACB_ERR_ARG for K < 1 or taps outside 1..ACB_MAXTAPS_PER_K*K. */
int acb_build_lowpass(int K, int taps, float *h);
/* The planners' tables for taps > K (2*taps floats, re/im): w[i] = h[i] * mixer(i - H) * scale with h from
 * acb_build_lowpass and H = taps - K, so tap i meets sample m*K - H + i of row m.  Each front-end's own mixer: the float
 * images of the stored Fr and of Fc (rtl.c:283) and /127.5 for u8; soapy.c / sdrplay.c with the folded power-of-two
 * scale for CS16 (as acb_cs16_build_wf); air.c's IF at rate/4 for real input.  The offset is a whole number of Hz, so
 * the phase 2*pi*(offset*n mod rate)/rate is reduced exactly and evaluated in double (a float phase product, as the
 * reference's K-tap tables use, would be off by up to 1/128 rad at 16K taps); each weight is rounded to float once.
 * A carrier at the channel centre gives the reference's envelope level. */
void acb_build_wf_lp(int fr_stored, unsigned fc_hz, int K, int taps, float *wf);
void acb_cs16_build_wf_lp(int variant, unsigned freq_hz, unsigned fc_hz, int K, int taps, float *wf);
void acb_air_build_wf_lp(int fr_hz, int fc_hz, unsigned rate, int taps, float *wf);

/* ---- context ---- */

int  acb_create(const acb_config_t *cfg, acb_ctx_t **out);
void acb_destroy(acb_ctx_t *ctx);
const char *acb_last_error(void);
const char *acb_version(void);

/* Replaces the channel part of initRtl (rtl.c:243-287) for one stream: freqs in CLI order,
 * chooses Fc, builds and uploads the tables.  fc_out may be NULL. */
int acb_set_plan(acb_ctx_t *ctx, int stream, const unsigned *freqs_hz, int nch, unsigned *fc_out);
/* Same with the centre frequency given (a host that tuned already; a context that serves only SOME of the
 * channels chooseFc planned for — acb_multi_* in channel-split mode, the wide-stream case of SURVEY.md §8e). */
int acb_set_plan_at(acb_ctx_t *ctx, int stream, const unsigned *freqs_hz, int nch, unsigned fc_hz);
/* The channel part of initAirspy (air.c:165-285) for a real-input context. */
int acb_set_plan_air(acb_ctx_t *ctx, int stream, const unsigned *freqs_hz, int nch, unsigned *fc_out);
/* Same with the tuner centre given instead of acb_air_choose_fc's choice over these channels (a context that serves only
 * SOME of a receiver's channels: acb_multi_set_plan_air in channel-split mode).  Tables and fast plans as acb_set_plan_air
 * builds them; fc_hz = 0 is ACB_ERR_PLAN. */
int acb_set_plan_air_at(acb_ctx_t *ctx, int stream, const unsigned *freqs_hz, int nch, unsigned fc_hz);
/* The channel part of initSoapy (soapy.c:112-163) / initSdrplay (sdrplay.c:95-138) for a CS16
 * context; fc_hz = 0 lets chooseFc pick the centre (soapy.c:132-133 honours a user frequency). */
int acb_set_plan_cs16(acb_ctx_t *ctx, int stream, const unsigned *freqs_hz, int nch, int variant, unsigned fc_hz, unsigned *fc_out);
/* The planners (acb_set_plan, _at, _air, _cs16, and acb_multi_set_plan) build K-tap reference tables at taps = K and
 * the acb_build_wf_lp family's low-pass tables at taps > K; they fail with ACB_ERR_ARG at taps < K.
 * Same, with caller-supplied tables (nch x 2*taps floats; taps = K: e.g. taken from channel[].wf). */
int acb_set_wf(acb_ctx_t *ctx, int stream, const float *wf, int nch);
/* initMsk + initAcars for every channel of every stream (msk.c:30-51, acars.c:230-234).  Submits still in flight
 * are abandoned with their frames.  The streaming submits' carried remainder (the samples that did not fill a row)
 * and the taps > K history are discarded: row 0 after a reset starts with the next sample submitted. */
int acb_reset(acb_ctx_t *ctx);
/* initMsk + initAcars for one stream's channels only, for a receiver that was retuned, stalled or reconnected: its
 * carried remainder and taps > K history are discarded, its position returns to 0 (the next submit starts it at row 0,
 * as after acb_reset) and, with ACB_FLAG_DECODE_STATS, its counts restart from nothing: they cover the submits made after
 * the reset only.  Submits already made are still delivered (their messages, not their counts).  The other streams are
 * not touched and nothing waits on the device: the reset is queued behind the work already submitted.  To retune one receiver, call
 * acb_set_plan* (or acb_set_wf) for its stream, then acb_reset_stream; the planners wait for the submits in flight
 * before they replace the stream's tables. */
int acb_reset_stream(acb_ctx_t *ctx, int stream);

/* ---- processing ---- */

/* Replaces in_callback (rtl.c:314-361) for all streams at once.  Stream s's input is
 * `nblk` consecutive blocks of 1024*K*2 bytes (interleaved u8 I,Q) at iq + s*stream_stride.
 * Asynchronous: host->device copy, channelizer and demod are queued; call acb_sync to
 * collect.  `iq` should come from acb_host_alloc (pinned) for full PCIe overlap. */
int acb_submit_host(acb_ctx_t *ctx, const uint8_t *iq, size_t stream_stride, int nblk);
/* Same with the input already resident in device memory (no copy).
 * Input lifetime, both calls: up to three submits are in flight; when submit N+2 returns, the input of submit N
 * (the host buffer, or the device buffer) has been read and may be overwritten — as it may after an acb_collect /
 * acb_sync that covered submit N. */
int acb_submit_device(acb_ctx_t *ctx, const uint8_t *iq_dev, size_t stream_stride, int nblk);
/* Replaces rx_callback (air.c:291-341): `nsamples` float32 real samples per stream (stream s at
 * x + s*stream_stride_samples), ANY count per call — what does not fill a K-sample output row is
 * carried to the next call, the equivalent of the reference's carried partial sum ch->D / ind.
 * Returns the number of envelope samples produced per channel (>= 0) or a negative error. */
int acb_submit_real_host(acb_ctx_t *ctx, const float *x, size_t stream_stride_samples, size_t nsamples);
/* Replaces the channelizer loops of soapy.c:232-254 (interleaved CS16) and sdrplay.c:215-236
 * (planar xi/xq): `nsamples` complex int16 samples per stream, any count per call, remainder
 * carried (the reference carries ch->D and the tap index).  Returns envelope samples produced. */
int acb_submit_cs16_host(acb_ctx_t *ctx, const int16_t *iq, size_t stream_stride_samples, size_t nsamples);
int acb_submit_cs16_planar_host(acb_ctx_t *ctx, const int16_t *xi, const int16_t *xq, size_t stream_stride_samples, size_t nsamples);
/* Input lifetime, the three streaming calls (real, CS16, CS16 planar): the context copies what it needs (the carried
 * remainder and history live on the device), so:
 *   - pageable memory may be overwritten as soon as the call returns;
 *   - pinned memory (acb_host_alloc) is read asynchronously.  It may be overwritten once an acb_collect or acb_sync has
 *     covered the submit.  Submits that produced rows are covered in call order, one per acb_collect (the oldest first),
 *     and all of them by acb_sync.  A submit that produced no row (returned 0) is covered only by the next acb_sync.
 * A refused call (negative return) has read nothing, and the carried remainder is unchanged. */
/* The same three with the input already in device memory (a GPU-native source, or the broadcast buffer of a wide stream
 * served by several GPUs): arguments, return value, carried remainder, taps > K history, emission groups and every
 * channelizer form are the host calls', and a context may mix host and device submits of its kind freely — the result is
 * the one all-host submits give.  A small kernel appends each stream's samples behind its carried remainder on the
 * device: no host round trip, no synchronisation, no allocation.
 *   - Where the input may live: device memory of the context's device, or managed memory (cudaPointerGetAttributes
 *     decides).  Host memory, pinned or pageable, and another device's memory are refused with ACB_ERR_ARG.  The
 *     interleaved forms need 4-byte aligned input, the planar planes 2-byte aligned ones.
 *   - The host calls' refusals hold unchanged (wrong context kind, nsamples 0 or beyond max_blocks*1024*K, a stride
 *     smaller than nsamples with several streams); a refused call reads nothing and leaves the carry unchanged.
 *   - Input lifetime: that of pinned host memory above.  The input may be overwritten once an acb_collect or acb_sync
 *     has covered the submit; a submit that returned 0 is covered only by the next acb_sync.
 *   - Ordering: acb_wait_event orders the next device submit's read of its input behind the event (see there). */
int acb_submit_real_device(acb_ctx_t *ctx, const float *x_dev, size_t stream_stride_samples, size_t nsamples);
int acb_submit_cs16_device(acb_ctx_t *ctx, const int16_t *iq_dev, size_t stream_stride_samples, size_t nsamples);
int acb_submit_cs16_planar_device(acb_ctx_t *ctx, const int16_t *xi_dev, const int16_t *xq_dev,
                                  size_t stream_stride_samples, size_t nsamples);
/* Independent receivers: the ragged form of every submit above takes a count per stream — nblk[s] blocks, or
 * nsamples[s] samples — so that each stream advances at its own pace.  Arguments are otherwise the lockstep calls':
 *   - A count of 0 is allowed: the stream does not advance.  A call whose counts are all 0 is refused (ACB_ERR_ARG).
 *   - The lockstep refusals hold per stream (wrong kind, a count above the cap, alignment), and with several streams the
 *     stride must hold the largest count.  A refused call reads nothing and leaves every carry unchanged.
 *   - The streaming calls write each stream's new envelope rows to nout[s] (nout may be NULL) and return the largest of
 *     them, or a negative error.
 *   - Stream s's envelope rows, messages, chain states and decode statistics are bit-identical to those of a one-stream
 *     context of the same configuration fed only stream s's samples with the same cuts, for every input kind and
 *     channelizer form.  With every count equal a ragged call is the lockstep call, bits and emission order alike, and a
 *     context may mix lockstep and ragged calls, host and device.
 *   - Input: the host calls read each stream's own count, except that every stream but the last is read up to the
 *     largest count (within its stride).  acb_submit_device_ragged's channelizer reads every stream, the last one
 *     included, for the largest nblk: each stream's region must be readable that far (the rows past its own count are
 *     computed and never used).  The streaming device calls read each stream's own count.
 *   - acb_read_dm keeps its layout with nsamp = the largest count of rows; stream s's rows at or beyond its own count are
 *     unspecified.
 *   - Lifetime and ordering: those of the lockstep calls. */
int acb_submit_host_ragged(acb_ctx_t *ctx, const uint8_t *iq, size_t stream_stride, const int *nblk);
int acb_submit_device_ragged(acb_ctx_t *ctx, const uint8_t *iq_dev, size_t stream_stride, const int *nblk);
int acb_submit_real_host_ragged(acb_ctx_t *ctx, const float *x, size_t stream_stride_samples, const size_t *nsamples, size_t *nout);
int acb_submit_cs16_host_ragged(acb_ctx_t *ctx, const int16_t *iq, size_t stream_stride_samples, const size_t *nsamples, size_t *nout);
int acb_submit_cs16_planar_host_ragged(acb_ctx_t *ctx, const int16_t *xi, const int16_t *xq, size_t stream_stride_samples,
                                       const size_t *nsamples, size_t *nout);
int acb_submit_real_device_ragged(acb_ctx_t *ctx, const float *x_dev, size_t stream_stride_samples, const size_t *nsamples,
                                  size_t *nout);
int acb_submit_cs16_device_ragged(acb_ctx_t *ctx, const int16_t *iq_dev, size_t stream_stride_samples, const size_t *nsamples,
                                  size_t *nout);
int acb_submit_cs16_planar_device_ragged(acb_ctx_t *ctx, const int16_t *xi_dev, const int16_t *xq_dev, size_t stream_stride_samples,
                                         const size_t *nsamples, size_t *nout);
/* Emission order of the streaming front-ends (SURVEY H5).  The reference runs demodMSK channel by channel on
 * whatever a transfer (air.c:336) or a full dm_buffer (soapy.c:247: 1024 outputs; sdrplay.c:229: 512) delivered, so
 * its messages leave in (group, channel, time) order.  A submit may carry many such groups; tell the context how
 * they are cut and acb_sync / acb_collect queue the frames exactly in the reference's order:
 *   ACB_GROUP_SUBMIT   one group per submit call (default);
 *   ACB_GROUP_OUTPUTS  a group every `period` envelope samples, counted from the start of the stream;
 *   ACB_GROUP_INPUT    a group per transfer of `period` input samples, counted from the start of the stream.
 * (u8 IQ contexts always group per 1024-sample block, rtl.c:357-360.)
 * Every stream counts its groups from its own start (acb_create, acb_reset, acb_reset_stream).  Within a submit the frames
 * leave in (group number, stream, channel, time) order, the group number being the stream's 1024-row block (u8), the
 * `period`-output group or the transfer (the first output each transfer completes) it lies in; with ACB_GROUP_SUBMIT
 * the submit is one group.  When every stream is at the same position, as with lockstep calls only, this is the order
 * above. */
enum { ACB_GROUP_SUBMIT = 0, ACB_GROUP_OUTPUTS = 1, ACB_GROUP_INPUT = 2 };
int acb_set_emission_groups(acb_ctx_t *ctx, int unit, uint64_t period);
/* Replaces demodMSK's input side (msk.c:67; soundfile.c:71-77): 12.5 kS/s envelope samples,
 * dm[(s*nsamp + n)*nch + c], fed straight to the demodulator (no channelizer). */
int acb_submit_dm_host(acb_ctx_t *ctx, const float *dm, int nsamp);
/* Order the next acb_submit_device behind work of ANOTHER CUDA stream: `cuda_event` is a cudaEvent_t recorded there
 * (e.g. behind the NCCL broadcast that fills the input buffer; torch.cuda.Event.cuda_event).  No host sync.
 * On real-input and CS16 contexts it also orders the next acb_submit_real_device / acb_submit_cs16_device /
 * acb_submit_cs16_planar_device's read of its input behind the event as recorded at this call (the host submits'
 * copies are not held up by it).  Every later submit is ordered behind that one, so one wait covers a device buffer
 * for as long as it is not refilled. */
int acb_wait_event(acb_ctx_t *ctx, void *cuda_event);
/* Wait for the OLDEST submit still in flight only (at most three are), run the block FEC on its
 * frames and queue the survivors; later submits keep running.  This is what lets the H2D copy
 * of step i+1 overlap the kernels of step i.  Returns the number of messages waiting. */
int acb_collect(acb_ctx_t *ctx);
/* Wait for everything queued, run the block FEC (blk_thread, acars.c:93-215) on what the
 * device decoded, and append the survivors to the output queue in the reference's emission
 * order (block-major, then stream, then channel, then time; rtl.c:357-360).
 * Returns the number of messages waiting, or a negative error. */
int acb_sync(acb_ctx_t *ctx);
/* Pop up to `max` messages from the output queue (the outputmsg() feed, acars.c:209). */
int acb_drain(acb_ctx_t *ctx, acb_msg_t *out, int max);
/* Messages currently waiting in the output queue. */
int acb_pending(acb_ctx_t *ctx);

/* Pinned host memory for submit_host callers. */
void *acb_host_alloc(size_t bytes);
void  acb_host_free(void *p);
/* Device memory for submit_device callers (benchmarks keep the input resident in HBM). */
void *acb_device_alloc(acb_ctx_t *ctx, size_t bytes);
void  acb_device_free(acb_ctx_t *ctx, void *p);
int   acb_copy_to_device(acb_ctx_t *ctx, void *dst_dev, const void *src_host, size_t bytes);

/* ---- inspection (parity tests, the compat shim, bench instrumentation) ---- */

/* Tolerance of what these return (default, exact channelizer): envelope samples and messages are bit-identical to the
 * reference's; the demodulator state is bit-identical on every fixture of the test suite, and structurally within 1 ulp of
 * a float ring entry with probability ~2^-29 per sample (the device's VCO sincos is a table evaluation of at most 1.75 ulp,
 * glibc's is 0.52 ulp, and the product is rounded to float, msk.c:90; tests/test_demod_primitives.py asserts the bound and
 * finds 0 float mismatches in 2^24 seeded mixer pairs) — far inside the stated bar of 1e-5 relative.  With
 * ACB_FLAG_FAST_CHANNELIZER: messages identical, intermediates as documented in DESIGN.md §2. */
/* Envelope samples the channelizer produced for the last submit: out[(s*nsamp+n)*nch + c]. */
int acb_read_dm(acb_ctx_t *ctx, float *out, size_t nfloats);
/* The state is the demodulator's and the frame synchroniser's only: a round trip does not carry the channelizer's input
 * side — the streaming front-ends' carried remainder, or the window history of a taps > K context — nor the stream's
 * position, tables or statistics.  To move a whole stream use acb_save_streams / acb_load_streams below. */
int acb_get_state(acb_ctx_t *ctx, int stream, int chn, acb_chan_state_t *out);
int acb_set_state(acb_ctx_t *ctx, int stream, int chn, const acb_chan_state_t *in);

/* ---- moving streams: a stream's whole decoding state, to another slot, context, device or process ----
 *
 * A blob holds `count` records behind a 64-byte header; record i is one stream's state:
 *   - its position (envelope rows since its start), carried remainder count and whether its plan is on the raster;
 *   - its nch chain states (the frame being assembled, the PLL, the bit clock);
 *   - the channelizer's input side: the u8 taps > K history, or the streaming kinds' history and carried remainder;
 *   - its channel tables and fast plan, copied as the context holds them (no replanning);
 *   - with ACB_FLAG_DECODE_STATS its decode counts, with ACB_FLAG_LEVEL_STATS its level tables and open 1024-row windows,
 *     with ACB_FLAG_FREQ_STATS its chains' frequency sums, planned frequencies and NCO steps.
 * Records have one size per configuration.  The exact tables dominate it: nch * taps_pad * 8 bytes (taps_pad: taps
 * rounded up to 16 bytes of input), e.g. about 52 MB per stream at K = 1600, 256 channels, taps = 16K.
 * The format is little-endian and opaque; it carries a magic, a format version, the fingerprint below and a CRC-32, and
 * moves between builds of the same format version.
 *
 * The promise: stream s saved from one context and loaded into stream t of another, then fed what s would have been fed,
 * gives bit for bit what s would have given had it stayed — envelope rows, messages (every field but `stream`), chain
 * states, decode and level statistics, emission group numbers.  It holds for every input kind and channelizer form,
 * taps = K and taps > K, lockstep and ragged, host and device submits, the same or another device or process.  One
 * condition: both contexts must run the same channelizer form for the rows compared.  The fast forms run only while
 * every stream of a context is planned on the raster (otherwise the whole context runs EXACT), so a stream's envelope
 * can depend on its neighbours' plans; under a fast flag, give both contexts raster plans (or neither). */
/* bytes a blob of n streams of this context takes */
size_t acb_streams_blob_bytes(acb_ctx_t *ctx, int n);
/* Save streams[0..n) into blob (cap >= acb_streams_blob_bytes(ctx, n)); record i is streams[i].  The submits in flight
 * are collected first, as acb_sync collects them (their messages wait in the output queue, their counts are added; a
 * ring overflow is left for the next acb_collect / acb_sync to report), so the blob holds each stream's state after every
 * submit made so far, and a continuation produces only later messages.  The context is not changed.  To move a stream:
 * save it, load it elsewhere, then stop feeding (or acb_reset_stream) the source slot.  Returns ACB_OK. */
int acb_save_streams(acb_ctx_t *ctx, const int *streams, int n, void *blob, size_t cap);
/* Load record i of blob into stream streams[i]: n must be the blob's record count, streams distinct and in range.  Like
 * acb_reset_stream the load is queued behind the work in flight and touches no other stream: submits made before it
 * still deliver that slot's messages (not their counts), and the slot's statistics become the blob's.  The bytes are
 * staged before the call returns (the caller may free the blob); the host waits only for an earlier load's staging,
 * and, when a save or load needs more staging than the context has used so far, for the allocation (which synchronises
 * the device: save or load the largest set once up front to avoid it in a live pipeline).
 * Refused with ACB_ERR_ARG, the context unchanged, unless the format version and the CRC match, and the input kind, K,
 * taps, nch, channelizer form, the ACB_FLAG_DECODE_STATS, ACB_FLAG_LEVEL_STATS and ACB_FLAG_FREQ_STATS bits and (streaming kinds) the
 * emission-group unit and period match the context's.  nstreams, max_blocks and the device may differ. */
int acb_load_streams(acb_ctx_t *ctx, const int *streams, int n, const void *blob, size_t size);
/* A blob's fingerprint; host only (no device, no context).  ACB_ERR_ARG for a wrong magic or version, a size that does
 * not match the header, or a CRC mismatch. */
typedef struct {
	int in_kind;              /* 0 u8 IQ, 1 real, 2 CS16 */
	int K, taps, nch;         /* taps as the context runs it (K for taps = 0) */
	int form;                 /* the channelizer form: 0 EXACT, 1 GENERIC, 2 DFT, 3 RDFT, 4 OVL_FAST, 5 OVL_RDFT, 6 WB, 7 WB_REAL */
	int flags;                /* ACB_FLAG_DECODE_STATS | ACB_FLAG_LEVEL_STATS | ACB_FLAG_FREQ_STATS bits of the context */
	int group_unit;           /* streaming kinds: ACB_GROUP_*; u8: 0 */
	uint64_t group_period;
	int count;                /* records */
	uint64_t record_bytes;
} acb_streams_blob_info_t;
int acb_streams_blob_check(const void *blob, size_t size, acb_streams_blob_info_t *out);

/* CUDA-event stopwatch on the context's compute stream (the stream the kernels run on):
 * acb_mark(ctx,0) ... submits ... acb_mark(ctx,1); acb_elapsed_ms waits for mark 1. */
int acb_mark(acb_ctx_t *ctx, int which);
int acb_elapsed_ms(acb_ctx_t *ctx, float *ms);

typedef struct {
	uint64_t submits;           /* submit calls */
	uint64_t kernel_launches;   /* CUDA kernels launched by this context */
	uint64_t blocks;            /* stream-blocks processed */
	uint64_t raw_frames;        /* frames handed from the device to the FEC */
	uint64_t fec_dropped;       /* frames the FEC rejected */
	double   chan_ms;           /* accumulated device time of the channelizer kernel (CUDA events) */
	double   demod_ms;          /* accumulated device time from a demod kernel's start to the end of its block FEC */
	uint64_t chan_launches, demod_launches;
	uint64_t fast_chan_launches; /* channelizer launches that took a fast form: ACB_FLAG_FAST_CHANNELIZER's (taps = K) or
	                                ACB_FLAG_FAST_FILTER's or ACB_FLAG_FAST_FILTER_REAL's (taps > K),
	                                or ACB_FLAG_FAST_WIDEBAND's or ACB_FLAG_FAST_WIDEBAND_REAL's (either) */
	uint64_t frames_lost;       /* frames that found the device ring full (ACB_ERR_OVERFLOW was returned once per submit) */
	double   host_ms;           /* accumulated wall time the consumer thread spent ordering and queuing frames */
} acb_stats_t;
int acb_get_stats(acb_ctx_t *ctx, acb_stats_t *out, int reset);

/* Per-chain decode statistics (ACB_FLAG_DECODE_STATS): for one (stream, channel), how many times each event of the
 * frame synchroniser (decodeAcars) and of the block FEC (blk_thread) occurred — the reference's -v output as counts
 * (one count per kind of line and channel; the log itself is not produced).  Each field names its event:
 *   preamble            two SYN seen, waiting for SOH (acars.c:267-271)
 *   started             SOH accepted, a block is being assembled (acars.c:281-298)
 *   txt_parity          block abandoned: more than MAXPERR+1 bad bytes (acars.c:307-317, "too many parity errors")
 *   txt_long            block abandoned: over 240 bytes (acars.c:334-338, "too long")
 *   txt_missed_end      DLE after 20 bytes, emitted anyway (acars.c:324-332, "miss txt end")
 *   emitted             handed to the block FEC (acars.c:350-366, "put message")
 *   fec_short           shorter than 13 bytes (acars.c:124-129, "too short")
 *   fec_parity_excess   more than MAXPERR parity errors (acars.c:145-152, "too many parity errors: %d")
 *   fec_parity          1..MAXPERR parity errors (acars.c:153-155, "parity error(s)")
 *   fec_crc             CRC non-zero (acars.c:166-167, "crc error")
 *   fec_fixed           repaired (acars.c:177-178, 189-190, "errors fixed")
 *   fec_unfixable       not repairable (acars.c:172-173, 184-185, "not able to fix errors")
 *   fec_parity_problem  the final parity re-check failed (acars.c:202-206, "parity check problem")
 *   delivered           queued for acb_drain (outputmsg, acars.c:209)
 *   lost                found the device ring full (this chain's part of acb_stats_t.frames_lost)
 * Per chain, at any time:
 *   emitted   = fec_short + fec_parity_excess + fec_unfixable + fec_parity_problem + delivered + lost
 *   started   = emitted + txt_parity + txt_long + (1 while a block is open: Acarsstate TXT, CRC1 or CRC2)
 *   delivered = the messages acb_drain returns for the chain
 * (the second holds for chain states the context produced itself; acb_set_state can open or close a block). */
typedef struct {
	uint64_t preamble, started, txt_parity, txt_long, txt_missed_end, emitted;
	uint64_t fec_short, fec_parity_excess, fec_parity, fec_crc, fec_fixed, fec_unfixable, fec_parity_problem;
	uint64_t delivered, lost;
} acb_decode_stats_t;
/* Fills out[s*nch + c] for every chain; n >= nstreams*nch.  The counts cover exactly the submits acb_collect / acb_sync
 * have covered (the ones whose messages acb_drain returns); a submit abandoned by acb_reset contributes nothing, and
 * acb_reset clears the counts along with the undrained messages.  reset != 0 clears them after reading.  ACB_ERR_ARG
 * without ACB_FLAG_DECODE_STATS. */
int acb_get_decode_stats(acb_ctx_t *ctx, acb_decode_stats_t *out, size_t n, int reset);

/* Levels (ACB_FLAG_LEVEL_STATS): how loud each receiver's input is and whether its ADC clips, and how much power and
 * noise each channel's envelope carries — the receiver side of frames that were never started.
 *
 * Input, per stream.  The samples counted are, for every output row m a covered submit produced for the stream, the K
 * input samples [m*K, (m+1)*K): each sample exactly once, whatever the cuts (a streaming kind's carried remainder counts
 * when its row completes; the history of taps > K is not counted again).  A sample's components are converted as the
 * channelizer converts them: u8 (float)b - 127.37f, CS16 (float)int16, real the float itself.  A sample is clipped when
 * a component is full scale: u8 0 or 255, CS16 -32768 or 32767, real x <= -1 or x >= 2047/2048 (the end codes of a 12-bit
 * converter scaled (code - 2048)/2048).  The full-scale amplitude fs is 127.5 (u8), 32768 (CS16), 1.0 (real): the mean
 * power in dBFS is 10*log10(power_sum / samples / fs^2).  Ragged submits count each stream's own rows only; envelope
 * input (acb_submit_dm_host) leaves this table untouched. */
typedef struct {
	uint64_t samples;      /* input samples of the rows produced: rows * K (complex for u8 / CS16, real for real input) */
	uint64_t clipped;      /* samples with a full-scale component */
	double   power_sum;    /* sum over those samples of I^2 + Q^2 (real: x^2), converted as above */
	float    peak;         /* largest |component| of a converted sample (0 before any) */
	float    pad;
} acb_input_level_t;
/* Envelope, per chain, in the envelope's own units (the reference's scale).  Windows are the rows [1024*j, 1024*(j+1))
 * counted from the stream's own start (acb_create, acb_reset, acb_reset_stream); a window may span submits and counts for
 * the submit that completes it. */
typedef struct {
	uint64_t rows;         /* envelope samples */
	double   power_sum;    /* sum of dm^2 */
	float    peak;         /* largest dm (0 before any) */
	float    pad;
	uint64_t windows;      /* windows of 1024 rows completed */
	double   floor;        /* smallest window mean of dm^2 among them; 0 when windows == 0 */
} acb_chan_level_t;
/* Fills in[s] (n_in >= nstreams) and ch[s*nch + c] (n_ch >= nstreams*nch); either may be NULL.  The tables cover exactly
 * the submits acb_collect / acb_sync have covered; reset != 0 clears them after reading (an open window's partial sum is
 * kept, so the window alignment stays); acb_reset clears everything; acb_reset_stream clears that stream's rows and open
 * window, queued behind the work in flight, and no other stream's.  ACB_ERR_ARG without ACB_FLAG_LEVEL_STATS. */
int acb_get_level_stats(acb_ctx_t *ctx, acb_input_level_t *in, size_t n_in, acb_chan_level_t *ch, size_t n_ch, int reset);

/* Frequency error (ACB_FLAG_FREQ_STATS): how far each channel's AM carrier sits from the frequency the planner placed it
 * at, and so how far off frequency the receiver is tuned.
 *
 * Per chain (s, c), over the same rows the level tables count (every output row m a covered submit produced for stream
 * s, with its own K input samples [m*K, (m+1)*K), converted as acb_input_level_t documents; the taps > K history is not
 * used).  With h = K/2 (rounded down: an odd K leaves the row's last sample out) and w the chain's NCO table,
 *   a_m = sum_{n<h} x[mK+n] w[n],   b_m = sum_{n<h} x[mK+h+n] w[h+n],   w[n] = (float)cos(step n) - j (float)sin(step n),
 * a_m and b_m in float, the row's terms and the sums in double:
 *   pairs += 1,  s_re + j s_im += b_m conj(a_m),  mag_sum += |a_m| |b_m|,  power_sum += |a_m|^2 + |b_m|^2.
 * step is the offset, in radians per input sample, of the channel from the tuner centre that the chain's mixer removes:
 * 2 pi ((float)Fr - (float)Fc) / rate for the IQ planners (acb_set_plan*, acb_set_plan_cs16), and for real input the
 * mirror image of air.c's IF, -2 pi (Fc - Fr + rate/4) / rate, since the real front-end's IF is spectrally inverted.
 * Either way a carrier above freq_hz turns s positive (counter-clockwise) for every input kind.  freq_hz is the RF
 * frequency the mixer centres: Fc plus the IQ offset, or Fr for real input.  The planners record both for every chain;
 * a stream whose table came from acb_set_wf has freq_hz = step = 0 and is not measured (pairs stays 0).  A re-plan
 * takes effect for the rows after it.
 *
 * The offset of a chain is rate * atan2(s_im, s_re) / (2 pi h) Hz, with rate = K * 12500: unambiguous within
 * +-rate / (2h), +-12.5 kHz at even K; a carrier further out aliases by multiples of rate / h.  |s| / mag_sum is in
 * [0, 1]: near 1 for a chain with a carrier, near 0 for one with noise only.  The tables cover exactly the submits
 * acb_collect / acb_sync have covered; envelope input (acb_submit_dm_host) adds nothing. */
typedef struct {
	uint64_t pairs;        /* rows measured */
	double   s_re, s_im;   /* sum of b_m conj(a_m) */
	double   mag_sum;      /* sum of |a_m| |b_m| */
	double   power_sum;    /* sum of |a_m|^2 + |b_m|^2 */
	double   freq_hz;      /* the chain's planned RF frequency (0: not measured) */
	double   step;         /* the NCO's step, radians per input sample */
} acb_chan_freq_t;
/* Fills out[s*nch + c] for every chain; n >= nstreams*nch.  reset != 0 clears the sums after reading (freq_hz and step
 * describe the plan and stay); acb_reset clears every chain's sums, acb_reset_stream that stream's, queued behind the
 * work in flight.  ACB_ERR_ARG without ACB_FLAG_FREQ_STATS. */
int acb_get_freq_stats(acb_ctx_t *ctx, acb_chan_freq_t *out, size_t n, int reset);
/* The offsets, coherences and frequency error of one stream's nch chains (host only): offset_hz[c] and coherence[c] as
 * above (0 for a chain with pairs == 0), and *ppm = 1e6 * sum_c |s_c| offset_c / freq_hz_c / sum_c |s_c| over the chains
 * with pairs > 0 (0 when there is none).  Any output may be NULL.  K is the context's (the offset's scale is
 * K * 12500 / (2 pi floor(K/2))).  ACB_ERR_ARG for a NULL table, nch < 1 or K < 2. */
int acb_freq_error(const acb_chan_freq_t *ch, int nch, int K, double *offset_hz, double *coherence, double *ppm);

/* ---- one process, several GPUs (the C host's way to a whole node; SURVEY.md §8e) ----
 *
 * acb_multi_* fronts one context per device.  Two ways to cut the work, neither with any device-to-device
 * traffic (channels and streams share nothing):
 *   ACB_MULTI_SPLIT_STREAMS   device d serves a contiguous range of the streams (BASELINE config 4);
 *   ACB_MULTI_SPLIT_CHANNELS  every device sees every stream and serves a contiguous range of its channels
 *                             (one wide stream, configs 3/5); each device fetches the block over its own PCIe link.
 * Every input kind: u8 IQ (acb_multi_set_plan, acb_multi_submit_host), real input (cfg->flags ACB_FLAG_REAL_INPUT:
 * acb_multi_set_plan_air, acb_multi_submit_real_host) and CS16 (ACB_FLAG_CS16_INPUT: acb_multi_set_plan_cs16,
 * acb_multi_submit_cs16_host, acb_multi_submit_cs16_planar_host).  Each part is an ordinary context of cfg's kind and
 * flags, so it runs the kernels (fast and wideband forms included) a single context would; a submit of the wrong kind
 * is refused as the single-context call refuses it.  Arguments, return values and input lifetime are the single-context
 * calls'; in a channel split every part reads the whole input, in a stream split part p reads from stream s0(p).  The
 * planners choose the centre once over all channels of the stream and give it to every part.  The streaming submits
 * return the envelope samples produced, which every part must agree on (ACB_ERR_CUDA otherwise).
 * Stream / channel indices in the API and in the messages are global; messages are merged into the emission order one
 * context gives: u8 IQ (block, stream, channel, time; rtl.c:357-360), the streaming kinds (emission group, stream,
 * channel, time) with the groups of acb_multi_set_emission_groups (acb_set_emission_groups's units and rule), which the
 * multi-context tracks itself; acb_multi_reset restarts them with the parts.  cfg->device is ignored, `devices` names the
 * CUDA ordinals (repeats allowed: two contexts on one GPU).  ACB_MAXSTREAMS applies to each part: a stream split
 * accepts up to ndev * 65535 streams (the parts differ by at most one stream), a channel split 65535; a part over the
 * limit fails acb_multi_create with ACB_ERR_ARG.  Devices beyond the number of streams (channels) stay idle.
 * Input comes from the host only: a device pointer belongs to one GPU.  Several GPUs reading one wide stream from
 * device memory broadcast it and give each context its copy (acb_wait_event + the device submits; Python:
 * acarsdec_b200.wide.WideStream). */
typedef struct acb_multi acb_multi_t;
enum { ACB_MULTI_SPLIT_STREAMS = 0, ACB_MULTI_SPLIT_CHANNELS = 1 };
int  acb_multi_create(const acb_config_t *cfg, const int *devices, int ndev, int mode, acb_multi_t **out);
void acb_multi_destroy(acb_multi_t *m);
int  acb_multi_parts(acb_multi_t *m);                        /* number of per-device contexts */
acb_ctx_t *acb_multi_part(acb_multi_t *m, int i);            /* the i-th one (stats, inspection) */
int  acb_multi_set_plan(acb_multi_t *m, int stream, const unsigned *freqs_hz, int nch, unsigned *fc_out);
int  acb_multi_set_wf(acb_multi_t *m, int stream, const float *wf, int nch);
int  acb_multi_reset(acb_multi_t *m);
int  acb_multi_submit_host(acb_multi_t *m, const uint8_t *iq, size_t stream_stride, int nblk);
int  acb_multi_set_plan_air(acb_multi_t *m, int stream, const unsigned *freqs_hz, int nch, unsigned *fc_out);
int  acb_multi_set_plan_cs16(acb_multi_t *m, int stream, const unsigned *freqs_hz, int nch, int variant, unsigned fc_hz, unsigned *fc_out);
int  acb_multi_submit_real_host(acb_multi_t *m, const float *x, size_t stream_stride_samples, size_t nsamples);
int  acb_multi_submit_cs16_host(acb_multi_t *m, const int16_t *iq, size_t stream_stride_samples, size_t nsamples);
int  acb_multi_submit_cs16_planar_host(acb_multi_t *m, const int16_t *xi, const int16_t *xq, size_t stream_stride_samples, size_t nsamples);
/* The ragged forms (see acb_submit_host_ragged).  A stream split hands each part its streams' counts; a part whose counts
 * are all 0 sits the submit out.  A channel split hands every part all the counts, and the parts must agree on every
 * nout[s] (ACB_ERR_CUDA otherwise).  The counts are checked before any part reads anything. */
int  acb_multi_submit_host_ragged(acb_multi_t *m, const uint8_t *iq, size_t stream_stride, const int *nblk);
int  acb_multi_submit_real_host_ragged(acb_multi_t *m, const float *x, size_t stream_stride_samples, const size_t *nsamples, size_t *nout);
int  acb_multi_submit_cs16_host_ragged(acb_multi_t *m, const int16_t *iq, size_t stream_stride_samples, const size_t *nsamples,
                                       size_t *nout);
int  acb_multi_submit_cs16_planar_host_ragged(acb_multi_t *m, const int16_t *xi, const int16_t *xq, size_t stream_stride_samples,
                                              const size_t *nsamples, size_t *nout);
/* acb_reset_stream on the parts serving `stream`.  The submits in flight are collected first, as acb_multi_sync collects
 * them (their messages wait in the output queue): the merge tells a message's submit by its stream's position. */
int  acb_multi_reset_stream(acb_multi_t *m, int stream);
int  acb_multi_set_emission_groups(acb_multi_t *m, int unit, uint64_t period);
int  acb_multi_collect(acb_multi_t *m);
int  acb_multi_sync(acb_multi_t *m);
int  acb_multi_drain(acb_multi_t *m, acb_msg_t *out, int max);
int  acb_multi_get_state(acb_multi_t *m, int stream, int chn, acb_chan_state_t *out);
int  acb_multi_set_state(acb_multi_t *m, int stream, int chn, const acb_chan_state_t *in);
/* acb_get_decode_stats over the parts, indexed by global stream and channel: out[s*nch + c], n >= nstreams*nch */
int  acb_multi_get_decode_stats(acb_multi_t *m, acb_decode_stats_t *out, size_t n, int reset);
/* acb_get_level_stats over the parts, indexed globally.  A stream split takes each part's streams.  In a channel split
 * every part reads the same samples, so in[] comes from part 0; ch[] from each part's channels. */
int  acb_multi_get_level_stats(acb_multi_t *m, acb_input_level_t *in, size_t n_in, acb_chan_level_t *ch, size_t n_ch, int reset);
/* acb_get_freq_stats over the parts, indexed by global stream and channel: out[s*nch + c], n >= nstreams*nch */
int  acb_multi_get_freq_stats(acb_multi_t *m, acb_chan_freq_t *out, size_t n, int reset);
/* acb_save_streams / acb_load_streams over the parts.  A blob is the one a single context of cfg would give, whatever the
 * split, so streams move freely between single contexts, stream splits and channel splits.  A stream split takes each
 * stream's record from (gives it to) the part that owns it.  A channel split assembles each stream's nch chains, tables
 * and counts from the parts' channels, and the input side and input levels from part 0 (every part reads the same
 * samples); a stream is on the raster only when every part's channels are.  The envelope level sums of a channel split
 * (acb_chan_level_t power_sum and floor, and the open windows' sums) follow its parts' channel tiling, as
 * acb_multi_get_level_stats's do: within 1e-10 relative of a single context's, everything else bit for bit.  Load checks
 * every part's share before any
 * part changes, collects the submits in flight first (as acb_multi_reset_stream) and sets each stream's position to
 * the blob's. */
size_t acb_multi_streams_blob_bytes(acb_multi_t *m, int n);
int  acb_multi_save_streams(acb_multi_t *m, const int *streams, int n, void *blob, size_t cap);
int  acb_multi_load_streams(acb_multi_t *m, const int *streams, int n, const void *blob, size_t size);

/* Block FEC on one frame in place on the HOST (acars.c:123-207): 1 = deliver, 0 = drop.  The
 * processing path runs the same repair on the device (k_block_fec, one thread per frame, right
 * behind the demod); this entry serves the shim's host-side decodeAcars and callers with their own
 * queue. */
int acb_block_fec(acb_msg_t *m);
/* The device block FEC on a batch of raw frames (len, txt with parity bits, crc): repairs msgs[i]
 * in place, keep[i] = 1 where the reference would call outputmsg().  Returns the number kept. */
int acb_block_fec_batch(acb_ctx_t *ctx, acb_msg_t *msgs, int n, int *keep);
/* Tables behind it, generated rather than stored (syndrom.h:4-13, 15-49, 52-295). */
uint16_t acb_crc_update(uint16_t crc, uint8_t c);
uint16_t acb_syndrome(int index);      /* index = bit + 8*bytes_from_end, 0..1935 */

/* The bit/byte frame synchroniser (decodeAcars, acars.c:246-375) as a host call, over caller-owned
 * state: the same definition (csrc/frame_sm.h) the demod kernel runs per channel on the device.
 * Used by the compat shim's decodeAcars(channel_t*).  Integer-only. */
typedef struct {
	int *state, *nbits, *bitcount, *blk_len, *blk_err;
	unsigned *msk_s;
	double *msk_df, *lvlsum;
	unsigned char *txt;                 /* >= 250 bytes */
	unsigned char *crc;                 /* 2 bytes */
	int (*frame_begin)(void *user);     /* SOH seen; return 0 to refuse (no storage) */
	void (*frame_emit)(void *user);     /* frame complete */
	void *user;
} acb_frame_view_t;
void acb_frame_byte(acb_frame_view_t *v, unsigned char r);

#ifdef __cplusplus
}
#endif
#endif
