/*
 * libacarsdec_compat — the reference's own symbols for the hot path, as a thin shim over the
 * context API of libacars_b200 (include/acars_b200.h).  acarsdec.c and the untouched front-ends
 * link against this instead of msk.c + acars.c (+ rtl.c and librtlsdr).
 *
 *   initMsk / demodMSK             msk.c:30, msk.c:67      -> one-channel GPU context, stateless calls
 *   initAcars / decodeAcars /      acars.c:218, 246, 378   -> consumer thread feeding outputmsg();
 *   deinitAcars                                               the host-side frame sync entry
 *   initRtl / runRtlSample /       rtl.c:193, 371, 406,413 -> nbch-channel GPU context fed from a
 *   runRtlCancel / runRtlClose                                raw u8 IQ capture instead of a dongle
 *
 * channel_t stays the carrier of all per-channel state, exactly like in the reference: demodMSK
 * uploads it, runs the CUDA demodulator over ch->dm_buffer and writes the new state back, so any
 * chunking of the stream gives the same result and the host may inspect or reset the fields.
 * The RTL path keeps the state resident on the device between blocks (that is the fast path) and
 * writes it back to channel[] when the run ends.
 *
 * Build with the same WITH_* macros as the host (channel_t's layout depends on them,
 * acarsdec.h:62-74) and, to use the host's real header, -DACB_USE_REFERENCE_HEADER -I<acarsdec>.
 */
#define _GNU_SOURCE
#include <errno.h>
#include <math.h>
#include <pthread.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/time.h>
#include <unistd.h>

#include "../../include/acarsdec_compat.h"
#include "../../include/acars_b200.h"

#define FLEN 11                 /* msk.c:25 */
#define RTLOUTBUFSZ 1024        /* rtl.c:49 */
#define RTLMULTMAX 320          /* rtl.c:39 */

/* ---------------------------------------------------------------- output queue + consumer */

static pthread_mutex_t q_mtx = PTHREAD_MUTEX_INITIALIZER;
static pthread_cond_t q_cnd = PTHREAD_COND_INITIALIZER;
static msgblk_t *q_head, *q_tail;      /* FIFO through ->prev, like acars.c:30-33 */
static pthread_t q_thread;
static int q_running, q_shutdown;

static void *consumer(void *arg)
{
	(void)arg;
	for (;;) {
		pthread_mutex_lock(&q_mtx);
		while (!q_head && !q_shutdown) pthread_cond_wait(&q_cnd, &q_mtx);
		msgblk_t *b = q_head;
		if (!b) {                       /* shutdown and empty */
			pthread_mutex_unlock(&q_mtx);
			return NULL;
		}
		q_head = b->prev;
		if (!q_head) q_tail = NULL;
		pthread_mutex_unlock(&q_mtx);
		outputmsg(b);                   /* acars.c:209 */
		free(b);
	}
}

static void q_push(msgblk_t *b)
{
	pthread_mutex_lock(&q_mtx);
	b->prev = NULL;
	if (q_tail) q_tail->prev = b; else q_head = b;
	q_tail = b;
	pthread_cond_signal(&q_cnd);
	pthread_mutex_unlock(&q_mtx);
}

/* Wall-clock time of an envelope sample.  The reference stamps a block with gettimeofday() when its loop reaches
 * the SOH byte (acars.c:290), i.e. when the transfer holding that sample is processed.  The shim processes
 * batches of transfers, so it stamps every batch when its input has been read and places a sample inside its
 * batch at the stream's own rate (12.5 kS/s per channel): the last sample of a batch arrived at the stamp. */
#define NSTAMP 8
static struct { uint64_t end_pos; struct timeval tv; } stamps[NSTAMP];
static unsigned nstamps;

static void stamp_reset(void) { nstamps = 0; }

static void stamp_batch(uint64_t end_pos)
{
	gettimeofday(&stamps[nstamps % NSTAMP].tv, NULL);
	stamps[nstamps % NSTAMP].end_pos = end_pos;
	nstamps++;
}

static struct timeval stamp_time(uint64_t pos)
{
	struct timeval tv;
	if (nstamps == 0) { gettimeofday(&tv, NULL); return tv; }
	unsigned first = nstamps > NSTAMP ? nstamps - NSTAMP : 0, pick = nstamps - 1;
	for (unsigned i = first; i < nstamps; i++)
		if (stamps[i % NSTAMP].end_pos > pos) { pick = i; break; }
	const uint64_t end = stamps[pick % NSTAMP].end_pos;
	tv = stamps[pick % NSTAMP].tv;
	if (end > pos + 1) {
		const uint64_t us = (end - 1 - pos) * 1000000ull / INTRATE;
		const long long t = (long long)tv.tv_sec * 1000000ll + tv.tv_usec - (long long)us;
		tv.tv_sec = (time_t)(t / 1000000ll);
		tv.tv_usec = (suseconds_t)(t % 1000000ll);
	}
	return tv;
}

/* a repaired block from the library -> msgblk_t on the consumer queue */
static void deliver(const acb_msg_t *m, int chn, const struct timeval *tv)
{
	msgblk_t *b = calloc(1, sizeof(*b));
	if (!b) return;
	b->chn = chn;
	b->tv = *tv;
	b->len = m->len;
	b->err = m->err;
	b->lvl = m->lvl;
	memcpy(b->txt, m->txt, sizeof(b->txt));
	b->crc[0] = m->crc[0];
	b->crc[1] = m->crc[1];
	q_push(b);
}

/* everything the library has queued -> the consumer, stamped with the time of its SOH sample */
static void deliver_ready(acb_multi_t *m) __attribute__((unused));
static void deliver_ready(acb_multi_t *m)
{
	acb_msg_t out[16];
	for (int n; (n = acb_multi_drain(m, out, 16)) > 0;)
		for (int i = 0; i < n; i++) {
			const struct timeval tv = stamp_time(out[i].soh_pos);      /* acars.c:290 */
			deliver(&out[i], out[i].chn, &tv);
		}
}

/* The front-ends serve one stream with nbch channels: on one GPU, or with ACARSDEC_B200_DEVICES=0,1,... the channels
 * split over several (acb_multi_*, channel-split mode): the unmodified C host reaches a whole node this way.  Without
 * the list, ACARSDEC_B200_DEVICE names the one device (default 0). */
static int parse_devices(int *dev, int max) __attribute__((unused));
static int parse_devices(int *dev, int max)
{
	const char *e = getenv("ACARSDEC_B200_DEVICES");
	int n = 0;
	if (e && *e) {
		char *dup = strdup(e), *save = NULL;
		for (char *t = strtok_r(dup, ",", &save); t && n < max; t = strtok_r(NULL, ",", &save)) dev[n++] = atoi(t);
		free(dup);
	}
	if (n == 0) {
		e = getenv("ACARSDEC_B200_DEVICE");
		dev[n++] = e ? atoi(e) : 0;
	}
	return n;
}

/* one stream, nbch channels, split over the devices parse_devices names */
static acb_multi_t *front_end_create(acb_config_t *cfg) __attribute__((unused));
static acb_multi_t *front_end_create(acb_config_t *cfg)
{
	int devs[MAXNBCHANNELS];
	const int ndev = parse_devices(devs, MAXNBCHANNELS);
	acb_multi_t *m = NULL;
	if (acb_multi_create(cfg, devs, ndev, ACB_MULTI_SPLIT_CHANNELS, &m) != ACB_OK) {
		fprintf(stderr, "acarsdec_b200: %s\n", acb_last_error());
		if (m) acb_multi_destroy(m);
		return NULL;
	}
	return m;
}

/* ---------------------------------------------------------------- initAcars / deinitAcars */

int initAcars(channel_t *ch)
{
	if (ch->chn == 0 && !q_running) {          /* acars.c:220-228 */
		q_shutdown = 0;
		q_head = q_tail = NULL;
		if (pthread_create(&q_thread, NULL, consumer, NULL)) return -1;
		q_running = 1;
	}
	ch->outbits = 0;                            /* acars.c:230-234 */
	ch->nbits = 8;
	ch->Acarsstate = WSYN;
	ch->blk = NULL;
	return 0;
}

int deinitAcars(void)
{
	if (!q_running) return 0;
	pthread_mutex_lock(&q_mtx);
	q_shutdown = 1;
	pthread_cond_signal(&q_cnd);
	pthread_mutex_unlock(&q_mtx);
	pthread_join(q_thread, NULL);
	q_running = 0;
	return 0;
}

/* ---------------------------------------------------------------- decodeAcars on the host */

static int view_begin(void *u)
{
	channel_t *ch = u;
	if (!ch->blk) ch->blk = malloc(sizeof(msgblk_t));      /* acars.c:283-289 */
	if (!ch->blk) return 0;
	gettimeofday(&ch->blk->tv, NULL);
	ch->blk->chn = ch->chn;
	return 1;
}

static void view_emit(void *u)
{
	channel_t *ch = u;
	acb_msg_t m;
	memset(&m, 0, sizeof(m));
	m.chn = ch->chn;
	m.len = ch->blk->len;
	m.err = ch->blk->err;
	m.lvl = (float)(10 * log10(ch->MskLvlSum / ch->MskBitCount));    /* acars.c:351 */
	memcpy(m.txt, ch->blk->txt, sizeof(ch->blk->txt));
	m.crc[0] = ch->blk->crc[0];
	m.crc[1] = ch->blk->crc[1];
	if (acb_block_fec(&m)) deliver(&m, ch->chn, &ch->blk->tv);      /* blk_thread, acars.c:123-209 */
	free(ch->blk);
	ch->blk = NULL;
}

/* acars.c:246 — the byte-level state machine on host-side state.  The GPU demodulator runs the
 * same definition per channel on the device; this entry exists for API completeness (a host that
 * assembles bits itself). */
void decodeAcars(channel_t *ch)
{
	static __thread unsigned char scratch_txt[256], scratch_crc[2];
	int st = (int)ch->Acarsstate, no_len = 0, no_err = 0;
	acb_frame_view_t v;
	if (st == SOH1 && ch->outbits == 0x01 && !view_begin(ch)) {   /* acars.c:285-288: no memory */
		ch->Acarsstate = WSYN; ch->MskDf = 0; ch->nbits = 1;
		return;
	}
	v.state = &st; v.nbits = &ch->nbits; v.bitcount = &ch->MskBitCount;
	v.msk_s = &ch->MskS; v.msk_df = &ch->MskDf; v.lvlsum = &ch->MskLvlSum;
	v.blk_len = ch->blk ? &ch->blk->len : &no_len;
	v.blk_err = ch->blk ? &ch->blk->err : &no_err;
	v.txt = ch->blk ? (unsigned char *)ch->blk->txt : scratch_txt;
	v.crc = ch->blk ? ch->blk->crc : scratch_crc;
	v.frame_begin = view_begin; v.frame_emit = view_emit; v.user = ch;
	acb_frame_byte(&v, ch->outbits);
	ch->Acarsstate = st;
}

/* ---------------------------------------------------------------- initMsk / demodMSK */

static acb_ctx_t *one_ctx;          /* 1 stream x 1 channel, envelope input */
static pthread_mutex_t one_mtx = PTHREAD_MUTEX_INITIALIZER;
#define ONE_MAXBLK 4                /* 4096 samples per launch: soundfile.c's MAXNBFRAMES */

static int one_ctx_get(void)
{
	if (one_ctx) return 0;
	acb_config_t cfg = { 0, 160, 1, 1, ONE_MAXBLK, ACB_FLAG_NO_INPUT_STAGING, 0 };
	const char *dev = getenv("ACARSDEC_B200_DEVICE");
	if (dev) cfg.device = atoi(dev);
	if (acb_create(&cfg, &one_ctx) != ACB_OK) {
		fprintf(stderr, "acarsdec_b200: %s\n", acb_last_error());
		if (one_ctx) acb_destroy(one_ctx);
		one_ctx = NULL;
		return -1;
	}
	return 0;
}

int initMsk(channel_t *ch)
{
	ch->MskPhi = ch->MskClk = 0;            /* msk.c:34-40 */
	ch->MskS = 0;
	ch->MskDf = 0;
	ch->idx = 0;
	ch->inb = calloc(FLEN, sizeof(float complex));
	if (ch->inb == NULL) return -1;
	pthread_mutex_lock(&one_mtx);
	int r = one_ctx_get();                  /* fails loudly when there is no H100: no CPU fallback */
	pthread_mutex_unlock(&one_mtx);
	return r;
}

static void state_pack(const channel_t *ch, acb_chan_state_t *s)
{
	memset(s, 0, sizeof(*s));
	s->MskPhi = ch->MskPhi; s->MskDf = ch->MskDf; s->MskLvlSum = ch->MskLvlSum; s->MskClk = ch->MskClk;
	s->MskBitCount = ch->MskBitCount; s->MskS = ch->MskS; s->idx = ch->idx;
	s->nbits = ch->nbits; s->Acarsstate = (int)ch->Acarsstate; s->outbits = ch->outbits;
	for (int i = 0; i < FLEN; i++) { s->inb_re[i] = crealf(ch->inb[i]); s->inb_im[i] = cimagf(ch->inb[i]); }
	if (ch->blk) {
		s->blk_len = ch->blk->len; s->blk_err = ch->blk->err;
		memcpy(s->blk_txt, ch->blk->txt, sizeof(ch->blk->txt));
		s->blk_crc[0] = ch->blk->crc[0]; s->blk_crc[1] = ch->blk->crc[1];
	}
}

static void state_unpack(const acb_chan_state_t *s, channel_t *ch)
{
	ch->MskPhi = s->MskPhi; ch->MskDf = s->MskDf; ch->MskLvlSum = s->MskLvlSum; ch->MskClk = s->MskClk;
	ch->MskBitCount = s->MskBitCount; ch->MskS = s->MskS; ch->idx = s->idx;
	ch->nbits = s->nbits; ch->Acarsstate = s->Acarsstate; ch->outbits = (unsigned char)s->outbits;
	for (int i = 0; i < FLEN; i++) ch->inb[i] = s->inb_re[i] + s->inb_im[i] * I;
	if (s->Acarsstate >= TXT && s->Acarsstate <= CRC2) {      /* a frame is being assembled */
		if (!ch->blk) {
			ch->blk = calloc(1, sizeof(msgblk_t));
			if (ch->blk) { gettimeofday(&ch->blk->tv, NULL); ch->blk->chn = ch->chn; }
		}
		if (ch->blk) {
			ch->blk->len = s->blk_len; ch->blk->err = s->blk_err;
			memcpy(ch->blk->txt, s->blk_txt, sizeof(ch->blk->txt));
			ch->blk->crc[0] = s->blk_crc[0]; ch->blk->crc[1] = s->blk_crc[1];
		}
	}
}

void demodMSK(channel_t *ch, int len)
{
	struct timeval now;
	acb_chan_state_t st;
	acb_msg_t out[8];
	pthread_mutex_lock(&one_mtx);
	if (one_ctx_get()) { pthread_mutex_unlock(&one_mtx); return; }
	gettimeofday(&now, NULL);
	state_pack(ch, &st);
	int rc = acb_set_state(one_ctx, 0, 0, &st);
	for (int off = 0; rc == ACB_OK && off < len; off += ONE_MAXBLK * RTLOUTBUFSZ) {
		int n = len - off < ONE_MAXBLK * RTLOUTBUFSZ ? len - off : ONE_MAXBLK * RTLOUTBUFSZ;
		rc = acb_submit_dm_host(one_ctx, ch->dm_buffer + off, n);
		if (rc == ACB_OK) rc = acb_sync(one_ctx);
		if (rc > 0) rc = ACB_OK;
	}
	if (rc == ACB_OK) rc = acb_get_state(one_ctx, 0, 0, &st);
	if (rc != ACB_OK) {
		fprintf(stderr, "acarsdec_b200: demodMSK: %s\n", acb_last_error());
		pthread_mutex_unlock(&one_mtx);
		return;
	}
	int had_blk = ch->blk != NULL;
	struct timeval tv = had_blk ? ch->blk->tv : now;
	state_unpack(&st, ch);
	if (!(st.Acarsstate >= TXT && st.Acarsstate <= CRC2) && ch->blk) {   /* frame finished or dropped */
		free(ch->blk);
		ch->blk = NULL;
	}
	for (int n; (n = acb_drain(one_ctx, out, 8)) > 0;)
		for (int i = 0; i < n; i++) deliver(&out[i], ch->chn, &tv);
	pthread_mutex_unlock(&one_mtx);
}

/* ACARSDEC_B200_TAPS=<n>: the channel filter length of every front-end (acb_config_t.taps).  Unset, or n == K: the
 * reference's boxcar; K < n <= ACB_MAXTAPS_PER_K*K: the planner's low-pass over an overlapping window
 * (acb_build_lowpass), which keeps a strong neighbour channel out of a weak one.  Anything else is an init error. */
static int env_taps(int K, int *taps)
{
	const char *e = getenv("ACARSDEC_B200_TAPS");
	*taps = 0;
	if (!e || !*e) return 0;
	char *end;
	const long v = strtol(e, &end, 10);
	if (*end || v < K || v > (long)ACB_MAXTAPS_PER_K * K) {
		fprintf(stderr, "acarsdec_b200: ACARSDEC_B200_TAPS=%s: need a number of taps from %d (the reference's boxcar) to %d\n",
		        e, K, ACB_MAXTAPS_PER_K * K);
		return -1;
	}
	*taps = v == K ? 0 : (int)v;
	return 0;
}

/* ---------------------------------------------------------------- RTL front-end on a capture file */

#ifdef WITH_RTL

static acb_multi_t *rtl_ctx;
static FILE *rtl_src;

static int rtl_batch = 16;              /* blocks per submit; ACARSDEC_B200_BLOCKS */
static volatile int rtl_cancel;
static size_t rtl_inbufsize;

int initRtl(char **argv, int optind)
{
	unsigned Fd[MAXNBCHANNELS];
	char *argF;
	if (argv[optind] == NULL) {
		fprintf(stderr, "Need a raw u8 IQ capture file (or - for stdin) after -r\n");
		exit(1);
	}
	const char *path = argv[optind++];
	if (rtlMult > RTLMULTMAX || rtlMult < 1) {          /* rtl.c:208-211 */
		fprintf(stderr, "rtlMult can't be larger than 360\n");
		return 1;
	}
	rtl_inbufsize = (size_t)RTLOUTBUFSZ * rtlMult * 2;   /* rtl.c:213 */
	rtl_src = strcmp(path, "-") ? fopen(path, "rb") : stdin;
	if (!rtl_src) {
		fprintf(stderr, "Failed to open IQ capture %s: %s\n", path, strerror(errno));
		return -1;
	}
	nbch = 0;
	while ((argF = argv[optind]) && nbch < MAXNBCHANNELS) {      /* rtl.c:243-257 */
		Fd[nbch] = (unsigned)acb_round_freq(atof(argF));
		optind++;
		if (Fd[nbch] < 118000000 || Fd[nbch] > 138000000) {
			fprintf(stderr, "WARNING: Invalid frequency %d\n", Fd[nbch]);
			continue;
		}
		channel[nbch].chn = nbch;
		channel[nbch].Fr = acb_stored_fr(Fd[nbch]);
		nbch++;
	}
	if (nbch == 0) {
		fprintf(stderr, "Need a least one frequency\n");
		return 1;
	}
	unsigned Fc = acb_choose_fc(Fd, nbch, rtlMult);              /* rtl.c:268-270 */
	if (Fc == 0) {
		fprintf(stderr, "Frequencies too far apart\n");
		return 1;
	}
	const char *e = getenv("ACARSDEC_B200_BLOCKS");
	if (e && atoi(e) > 0) rtl_batch = atoi(e);
	acb_config_t cfg = { 0, rtlMult, 1, (int)nbch, rtl_batch, 0, 0 };
	if (env_taps(rtlMult, &cfg.taps)) return 1;
	if (!(rtl_ctx = front_end_create(&cfg))) return 1;
	float *wf = malloc(sizeof(float) * 2 * rtlMult * nbch);
	if (!wf) return 1;
	for (unsigned n = 0; n < nbch; n++) {                        /* rtl.c:272-287 */
		channel_t *ch = &channel[n];
		ch->wf = malloc(rtlMult * sizeof(float complex));
		ch->dm_buffer = malloc(RTLOUTBUFSZ * sizeof(float));
		if (ch->wf == NULL || ch->dm_buffer == NULL) {
			fprintf(stderr, "ERROR : malloc\n");
			return 1;
		}
		acb_build_wf(ch->Fr, Fc, rtlMult, wf + (size_t)n * 2 * rtlMult);
		for (int i = 0; i < rtlMult; i++)
			ch->wf[i] = wf[((size_t)n * rtlMult + i) * 2] + wf[((size_t)n * rtlMult + i) * 2 + 1] * I;
	}
	/* channel[].wf keeps the reference's K-entry table either way; with a longer filter the library plans its own */
	int rc = cfg.taps ? acb_multi_set_plan(rtl_ctx, 0, Fd, (int)nbch, NULL) : acb_multi_set_wf(rtl_ctx, 0, wf, (int)nbch);
	free(wf);
	if (rc != ACB_OK) {
		fprintf(stderr, "acarsdec_b200: %s\n", acb_last_error());
		return 1;
	}
	if (verbose) fprintf(stderr, "Set center freq. to %dHz\n", (int)Fc);
	fprintf(stderr, "Setting sample rate: %.4f MS/s\n", INTRATE * rtlMult / 1e6);    /* rtl.c:298 */
	return 0;
}

int runRtlSample(void)
{
	if (!rtl_ctx || !rtl_src) return 1;
	uint8_t *buf[2];
	for (int i = 0; i < 2; i++) {
		buf[i] = acb_host_alloc(rtl_inbufsize * rtl_batch);
		if (!buf[i]) { fprintf(stderr, "acarsdec_b200: %s\n", acb_last_error()); return 1; }
	}
	/* demodulator state as the host initialised it (initMsk/initAcars) goes to the device */
	acb_chan_state_t st;
	for (unsigned n = 0; n < nbch; n++) {
		state_pack(&channel[n], &st);
		acb_multi_set_state(rtl_ctx, 0, (int)n, &st);
	}
	int which = 0, rc = ACB_OK, inflight = 0;
	uint64_t pos = 0;
	stamp_reset();
	while (!signalExit && !rtl_cancel) {
		if (inflight == 2) {
			/* buf[which] was the source of the submit two back: it must have been consumed */
			rc = acb_multi_collect(rtl_ctx);
			if (rc < 0) break;
			inflight--;
			deliver_ready(rtl_ctx);
		}
		size_t got = fread(buf[which], 1, rtl_inbufsize * rtl_batch, rtl_src);
		int nblk = (int)(got / rtl_inbufsize);
		if (got % rtl_inbufsize) fprintf(stderr, "warning: partial read\n");     /* rtl.c:322-326 */
		if (nblk == 0) break;
		pos += (uint64_t)nblk * RTLOUTBUFSZ;
		stamp_batch(pos);
		rc = acb_multi_submit_host(rtl_ctx, buf[which], rtl_inbufsize * nblk, nblk);
		if (rc != ACB_OK) break;
		which ^= 1;
		inflight++;
		if (nblk < rtl_batch) break;
	}
	if (rc >= 0) rc = acb_multi_sync(rtl_ctx);
	if (rc < 0) fprintf(stderr, "acarsdec_b200: %s\n", acb_last_error());
	deliver_ready(rtl_ctx);
	for (unsigned n = 0; n < nbch; n++)
		if (acb_multi_get_state(rtl_ctx, 0, (int)n, &st) == ACB_OK) state_unpack(&st, &channel[n]);
	for (int i = 0; i < 2; i++) acb_host_free(buf[i]);
	signalExit = 1;                                     /* rtl.c:366: the reader thread ended */
	return rc < 0 ? 1 : 0;
}

int runRtlCancel(void)
{
	rtl_cancel = 1;
	return 0;
}

int runRtlClose(void)
{
	if (rtl_ctx) { acb_multi_destroy(rtl_ctx); rtl_ctx = NULL; }
	if (rtl_src && rtl_src != stdin) fclose(rtl_src);
	rtl_src = NULL;
	return 0;
}

#endif /* WITH_RTL */

/* ---------------------------------------------------------------- Airspy front-end on a capture file */

#ifdef WITH_AIR

static acb_multi_t *air_ctx;
static FILE *air_src;
static unsigned air_rate, air_mult;
static volatile int air_cancel;
#define AIR_TRANSFER 65536          /* samples per read: libairspy's float32-real transfer size */

/* air.c:66 initAirspy — argv[optind] names a raw float32 capture of REAL samples (what libairspy
 * delivers with AIRSPY_SAMPLE_FLOAT32_REAL); its rate comes from ACARSDEC_B200_AIRRATE (default
 * 2500000; the reference takes the first device rate <= 10 MS/s that is a multiple of 12500). */
int initAirspy(char **argv, int optind)
{
	unsigned Fd[MAXNBCHANNELS];
	char *argF;
	if (argv[optind] == NULL) { fprintf(stderr, "Need a float32 capture file after -s\n"); return -1; }
	const char *path = argv[optind++];
	const char *e = getenv("ACARSDEC_B200_AIRRATE");
	air_rate = e ? (unsigned)atoi(e) : 2500000u;
	air_mult = air_rate / INTRATE;
	if (air_rate > 10000000 || air_mult * INTRATE != air_rate) {          /* air.c:211-216 */
		fprintf(stderr, "did not find needed sampling rate\n");
		return -1;
	}
	air_src = strcmp(path, "-") ? fopen(path, "rb") : stdin;
	if (!air_src) { fprintf(stderr, "Failed to open capture %s: %s\n", path, strerror(errno)); return -1; }
	nbch = 0;
	while ((argF = argv[optind]) && nbch < MAXNBCHANNELS) {               /* air.c:165-183 */
		Fd[nbch] = (unsigned)acb_round_freq(atof(argF));
		optind++;
		if (Fd[nbch] < 118000000 || Fd[nbch] > 138000000) {
			fprintf(stderr, "WARNING: Invalid frequency %d\n", Fd[nbch]);
			continue;
		}
		channel[nbch].chn = nbch;
		channel[nbch].Fr = (int)Fd[nbch];
		nbch++;
	}
	if (nbch == 0) { fprintf(stderr, "Need a least one frequency\n"); return 1; }
	if (air_rate == 5000000) { fprintf(stderr, "5 MS/s needs the R820T IF filter path (air.c:47-61): not available on a capture\n"); return 1; }
	unsigned lo = Fd[0], hi = Fd[0];
	for (unsigned n = 1; n < nbch; n++) { if (Fd[n] < lo) lo = Fd[n]; if (Fd[n] > hi) hi = Fd[n]; }
	const unsigned Fc = acb_air_choose_fc(lo, hi);
	if (Fc == 0) { fprintf(stderr, "Frequencies too far apart\n"); return 1; }
	if (verbose) fprintf(stderr, "Using %d sampling rate\nSet freq. to %d hz\n", air_rate, Fc);
	const int maxblk = (AIR_TRANSFER * 8 / (int)air_mult) / RTLOUTBUFSZ + 2;
	acb_config_t cfg = { 0, (int)air_mult, 1, (int)nbch, maxblk, ACB_FLAG_REAL_INPUT, 0 };
	if (env_taps((int)air_mult, &cfg.taps)) return -1;
	if (!(air_ctx = front_end_create(&cfg))) return -1;
	float *wf = malloc(sizeof(float) * 2 * air_mult * nbch);
	if (!wf) return -1;
	for (unsigned n = 0; n < nbch; n++) {                                 /* air.c:263-285 */
		channel_t *ch = &channel[n];
		ch->wf = malloc(air_mult * sizeof(float complex));
		ch->dm_buffer = malloc(512 * sizeof(double));
		if (ch->wf == NULL || ch->dm_buffer == NULL) { fprintf(stderr, "malloc error\n"); return -1; }
		ch->D = 0;
		acb_air_build_wf(ch->Fr, (int)Fc, air_rate, wf + (size_t)n * 2 * air_mult);
		for (unsigned i = 0; i < air_mult; i++)
			ch->wf[i] = wf[((size_t)n * air_mult + i) * 2] + wf[((size_t)n * air_mult + i) * 2 + 1] * I;
	}
	int rc = cfg.taps ? acb_multi_set_plan_air(air_ctx, 0, Fd, (int)nbch, NULL) : acb_multi_set_wf(air_ctx, 0, wf, (int)nbch);
	free(wf);
	if (rc != ACB_OK) { fprintf(stderr, "acarsdec_b200: %s\n", acb_last_error()); return -1; }
	return 0;
}

/* air.c:344 runAirspySample — batches of 8 transfers per submit, two pinned buffers so that reading batch i+1
 * overlaps the device work of batch i; any length is fine, the library carries what does not fill an output
 * row (the reference carries ch->D / ind).  Frames are queued in the reference's order: per 65536-sample
 * transfer, channel by channel (air.c:336). */
int runAirspySample(void)
{
	if (!air_ctx || !air_src) return -1;
	const size_t cap = (size_t)AIR_TRANSFER * 8;
	float *buf[2] = { acb_host_alloc(cap * sizeof(float)), acb_host_alloc(cap * sizeof(float)) };
	if (!buf[0] || !buf[1]) { fprintf(stderr, "acarsdec_b200: %s\n", acb_last_error()); return -1; }
	acb_chan_state_t st;
	for (unsigned n = 0; n < nbch; n++) { state_pack(&channel[n], &st); acb_multi_set_state(air_ctx, 0, (int)n, &st); }
	acb_multi_set_emission_groups(air_ctx, ACB_GROUP_INPUT, AIR_TRANSFER);
	int rc = ACB_OK, which = 0, inflight = 0;
	uint64_t pos = 0;
	stamp_reset();
	while (!signalExit && !air_cancel) {
		if (inflight == 2) {                 /* buf[which] fed the submit two back: it has been consumed */
			rc = acb_multi_collect(air_ctx);
			if (rc < 0) break;
			inflight--;
			deliver_ready(air_ctx);
		}
		size_t got = fread(buf[which], sizeof(float), cap, air_src);
		if (got == 0) break;
		rc = acb_multi_submit_real_host(air_ctx, buf[which], got, got);
		if (rc < 0) break;
		if (rc > 0) { pos += (uint64_t)rc; inflight++; which ^= 1; }
		else if ((rc = acb_multi_sync(air_ctx)) < 0) break;             /* fewer samples than one output row: copy done before reuse */
		else inflight = 0;
		stamp_batch(pos);
		if (got < cap) break;
	}
	if (rc >= 0) rc = acb_multi_sync(air_ctx);
	if (rc < 0) fprintf(stderr, "acarsdec_b200: %s\n", acb_last_error());
	deliver_ready(air_ctx);
	for (unsigned n = 0; n < nbch; n++)
		if (acb_multi_get_state(air_ctx, 0, (int)n, &st) == ACB_OK) state_unpack(&st, &channel[n]);
	acb_host_free(buf[0]);
	acb_host_free(buf[1]);
	acb_multi_destroy(air_ctx);
	air_ctx = NULL;
	return rc < 0 ? -1 : 0;
}

#endif /* WITH_AIR */

/* ---------------------------------------------------------------- CS16 front-ends on a capture file */

#if defined(WITH_SOAPY) || defined(WITH_SDRPLAY)

static acb_multi_t *cs_ctx;
static FILE *cs_src;
static int cs_mult;
#define CS_BATCH 8                  /* blocks of 1024*mult complex samples per submit */

/* the channel part shared by initSoapy (soapy.c:112-163) and initSdrplay (sdrplay.c:95-138) */
static int cs16_setup(const char *path, char **argv, int optind, int mult, int variant, unsigned fc_user, const char *range_fmt)
{
	unsigned Fd[MAXNBCHANNELS];
	char *argF;
	cs_mult = mult;
	cs_src = strcmp(path, "-") ? fopen(path, "rb") : stdin;
	if (!cs_src) { fprintf(stderr, "Failed to open CS16 capture %s: %s\n", path, strerror(errno)); return -1; }
	nbch = 0;
	while ((argF = argv[optind]) && nbch < MAXNBCHANNELS) {
		Fd[nbch] = (unsigned)acb_round_freq(atof(argF));
		optind++;
		if (Fd[nbch] < 118000000 || Fd[nbch] > 138000000) {
			fprintf(stderr, range_fmt, Fd[nbch]);
			continue;
		}
		channel[nbch].chn = nbch;
		channel[nbch].Fr = (float)Fd[nbch];
		nbch++;
	}
	if (nbch == 0) { fprintf(stderr, "Need a least one frequency\n"); return 1; }
	acb_config_t cfg = { 0, mult, 1, (int)nbch, CS_BATCH, ACB_FLAG_CS16_INPUT, 0 };
	if (env_taps(mult, &cfg.taps)) return -1;
	if (!(cs_ctx = front_end_create(&cfg))) return -1;
	unsigned Fc = 0;
	if (acb_multi_set_plan_cs16(cs_ctx, 0, Fd, (int)nbch, variant, fc_user, &Fc) != ACB_OK) {
		fprintf(stderr, "%s\n", acb_last_error());            /* "Frequencies too far apart" */
		return 1;
	}
	/* channel[] as the reference leaves it: the unscaled oscillator (the library's table carries an
	 * exact power-of-two factor on top, see acb_cs16_build_wf) */
	const float unscale = variant == ACB_CS16_SOAPY ? 32768.0f : 4.0f;
	float *wf = malloc(sizeof(float) * 2 * mult);
	if (!wf) return -1;
	for (unsigned n = 0; n < nbch; n++) {
		channel_t *ch = &channel[n];
		ch->counter = 0;
		ch->D = 0;
		ch->oscillator = malloc(mult * sizeof(float complex));
		ch->dm_buffer = malloc(RTLOUTBUFSZ * sizeof(float));
		if (!ch->oscillator || !ch->dm_buffer) { fprintf(stderr, "ERROR : malloc\n"); free(wf); return -1; }
		acb_cs16_build_wf(variant, (unsigned)ch->Fr, Fc, mult, wf);
		for (int i = 0; i < mult; i++) ch->oscillator[i] = wf[2 * i] * unscale + wf[2 * i + 1] * unscale * I;
	}
	free(wf);
	return (int)-(long)Fc;                                   /* <= -1: success, the centre frequency negated */
}

static int cs16_run(int group_outputs)
{
	if (!cs_ctx || !cs_src) return -1;
	const size_t cap = (size_t)RTLOUTBUFSZ * cs_mult * CS_BATCH;          /* complex samples per submit */
	int16_t *buf[2] = { acb_host_alloc(cap * 2 * sizeof(int16_t)), acb_host_alloc(cap * 2 * sizeof(int16_t)) };
	if (!buf[0] || !buf[1]) { fprintf(stderr, "acarsdec_b200: %s\n", acb_last_error()); return -1; }
	acb_chan_state_t st;
	for (unsigned n = 0; n < nbch; n++) { state_pack(&channel[n], &st); acb_multi_set_state(cs_ctx, 0, (int)n, &st); }
	/* the reference runs demodMSK channel by channel whenever dm_buffer is full (soapy.c:247: 1024 outputs,
	 * sdrplay.c:229: 512): frames are queued in that order */
	acb_multi_set_emission_groups(cs_ctx, ACB_GROUP_OUTPUTS, (uint64_t)group_outputs);
	int rc = ACB_OK, which = 0, inflight = 0;
	uint64_t pos = 0;
	stamp_reset();
	while (!signalExit) {
		if (inflight == 2) {                 /* buf[which] fed the submit two back: it has been consumed */
			rc = acb_multi_collect(cs_ctx);
			if (rc < 0) break;
			inflight--;
			deliver_ready(cs_ctx);
		}
		size_t got = fread(buf[which], 2 * sizeof(int16_t), cap, cs_src);
		if (got == 0) break;
		rc = acb_multi_submit_cs16_host(cs_ctx, buf[which], got, got);      /* any count: the remainder is carried */
		if (rc < 0) break;
		if (rc > 0) { pos += (uint64_t)rc; inflight++; which ^= 1; }
		else if ((rc = acb_multi_sync(cs_ctx)) < 0) break;
		else inflight = 0;
		stamp_batch(pos);
		if (got < cap) break;
	}
	if (rc >= 0) rc = acb_multi_sync(cs_ctx);
	if (rc < 0) fprintf(stderr, "acarsdec_b200: %s\n", acb_last_error());
	deliver_ready(cs_ctx);
	for (unsigned n = 0; n < nbch; n++)
		if (acb_multi_get_state(cs_ctx, 0, (int)n, &st) == ACB_OK) state_unpack(&st, &channel[n]);
	acb_host_free(buf[0]);
	acb_host_free(buf[1]);
	signalExit = 1;
	return rc < 0 ? -1 : 0;
}

static void cs16_close(void)
{
	if (cs_ctx) { acb_multi_destroy(cs_ctx); cs_ctx = NULL; }
	if (cs_src && cs_src != stdin) fclose(cs_src);
	cs_src = NULL;
}
#endif

#ifdef WITH_SOAPY
/* soapy.c:69 initSoapy — argv[optind] (the "device string" after -d) names a raw interleaved CS16
 * capture sampled at rateMult*12500 Hz; -c freq is honoured, -g/-p/--antenna are accepted. */
int initSoapy(char **argv, int optind)
{
	if (argv[optind] == NULL) {
		fprintf(stderr, "Need a CS16 capture file after -d\n");
		exit(1);                                             /* soapy.c:76-79 */
	}
	const char *path = argv[optind++];
	int r = cs16_setup(path, argv, optind, rateMult, ACB_CS16_SOAPY, (unsigned)freq,
	                   "WARNING: frequency not in range 118-138 MHz: %d\n");
	if (r >= 0 || r == -1) return r;
	freq = -r;                                               /* soapy.c:132-133 */
	const int rate = INTRATE * rateMult;
	for (unsigned n = 0; n < nbch; n++) {                    /* soapy.c:138-144 */
		const int f = (int)channel[n].Fr;
		if (f < freq - rate / 2 || f > freq + rate / 2)
			fprintf(stderr, "WARNING: frequency not in tuned range %d-%d: %d\n", freq - rate / 2, freq + rate / 2, f);
	}
	if (verbose) fprintf(stderr, "Set center freq. to %dHz\nSetting sample rate: %.4f MS/s\n", freq, rate / 1e6);
	return 0;
}

int soapySetAntenna(const char *antenna)
{
	if (cs_ctx == NULL) { fprintf(stderr, "soapySetAntenna: SoapySDR not init'd\n"); return 1; }    /* soapy.c:183-186 */
	if (antenna == NULL) { fprintf(stderr, "soapySetAntenna: antenna is NULL\n"); return 1; }
	return 0;                                                /* nothing to switch on a capture */
}

int runSoapySample(void) { return cs16_run(RTLOUTBUFSZ) < 0 ? 1 : 0; }   /* soapy.c:263; SOAPYOUTBUFSZ = 1024 */

int runSoapyClose(void) { cs16_close(); return 0; }           /* soapy.c:297 */
#endif /* WITH_SOAPY */

#ifdef WITH_SDRPLAY
/* sdrplay.c:95 initSdrplay — the reference takes no device argument (-s f1 f2 ...), so the capture
 * (raw interleaved CS16 at 2 MS/s) is named by ACARSDEC_B200_CAPTURE. */
int initSdrplay(char **argv, int optind)
{
	const char *path = getenv("ACARSDEC_B200_CAPTURE");
	if (!path) { fprintf(stderr, "Sorry, no device found (set ACARSDEC_B200_CAPTURE to a CS16 capture)\n"); exit(2); }   /* sdrplay.c:173-176 */
	int r = cs16_setup(path, argv, optind, 160, ACB_CS16_SDRPLAY, 0, "WARNING: Invalid frequency %d\n");
	if (r >= 0 || r == -1) return r;
	fprintf(stderr, "SDRplay capture selects freq %d\n", -r);
	return 0;
}

/* sdrplay.c:238 runSdrplaySample never returns in the reference (while(1) sleep); here it returns at
 * the end of the capture with signalExit set */
int runSdrplaySample(void)
{
	int r = cs16_run(512);                                  /* sdrplay.c:229 */
	cs16_close();
	return r;
}
#endif /* WITH_SDRPLAY */
