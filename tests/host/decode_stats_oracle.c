/*
 * TEST INFRASTRUCTURE — NOT PRODUCT CODE.
 *
 * The restatement's decode statistics (ACB_FLAG_DECODE_STATS): per channel, how often each event occurs that the
 * reference's decodeAcars and blk_thread print a -v line for (acars.c:101-206, 311-354), in the field order of
 * acb_decode_stats_t.  Built on the pinned restatement (oracle/libacars_oracle.so) without changing it:
 *
 *   dso_demod      orc_demod over a chunk of envelope with its raw-bit trace on, then the frame synchroniser
 *                  (acars.c:246-375) replayed over those bits with the counts.  The demodulator's feedback from the
 *                  synchroniser (MskS ^= 2, MskDf = 0) is already in the bits orc_demod produced, so the replay sees
 *                  exactly the bytes decodeAcars saw; its state is carried across chunks (dso_sync_t) and the tests
 *                  hold it to orc_demod's own after every chunk.
 *   dso_block_fec  blk_thread (acars.c:123-209) with the lines it prints counted; the tests hold its keep decision and
 *                  repaired text to orc_block_fec's.
 *
 * Built by tests/decode_stats_refs.py with gcc -O2 -ffp-contract=off against oracle/libacars_oracle.so.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../../oracle/acars_oracle.h"

typedef struct {                 /* acb_decode_stats_t, field for field */
	uint64_t preamble, started, txt_parity, txt_long, txt_missed_end, emitted;
	uint64_t fec_short, fec_parity_excess, fec_parity, fec_crc, fec_fixed, fec_unfixable, fec_parity_problem;
	uint64_t delivered, lost;
} dso_counts_t;

typedef struct {                 /* the frame synchroniser's state of the replay (channel_t's part, acarsdec.h:76-89) */
	int state, nbits, blk_len, blk_err;
	unsigned outbits;
} dso_sync_t;

#define SYN 0x16
#define SOH 0x01
#define ETX 0x83
#define ETB 0x97
#define DLE 0x7f
#define MAXPERR 3

void dso_sync_init(dso_sync_t *s)
{
	memset(s, 0, sizeof(*s));
	s->nbits = 8;                /* acars.c:230-234 */
	s->state = ORC_WSYN;
}

static void resync(dso_sync_t *s)   /* acars.c:239-244 (MskDf = 0 is the demodulator's: already in the bits) */
{
	s->state = ORC_WSYN;
	s->nbits = 1;
}

static void put_msg(dso_sync_t *s, dso_counts_t *k)   /* acars.c:350-369, "put message" */
{
	k->emitted++;
	s->state = ORC_END;
	s->nbits = 8;
}

/* acars.c:246-375 on the byte r; only what the counts and the control flow need */
static void sync_byte(dso_sync_t *s, unsigned char r, dso_counts_t *k)
{
	switch (s->state) {
	case ORC_WSYN:
		if (r == SYN || r == (unsigned char)~SYN) { s->state = ORC_SYN2; s->nbits = 8; }
		else s->nbits = 1;
		return;
	case ORC_SYN2:
		if (r == SYN) { k->preamble++; s->state = ORC_SOH1; s->nbits = 8; return; }
		if (r == (unsigned char)~SYN) { s->nbits = 8; return; }
		resync(s);
		return;
	case ORC_SOH1:
		if (r != SOH) { resync(s); return; }
		k->started++;
		s->state = ORC_TXT; s->blk_len = 0; s->blk_err = 0; s->nbits = 8;
		return;
	case ORC_TXT:
		s->blk_len++;
		if (!orc_odd_parity(r) && ++s->blk_err > MAXPERR + 1) { k->txt_parity++; resync(s); return; }   /* "too many parity errors" */
		if (r == ETX || r == ETB) { s->state = ORC_CRC1; s->nbits = 8; return; }
		if (s->blk_len > 20 && r == DLE) { k->txt_missed_end++; s->blk_len -= 3; put_msg(s, k); return; }   /* "miss txt end" */
		if (s->blk_len > 240) { k->txt_long++; resync(s); return; }                                       /* "too long" */
		s->nbits = 8;
		return;
	case ORC_CRC1:
		s->state = ORC_CRC2; s->nbits = 8;
		return;
	case ORC_CRC2:
		put_msg(s, k);
		return;
	default:                     /* ORC_END */
		resync(s);
		s->nbits = 8;
		return;
	}
}

/* orc_demod over dm[0..len) with the synchroniser replayed over its bits; the pre-FEC blocks go to *sink as orc_demod
 * leaves them.  Returns the number of bits, or -1 when the trace could not be allocated. */
long dso_demod(orc_chan_t *c, const float *h, const float *dm, int len, orc_sink_t *sink, dso_sync_t *s, dso_counts_t *k)
{
	const int64_t cap = len / 4 + 8;        /* a bit every 5.2 samples at the least */
	uint8_t *bits = malloc(cap);
	if (!bits) return -1;
	orc_sink_t local = *sink;
	local.bits = bits;
	local.nbits = 0;
	local.capbits = cap;
	orc_demod(c, h, dm, len, &local);
	for (int64_t i = 0; i < local.nbits; i++) {        /* putbit, msk.c:53-63 */
		s->outbits = (s->outbits >> 1) | (bits[i] ? 0x80u : 0u);
		if (--s->nbits <= 0) sync_byte(s, (unsigned char)s->outbits, k);
	}
	sink->msgs = local.msgs;
	sink->nmsg = local.nmsg;
	sink->capmsg = local.capmsg;
	free(bits);
	return (long)local.nbits;
}

/* acars.c:39-64 */
static int fixprerr(orc_msg_t *m, uint16_t crc, const int *pr, int pn)
{
	if (pn > 0) {
		for (int i = 0; i < 8; i++)
			if (fixprerr(m, crc ^ orc_syndrome(i, m->len - *pr + 1), pr + 1, pn - 1)) {
				m->txt[*pr] ^= (1 << i);
				return 1;
			}
		return 0;
	}
	if (crc == 0) return 1;
	for (int i = 0; i < 16; i++)
		if (orc_syndrome(i & 7, i >> 3) == crc) return 1;
	return 0;
}

/* acars.c:66-90 */
static int fixdberr(orc_msg_t *m, uint16_t crc)
{
	for (int i = 0; i < 16; i++)
		if (orc_syndrome(i & 7, i >> 3) == crc) return 1;
	for (int j = 0; j < m->len; j++) {
		const int p = m->len - j + 1;
		for (int a = 0; a < 8; a++)
			for (int b = 0; b < 8; b++) {
				if (a == b) continue;
				if ((crc ^ orc_syndrome(a, p) ^ orc_syndrome(b, p)) == 0) {
					m->txt[j] ^= (1 << a);
					m->txt[j] ^= (1 << b);
					return 1;
				}
			}
	}
	return 0;
}

/* blk_thread on one block (acars.c:123-209), its -v lines counted: 1 = outputmsg(), 0 = dropped */
int dso_block_fec(orc_msg_t *m, dso_counts_t *k)
{
	int pr[MAXPERR], pn = 0;
	uint16_t crc = 0;
	if (m->len < 13) { k->fec_short++; return 0; }                        /* "too short" */
	m->txt[12] &= (ETX | 0x02);
	m->txt[12] |= (ETX & 0x02);
	for (int i = 0; i < m->len; i++)
		if (!orc_odd_parity(m->txt[i])) { if (pn < MAXPERR) pr[pn] = i; pn++; }
	if (pn > MAXPERR) { k->fec_parity_excess++; return 0; }               /* "too many parity errors: %d" */
	if (pn) k->fec_parity++;                                              /* "parity error(s): %d" */
	m->err = pn;
	for (int i = 0; i < m->len; i++) crc = orc_crc_step(crc, m->txt[i]);
	crc = orc_crc_step(crc, m->crc[0]);
	crc = orc_crc_step(crc, m->crc[1]);
	if (crc) k->fec_crc++;                                                /* "crc error" */
	if (pn || crc) {
		if (pn ? !fixprerr(m, crc, pr, pn) : !fixdberr(m, crc)) { k->fec_unfixable++; return 0; }   /* "not able to fix errors" */
		k->fec_fixed++;                                                   /* "errors fixed" */
	}
	pn = 0;
	for (int i = 0; i < m->len; i++) {
		if (!orc_odd_parity(m->txt[i])) pn++;
		m->txt[i] &= 0x7f;
	}
	if (pn) { k->fec_parity_problem++; return 0; }                        /* "parity check problem" */
	k->delivered++;
	return 1;
}
