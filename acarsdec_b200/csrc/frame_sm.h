/*
 * ACARS bit/byte frame synchroniser — the per-byte state machine that sits INSIDE the
 * demodulator's serial recurrence (it resets the PLL and flips the bit polarity).
 * Behaviour follows decodeAcars()/resetAcars() of the reference (acars.c:239-375).
 *
 * One definition serves the CUDA demod kernel (state in registers, text in HBM) and the
 * host-side decodeAcars() symbol of the compat shim (state in channel_t): the template
 * parameter is an accessor with these members
 *
 *   int &state(), &nbits(), &bitcount(), &blk_len(), &blk_err();
 *   unsigned &msk_s();  double &msk_df(), &lvlsum();
 *   void txt_put(int i, unsigned char r);  unsigned char txt_get(int i);
 *   void crc_put(int i, unsigned char r);
 *   bool frame_begin();   // SOH seen: claim storage / note the time; false = no storage
 *   void frame_emit();    // frame complete: hand over (level is computed from lvlsum/bitcount)
 *
 * and optionally
 *
 *   void event(int e);    // a FrameEvent below occurred (the decode statistics, ACB_FLAG_DECODE_STATS)
 *
 * An accessor without event() gets nothing: the calls compile away, so its code is what it was before the hook.
 *
 * Integer-only apart from zeroing two doubles, so host and device agree trivially.
 */
#ifndef ACB_FRAME_SM_H
#define ACB_FRAME_SM_H

#if defined(__CUDACC__)
#define ACB_HD __host__ __device__ __forceinline__
#else
#define ACB_HD inline
#endif

namespace acb {

enum FrameState { F_WSYN = 0, F_SYN2, F_SOH1, F_TXT, F_CRC1, F_CRC2, F_END };   /* acarsdec.h:88 */

constexpr unsigned char C_SYN = 0x16, C_NSYN = 0xE9, C_SOH = 0x01, C_STX = 0x02;
constexpr unsigned char C_ETX = 0x83, C_ETB = 0x97, C_DLE = 0x7f;               /* acars.c:22-27 */
constexpr int MAX_PARITY_ERR = 3;                                               /* acars.c:92 */

/* The frame synchroniser's events (acb_decode_stats_t).  The first six are raised here; EV_SHORT and EV_LOST are the
 * accessor's own, from where its frame_emit put the frame (a block under 13 bytes, acars.c:124-129; a full device ring). */
enum FrameEvent {
	EV_PREAMBLE = 0,       /* two SYN seen, waiting for SOH (acars.c:267-271) */
	EV_STARTED,            /* SOH accepted, a block is assembled (acars.c:281-298) */
	EV_TXT_PARITY,         /* block abandoned: too many parity errors (acars.c:307-317) */
	EV_TXT_LONG,           /* block abandoned: over 240 bytes (acars.c:334-338) */
	EV_TXT_MISSED_END,     /* DLE after 20 bytes, emitted anyway (acars.c:324-332) */
	EV_EMITTED,            /* handed to the block FEC (acars.c:350-366) */
	EV_SHORT,              /* emitted, shorter than 13 bytes */
	EV_LOST,               /* emitted, found the device ring full */
	EV_COUNT
};

template <class A> ACB_HD auto frame_event_(A &a, int e, int) -> decltype(a.event(e), void()) { a.event(e); }
template <class A> ACB_HD void frame_event_(A &, int, long) {}
template <class A> ACB_HD void frame_event(A &a, int e) { frame_event_(a, e, 0); }

/* numbits[c] & 1 (syndrom.h:4-13): odd number of ones = parity ok */
ACB_HD bool parity_ok(unsigned char c)
{
	unsigned v = c;
	v ^= v >> 4; v ^= v >> 2; v ^= v >> 1;
	return (v & 1u) != 0;
}

/* acars.c:239-244 */
template <class A> ACB_HD void frame_resync(A &a)
{
	a.state() = F_WSYN;
	a.msk_df() = 0.0;
	a.nbits() = 1;
}

template <class A> ACB_HD void frame_finish(A &a)
{
	frame_event(a, EV_EMITTED);
	a.frame_emit();                         /* acars.c:350-366 */
	a.state() = F_END;
	a.nbits() = 8;
}

/* acars.c:246-375 — called by putbit when nbits reaches 0 with the assembled byte r */
template <class A> ACB_HD void frame_byte(A &a, unsigned char r)
{
	/* WSYN first and without the switch: while hunting for SYN this runs once per BIT inside the
	 * demodulator's serial loop, and a 7-way switch compiles to an indirect branch there */
	if (a.state() == F_WSYN) {              /* sliding one bit at a time */
		if (r == C_SYN || r == C_NSYN) {
			if (r == C_NSYN) a.msk_s() ^= 2u;   /* inverted polarity */
			a.state() = F_SYN2;
			a.nbits() = 8;
		} else {
			a.nbits() = 1;
		}
		return;
	}
	switch (a.state()) {
	case F_SYN2:
		if (r == C_SYN) { frame_event(a, EV_PREAMBLE); a.state() = F_SOH1; a.nbits() = 8; return; }
		if (r == C_NSYN) { a.msk_s() ^= 2u; a.nbits() = 8; return; }
		frame_resync(a);
		return;
	case F_SOH1:
		if (r != C_SOH || !a.frame_begin()) { frame_resync(a); return; }
		frame_event(a, EV_STARTED);
		a.state() = F_TXT;
		a.blk_len() = 0;
		a.blk_err() = 0;
		a.nbits() = 8;
		a.lvlsum() = 0.0;
		a.bitcount() = 0;
		return;
	case F_TXT: {
		int n = a.blk_len();
		a.txt_put(n, r);
		a.blk_len() = ++n;
		if (!parity_ok(r)) {
			if (++a.blk_err() > MAX_PARITY_ERR + 1) { frame_event(a, EV_TXT_PARITY); frame_resync(a); return; }
		}
		if (r == C_ETX || r == C_ETB) { a.state() = F_CRC1; a.nbits() = 8; return; }
		if (n > 20 && r == C_DLE) {         /* end of text was missed: the BCS is already in txt */
			frame_event(a, EV_TXT_MISSED_END);
			n -= 3;
			a.blk_len() = n;
			a.crc_put(0, a.txt_get(n));
			a.crc_put(1, a.txt_get(n + 1));
			frame_finish(a);
			return;
		}
		if (n > 240) { frame_event(a, EV_TXT_LONG); frame_resync(a); return; }
		a.nbits() = 8;
		return;
	}
	case F_CRC1:
		a.crc_put(0, r);
		a.state() = F_CRC2;
		a.nbits() = 8;
		return;
	case F_CRC2:
		a.crc_put(1, r);
		frame_finish(a);
		return;
	default:                                /* F_END */
		frame_resync(a);
		a.nbits() = 8;
		return;
	}
}

} // namespace acb
#endif
