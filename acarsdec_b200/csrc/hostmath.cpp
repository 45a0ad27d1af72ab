/*
 * Host-side pieces of the hot path that the reference also runs on the host, written so that
 * their results are bit-identical to the reference's when built against the same glibc:
 *
 *   front-end planning  — frequency rounding, chooseFc, the per-channel mixer/boxcar table
 *                         (initRtl, rtl.c:243-287) and the matched filter (initMsk, msk.c:44-48);
 *                         these run once and use libm (sincosf, cosf), so they stay on the CPU
 *                         and the tables are uploaded;
 *   block FEC           — blk_thread's parity/CRC/syndrome repair (acars.c:39-215), integer
 *                         only, one call per decoded frame; CRC and syndrome tables are
 *                         generated at start-up instead of stored (syndrom.h).
 *
 * Must be compiled without FMA contraction / fast-math (build uses -ffp-contract=off).
 */
#ifndef _GNU_SOURCE
#define _GNU_SOURCE
#endif
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <mutex>
#include <vector>

#include "../../include/acars_b200.h"
#include "frame_sm.h"
#include "acb_internal.h"

/* cos/sin(k*pi/32), k < 64, as double-double (hi, lo) pairs for the demod kernel's VCO sincos
 * (demod_core.h sincos_vco); long double (64-bit mantissa) is ample for the non-zero entries, the
 * multiples of pi/2 are set exactly.  Internal (not in the public header): context.cu uploads it, the CPU
 * tests' host emulation of the demod loop reads it. */
extern "C" void acb_build_sincos_table(double *tc, double *ts)
{
	const long double pi = 3.14159265358979323846264338327950288L;
	for (int k = 0; k < 64; k++) {
		const long double c = cosl(k * pi / 32), s = sinl(k * pi / 32);
		tc[2 * k] = (double)c; tc[2 * k + 1] = (double)(c - (long double)tc[2 * k]);
		ts[2 * k] = (double)s; ts[2 * k + 1] = (double)(s - (long double)ts[2 * k]);
		if (k % 16 == 0) {
			static const double qc[4] = { 1, 0, -1, 0 }, qs[4] = { 0, 1, 0, -1 };
			tc[2 * k] = qc[k / 16]; tc[2 * k + 1] = 0; ts[2 * k] = qs[k / 16]; ts[2 * k + 1] = 0;
		}
	}
}

/* ------------------------------------------------------------------ front-end planning */

extern "C" int acb_round_freq(double mhz)
{
	/* rtl.c:245-247: nearest multiple of INTRATE, computed in int */
	return ((int)(1000000 * mhz + ACB_INTRATE / 2) / ACB_INTRATE) * ACB_INTRATE;
}

extern "C" int acb_stored_fr(unsigned freq_hz)
{
	/* rtl.c:255: channel[].Fr (an int) receives (float)Fd — frequencies off the 8 Hz float
	 * grid above 2^27 move by up to 4 Hz, and the table below is built from the moved value */
	return (int)(float)freq_hz;
}

extern "C" unsigned acb_choose_fc(const unsigned *freqs_hz, int n, int K)
{
	/* rtl.c:131-168.  Candidates run downward in 1 Hz steps from (highest + 2*INTRATE); the
	 * first that keeps every channel inside [2*INTRATE, rate/2 - 2*INTRATE] of the centre
	 * with no channel the mirror image of its lower neighbour wins. */
	if (n <= 0 || !freqs_hz) return 0;
	std::vector<long long> f(freqs_hz, freqs_hz + n);
	std::sort(f.begin(), f.end());
	const long long rate = (long long)ACB_INTRATE * K, guard = 2 * ACB_INTRATE;
	if (f.back() - f.front() > rate - 2 * guard) return 0;
	long long fc = f.back() + guard;
	for (; fc > f.front() - guard; fc--) {
		bool ok = true;
		for (int i = 0; i < n && ok; i++) {
			const long long d = llabs(fc - f[i]);
			ok = d <= rate / 2 - guard && d >= guard && !(i > 0 && fc - f[i - 1] == f[i] - fc);
		}
		if (ok) break;
	}
	return (unsigned)fc;      /* like the reference, an exhausted scan returns its last candidate */
}

/* Band planner for channel sets one tuner cannot cover.  chooseFc (rtl.c:149-152) gives up when the span
 * exceeds rate - 4*INTRATE; the scan script of the reference (scan.sh:1-16) then walks the band with one
 * dongle, eight channels and five minutes at a time.  Here the whole set is cut into the FEWEST receiver bands
 * (greedy over the sorted frequencies: extend the current band while its span still fits — optimal for
 * interval covering), each with the centre chooseFc picks for its members.  group_of[i] is the band of
 * freqs_hz[i] (CLI order kept inside a band), fc_out[g] its centre.  Returns the number of bands, or
 * ACB_ERR_PLAN when more than max_groups are needed / ACB_ERR_ARG. */
extern "C" int acb_plan_bands(const unsigned *freqs_hz, int n, int K, int *group_of, unsigned *fc_out, int max_groups)
{
	if (!freqs_hz || !group_of || !fc_out || n < 1 || K < 1 || max_groups < 1) return ACB_ERR_ARG;
	std::vector<int> order(n);
	for (int i = 0; i < n; i++) order[i] = i;
	std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return freqs_hz[a] < freqs_hz[b]; });
	const long long span = (long long)ACB_INTRATE * K - 4LL * ACB_INTRATE;
	int ng = 0;
	size_t i = 0;
	while (i < order.size()) {
		if (ng == max_groups) return ACB_ERR_PLAN;
		size_t j = i;
		std::vector<unsigned> members;
		unsigned fc = 0;
		/* longest run that fits AND that chooseFc can centre (the mirror rule can refuse a set that fits) */
		for (size_t e = i; e < order.size() && (long long)freqs_hz[order[e]] - (long long)freqs_hz[order[i]] <= span; e++) {
			members.push_back(freqs_hz[order[e]]);
			const unsigned c = acb_choose_fc(members.data(), (int)members.size(), K);
			/* an exhausted scan returns its last candidate (rtl.c:154-167 does): only a centre that really keeps
			 * every member off DC, inside the band and off its neighbour's mirror image counts */
			bool ok = c != 0;
			const long long rate = (long long)ACB_INTRATE * K, guard = 2 * ACB_INTRATE;
			for (size_t m = 0; ok && m < members.size(); m++) {
				const long long d = llabs((long long)c - (long long)members[m]);
				ok = d <= rate / 2 - guard && d >= guard && !(m > 0 && (long long)c - (long long)members[m - 1] == (long long)members[m] - (long long)c);
			}
			if (ok) { fc = c; j = e + 1; }
		}
		if (fc == 0) return ACB_ERR_PLAN;             /* not even the first channel alone: K too small for the guard bands */
		for (size_t e = i; e < j; e++) group_of[order[e]] = ng;
		fc_out[ng++] = fc;
		i = j;
	}
	return ng;
}

extern "C" void acb_build_wf(int fr_stored, unsigned fc_hz, int K, float *wf)
{
	/* rtl.c:283-286.  Types matter: the offset is a float difference divided by a float rate,
	 * scaled by 2*pi in double and stored back to float; the phase of tap `ind` is the float
	 * product AMFreq*ind; the unit vector comes from cexpf (= sincosf of the imaginary part);
	 * "/rtlMult" is a float division, "/127.5" a double division rounded to float. */
	const float rate = (float)(ACB_INTRATE * K);
	const float step = (float)(((float)fr_stored - (float)fc_hz) / rate * 2.0 * M_PI);
	for (int ind = 0; ind < K; ind++) {
		const float ph = step * (float)ind;
		float sn, cs;
		sincosf(-ph, &sn, &cs);
		wf[2 * ind] = (float)((double)(cs / (float)K) / 127.5);
		wf[2 * ind + 1] = (float)((double)(sn / (float)K) / 127.5);
	}
}

extern "C" unsigned acb_air_choose_fc(unsigned min_hz, unsigned max_hz)
{
	/* air.c:42-64 with filter == 0 (all Airspy rates except 5 MS/s, where the reference also
	 * programs the R820T IF filters — a device matter with no file-replay equivalent) */
	return ((max_hz + min_hz) / 2 + ACB_INTRATE / 2) / ACB_INTRATE * ACB_INTRATE;
}

extern "C" void acb_air_build_wf(int fr_hz, int fc_hz, unsigned rate, float *wf)
{
	/* air.c:263-285: IF = rate/4 above (Fc - Fr); the phase is a double accumulator kept inside
	 * +-2*pi; the unit vector is cexpf of the float-rounded phase (= sincosf); "/AIRMULT" divides
	 * by the float image of the unsigned tap count */
	const unsigned K = rate / ACB_INTRATE;
	const double step = 2.0 * M_PI * (double)(unsigned)(fc_hz - fr_hz + rate / 4) / (double)rate;
	double ph = 0;
	for (unsigned i = 0; i < K; i++) {
		float sn, cs;
		sincosf((float)-ph, &sn, &cs);
		wf[2 * i] = cs / (float)K;
		wf[2 * i + 1] = sn / (float)K;
		ph += step;
		if (ph > 2.0 * M_PI) ph -= 2.0 * M_PI;
		if (ph < -2.0 * M_PI) ph += 2.0 * M_PI;
	}
}

extern "C" void acb_cs16_build_wf(int variant, unsigned freq_hz, unsigned fc_hz, int K, float *wf)
{
	/* soapy.c:159-162 / sdrplay.c:133-137: oscillator[ind] = cexpf(-j*phase*ind)/K, where the
	 * per-tap phase is a FLOAT product in soapy.c (float AMFreq) and a DOUBLE product rounded to
	 * float by cexpf's argument conversion in sdrplay.c (double correctionPhase); channel[].Fr is a
	 * float in both.  What the kernel needs on top is folded in exactly (powers of two commute with
	 * every rounding here): soapy.c:242 divides each product by 32768.0 before accumulating, and
	 * sdrplay.c:225 divides the envelope by 4. */
	const float fr = (float)freq_hz;
	const float rate = (float)(ACB_INTRATE * K);
	const double dstep = (fr - (float)fc_hz) / rate * 2.0 * M_PI;
	const float fstep = (float)dstep;
	const float scale = variant == ACB_CS16_SOAPY ? 1.0f / 32768.0f : 0.25f;
	for (int ind = 0; ind < K; ind++) {
		const float ph = variant == ACB_CS16_SOAPY ? fstep * (float)ind : (float)(dstep * ind);
		float sn, cs;
		sincosf(-ph, &sn, &cs);
		wf[2 * ind] = cs / (float)K * scale;
		wf[2 * ind + 1] = sn / (float)K * scale;
	}
}

/* ------------------------------------------------------------------ overlapping-window channel filter (taps > K) */

/* modified Bessel function of the first kind, order 0: its power series, to the last double bit for the small
 * arguments a Kaiser window needs (|x| <= beta = 6: terms fall below 1e-17 of the sum after ~25 of them) */
static double bessel_i0(double x)
{
	const double q = x * x / 4;
	double term = 1, sum = 1;
	for (int k = 1; k < 200 && term > sum * 1e-18; k++) {
		term *= q / ((double)k * k);
		sum += term;
	}
	return sum;
}

extern "C" int acb_build_lowpass(int K, int taps, float *h)
{
	if (!h || K < 1 || taps < 1 || taps > ACB_MAXTAPS_PER_K * K) return ACB_ERR_ARG;
	const double beta = 6.0, fcut = 0.5 / K;          /* cutoff in cycles per input sample: ACB_INTRATE/2 */
	const double mid = (taps - 1) / 2.0, i0b = bessel_i0(beta);
	std::vector<double> v(taps);
	double sum = 0;
	for (int n = 0; n < taps; n++) {
		const double t = n - mid, x = 2 * fcut * t;
		const double ideal = t == 0 ? 2 * fcut : 2 * fcut * sin(M_PI * x) / (M_PI * x);
		const double r = taps > 1 ? 2.0 * n / (taps - 1) - 1 : 0;
		v[n] = ideal * bessel_i0(beta * sqrt(std::max(0.0, 1 - r * r))) / i0b;
		sum += v[n];
	}
	for (int n = 0; n < taps; n++) h[n] = (float)(v[n] / sum);
	return ACB_OK;
}

/* w[i] = h[i] * exp(-j*2*pi*off*(i - H)/rate) * scale, off a whole number of Hz: the phase is reduced exactly in
 * integers, then evaluated and multiplied in double and rounded to float once */
static void build_wf_lp(long long off, long long rate, int K, int taps, double scale, float *wf)
{
	std::vector<float> h(taps);
	acb_build_lowpass(K, taps, h.data());
	const int H = taps - K;
	for (int i = 0; i < taps; i++) {
		const long long r = (off * (long long)(i - H)) % rate;
		const double ph = 2.0 * M_PI * (double)r / (double)rate;
		wf[2 * i] = (float)((double)h[i] * cos(ph) * scale);
		wf[2 * i + 1] = (float)(-(double)h[i] * sin(ph) * scale);
	}
}

extern "C" void acb_build_wf_lp(int fr_stored, unsigned fc_hz, int K, int taps, float *wf)
{
	/* rtl.c:283: the offset is the float image of the stored Fr minus the float image of Fc (both whole numbers) */
	const float off = (float)fr_stored - (float)fc_hz;
	build_wf_lp((long long)off, (long long)ACB_INTRATE * K, K, taps, 1.0 / 127.5, wf);
}

extern "C" void acb_cs16_build_wf_lp(int variant, unsigned freq_hz, unsigned fc_hz, int K, int taps, float *wf)
{
	/* soapy.c:159-162 / sdrplay.c:133-137: (float)Fr - (float)Fc; soapy.c:242's /32768.0 or sdrplay.c:225's /4 folded in */
	const float off = (float)freq_hz - (float)fc_hz;
	build_wf_lp((long long)off, (long long)ACB_INTRATE * K, K, taps, variant == ACB_CS16_SOAPY ? 1.0 / 32768.0 : 0.25, wf);
}

extern "C" void acb_air_build_wf_lp(int fr_hz, int fc_hz, unsigned rate, int taps, float *wf)
{
	/* air.c:263-285: the IF of the channel, Fc - Fr + rate/4 */
	const unsigned K = rate / ACB_INTRATE;
	build_wf_lp((long long)(unsigned)(fc_hz - fr_hz + rate / 4), (long long)rate, (int)K, taps, 1.0, wf);
}

extern "C" int acb_fast_plan(const unsigned *freqs_hz, int nch, int K, unsigned fc_hz, int *k_out, float *tw)
{
	/* The reference's table wf[ind] = cexpf(-j*AMFreq*ind)/K/127.5 (rtl.c:283-286) is a sampled complex
	 * exponential; when the offset it mixes with — the float image of the stored Fr minus the float
	 * image of Fc (rtl.c:255, 283) — is a whole number k of 12.5 kHz steps, D is bin k of a K-point DFT of
	 * the row and k_channelize_dft applies.  Both float images are multiples of 8 Hz, so k is even.
	 * T_c[n2] = exp(-j*2*pi*k*n2/K)/K/127.5 for n2 < K/4, evaluated in double. */
	if (!freqs_hz || nch <= 0 || K <= 0 || (K & 3)) return 0;
	const int N2 = K / 4;
	for (int ch = 0; ch < nch; ch++) {
		const float d = (float)acb_stored_fr(freqs_hz[ch]) - (float)fc_hz;
		const float kf = d / (float)ACB_INTRATE;
		const int k = (int)kf;
		if ((float)k != kf || (k & 1) || k == 0 || k <= -K / 2 || k >= K / 2) return 0;
		if (k_out) k_out[ch] = k;
		if (!tw) continue;
		for (int n2 = 0; n2 < N2; n2++) {
			const double ph = -2.0 * M_PI * (double)(((long long)k * n2) % K) / (double)K;
			tw[((size_t)ch * N2 + n2) * 2] = (float)(cos(ph) / K / 127.5);
			tw[((size_t)ch * N2 + n2) * 2 + 1] = (float)(sin(ph) / K / 127.5);
		}
	}
	return 1;
}

extern "C" int acb_fast_plan_cs16(int variant, const unsigned *freqs_hz, int nch, int K, unsigned fc_hz, int *k_out, float *tw)
{
	/* soapy.c:159-165 / sdrplay.c:133-137: the oscillator is a sampled exponential of (float)Fr - (float)Fc over the input
	 * rate; when that offset is a whole EVEN number k of 12.5 kHz steps, D is bin k of the row's K-point DFT and the
	 * folded kernel applies.  The variant's power-of-two scale (acb_cs16_build_wf) goes into the twiddles. */
	if (!freqs_hz || nch <= 0 || K <= 0 || (K & 7)) return 0;
	if (variant != ACB_CS16_SOAPY && variant != ACB_CS16_SDRPLAY) return 0;
	const int N2 = K / 4;
	const double scale = variant == ACB_CS16_SOAPY ? 1.0 / 32768.0 : 0.25;
	for (int ch = 0; ch < nch; ch++) {
		const float d = (float)freqs_hz[ch] - (float)fc_hz;
		const float kf = d / (float)ACB_INTRATE;
		const int k = (int)kf;
		if ((float)k != kf || (k & 1) || k == 0 || k <= -K / 2 || k >= K / 2) return 0;
		if (k_out) k_out[ch] = k;
		if (!tw) continue;
		for (int n2 = 0; n2 < N2; n2++) {
			const double ph = -2.0 * M_PI * (double)(((long long)k * n2) % K) / (double)K;
			tw[((size_t)ch * N2 + n2) * 2] = (float)(cos(ph) / K * scale);
			tw[((size_t)ch * N2 + n2) * 2 + 1] = (float)(sin(ph) / K * scale);
		}
	}
	return 1;
}

extern "C" int acb_wb_twiddles(int variant, int K, float *E)
{
	/* Every twiddle the two planners above write depends on k and n2 only through r = (k*n2) % K (C remainder: the sign of
	 * k), so one table indexed by r in (-K, K) serves every channel of a context (k_channelize_wb).  Both signs are kept:
	 * cos(2*pi*(r + K)/K) need not round like cos(2*pi*r/K).  The expressions are the planners' own, token for token.
	 * Real input (acb_fast_plan_air below, k_channelize_wb_real): 0 < k < K, so only r in [0, K) occurs; the table keeps
	 * the same layout. */
	if (!E || K <= 0 || K > ACB_MAXK || (K & 3)) return 0;
	if (variant != -1 && variant != ACB_CS16_SOAPY && variant != ACB_CS16_SDRPLAY && variant != ACB_WB_TW_REAL) return 0;
	if (variant == ACB_WB_TW_REAL && (K & 7)) return 0;
	const double scale = variant == ACB_CS16_SOAPY ? 1.0 / 32768.0 : 0.25;
	for (int r = -(K - 1); r < K; r++) {
		const double ph = -2.0 * M_PI * (double)r / (double)K;
		float *o = E + (size_t)(r + K - 1) * 2;
		if (variant == -1) {
			o[0] = (float)(cos(ph) / K / 127.5);
			o[1] = (float)(sin(ph) / K / 127.5);
		} else if (variant == ACB_WB_TW_REAL) {
			o[0] = (float)(cos(ph) / K);
			o[1] = (float)(sin(ph) / K);
		} else {
			o[0] = (float)(cos(ph) / K * scale);
			o[1] = (float)(sin(ph) / K * scale);
		}
	}
	return 1;
}

extern "C" int acb_fast_plan_air(const unsigned *freqs_hz, int nch, int K, unsigned fc_hz, int *k_out, float *tw)
{
	/* air.c:278-285: AMFreq = 2*pi*(Fc - Fr + rate/4)/rate, wf[i] = cexpf(-j*i*AMFreq)/K: bin k = (Fc - Fr + rate/4)/12500
	 * of the K-point DFT of the real row when that is a whole number (air.c:66 puts Fc on the 12.5 kHz raster). */
	if (!freqs_hz || nch <= 0 || K <= 0 || (K & 7)) return 0;
	const unsigned rate = (unsigned)K * ACB_INTRATE;
	const int N2 = K / 4;
	for (int ch = 0; ch < nch; ch++) {
		const unsigned off = (unsigned)((int)fc_hz - (int)freqs_hz[ch] + (int)(rate / 4));
		if (off % ACB_INTRATE) return 0;
		const int k = (int)(off / ACB_INTRATE);
		if (k <= 0 || k >= K) return 0;
		if (k_out) k_out[ch] = k;
		if (!tw) continue;
		for (int n2 = 0; n2 < N2; n2++) {
			const double ph = -2.0 * M_PI * (double)(((long long)k * n2) % K) / (double)K;
			tw[((size_t)ch * N2 + n2) * 2] = (float)(cos(ph) / K);
			tw[((size_t)ch * N2 + n2) * 2 + 1] = (float)(sin(ph) / K);
		}
	}
	return 1;
}

extern "C" void acb_build_h(float *h)
{
	/* msk.c:44-48: cos(2*pi*600/INTRATE/12 * (i - 66)) evaluated by cosf on the float-rounded
	 * double argument, negative lobes clamped to zero */
	for (int i = 0; i < 133; i++) {
		const double arg = 2.0 * M_PI * 600.0 / ACB_INTRATE / 12 * (i - 66);
		const float v = cosf((float)arg);
		h[i] = v < 0 ? 0.0f : v;
	}
}

/* ------------------------------------------------------------------ block FEC */

namespace {

struct FecTables {
	uint16_t crc[256];
	uint16_t syn[8 * 252];            /* syndrom.h:52-295 has 1936 = 8 x 242 entries; a 241-byte
	                                     block (acars.c:319 precedes the length check) indexes just past
	                                     that in the reference — keep the lookups in bounds here */
	FecTables()
	{
		for (int b = 0; b < 256; b++) {       /* reflected CCITT, poly 0x8408 (syndrom.h:15-48) */
			uint16_t r = (uint16_t)b;
			for (int k = 0; k < 8; k++) r = (r & 1) ? (uint16_t)((r >> 1) ^ 0x8408) : (uint16_t)(r >> 1);
			crc[b] = r;
		}
		/* syndrome of one wrong bit: CRC (init 0) of that bit followed by p zero bytes */
		for (int bit = 0; bit < 8; bit++) {
			uint16_t r = crc[1u << bit];
			for (int p = 0; p < 252; p++) {
				syn[bit + 8 * p] = r;
				r = (uint16_t)((r >> 8) ^ crc[r & 0xff]);
			}
		}
	}
};

const FecTables &tables()
{
	static const FecTables t;
	return t;
}

inline bool odd_parity(unsigned char c)
{
	return __builtin_parity(c) != 0;      /* numbits[c] & 1, syndrom.h:4-13 */
}

inline uint16_t crc_step(const FecTables &t, uint16_t crc, unsigned char c)
{
	return (uint16_t)((crc >> 8) ^ t.crc[(crc ^ c) & 0xff]);      /* update_crc, syndrom.h:49 */
}

bool crc_bytes_hit(const FecTables &t, uint16_t crc)
{
	/* a single wrong bit inside the two BCS bytes (acars.c:57-62, 70-74): accepted, not repaired */
	for (int i = 0; i < 16; i++)
		if (t.syn[i] == crc) return true;
	return false;
}

/* acars.c:39-64: try every bit of each parity-failing byte, depth-first in the reference's order */
bool repair_parity(const FecTables &t, acb_msg_t *m, uint16_t crc, const int *pos, int npos)
{
	if (npos == 0) return crc == 0 || crc_bytes_hit(t, crc);
	const int base = 8 * (m->len - pos[0] + 1);
	for (int bit = 0; bit < 8; bit++)
		if (repair_parity(t, m, crc ^ t.syn[bit + base], pos + 1, npos - 1)) {
			m->txt[pos[0]] ^= (unsigned char)(1u << bit);
			return true;
		}
	return false;
}

/* acars.c:66-90: no parity error but CRC fails -> two wrong bits in one byte */
bool repair_double(const FecTables &t, acb_msg_t *m, uint16_t crc)
{
	if (crc_bytes_hit(t, crc)) return true;
	for (int k = 0; k < m->len; k++) {
		const int base = 8 * (m->len - k + 1);
		for (int i = 0; i < 8; i++)
			for (int j = 0; j < 8; j++)
				if (i != j && (uint16_t)(crc ^ t.syn[i + base] ^ t.syn[j + base]) == 0) {
					m->txt[k] ^= (unsigned char)((1u << i) | (1u << j));
					return true;
				}
	}
	return false;
}

} // namespace

extern "C" uint16_t acb_crc_update(uint16_t crc, uint8_t c) { return crc_step(tables(), crc, c); }

extern "C" uint16_t acb_syndrome(int index)
{
	return (index >= 0 && index < 8 * 242) ? tables().syn[index] : 0;
}

extern "C" int acb_block_fec(acb_msg_t *m)
{
	/* acars.c:123-207 */
	const FecTables &t = tables();
	constexpr unsigned char ETX = 0x83, STX = 0x02;
	constexpr int MAXPERR = 3;
	if (m->len < 13 || m->len > ACB_TXTMAX) return 0;
	m->txt[12] = (unsigned char)((m->txt[12] & (ETX | STX)) | (ETX & STX));   /* acars.c:132-133 */

	int bad[MAXPERR], nbad = 0;
	for (int i = 0; i < m->len; i++)
		if (!odd_parity(m->txt[i])) {
			if (nbad < MAXPERR) bad[nbad] = i;
			nbad++;
		}
	if (nbad > MAXPERR) return 0;
	m->err = nbad;

	uint16_t crc = 0;
	for (int i = 0; i < m->len; i++) crc = crc_step(t, crc, m->txt[i]);
	crc = crc_step(t, crc, m->crc[0]);
	crc = crc_step(t, crc, m->crc[1]);

	if (nbad) {
		if (!repair_parity(t, m, crc, bad, nbad)) return 0;
	} else if (crc) {
		if (!repair_double(t, m, crc)) return 0;
	}

	int still = 0;
	for (int i = 0; i < m->len; i++) {          /* acars.c:194-207 */
		if (!odd_parity(m->txt[i])) still++;
		m->txt[i] &= 0x7f;
	}
	return still == 0;
}

/* ------------------------------------------------------------------ frame sync on the host */

namespace {
struct ViewAcc {
	acb_frame_view_t *v;
	int &state() { return *v->state; }
	int &nbits() { return *v->nbits; }
	int &bitcount() { return *v->bitcount; }
	int &blk_len() { return *v->blk_len; }
	int &blk_err() { return *v->blk_err; }
	unsigned &msk_s() { return *v->msk_s; }
	double &msk_df() { return *v->msk_df; }
	double &lvlsum() { return *v->lvlsum; }
	void txt_put(int i, unsigned char r) { v->txt[i] = r; }
	unsigned char txt_get(int i) { return v->txt[i]; }
	void crc_put(int i, unsigned char r) { v->crc[i] = r; }
	bool frame_begin() { return v->frame_begin ? v->frame_begin(v->user) != 0 : true; }
	void frame_emit() { if (v->frame_emit) v->frame_emit(v->user); }
};
} // namespace

extern "C" void acb_frame_byte(acb_frame_view_t *v, unsigned char r)
{
	ViewAcc a{ v };
	acb::frame_byte(a, r);
}
