/*
 * demodMSK + putbit + decodeAcars for one channel, written once for the CUDA kernel k_demod
 * (kernels.cu; L lanes of a warp per channel) and for the single-lane host emulation the CPU tests
 * build (tests/host/demod_emul.cpp, test infrastructure only — the shipped library has no CPU path).
 *
 * Reference: msk.c:67-137 (demodMSK), msk.c:53-63 (putbit), acars.c:239-375 (decodeAcars/resetAcars).
 * Numerics contract: SURVEY.md §8a — every rounding of the reference is replayed in its order; the
 * explicit round-to-nearest intrinsics below are never contracted by the compiler (the host build uses
 * -ffp-contract=off).
 *
 * Shape of one loop iteration = one bit period.  The bit clock fires every 5.19..5.23 envelope
 * samples (|MskDf| <= 0.0038: the PLL's error input is a normalised component, msk.c:110-130), and
 * after a fire MskClk restarts in [-s/2, s/2), so the next fire comes exactly 5 or 6 samples later.
 * The fast path checks that (two compares on the bit-clock chain) and then
 *   - advances the two cheap serial chains (VCO phase, bit clock) six steps, rounded step by step
 *     like the reference's loop,
 *   - lets the L lanes of the channel split the six in*cexp(-j phi) mixer evaluations (the
 *     expensive, mutually independent part of a bit period) and drop them into the channel's ring,
 *   - runs the matched filter / normalisation / decision / PLL once.
 * Anything else (start-up from a foreign state, the last samples of a launch) takes the general
 * path: the reference's loop as written, sample by sample.
 *
 * Instruction-count notes (the kernel is latency bound: one warp per scheduler issues one dependent
 * instruction every ~4 cycles, so time = instructions per bit):
 *   - the ring is kept twice (rows r and r+11) so the matched filter reads 11 consecutive rows from
 *     its start index with immediate offsets, no modulo;
 *   - h[o + 12 j] is stored transposed (h2[o][j]): three 16-byte loads instead of eleven;
 *   - only ONE of the two normalising divisions (msk.c:111) is evaluated: the decision needs the
 *     sign of one component and the PLL the value of the other; the sign of x/d is the sign of x
 *     unless the quotient underflows, which a guard sends to the exact path;
 *   - the matched-filter phase index uses 1/s from a 3-term series in MskDf and replays the
 *     reference's exact division only when the value lands within 1e-4 of an integer.
 */
#ifndef ACB_DEMOD_CORE_H
#define ACB_DEMOD_CORE_H

#include <math.h>
#include <stdint.h>
#include <string.h>

#include "acb_internal.h"
#include "frame_sm.h"

namespace acb {

/* loop unrolling is a request to nvcc's device pass; the host compilers that build the same loop (nvcc's host pass,
 * hostmath.cpp, the tests' emulation) are not asked */
#if defined(__CUDA_ARCH__)
#define DC_UNROLL _Pragma("unroll")
#else
#define DC_UNROLL
#endif

#if defined(__CUDA_ARCH__)
#define DC_DADD(a, b) __dadd_rn((a), (b))
#define DC_DMUL(a, b) __dmul_rn((a), (b))
#define DC_DDIV(a, b) __ddiv_rn((a), (b))
#define DC_DSQRT(a) __dsqrt_rn((a))
#define DC_FADD(a, b) __fadd_rn((a), (b))
#define DC_FMUL(a, b) __fmul_rn((a), (b))
#define DC_D2F(a) __double2float_rn((a))
#define DC_D2I_RZ(a) __double2int_rz((a))
#define DC_D2LL(a) __double_as_longlong((a))
#define DC_LL2D(a) __longlong_as_double((a))
#define DC_LOINT(a) __double2loint((a))
#else
/* host emulation: IEEE double/float arithmetic with contraction off is the same rounding */
#define DC_DADD(a, b) ((double)(a) + (double)(b))
#define DC_DMUL(a, b) ((double)(a) * (double)(b))
#define DC_DDIV(a, b) ((double)(a) / (double)(b))
#define DC_DSQRT(a) sqrt((double)(a))
#define DC_FADD(a, b) ((float)(a) + (float)(b))
#define DC_FMUL(a, b) ((float)(a) * (float)(b))
#define DC_D2F(a) ((float)(a))
static inline int dc_d2i_rz(double a) { return !(a == a) ? 0 : a <= -2147483648.0 ? INT32_MIN : a >= 2147483647.0 ? INT32_MAX : (int)a; }
static inline long long dc_d2ll(double a) { long long v; memcpy(&v, &a, 8); return v; }
static inline double dc_ll2d(long long a) { double v; memcpy(&v, &a, 8); return v; }
#define DC_D2I_RZ(a) dc_d2i_rz((a))
#define DC_D2LL(a) dc_d2ll((a))
#define DC_LL2D(a) dc_ll2d((a))
#define DC_LOINT(a) ((int)(uint32_t)dc_d2ll((a)))
#endif

struct DemodRegs {
	double phi, df, lvlsum;
	float clk;
	int bitcount;
	unsigned S, idx;
	int nbits, state;
	unsigned outbits;
	int blk_len, blk_err;
	unsigned long long pos, soh_pos;
	unsigned long long pos0;          /* pos at the start of the launch */
	int fire_n;                       /* sample of the launch that fired the current bit: its position is pos0 + fire_n */
};

struct alignas(8) DcF2 { float x, y; };            /* one ring entry: (re, im) of in*cexp(-j phi), msk.c:90 */
struct alignas(16) DcF4 { float x, y, z, w; };
struct alignas(16) DcD2 { double x, y; };          /* table entry (hi, lo) */

constexpr int DEMOD_LOOK = 6;         /* samples examined per iteration (bit period = 5.19..5.23) */
constexpr int RING_ROWS = 2 * FLEN;   /* the ring, kept twice */

/* one warp's (or the host emulation's single lane's) shared state: CPW = channels per warp */
template <int CPW> struct alignas(16) DemodShared {
	DcD2 tcos[64], tsin[64];          /* cos/sin(k*pi/32) as double-double */
	DcF4 h2[MFLTOVER + 1][3];         /* h2[o] = h[o + 12 j], j = 0..11 (msk.c:104-107; j = 11 unused): three 16-byte loads */
	DcF2 ring[RING_ROWS][CPW];
};

/* Double constants of the loop.  On the device they live in constant memory: a 64-bit immediate costs two
 * uniform-register moves per use in SASS (a sixth of the loop's instructions before this), a constant-bank
 * operand costs nothing. */
struct DcConsts {
	double two_pi, s0, thr, inv_s0, pllc, pllk;
	double sc_magic, k32_pi, pi32_a, pi32_b, pi32_c;      /* sincos_vco: 32/pi, three-part pi/32 */
	double s9, s7, s5, s3, c8, c6, c4, c2;               /* Taylor coefficients of sin r, cos r - 1 */
	double half, six, twelve, eps_d, guard_u, guard_df;
};
#define DC_CONSTS_INIT { \
	2.0 * M_PI, 1800.0 / 12500 * 2.0 * M_PI /* msk.c:81 */, 3 * M_PI / 2.0 /* msk.c:96,100 */, \
	1.0 / (1800.0 / 12500 * 2.0 * M_PI), (double)0.52f /* PLLC, msk.c:66 */, \
	(1.0 - (double)0.52f) * (double)38e-4f /* (1.0-PLLC)*PLLG, msk.c:130 */, \
	6755399441055744.0 /* 1.5 * 2^52 */, 0x1.45f306dc9c883p+3, 0x1.921fb54442d18p-4, 0x1.1a62633145c07p-58, -0x1.f1976b7ed8fbcp-114, \
	1.0 / 362880, -1.0 / 5040, 1.0 / 120, -1.0 / 6, 1.0 / 40320, -1.0 / 720, 1.0 / 24, -0.5, \
	0.5, 6.0, 12.0, 1e-8 /* msk.c:111 */, 1e-4, 0.01 }
#if defined(__CUDACC__)
static __constant__ DcConsts c_dcc = DC_CONSTS_INIT;
static __device__ DcConsts g_dcc = DC_CONSTS_INIT;      /* the same in global memory: see demod_run */
#endif
static const DcConsts h_dcc = DC_CONSTS_INIT;
#if defined(__CUDA_ARCH__)
#define DCK c_dcc
#else
#define DCK h_dcc
#endif

/* cos(p), sin(p) for p in [0, 2*pi] — the VCO phase after msk.c:82-83.  p = k*pi/32 + r with
 * |r| <= pi/64 (three-part pi/32, so r keeps full relative accuracy next to the zeros of sin and
 * cos, which are table points with exact entries); short Taylor polynomials for sin r and
 * cos r - 1; angle addition against the double-double table.  Max error 1.72 ulp (typ. < 0.6), i.e. the
 * class of CUDA's own sincos, also for p in [-4 pi, 8 pi] (a foreign MskPhi); tests/test_demod_primitives.py
 * asserts <= 1.75 ulp against mpmath / 80-bit references and that nvcc's build returns g++'s bits.  See
 * DESIGN.md for why ~1 ulp here is invisible after the (float) rounding of in*cexp(-j p) (msk.c:90). */
ACB_HD void sincos_vco(const DcConsts &DCK_, double p, const DcD2 *tcos, const DcD2 *tsin, double &sn, double &cs)
{
	const double t = fma(p, DCK_.k32_pi, DCK_.sc_magic);       /* p * 32/pi, rounded to integer */
	const int k = DC_LOINT(t) & 63;
	const double kd = t - DCK_.sc_magic;
	double r = fma(-kd, DCK_.pi32_a, p);
	r = fma(-kd, DCK_.pi32_b, r);
	r = fma(-kd, DCK_.pi32_c, r);
	const double r2 = r * r;
	double sp = fma(r2, DCK_.s9, DCK_.s7);
	sp = fma(sp, r2, DCK_.s5);
	sp = fma(sp, r2, DCK_.s3);
	const double sr = fma(r * r2, sp, r);                    /* sin r */
	double cp = fma(r2, DCK_.c8, DCK_.c6);
	cp = fma(cp, r2, DCK_.c4);
	cp = fma(cp, r2, DCK_.c2);
	const double cm = r2 * cp;                               /* cos r - 1 */
	const DcD2 C = tcos[k], S = tsin[k];
	cs = C.x + fma(-S.x, sr, fma(C.x, cm, C.y));
	sn = S.x + fma(C.x, sr, fma(S.x, cm, S.y));
}

/* Round a double to float precision, result kept as a double: (double)(float)x.  MskClk (msk.c:95) is a
 * float updated with a double addend, six times per bit.
 *   F2F = false: integer ops on the bit pattern, bit-identical to the conversion pair for zero and for
 *         every x with FLT_MIN <= |x| whose float image is finite (it rounds to 24 bits at every magnitude,
 *         so it differs below FLT_MIN, including the x that round up to FLT_MIN; MskClk lives in [-0.5, 5.3];
 *         differences of such values are zero or >= 2^-53 in magnitude, so neither range can occur): 5 ALU
 *         ops, ~22 cycles of latency.  tests/test_demod_primitives.py asserts both the identity and the range;
 *   F2F = true: the conversion pair itself: 2 instructions on the quarter-rate conversion unit, ~45 cycles. */
template <bool F2F> ACB_HD double round_to_f32(double x)
{
	if (F2F) return (double)DC_D2F(x);
	unsigned long long u = (unsigned long long)DC_D2LL(x);
	u += 0x0FFFFFFFull + ((u >> 29) & 1ull);
	u &= ~0x1FFFFFFFull;
	return DC_LL2D((long long)u);
}

/* one step of the VCO phase (msk.c:82-83) */
ACB_HD double phase_step(const DcConsts &DCK_, double p, double sv)
{
	p = DC_DADD(p, sv);
	return (p >= DCK_.two_pi) ? DC_DADD(p, -DCK_.two_pi) : p;
}

/* in * cexp(-j p) rounded to float complex (msk.c:86-91) */
ACB_HD DcF2 mix_sample(const DcConsts &DCK_, float x, double p, const DcD2 *tcos, const DcD2 *tsin)
{
	double sn, cs;
	sincos_vco(DCK_, p, tcos, tsin, sn, cs);
	const double xd = (double)x;
	DcF2 o;
	o.x = DC_D2F(DC_DMUL(xd, cs));
	o.y = DC_D2F(DC_DMUL(xd, -sn));
	return o;
}

/* msk.c:100-104 — the bit clock steps back by 3*pi/2 and the matched filter's phase index is
 * o = (int)(12*(MskClk/s + 0.5)), capped at 12.  1/s = (1/S0)(1 - x + x^2), x = MskDf/S0 (|x| < 5e-3 while
 * the PLL is in charge: 1e-7 relative) gives the value to ~1e-6; only when that lands within 1e-4 of an
 * integer (where the truncation could differ), or MskDf is outside the PLL's range, is the reference's exact
 * division sequence replayed. */
template <bool F2F> ACB_HD int bit_clock_fire(const DcConsts &DCK_, double &clkd, double sv, double df)
{
	clkd = round_to_f32<F2F>(DC_DADD(clkd, -DCK_.thr));
	const double xs = DC_DMUL(df, DCK_.inv_s0);
	const double inv_s = fma(DCK_.inv_s0, fma(xs, xs, -xs), DCK_.inv_s0);
	double u = fma(DC_DMUL(clkd, inv_s), DCK_.twelve, DCK_.six);
	if (!(fabs(u - rint(u)) >= DCK_.guard_u) || !(fabs(df) <= DCK_.guard_df))
		u = DC_DMUL(DCK_.twelve, DC_DADD(DC_DDIV(clkd, sv), DCK_.half));
	const int o = DC_D2I_RZ(u);
	return o < 0 ? 0 : (o > MFLTOVER ? MFLTOVER : o);
}

/* The loop.  `in` points at the channel's first envelope sample of this launch, samples nch floats
 * apart.  L lanes per channel: lane `sub` of group `grp`; all lanes of a group carry identical
 * registers and only differ in which mixer evaluations they contribute.  Env supplies the warp
 * collectives (identity on the host).  FrameAcc is frame_sm.h's accessor over `r`; it reads r.pos0 +
 * r.fire_n when it needs a sample position. */
template <int L, bool F2F, bool PIN, class Env, bool RAGGED = false, class FrameAcc, int CPW>
ACB_HD void demod_run(DemodRegs &r, DemodShared<CPW> &sm, const float *in, int nch, int nsamp, int sub, int grp,
                      FrameAcc &acc)
{
	constexpr int ROUNDS = (DEMOD_LOOK + L - 1) / L;         /* mixer evaluations per lane and bit */
	/* the loop's double constants, held in registers for the whole launch (left to itself the compiler re-reads
	 * them from the constant bank into uniform registers every iteration: 26 instructions of ~440) */
#if defined(__CUDA_ARCH__)
	/* PIN: read through a volatile global pointer — a value the compiler cannot re-create at its uses; costs ~50
	 * registers per thread, which matters when the kernel shares the SMs with the channelizer (contexts with
	 * many chains run the unpinned form) */
	DcConsts DCK_;
	if (!PIN) DCK_ = DCK;
	else {
		const volatile double *src = reinterpret_cast<const volatile double *>(&g_dcc);
		double *dst = reinterpret_cast<double *>(&DCK_);
DC_UNROLL
		for (int i = 0; i < (int)(sizeof(DcConsts) / sizeof(double)); i++) dst[i] = src[i];
	}
#else
	const DcConsts DCK_ = DCK;
#endif
	r.pos0 = r.pos;
	double clkd = (double)r.clk;             /* MskClk: a float value carried in a double register */
	int n = 0;
	/* This lane's envelope samples of the coming iteration (sample n + sub + i*L of round i), loaded one iteration
	 * ahead: an iteration's first sample is only known once the previous bit clock has fired, and a load issued then
	 * has a whole bit period (~2000 cycles) to come back from L2/HBM instead of stalling the mixer (the loads were
	 * 23 % of the kernel's cycles as `long scoreboard` stalls when they were issued where they are used).  Indices
	 * past the launch are clamped: such values are never stored (the general path loads its own). */
	float xn[ROUNDS];
	const int last = nsamp - 1;
DC_UNROLL
	for (int i = 0; i < ROUNDS; i++) {
		const int k = sub + i * L;
		xn[i] = nsamp > 0 ? in[(size_t)(k < last ? k : last) * nch] : 0.f;
	}
	/* Channels of a warp consume 5 or 6 samples per iteration each, so they finish a few iterations apart: finished
	 * groups idle through the general path (m <= 0).  The "does anybody still have samples" vote (a warp
	 * reconvergence point, 7 % of the kernel's cycles when taken every iteration) is only needed near the end: as long
	 * as the lane furthest ahead has 6*q samples left, q more iterations cannot exhaust anybody. */
	int budget = 0;                          /* iterations that need no vote */
	bool hunting = r.state == F_WSYN;        /* acars.c:254: the bit-sliding SYN search, tested once per bit */
	for (;;) {
		if (budget == 0) {
			if (!Env::any(n < nsamp)) break;
			/* RAGGED: the groups of a warp have different sample counts, so the budget must still be the same for the whole
			 * warp; any budget >= 1 is correct (a group that runs out idles through the general path), the largest
			 * remaining count keeps the votes as rare as in the even case */
			if constexpr (RAGGED) budget = Env::max(nsamp - n) / DEMOD_LOOK;
			else budget = (nsamp - Env::max(n)) / DEMOD_LOOK;
			if (budget < 1) budget = 1;
		}
		budget--;
		const int m = nsamp - n;
		/* VCO step is constant until the next bit (msk.c:81): MskDf only changes in the bit path */
		const double sv = DC_DADD(DCK_.s0, r.df);
		const double fire_at = fma(sv, -DCK_.half, DCK_.thr);    /* 3*pi/2 - s/2: the halving is exact */

		/* the two cheap serial chains: phase (msk.c:82-83) and bit clock (msk.c:95-96), each rounded
		 * step by step exactly like the reference's loop */
		double pk[DEMOD_LOOK], ck[DEMOD_LOOK];
		{
			double p = r.phi, c = clkd;
DC_UNROLL
			for (int k = 0; k < DEMOD_LOOK; k++) {
				p = phase_step(DCK_, p, sv);
				c = round_to_f32<F2F>(DC_DADD(c, sv));
				pk[k] = p;
				ck[k] = c;
			}
		}
		/* this lane's mixer evaluations, before anything is decided: they are the long pole of a bit period
		 * and depend on the phase chain only (lanes past the sixth sample, and everybody when the general
		 * path is taken, compute a value nobody stores) */
		DcF2 mv[ROUNDS];
		const bool inside = m >= DEMOD_LOOK;                   /* all six candidate samples exist */
DC_UNROLL
		for (int i = 0; i < ROUNDS; i++) {
			const int k0 = i * L;
			double ps = pk[k0];
DC_UNROLL
			for (int j = 1; j < L; j++)
				if (k0 + j < DEMOD_LOOK && sub == j) ps = pk[k0 + j];
			mv[i] = mix_sample(DCK_, xn[i], ps, sm.tcos, sm.tsin);
		}
		int cnt = 0;                 /* samples consumed this iteration */
		bool fired = false;
		int o = 0;
		/* the bit clock rises by sv > 0 per step, so "not before sample 5, at sample 6 at the latest" is
		 * two compares */
		const bool regular = inside & (ck[3] < fire_at) & (ck[5] >= fire_at);
		/* no vote: the lanes of a group carry identical registers, so the branch is uniform per group, and groups
		 * share nothing — a group on the general path just makes the warp run both arms once (both arms pass the
		 * same two warp barriers) */
		if (regular) {
			const bool five = ck[4] >= fire_at;
			cnt = five ? 5 : 6;
			fired = true;
			r.phi = five ? pk[4] : pk[5];
			clkd = five ? ck[4] : ck[5];
DC_UNROLL
			for (int i = 0; i < ROUNDS; i++) {                     /* next iteration's samples: in flight during the bit part */
				const int k = n + cnt + sub + i * L;
				xn[i] = in[(size_t)(k < last ? k : last) * nch];
			}
			o = bit_clock_fire<F2F>(DCK_, clkd, sv, r.df);
			if (L > 1) Env::sync();  /* the previous bit's matched filter has read the rows being replaced */
DC_UNROLL
			for (int i = 0; i < ROUNDS; i++) {
				const int k = i * L + sub;
				if (k < cnt) {
					unsigned row = r.idx + (unsigned)k;
					row = row >= (unsigned)FLEN ? row - FLEN : row;
					sm.ring[row][grp] = mv[i];
					sm.ring[row + FLEN][grp] = mv[i];
				}
			}
			if (L > 1) Env::sync();
			r.idx += (unsigned)cnt;
			r.idx = r.idx >= (unsigned)FLEN ? r.idx - FLEN : r.idx;
		} else {
			/* general path: msk.c:74-96 as written, one sample at a time, every lane for itself (lane 0
			 * of the group stores) */
			if (L > 1) Env::sync();
			const int mm = m < DEMOD_LOOK ? m : DEMOD_LOOK;
			double p = r.phi, c = clkd;
			for (int k = 0; k < mm; k++) {
				p = phase_step(DCK_, p, sv);
				const DcF2 v = mix_sample(DCK_, in[(size_t)(n + k) * nch], p, sm.tcos, sm.tsin);
				if (sub == 0) {
					sm.ring[r.idx][grp] = v;
					sm.ring[r.idx + FLEN][grp] = v;
				}
				r.idx = r.idx + 1 == (unsigned)FLEN ? 0u : r.idx + 1;
				c = round_to_f32<F2F>(DC_DADD(c, sv));
				cnt++;
				if (c >= fire_at) { fired = true; break; }
			}
			r.phi = p;
			clkd = c;
			if (fired) o = bit_clock_fire<F2F>(DCK_, clkd, sv, r.df);
DC_UNROLL
			for (int i = 0; i < ROUNDS; i++) {
				const int k = n + cnt + sub + i * L;
				xn[i] = last >= 0 ? in[(size_t)(k < last ? k : last) * nch] : 0.f;
			}
			if (L > 1) Env::sync();
		}
		r.fire_n = n + cnt - 1;                                /* the sample that fired the bit */

		if (fired) {
			/* matched filter (msk.c:103-107): 11 taps out of the x12 oversampled half cosine */
			float vr = 0.f, vi = 0.f;
			const DcF4 h0 = sm.h2[o][0], h1 = sm.h2[o][1], h2 = sm.h2[o][2];
			const float hh11[12] = { h0.x, h0.y, h0.z, h0.w, h1.x, h1.y, h1.z, h1.w, h2.x, h2.y, h2.z, h2.w };
			const DcF2 *rp = &sm.ring[r.idx][grp];
DC_UNROLL
			for (int j = 0; j < FLEN; j++) {
				const float hh = hh11[j];
				const DcF2 e = rp[(size_t)j * CPW];
				vr = DC_FADD(vr, DC_FMUL(hh, e.x));
				vi = DC_FADD(vi, DC_FMUL(hh, e.y));
			}
			/* normalise (msk.c:110-113): cabsf is (float)sqrt((double)x*x + (double)y*y) in glibc */
			const double dvr = (double)vr, dvi = (double)vi;
			const float lvl = DC_D2F(DC_DSQRT(DC_DADD(DC_DMUL(dvr, dvr), DC_DMUL(dvi, dvi))));
			const double d = DC_DADD((double)lvl, DCK_.eps_d);
			r.lvlsum = DC_DADD(r.lvlsum, (double)DC_FMUL(DC_FMUL(lvl, lvl), 0.25f));
			r.bitcount++;

			/* decision + phase error (msk.c:115-127).  v/(lvl+1e-8): the decision looks at the sign of one
			 * component, the PLL takes the value of the other */
			const bool odd = (r.S & 1u) != 0, inv = (r.S & 2u) != 0;
			const float vs = odd ? vi : vr;                        /* vo before the division */
			const float vq = DC_D2F(DC_DDIV(odd ? dvr : dvi, d));  /* the other component, normalised */
			bool vo_ge0, bit;
			if (fabsf(vs) >= 1e-30f && lvl < 1e6f) {               /* quotient cannot underflow: sign(vs/d) = sign(vs) */
				vo_ge0 = vs > 0.f;
				bit = vo_ge0 != inv;
			} else {
				const float vo = DC_D2F(DC_DDIV((double)vs, d));
				vo_ge0 = vo >= 0.f;
				bit = (inv ? -vo : vo) > 0.f;
			}
			const double dphi = (double)((vo_ge0 != odd) ? vq : -vq);

			/* putbit (msk.c:53-63) */
			r.outbits >>= 1;
			if (bit) r.outbits |= 0x80u;
			if (--r.nbits <= 0) {
				if (hunting) {
					/* decodeAcars' WSYN state (acars.c:254-268), the state a channel is in whenever nobody transmits: kept
					 * out of frame_byte's state dispatch, which compiles to an indirect branch */
					const unsigned ob = r.outbits & 0xffu;
					if (ob == C_SYN || ob == C_NSYN) {
						if (ob == C_NSYN) r.S ^= 2u;           /* inverted polarity */
						r.state = F_SYN2;
						r.nbits = 8;
						hunting = false;
					} else {
						r.nbits = 1;
					}
				} else {
					frame_byte(acc, (unsigned char)r.outbits);
					hunting = r.state == F_WSYN;
				}
#if defined(__CUDA_ARCH__)
				{
					int h = hunting;                     /* an opaque copy: the compiler must not fold the test back into the dispatch */
					asm volatile("" : "+r"(h));
					hunting = h != 0;
				}
#endif
			}
			r.S++;

			/* PLL filter (msk.c:130) — after putbit, so a frame resync's MskDf=0 is filtered too */
			r.df = DC_DADD(DC_DMUL(DCK_.pllc, r.df), DC_DMUL(DCK_.pllk, dphi));
		}
		n += cnt;
	}
	r.pos = r.pos0 + (unsigned long long)nsamp;
	r.clk = (float)clkd;
}

} // namespace acb
#endif
