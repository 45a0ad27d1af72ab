/*
 * TEST INFRASTRUCTURE — NOT PRODUCT CODE.
 *
 * CPU restatement of the overlapping-window channelizer (acb_config_t.taps > K, include/acars_b200.h).  There is no
 * reference counterpart, so this IS the definition, written literally: with H = taps - K, output row m of a stream is
 *
 *     dm[m] = | sum_{i<taps} x[m*K - H + i] * w[i] |
 *
 * over the whole stream given as one array, in ascending tap order, with the same rounded float operations as the
 * reference's boxcar (rtl.c:350-353: 4 products + 4 sums per complex tap; air.c:317-318: 2 + 2 per real tap), and the
 * terms whose sample index is negative OMITTED (not zero-filled: a zero u8 byte converts to -127.37).  |.| is cabsf
 * = hypotf.  At taps == K these reduce to orc_channelize, orc_channelize_real and orc_channelize_cs16's folded form
 * (variant 2), which tests/test_ovl_oracle.py asserts bit for bit.
 *
 * Built by tests/ovl_refs.py with -O2 -ffp-contract=off (no contraction: every product is rounded).
 */
#include <math.h>
#include <stddef.h>
#include <stdint.h>

/* u8 IQ (rtl.c): x = (float)u8 - 127.37f; wf: nch x 2*taps (re, im); dm: nch x nout */
void orc_channelize_ovl(const uint8_t *iq, long long nsamp, int K, int taps, int nch, const float *wf, float *dm)
{
	const long long nout = nsamp / K, H = taps - K;
	for (long long m = 0; m < nout; m++) {
		for (int ch = 0; ch < nch; ch++) {
			const float *w = wf + (size_t)ch * 2 * taps;
			float dr = 0, di = 0;
			for (int i = 0; i < taps; i++) {
				const long long n = m * K - H + i;
				if (n < 0) continue;
				float a = (float)iq[2 * n] - 127.37f, b = (float)iq[2 * n + 1] - 127.37f;
				float c = w[2 * i], d = w[2 * i + 1];
				float pr = a * c - b * d, pi = a * d + b * c;
				dr = dr + pr;
				di = di + pi;
			}
			dm[(size_t)ch * nout + m] = hypotf(dr, di);
		}
	}
}

/* CS16 IQ (soapy.c / sdrplay.c with the power-of-two scale folded into the table): x = (float)int16 */
void orc_channelize_ovl_cs16(const int16_t *iq, long long nsamp, int K, int taps, int nch, const float *wf, float *dm)
{
	const long long nout = nsamp / K, H = taps - K;
	for (long long m = 0; m < nout; m++) {
		for (int ch = 0; ch < nch; ch++) {
			const float *w = wf + (size_t)ch * 2 * taps;
			float dr = 0, di = 0;
			for (int i = 0; i < taps; i++) {
				const long long n = m * K - H + i;
				if (n < 0) continue;
				float a = (float)iq[2 * n], b = (float)iq[2 * n + 1];
				float c = w[2 * i], d = w[2 * i + 1];
				float pr = a * c - b * d, pi = a * d + b * c;
				dr = dr + pr;
				di = di + pi;
			}
			dm[(size_t)ch * nout + m] = hypotf(dr, di);
		}
	}
}

/* float32 real (air.c): D += w[i] * x */
void orc_channelize_ovl_real(const float *x, long long nsamp, int K, int taps, int nch, const float *wf, float *dm)
{
	const long long nout = nsamp / K, H = taps - K;
	for (long long m = 0; m < nout; m++) {
		for (int ch = 0; ch < nch; ch++) {
			const float *w = wf + (size_t)ch * 2 * taps;
			float dr = 0, di = 0;
			for (int i = 0; i < taps; i++) {
				const long long n = m * K - H + i;
				if (n < 0) continue;
				float pr = w[2 * i] * x[n], pi = w[2 * i + 1] * x[n];
				dr = dr + pr;
				di = di + pi;
			}
			dm[(size_t)ch * nout + m] = hypotf(dr, di);
		}
	}
}
