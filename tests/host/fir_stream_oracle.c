/*
 * TEST INFRASTRUCTURE — NOT PRODUCT CODE.
 *
 * CPU restatement of the short channel filter (acb_config_t.taps <= K, tables from acb_set_wf) for the two 4-byte input
 * kinds, the streaming front-ends' (air.c float32 real, soapy.c / sdrplay.c CS16 IQ).  The reference has no such mode,
 * so this IS the definition, written literally: output row m of a stream is
 *
 *     dm[m] = | sum_{i<taps} x[m*K + i] * w[i] |
 *
 * i.e. the FIRST `taps` samples of every K-sample row, over the whole stream given as one array, in ascending tap order,
 * with the reference's rounded float operations (air.c:317-318: 2 products + 2 sums per real tap; rtl.c:350-353's 4 + 4
 * per complex tap, which the CS16 front-ends use with the power-of-two scale folded into the table).  |.| is cabsf =
 * hypotf.  At taps == K these are orc_channelize_real and orc_channelize_ovl_cs16 at taps == K (the folded form), which
 * tests/test_fir_stream_oracle.py asserts bit for bit.
 *
 * (tests/host/ovl_oracle.c cannot stand in at taps < K: its H = taps - K is negative there, so it weights the LAST
 * `taps` samples of each row.)
 *
 * Built by tests/fir_stream_refs.py with -O2 -ffp-contract=off (no contraction: every product is rounded).
 */
#include <math.h>
#include <stddef.h>
#include <stdint.h>

/* float32 real (air.c): D += w[i] * x; wf: nch x 2*taps (re, im); dm: nch x nout */
void orc_channelize_fir_real(const float *x, long long nsamp, int K, int taps, int nch, const float *wf, float *dm)
{
	const long long nout = nsamp / K;
	for (long long m = 0; m < nout; m++) {
		const float *p = x + m * K;
		for (int ch = 0; ch < nch; ch++) {
			const float *w = wf + (size_t)ch * 2 * taps;
			float dr = 0, di = 0;
			for (int i = 0; i < taps; i++) {
				float pr = w[2 * i] * p[i], pi = w[2 * i + 1] * p[i];
				dr = dr + pr;
				di = di + pi;
			}
			dm[(size_t)ch * nout + m] = hypotf(dr, di);
		}
	}
}

/* CS16 IQ (interleaved I, Q): x = (float)int16 */
void orc_channelize_fir_cs16(const int16_t *iq, long long nsamp, int K, int taps, int nch, const float *wf, float *dm)
{
	const long long nout = nsamp / K;
	for (long long m = 0; m < nout; m++) {
		const int16_t *p = iq + 2 * m * K;
		for (int ch = 0; ch < nch; ch++) {
			const float *w = wf + (size_t)ch * 2 * taps;
			float dr = 0, di = 0;
			for (int i = 0; i < taps; i++) {
				float a = (float)p[2 * i], b = (float)p[2 * i + 1];
				float c = w[2 * i], d = w[2 * i + 1];
				float pr = a * c - b * d, pi = a * d + b * c;
				dr = dr + pr;
				di = di + pi;
			}
			dm[(size_t)ch * nout + m] = hypotf(dr, di);
		}
	}
}
