/*
 * TEST INFRASTRUCTURE — NOT PRODUCT CODE.
 *
 * CPU restatement of the pre-sum of the polyphase fast form of the overlapping-window channelizer for real input
 * (ACB_FLAG_FAST_FILTER_REAL, taps > K, include/acars_b200.h), operation for operation as k_channelize_ovl_rdft computes
 * it.  The kernel takes each channel's bin of a pre-summed row with k_channelize_rdft's operations, so the fast envelope
 * is the oracle's orc_channelize_rdft (oracle/acars_oracle.c) of these rows; tests/test_ovl_fast_real_oracle.py holds
 * that to the exact definition (tests/host/ovl_oracle.c) and to the definition evaluated in float64, and
 * tests/test_gpu_ovl_fast_real.py holds the GPU kernel to it bit for bit.
 *
 * Built by tests/ovl_fast_real_refs.py with -O2 -ffp-contract=off (no contraction: every FMA is an explicit fmaf).
 */
#include <math.h>
#include <stddef.h>
#include <stdlib.h>

/*   z[m*K + n] = sum_r p[n + H + r*K] * x[m*K + n + r*K],  p = fl(K*h), r <= 0 ascending (ascending tap order), one fmaf
 *                                                          per term, terms with a negative sample index omitted
 * for m < nsamp / K; h: taps floats (acb_build_lowpass), H = taps - K. */
void orc_ovl_presum_real(const float *x, long long nsamp, int K, int taps, const float *h, float *z)
{
	const int H = taps - K;
	const long long nout = nsamp / K;
	float *p = (float *)malloc((size_t)taps * sizeof(float));
	for (int i = 0; i < taps; i++) p[i] = (float)K * h[i];
	for (long long m = 0; m < nout; m++) {
		for (int n = 0; n < K; n++) {
			float a = 0;
			for (long long r = -((n + H) / K); r <= 0; r++) {
				const long long smp = m * K + n + r * K;
				if (smp < 0) continue;
				a = fmaf(p[n + H + r * K], x[smp], a);
			}
			z[m * K + n] = a;
		}
	}
	free(p);
}
