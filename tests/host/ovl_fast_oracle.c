/*
 * TEST INFRASTRUCTURE — NOT PRODUCT CODE.
 *
 * CPU restatement of the polyphase fast form of the overlapping-window channelizer (ACB_FLAG_FAST_FILTER, taps > K,
 * include/acars_b200.h), operation for operation as k_channelize_ovl_fast computes it, so the GPU kernel is held to it bit
 * for bit while tests/test_ovl_fast_oracle.py holds IT to the exact definition (tests/host/ovl_oracle.c) and to that
 * definition evaluated in float64.
 *
 * Built by tests/ovl_fast_refs.py with -O2 -ffp-contract=off (no contraction: every FMA is an explicit fmaf).
 */
#include <math.h>
#include <stddef.h>
#include <stdint.h>

/* Polyphase fast form (ACB_FLAG_FAST_FILTER, k_channelize_ovl_fast restated operation for operation).  With every
 * channel on the raster, w[i] = h[i] * exp(-j*2*pi*k*(i - H)/K) * scale, and
 *   z_m[n] = sum_r p[n + H + r*K] * x[m*K + n + r*K]      p = fl(K*h), r <= 0 ascending (ascending tap order), one fmaf
 *                                                         per component, terms with a negative tap or sample index omitted
 *   z'[n]  = z[n] + z[n + K/2]                             n < K/2 (k even)
 *   Y_r    = the 4-point DFT across the quarters of z' (as k_channelize_dft1), r = (k/2) mod 4
 *   D      = sum_{n2 < K/8} T[n2] * Y_r[n2]                four fmaf chains in n2 order, T = tw (acb_fast_plan*)
 * `h`: taps floats (acb_build_lowpass); `kbin`, `tw`: nch bins and nch x K/4 twiddles; `cvt` converts sample n. */
static void ovl_fast(int K, int taps, long long nout, int nch, const float *h, const int *kbin, const float *tw,
                     void (*cvt)(const void *, long long, float *, float *), const void *src, float *dm)
{
	const int H = taps - K, N2 = K / 4, N8 = K / 8, half = K / 2;
	float p[16 * 2048 + 1];
	float zr[2048], zi[2048];
	for (int i = 0; i < taps; i++) p[i] = (float)K * h[i];
	for (long long m = 0; m < nout; m++) {
		for (int n = 0; n < K; n++) {
			float a = 0, b = 0;
			for (long long r = -((n + H) / K); r <= 0; r++) {
				const long long smp = m * K + n + r * K;
				if (smp < 0) continue;
				float xr, xi;
				cvt(src, smp, &xr, &xi);
				const float pk = p[n + H + r * K];
				a = fmaf(pk, xr, a);
				b = fmaf(pk, xi, b);
			}
			zr[n] = a; zi[n] = b;
		}
		for (int n = 0; n < half; n++) { zr[n] = zr[n] + zr[n + half]; zi[n] = zi[n] + zi[n + half]; }
		for (int ch = 0; ch < nch; ch++) {
			const int res = (((kbin[ch] / 2) % 4) + 4) % 4;
			const float *t = tw + (size_t)ch * N2 * 2;
			float ax = 0, ay = 0, bx = 0, by = 0;
			for (int n2 = 0; n2 < N8; n2++) {
				const float z0r = zr[n2], z1r = zr[N8 + n2], z2r = zr[2 * N8 + n2], z3r = zr[3 * N8 + n2];
				const float z0i = zi[n2], z1i = zi[N8 + n2], z2i = zi[2 * N8 + n2], z3i = zi[3 * N8 + n2];
				const float s02r = z0r + z2r, s13r = z1r + z3r, s02i = z0i + z2i, s13i = z1i + z3i;
				const float d02r = z0r - z2r, d02i = z0i - z2i;
				const float wjr = z1i - z3i, wji = z3r - z1r;          /* -j (z1 - z3) */
				float yr, yi;
				switch (res) {
				case 0: yr = s02r + s13r; yi = s02i + s13i; break;
				case 2: yr = s02r - s13r; yi = s02i - s13i; break;
				case 1: yr = d02r + wjr; yi = d02i + wji; break;
				default: yr = d02r - wjr; yi = d02i - wji; break;
				}
				const float tr = t[2 * n2], ti = t[2 * n2 + 1];
				ax = fmaf(yr, tr, ax);
				ay = fmaf(yr, ti, ay);
				bx = fmaf(yi, tr, bx);
				by = fmaf(yi, ti, by);
			}
			const float re = ax - by, im = ay + bx;
			dm[(size_t)ch * nout + m] = sqrtf(fmaf(re, re, im * im));
		}
	}
}

static void cvt_u8(const void *src, long long n, float *a, float *b)
{
	const uint8_t *iq = (const uint8_t *)src;
	*a = (float)iq[2 * n] - 127.37f;
	*b = (float)iq[2 * n + 1] - 127.37f;
}

static void cvt_cs16(const void *src, long long n, float *a, float *b)
{
	const int16_t *iq = (const int16_t *)src;
	*a = (float)iq[2 * n];
	*b = (float)iq[2 * n + 1];
}

/* u8 IQ: x = (float)u8 - 127.37f (exact); dm: nch x nout */
void orc_channelize_ovl_fast(const uint8_t *iq, long long nsamp, int K, int taps, int nch, const float *h, const int *kbin,
                             const float *tw, float *dm)
{
	ovl_fast(K, taps, nsamp / K, nch, h, kbin, tw, cvt_u8, iq, dm);
}

/* CS16 IQ: x = (float)int16; the variant's scale is in tw (acb_fast_plan_cs16) */
void orc_channelize_ovl_fast_cs16(const int16_t *iq, long long nsamp, int K, int taps, int nch, const float *h, const int *kbin,
                                  const float *tw, float *dm)
{
	ovl_fast(K, taps, nsamp / K, nch, h, kbin, tw, cvt_cs16, iq, dm);
}
