/*
 * CUDA kernels of the acarsdec hot path for sm_90a (H100).
 *
 *  K1  k_channelize<MODE> : u8 IQ / float32 real / CS16 IQ samples -> per-channel NCO mix x
 *                     boxcar(K) -> decimate by K -> |.|  (reference: in_callback rtl.c:334-354;
 *                     rx_callback air.c:291-341; soapy.c:232-254, sdrplay.c:215-236).  FP32-issue bound by the
 *                     reference's rounding sequence: every complex MAC is 4 rounded products
 *                     and 4 rounded sums in tap order, no FMA contraction — reproduced exactly
 *                     (explicit __f*_rn intrinsics, never contracted) so dm is bit-identical
 *                     to the strict-IEEE build of the reference.
 *      k_channelize_dft   : opt-in fast form of the u8 path (ACB_FLAG_FAST_CHANNELIZER): the same bins as a
 *                     shared 4-point DFT across the row quarters + K/4 MACs per channel; HBM-bound
 *                     (bulk copies, FFMA); messages identical, envelope within tolerance.
 *  K2  k_demod<LANES>     : demodMSK + putbit + decodeAcars, 4 or 8 lanes per channel
 *                     (reference: msk.c:67-137, acars.c:246-375), state carried in HBM between
 *                     launches; serial recurrence per channel, parallel across channels/streams.
 *  K3  k_block_fec        : blk_thread's parity/CRC/syndrome repair, one thread per finished frame
 *                     (reference: acars.c:39-215).
 *
 * Numerics contract (SURVEY.md §8a): all order/rounding-sensitive arithmetic uses the
 * explicit round-to-nearest intrinsics, which the compiler never contracts; the TU is also
 * built with -fmad=false.
 */
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>

#include <algorithm>

#include "../../include/acars_b200.h"
#include "acb_internal.h"
#include "frame_sm.h"
#include "demod_core.h"

namespace acb {

__constant__ float c_h[FLENO];     /* matched filter, built on the host with glibc cosf (msk.c:44-48) */

/* stream-ordered uploads: the caller synchronises `stream` before it launches anything (the context's
 * streams are non-blocking, i.e. not ordered behind the legacy stream a plain cudaMemcpyToSymbol uses) */
int upload_matched_filter(const float *h, cudaStream_t stream);

/* Pairwise float2 arithmetic.  sm_90 has no packed FP32 instructions, so each is two scalar
 * round-to-nearest ops: one rounding per lane, the same result a packed form would give. */
__device__ __forceinline__ float2 fadd2_rn(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ float2 fmul2_rn(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c)
{
	return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}

/* ------------------------------------------------------------------------------------------
 * K1: channelizer
 * ---------------------------------------------------------------------------------------- */

/* (float)u8 - 127.37f  (rtl.c:338-339).  The byte is planted in the mantissa of 2^23, the
 * 2^23 removed (exact), then 127.37f subtracted — also exact: the result is a multiple of
 * 2^-17 below 2^7, so the reference's single rounding rounds nothing either. */
__device__ __forceinline__ float2 cvt_iq(unsigned w, int pair)
{
	float2 x;
	x.x = __uint_as_float(__byte_perm(w, 0x4B000000u, pair ? 0x7542 : 0x7540));
	x.y = __uint_as_float(__byte_perm(w, 0x4B000000u, pair ? 0x7543 : 0x7541));
	x = fadd2_rn(x, make_float2(-8388608.0f, -8388608.0f));
	return fadd2_rn(x, make_float2(-127.37f, -127.37f));
}

/* D += (a + jb) * (c + jd) with the reference's rounding: products rounded, (ac - bd) and
 * (ad + bc) rounded, then the accumulate rounded (rtl.c:351).  w = (c, d).  The -bd product is
 * b * (-d): negation is exact and round-to-nearest is symmetric, so it has the bits of a product with
 * a stored -d, zero weights' signed zeros included; the negation folds into the FMUL's operand.
 * Instruction shape: 4 FMUL + 4 FADD, none of them contracted into an FFMA (that would skip the
 * product rounding). */
__device__ __forceinline__ void cmac(float2 &acc, float a, float b, const float2 w)
{
	const float2 p1 = fmul2_rn(make_float2(a, a), make_float2(w.x, w.y));
	const float2 p2 = fmul2_rn(make_float2(b, b), make_float2(-w.y, w.x));
	const float2 t = make_float2(__fadd_rn(p1.x, p2.x), __fadd_rn(p1.y, p2.y));
	acc = fadd2_rn(acc, t);
}

/* cabsf (rtl.c:353): glibc hypotf is (float)sqrt((double)x*x + (double)y*y) for finite input */
__device__ __forceinline__ float envelope(float2 d)
{
	double x = (double)d.x, y = (double)d.y;
	return __double2float_rn(__dsqrt_rn(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y))));
}

__device__ __forceinline__ void cp_async16(void *smem, const void *gmem)
{
	unsigned s = (unsigned)__cvta_generic_to_shared(smem);
	asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(s), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

/* ------------------------------------------------------------------------------------------
 * K1 pipeline, float32 real input (air.c:314-333: D += wf[i]*S, table entries (c, d)), the two-rows form that
 * ACB_REAL_ROWS=2 selects in place of k_channelize_real4.  One CTA = one 1024-output block x one group of 8 channels;
 * 128 threads, two output rows per thread (rows t and t+128 of a 256-row tile) so every broadcast table load feeds two
 * MACs; the K taps are walked in chunks of 5 sixteen-byte units per row (5 is odd: the strided LDS.128 row reads are
 * conflict free without padding) staged by cp.async into a 2-deep ring together with the matching slice of the table,
 * so the copy of chunk i+1 runs under the arithmetic of chunk i.  Any K that keeps rows 16-byte aligned, up to ACB_MAXK.
 * ---------------------------------------------------------------------------------------- */

constexpr int C2_ROWS = 256;
enum { IN_U8IQ = 0, IN_F32REAL = 1, IN_CS16IQ = 2 };   /* input sample formats (acb_internal.h: InputKind) */

struct C2 {
	/* 16-byte units of a row per chunk: odd, so the strided per-thread LDS.128 row reads are conflict free with rows
	 * packed back to back.  (Whole-sector chunks of 6 units with a padded row stride were tried: no gain — the limit
	 * was elsewhere, see k_channelize_real4.) */
	static constexpr int UNITS = 5;
	static constexpr int ROW_UNITS = UNITS;                      /* shared-memory row stride in units */
	static constexpr int STAGES = 2;                             /* cp.async ring depth */
	static constexpr int TAP_BYTES = 4;                          /* input bytes per tap */
	static constexpr int TAPS_PER_UNIT = 16 / TAP_BYTES;
	static constexpr int W_BYTES = 8;                            /* table bytes per (tap, channel) */
	static constexpr int CHUNK_TAPS = UNITS * TAPS_PER_UNIT;
	static constexpr int TILE_BYTES = C2_ROWS * ROW_UNITS * 16;
	static constexpr int WF_BYTES = CHUNK_TAPS * CH_GROUP * W_BYTES;
	static constexpr int STAGE_BYTES = TILE_BYTES + WF_BYTES;
};

/* (float)int16 for both halves of a CS16 sample (soapy.c:239-240, sdrplay.c:218-219): x ^ 0x8000
 * planted in the mantissa of 2^23, then 2^23 + 2^15 removed — exact */
__device__ __forceinline__ float2 cvt_cs16(unsigned w)
{
	const unsigned v = w ^ 0x80008000u;
	float2 x;
	x.x = __uint_as_float(__byte_perm(v, 0x4B000000u, 0x7410));
	x.y = __uint_as_float(__byte_perm(v, 0x4B000000u, 0x7432));
	return fadd2_rn(x, make_float2(-8421376.0f, -8421376.0f));
}

/* air.c:317-318: D += wf[i] * S — (c*S, d*S) rounded, then the accumulate rounded. */
__device__ __forceinline__ void rmac(float2 &acc, float sv, const float2 w)
{
	acc = fadd2_rn(acc, make_float2(__fmul_rn(w.x, sv), __fmul_rn(w.y, sv)));
}

/* OVL (taps > K, DESIGN.md §4 "K1, overlapping window"): the window of a row starts `hbytes` (H_pad samples) before
 * the row and is `taps` (= K + H_pad) samples long.  A 16-byte unit that lies before the stream's input of this submit
 * is fetched from the history of the stream instead: `hist + s*hist_stride + hbytes` is where sample 0 of the submit
 * would sit if the history were laid out in front of it.  The choice is per unit: H_pad and every row are whole units. */
template <bool OVL>
__global__ void __launch_bounds__(CH_TILE)
k_channelize(const uint8_t *__restrict__ in, size_t stream_stride, const uint8_t *__restrict__ wf,
              float *__restrict__ dm, int K, int taps, int nch, int ngrp, size_t nsamp,
              const uint8_t *__restrict__ hist, size_t hist_stride, int hbytes)
{
	using T = C2;
	extern __shared__ __align__(16) unsigned char smem[];
	const int t = threadIdx.x;
	const int blk = blockIdx.x, s = blockIdx.y;
	const size_t rowbytes = (size_t)K * T::TAP_BYTES;
	const int U = taps * T::TAP_BYTES / 16;                          /* units of each row's window that carry taps */
	const int nchunk = (U + T::UNITS - 1) / T::UNITS;
	const uint8_t *src_blk = in + (size_t)s * stream_stride + (size_t)blk * OUTBLK * rowbytes;
	constexpr int NTILE = OUTBLK / C2_ROWS;
	const int nstep = NTILE * nchunk;

	{
		const int g = blockIdx.z;                                    /* channel group of 8: one CTA each */
		const uint8_t *wsrc = wf + ((size_t)s * ngrp + g) * taps * CH_GROUP * T::W_BYTES;

		auto issue = [&](int step) {
			const int tile = step / nchunk, ck = step - tile * nchunk;
			unsigned char *st = smem + (size_t)(step % T::STAGES) * T::STAGE_BYTES;
			const int uc = min(T::UNITS, U - ck * T::UNITS);         /* units of this chunk */
			const uint8_t *tsrc = src_blk + (size_t)tile * C2_ROWS * rowbytes + (size_t)ck * T::UNITS * 16;
			if constexpr (OVL) tsrc -= hbytes;
			{
				/* unit u = t + 128*i of the chunk tile lives at (row u/uc, column u%uc): one division
				 * per chunk, then incremental (the address arithmetic is a fifth of the kernel's
				 * instructions otherwise) */
				int row = t / uc, j = t - row * uc;
				const int drow = CH_TILE / uc, dj = CH_TILE - drow * uc;
				unsigned char *dst = st + ((size_t)row * T::ROW_UNITS + j) * 16;
				const uint8_t *src = tsrc + (size_t)row * rowbytes + (size_t)j * 16;
				const size_t dstep = ((size_t)drow * T::ROW_UNITS + dj) * 16, sstep = (size_t)drow * rowbytes + (size_t)dj * 16;
				const size_t dwrap = (size_t)(T::ROW_UNITS - uc) * 16, swrap = rowbytes - (size_t)uc * 16;
				for (int u = t; u < C2_ROWS * uc; u += CH_TILE) {
					if constexpr (OVL) {
						const uint8_t *sbase = in + (size_t)s * stream_stride;
						cp_async16(dst, src < sbase ? hist + (size_t)s * hist_stride + hbytes - (sbase - src) : src);
					} else {
						cp_async16(dst, src);
					}
					dst += dstep; src += sstep; j += dj;
					if (j >= uc) { j -= uc; dst += dwrap; src += swrap; }
				}
			}
			const int wunits = uc * T::TAPS_PER_UNIT * CH_GROUP * T::W_BYTES / 16;
			const uint8_t *ws = wsrc + (size_t)ck * T::CHUNK_TAPS * CH_GROUP * T::W_BYTES;
			for (int u = t; u < wunits; u += CH_TILE) cp_async16(st + T::TILE_BYTES + (size_t)u * 16, ws + (size_t)u * 16);
			cp_async_commit();
		};

		float2 accA[CH_GROUP], accB[CH_GROUP];
#pragma unroll
		for (int c = 0; c < CH_GROUP; c++) accA[c] = accB[c] = make_float2(0.f, 0.f);

		/* prologue: STAGES-1 chunks in flight; every iteration commits exactly one group (possibly
		 * empty) so that "all but the newest STAGES-1 groups" always means "chunk `step` landed" */
#pragma unroll
		for (int i = 0; i < T::STAGES - 1; i++) {
			if (i < nstep) issue(i); else cp_async_commit();
		}
		for (int step = 0; step < nstep; step++) {
			if (step + T::STAGES - 1 < nstep) issue(step + T::STAGES - 1); else cp_async_commit();
			asm volatile("cp.async.wait_group %0;" ::"n"(T::STAGES - 1) : "memory");
			__syncthreads();                                         /* chunk `step` visible to all */
			const int tile = step / nchunk, ck = step - tile * nchunk;
			const unsigned char *st = smem + (size_t)(step % T::STAGES) * T::STAGE_BYTES;
			const int uc = min(T::UNITS, U - ck * T::UNITS);
			const uint4 *rowA = reinterpret_cast<const uint4 *>(st) + (size_t)t * T::ROW_UNITS;
			const uint4 *rowB = reinterpret_cast<const uint4 *>(st) + (size_t)(t + CH_TILE) * T::ROW_UNITS;
			for (int j = 0; j < uc; j++) {
				const uint4 qa = rowA[j], qb = rowB[j];
				const unsigned wa[4] = { qa.x, qa.y, qa.z, qa.w }, wb[4] = { qb.x, qb.y, qb.z, qb.w };
				const float2 *wj = reinterpret_cast<const float2 *>(st + T::TILE_BYTES) + (size_t)j * 4 * CH_GROUP;
#pragma unroll
				for (int e = 0; e < 4; e++) {
					const float sa = __uint_as_float(wa[e]), sb = __uint_as_float(wb[e]);
#pragma unroll
					for (int c = 0; c < CH_GROUP; c++) {
						const float2 w = wj[e * CH_GROUP + c];
						rmac(accA[c], sa, w);
						rmac(accB[c], sb, w);
					}
				}
			}
			if (ck == nchunk - 1) {                                  /* row complete: |D| out, restart */
				const int nc = min(CH_GROUP, nch - g * CH_GROUP);
#pragma unroll
				for (int half = 0; half < 2; half++) {
					float2 *acc = half ? accB : accA;
					const size_t m = (size_t)blk * OUTBLK + (size_t)tile * C2_ROWS + t + half * CH_TILE;
					float *o = dm + ((size_t)s * nsamp + m) * nch + g * CH_GROUP;
					if (nc == CH_GROUP && (nch & 3) == 0) {
						reinterpret_cast<float4 *>(o)[0] = make_float4(envelope(acc[0]), envelope(acc[1]), envelope(acc[2]), envelope(acc[3]));
						reinterpret_cast<float4 *>(o)[1] = make_float4(envelope(acc[4]), envelope(acc[5]), envelope(acc[6]), envelope(acc[7]));
					} else {
#pragma unroll
						for (int c = 0; c < CH_GROUP; c++)
							if (c < nc) o[c] = envelope(acc[c]);
					}
#pragma unroll
					for (int c = 0; c < CH_GROUP; c++) acc[c] = make_float2(0.f, 0.f);
				}
			}
			__syncthreads();                                         /* stage may be refilled by issue(step+2) */
		}
	}
}

/* ------------------------------------------------------------------------------------------
 * K1 for IQ input: u8 (rtl.c:334-354) and CS16 (soapy.c:239-242 with the /32768.0 folded into the table,
 * sdrplay.c:218-222), D += (a + jb)(c + jd) per tap in tap order (cmac).
 *
 * One CTA = 512 output rows (half a 1024-row block) x one group of 8 channels; 128 threads, FOUR rows per thread (rows
 * t + 128 r), so each warp-uniform LDS.128 of the table — (c, d) of two channels — feeds 4 rows x 2 channels = 8 complex
 * MACs.  The instruction stream is the FP32 pipe's: per 32-bit word of the rows (u8: 2 taps) and thread, 64 complex MACs
 * = 512 FMUL/FADD, 48 conversion instructions and 8 table loads.
 *
 * Only the table goes through shared memory, in a 2-deep cp.async ring of IQ4_CU-unit chunks (2 x 2 KB for u8, 2 x 1 KB
 * for CS16, whatever K or taps): K1 then fits on an SM beside the co-resident demodulator's CTAs.  Each thread loads its
 * rows' 16-byte units straight from global memory into registers (qb), one unit ahead of the arithmetic on qa.  The two
 * units of a 32-byte sector are consecutive loads of the same thread, so DRAM is read once.  OVL: the window and the
 * per-unit choice between input and history are those of k_channelize.
 * ---------------------------------------------------------------------------------------- */
constexpr int IQ4_THREADS = 128, IQ4_RPT = 4, IQ4_ROWS = IQ4_THREADS * IQ4_RPT;
constexpr int IQ4_CU = 4;            /* table chunk in units of the row */
constexpr int IQ4_STAGES = 2;

template <int MODE, bool OVL>
__global__ void __launch_bounds__(IQ4_THREADS, 3)
k_channelize_iq4(const uint8_t *__restrict__ in, size_t stream_stride, const float2 *__restrict__ wf,
                 float *__restrict__ dm, int K, int taps, int nch, int ngrp, size_t nsamp,
                 const uint8_t *__restrict__ hist, size_t hist_stride, int hbytes)
{
	constexpr int TB = MODE == IN_U8IQ ? 2 : 4, TPU = 16 / TB;        /* input bytes per tap, taps per unit */
	constexpr int TPW = TPU / 4;                                       /* taps per 32-bit word */
	constexpr int WCH = IQ4_CU * TPU * CH_GROUP;                       /* (c, d) entries per table chunk */
	__shared__ __align__(16) float2 wsm[IQ4_STAGES][WCH];
	const int t = threadIdx.x, s = blockIdx.y, g = blockIdx.z;
	const size_t rowbytes = (size_t)K * TB;
	const int U = taps / TPU;                                          /* units of each row's window (taps padded to whole units) */
	const int nchunk = (U + IQ4_CU - 1) / IQ4_CU;
	const size_t m0 = (size_t)blockIdx.x * IQ4_ROWS + t;               /* the thread's rows: m0 + 128 r */
	const uint8_t *sbase = in + (size_t)s * stream_stride;
	const uint8_t *hbase = OVL ? hist + (size_t)s * hist_stride + hbytes : nullptr;
	const float2 *wsrc = wf + ((size_t)s * ngrp + g) * taps * CH_GROUP;
	const uint8_t *rp[IQ4_RPT];                                        /* the rows' unit under the arithmetic */
#pragma unroll
	for (int r = 0; r < IQ4_RPT; r++) rp[r] = sbase + (m0 + (size_t)r * IQ4_THREADS) * rowbytes - (OVL ? hbytes : 0);

	auto issue = [&](int ck) {                                         /* table chunk ck into its stage; always one commit */
		if (ck < nchunk) {
			const int n = min(IQ4_CU, U - ck * IQ4_CU) * TPU * CH_GROUP / 2;
			const float2 *src = wsrc + (size_t)ck * WCH;
			for (int i = t; i < n; i += IQ4_THREADS) cp_async16(&wsm[ck % IQ4_STAGES][2 * i], src + 2 * i);
		}
		cp_async_commit();
	};
	auto load = [&](uint4 (&q)[IQ4_RPT], int off) {                    /* the rows' unit at byte `off` past rp */
#pragma unroll
		for (int r = 0; r < IQ4_RPT; r++) {
			const uint8_t *p = rp[r] + off;
			if (OVL && p < sbase) p = hbase - (sbase - p);
			q[r] = __ldg(reinterpret_cast<const uint4 *>(p));
		}
	};

	float2 acc[IQ4_RPT][CH_GROUP];
#pragma unroll
	for (int r = 0; r < IQ4_RPT; r++)
#pragma unroll
		for (int c = 0; c < CH_GROUP; c++) acc[r][c] = make_float2(0.f, 0.f);

	auto word = [&](const unsigned (&v)[IQ4_RPT], const float2 *wj) {    /* the TPW taps of one 32-bit word of the rows */
#pragma unroll
		for (int h = 0; h < TPW; h++) {
			float2 x[IQ4_RPT];
#pragma unroll
			for (int r = 0; r < IQ4_RPT; r++) x[r] = MODE == IN_U8IQ ? cvt_iq(v[r], h) : cvt_cs16(v[r]);
			const float4 *wt = reinterpret_cast<const float4 *>(wj + h * CH_GROUP);
#pragma unroll
			for (int c2 = 0; c2 < CH_GROUP / 2; c2++) {
				const float4 w = wt[c2];
#pragma unroll
				for (int r = 0; r < IQ4_RPT; r++) {
					cmac(acc[r][2 * c2], x[r].x, x[r].y, make_float2(w.x, w.y));
					cmac(acc[r][2 * c2 + 1], x[r].x, x[r].y, make_float2(w.z, w.w));
				}
			}
		}
	};

	uint4 qa[IQ4_RPT], qb[IQ4_RPT];
	issue(0);
	load(qa, 0);
	int u = 0;                                                         /* unit in qa */
	for (int ck = 0; ck < nchunk; ck++) {
		issue(ck + 1);
		asm volatile("cp.async.wait_group 1;" ::: "memory");
		__syncthreads();                                               /* chunk ck visible to all */
		const float2 *w = wsm[ck % IQ4_STAGES];
		const int uc = min(IQ4_CU, U - ck * IQ4_CU);
		/* rolled loops over units and over the 4 words of a unit: a body of one word (~580 instructions) stays in the
		 * instruction cache, where a fully unrolled unit (~2300) or unit pair did not and ran 1.2x / 1.6x slower */
#pragma unroll 1
		for (int j = 0; j < uc; j++, u++) {
			if (u + 1 < U) load(qb, 16);
#pragma unroll 1
			for (int e = 0; e < 4; e++, w += TPW * CH_GROUP) {
				const unsigned v[IQ4_RPT] = { qa[0].x, qa[1].x, qa[2].x, qa[3].x };
				word(v, w);
#pragma unroll
				for (int r = 0; r < IQ4_RPT; r++) { qa[r].x = qa[r].y; qa[r].y = qa[r].z; qa[r].z = qa[r].w; }
			}
#pragma unroll
			for (int r = 0; r < IQ4_RPT; r++) { qa[r] = qb[r]; rp[r] += 16; }
		}
		__syncthreads();                                               /* stage may be refilled by issue(ck + 2) */
	}

	const int nc = min(CH_GROUP, nch - g * CH_GROUP);
#pragma unroll
	for (int r = 0; r < IQ4_RPT; r++) {
		float *o = dm + ((size_t)s * nsamp + m0 + (size_t)r * IQ4_THREADS) * nch + g * CH_GROUP;
		if (nc == CH_GROUP && (nch & 3) == 0) {
			reinterpret_cast<float4 *>(o)[0] = make_float4(envelope(acc[r][0]), envelope(acc[r][1]), envelope(acc[r][2]), envelope(acc[r][3]));
			reinterpret_cast<float4 *>(o)[1] = make_float4(envelope(acc[r][4]), envelope(acc[r][5]), envelope(acc[r][6]), envelope(acc[r][7]));
		} else {
#pragma unroll
			for (int c = 0; c < CH_GROUP; c++)
				if (c < nc) o[c] = envelope(acc[r][c]);
		}
	}
}

/* The float32 real-input form of the same pipeline with FOUR output rows per thread (64 threads per 256-row tile).
 * air.c:317-318 is D += wf[i]*S: half the arithmetic of a complex tap per table entry, so with two rows per thread the
 * warp-uniform table loads (64 bytes per tap) were a fifth of the instruction stream and the shared-memory pipe, not the
 * FP32 pipe, set the pace.  Four rows per thread
 * halve the table traffic per MAC; same arithmetic, same order, bit-identical results. */
constexpr int R4_THREADS = 64, R4_RPT = C2_ROWS / R4_THREADS;

template <bool OVL>                                                  /* OVL: as in k_channelize */
__global__ void __launch_bounds__(R4_THREADS)
k_channelize_real4(const uint8_t *__restrict__ in, size_t stream_stride, const uint8_t *__restrict__ wf,
                   float *__restrict__ dm, int K, int taps, int nch, int ngrp, size_t nsamp,
                   const uint8_t *__restrict__ hist, size_t hist_stride, int hbytes)
{
	constexpr int UNITS = 5, TAPS_PER_UNIT = 4, W_BYTES = 8, CHUNK_TAPS = UNITS * TAPS_PER_UNIT, STAGES = 2;
	constexpr int TILE_BYTES = C2_ROWS * UNITS * 16, STAGE_BYTES = TILE_BYTES + CHUNK_TAPS * CH_GROUP * W_BYTES;
	extern __shared__ __align__(16) unsigned char smem[];
	const int t = threadIdx.x;
	const int blk = blockIdx.x, s = blockIdx.y, g = blockIdx.z;
	const size_t rowbytes = (size_t)K * 4;
	const int U = taps / TAPS_PER_UNIT;                              /* taps is padded to whole units by the caller */
	const int nchunk = (U + UNITS - 1) / UNITS;
	const uint8_t *src_blk = in + (size_t)s * stream_stride + (size_t)blk * OUTBLK * rowbytes;
	constexpr int NTILE = OUTBLK / C2_ROWS;
	const int nstep = NTILE * nchunk;
	const uint8_t *wsrc = wf + ((size_t)s * ngrp + g) * taps * CH_GROUP * W_BYTES;

	auto issue = [&](int step) {
		const int tile = step / nchunk, ck = step - tile * nchunk;
		unsigned char *st = smem + (size_t)(step % STAGES) * STAGE_BYTES;
		const int uc = min(UNITS, U - ck * UNITS);
		const uint8_t *tsrc = src_blk + (size_t)tile * C2_ROWS * rowbytes + (size_t)ck * UNITS * 16;
		if constexpr (OVL) tsrc -= hbytes;
		int row = t / uc, j = t - row * uc;
		const int drow = R4_THREADS / uc, dj = R4_THREADS - drow * uc;
		unsigned char *dst = st + ((size_t)row * UNITS + j) * 16;
		const uint8_t *src = tsrc + (size_t)row * rowbytes + (size_t)j * 16;
		const size_t dstep = ((size_t)drow * UNITS + dj) * 16, sstep = (size_t)drow * rowbytes + (size_t)dj * 16;
		const size_t dwrap = (size_t)(UNITS - uc) * 16, swrap = rowbytes - (size_t)uc * 16;
		for (int u = t; u < C2_ROWS * uc; u += R4_THREADS) {
			if constexpr (OVL) {
				const uint8_t *sbase = in + (size_t)s * stream_stride;
				cp_async16(dst, src < sbase ? hist + (size_t)s * hist_stride + hbytes - (sbase - src) : src);
			} else {
				cp_async16(dst, src);
			}
			dst += dstep; src += sstep; j += dj;
			if (j >= uc) { j -= uc; dst += dwrap; src += swrap; }
		}
		const int wunits = uc * TAPS_PER_UNIT * CH_GROUP * W_BYTES / 16;
		const uint8_t *ws = wsrc + (size_t)ck * CHUNK_TAPS * CH_GROUP * W_BYTES;
		for (int u = t; u < wunits; u += R4_THREADS) cp_async16(st + TILE_BYTES + (size_t)u * 16, ws + (size_t)u * 16);
		cp_async_commit();
	};

	float2 acc[R4_RPT][CH_GROUP];
#pragma unroll
	for (int r = 0; r < R4_RPT; r++)
#pragma unroll
		for (int c = 0; c < CH_GROUP; c++) acc[r][c] = make_float2(0.f, 0.f);

	if (0 < nstep) issue(0); else cp_async_commit();
	for (int step = 0; step < nstep; step++) {
		if (step + 1 < nstep) issue(step + 1); else cp_async_commit();
		asm volatile("cp.async.wait_group %0;" ::"n"(STAGES - 1) : "memory");
		__syncthreads();
		const int tile = step / nchunk, ck = step - tile * nchunk;
		const unsigned char *st = smem + (size_t)(step % STAGES) * STAGE_BYTES;
		const int uc = min(UNITS, U - ck * UNITS);
		const uint4 *rows = reinterpret_cast<const uint4 *>(st) + (size_t)t * UNITS;
		for (int j = 0; j < uc; j++) {
			uint4 q[R4_RPT];
#pragma unroll
			for (int r = 0; r < R4_RPT; r++) q[r] = rows[(size_t)r * R4_THREADS * UNITS + j];
			const float2 *wj = reinterpret_cast<const float2 *>(st + TILE_BYTES) + (size_t)j * 4 * CH_GROUP;
#pragma unroll
			for (int e = 0; e < 4; e++) {
				float sv[R4_RPT];
#pragma unroll
				for (int r = 0; r < R4_RPT; r++) sv[r] = __uint_as_float(e == 0 ? q[r].x : e == 1 ? q[r].y : e == 2 ? q[r].z : q[r].w);
#pragma unroll
				for (int c = 0; c < CH_GROUP; c++) {
					const float2 w = wj[e * CH_GROUP + c];
#pragma unroll
					for (int r = 0; r < R4_RPT; r++) rmac(acc[r][c], sv[r], w);
				}
			}
		}
		if (ck == nchunk - 1) {                                  /* rows complete: |D| out, restart */
			const int nc = min(CH_GROUP, nch - g * CH_GROUP);
#pragma unroll
			for (int r = 0; r < R4_RPT; r++) {
				const size_t m = (size_t)blk * OUTBLK + (size_t)tile * C2_ROWS + t + r * R4_THREADS;
				float *o = dm + ((size_t)s * nsamp + m) * nch + g * CH_GROUP;
				if (nc == CH_GROUP && (nch & 3) == 0) {
					reinterpret_cast<float4 *>(o)[0] = make_float4(envelope(acc[r][0]), envelope(acc[r][1]), envelope(acc[r][2]), envelope(acc[r][3]));
					reinterpret_cast<float4 *>(o)[1] = make_float4(envelope(acc[r][4]), envelope(acc[r][5]), envelope(acc[r][6]), envelope(acc[r][7]));
				} else {
#pragma unroll
					for (int c = 0; c < CH_GROUP; c++)
						if (c < nc) o[c] = envelope(acc[r][c]);
				}
#pragma unroll
				for (int c = 0; c < CH_GROUP; c++) acc[r][c] = make_float2(0.f, 0.f);
			}
		}
		__syncthreads();
	}
}

/* a kernel's launch attributes: up to `smem` bytes of dynamic shared memory, and the largest shared-memory carve-out */
template <typename F>
static cudaError_t smem_max_carveout(F *kern, int smem)
{
	const cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
	return e != cudaSuccess ? e : cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
}

template <bool OVL>
static int launch_channelize_real4(const void *in, size_t stream_stride, const void *wf, float *dm,
                                   int K, int taps, int nch, int nstreams, int nblk, size_t nsamp, const Hist &h, cudaStream_t stream)
{
	if (nblk == 0) return 0;
	const int ngrp = (nch + CH_GROUP - 1) / CH_GROUP;
	const size_t smem = 2 * (size_t)(C2_ROWS * 5 * 16 + 20 * CH_GROUP * 8);
	if (cudaError_t e = smem_max_carveout(k_channelize_real4<OVL>, (int)smem)) return (int)e;
	dim3 grid(nblk, nstreams, ngrp);
	k_channelize_real4<OVL><<<grid, R4_THREADS, smem, stream>>>(reinterpret_cast<const uint8_t *>(in), stream_stride,
	                                                           reinterpret_cast<const uint8_t *>(wf), dm, K, taps, nch, ngrp, nsamp,
	                                                           reinterpret_cast<const uint8_t *>(h.base), h.stride, h.hpad * 4);
	return (int)cudaGetLastError();
}

template <bool OVL>
static int launch_channelize_real2(const void *in, size_t stream_stride, const void *wf, float *dm,
                                   int K, int taps, int nch, int nstreams, int nblk, size_t nsamp, const Hist &h, cudaStream_t stream)
{
	if (nblk == 0) return 0;
	const int ngrp = (nch + CH_GROUP - 1) / CH_GROUP;
	const size_t smem = (size_t)C2::STAGES * C2::STAGE_BYTES;
	/* the largest shared-memory carve-out: the staging ring is this kernel's working set.  (Kernels that prefer
	 * different splits do share an SM — the demod of submit i runs underneath the channelizer of submit i+1 whatever
	 * the two ask for, see launch_channelize_iq4.) */
	if (cudaError_t e = smem_max_carveout(k_channelize<OVL>, (int)smem)) return (int)e;
	dim3 grid(nblk, nstreams, ngrp);
	k_channelize<OVL><<<grid, CH_TILE, smem, stream>>>(reinterpret_cast<const uint8_t *>(in), stream_stride,
	                                                   reinterpret_cast<const uint8_t *>(wf), dm, K, taps, nch, ngrp, nsamp,
	                                                   reinterpret_cast<const uint8_t *>(h.base), h.stride, h.hpad * C2::TAP_BYTES);
	return (int)cudaGetLastError();
}

template <int MODE, bool OVL>
static int launch_channelize_iq4(const void *in, size_t stream_stride, const float *wf, float *dm,
                                 int K, int taps, int nch, int nstreams, int nblk, size_t nsamp, const Hist &h, cudaStream_t stream)
{
	if (nblk == 0) return 0;
	const int ngrp = (nch + CH_GROUP - 1) / CH_GROUP;
	/* a quarter of the shared-memory maximum, the rest L1: every lane of a row load touches its own 128-byte line, and
	 * with the 28 KB of L1 the largest carve-out leaves, the kernel ran 1.2x slower (DESIGN.md §4).  The demodulator runs
	 * underneath this kernel and asks for a larger configuration, sized for its own CTAs plus three of these (4 KB + 1 KB
	 * reserved each; the whole budget, registers included, is at launch_demod_t).  Kernels of different preferences do
	 * share an SM: with 100 KB asked for here instead, neither this kernel alone nor the pipelined step moved (13.59
	 * against 13.54 ms, 15.35 against 15.31 ms; H100 SXM 700 W, 4224 streams x 8 blocks). */
	cudaError_t e = cudaFuncSetAttribute(k_channelize_iq4<MODE, OVL>, cudaFuncAttributePreferredSharedMemoryCarveout, 25);
	if (e != cudaSuccess) return (int)e;
	dim3 grid(nblk * (OUTBLK / IQ4_ROWS), nstreams, ngrp);
	k_channelize_iq4<MODE, OVL><<<grid, IQ4_THREADS, 0, stream>>>(reinterpret_cast<const uint8_t *>(in), stream_stride,
	                                                             reinterpret_cast<const float2 *>(wf), dm, K, taps, nch, ngrp, nsamp,
	                                                             reinterpret_cast<const uint8_t *>(h.base), h.stride,
	                                                             h.hpad * (MODE == IN_U8IQ ? 2 : 4));
	return (int)cudaGetLastError();
}

template <bool OVL>
static int launch_channelize_k(int mode, const void *in, size_t stream_stride_bytes, const float *wf, float *dm,
                               int K, int taps, int nch, int nstreams, int nblk, size_t nsamp, const Hist &h, cudaStream_t stream)
{
	switch (mode) {
	case IN_F32REAL: {
		const bool two_rows = getenv("ACB_REAL_ROWS") && atoi(getenv("ACB_REAL_ROWS")) == 2;     /* A/B switch: the 2-rows-per-thread form */
		return two_rows ? launch_channelize_real2<OVL>(in, stream_stride_bytes, wf, dm, K, taps, nch, nstreams, nblk, nsamp, h, stream)
		                : launch_channelize_real4<OVL>(in, stream_stride_bytes, wf, dm, K, taps, nch, nstreams, nblk, nsamp, h, stream);
	}
	case IN_CS16IQ: return launch_channelize_iq4<IN_CS16IQ, OVL>(in, stream_stride_bytes, wf, dm, K, taps, nch, nstreams, nblk, nsamp, h, stream);
	default: return launch_channelize_iq4<IN_U8IQ, OVL>(in, stream_stride_bytes, wf, dm, K, taps, nch, nstreams, nblk, nsamp, h, stream);
	}
}

/* whole 1024-row blocks of any input kind; the caller sends remaining rows to the generic kernel.  h.hpad > 0 selects
 * the overlapping-window instantiations (taps = K + h.hpad) */
static int launch_channelize(int mode, const void *in, size_t stream_stride_bytes, const float *wf, float *dm,
                             int K, int taps, int nch, int nstreams, int nblk, size_t nsamp, const Hist &h, cudaStream_t stream)
{
	return h.hpad ? launch_channelize_k<true>(mode, in, stream_stride_bytes, wf, dm, K, taps, nch, nstreams, nblk, nsamp, h, stream)
	              : launch_channelize_k<false>(mode, in, stream_stride_bytes, wf, dm, K, taps, nch, nstreams, nblk, nsamp, h, stream);
}

/* ------------------------------------------------------------------------------------------
 * K1, fast form (ACB_FLAG_FAST_CHANNELIZER).  The reference's mixer table is a sampled complex
 * exponential: when (Fr - Fc) is a whole number k of 12.5 kHz steps — the planner's normal outcome,
 * frequencies are rounded to that raster (rtl.c:245-247) — wf[ind] = g*exp(-j*2*pi*k*ind/K) and the
 * boxcar sum D = sum_ind x[ind]*wf[ind] is bin k of a K-point DFT of the row.  Split ind = (K/4)*n1 + n2:
 *
 *     D_c = sum_{n2 < K/4} T_c[n2] * Y_{k_c mod 4}[n2],   Y_r[n2] = sum_{n1 < 4} x[(K/4)*n1 + n2] * (-j)^(r*n1)
 *
 * (k is always even: the float images of Fr and Fc that the reference mixes with are multiples of 8 Hz,
 * so only Y_0 = x0+x1+x2+x3 and Y_2 = x0-x1+x2-x3 occur.)
 *
 * Y_r is a 4-point DFT across the four quarters of the row: additions only, EXACT in float (integer
 * samples), and shared by every channel of the stream; each channel then needs K/4 complex MACs instead
 * of K.  The -127.37 offset of rtl.c:338-339 drops out (a channel is never at bin 0: chooseFc keeps it
 * 25 kHz from the centre).  FP32 work per input sample falls from 8*C to 2.5 + C lane-ops (C = 8: 64 ->
 * 10.5), which moves the kernel from the FP32 roof towards the HBM roof.
 *
 * This is NOT the reference's operation order: the envelope differs from the reference's in the last
 * bits.  Measured (tests/test_gpu_fast.py, tests/test_fast_oracle.py), relative to the total in-band
 * signal: 3e-7 from the exact double-precision DFT bin — the reference, whose table carries float phase
 * rounding (float AMFreq*ind), sits at 1.8e-6 — bit-identical to its CPU restatement
 * (oracle: orc_channelize_dft), and decoded messages identical on every fixture.  The default (exact)
 * kernel above stays bit-identical; this one is what the north star's tolerance (messages bit-exact,
 * float intermediates within tolerance) buys.
 *
 * Shape: one CTA = one 1024-row block of one stream for 8 channels, 16 tiles of 64 rows dealt round-robin
 * to its warps; lane l owns rows l and l+32 of a tile, and every FP32 step is done for both rows (float2
 * pairs, one scalar instruction per row on sm_90; the twiddle is the same scalar for both).
 * Whole rows are fetched by bulk copies (cp.async.bulk of one or two rows, completion on the warp's
 * mbarrier) issued by one lane: every 32-byte sector fetched is used, no per-unit addressing.
 * Warps do not synchronise with each other after the twiddles are in shared memory; with one private
 * buffer per warp, the copy of a warp's next tile hides under the other warps' arithmetic.
 * ---------------------------------------------------------------------------------------- */

constexpr int DFT_ROWS = 64;                     /* rows per tile: 2 per lane */

__device__ __forceinline__ float2 fsub2(float2 a, float2 b) { return fadd2_rn(a, make_float2(-b.x, -b.y)); }

/* byte `k` of word wa / wb as 32768 + u, packed (row A, row B): the byte lands in bits 8..15 of the
 * mantissa of 2^15, where the unit weight is */
template <int KB> __device__ __forceinline__ float2 dft_cvt(unsigned wa, unsigned wb)
{
	constexpr unsigned sel = 0x7404u | (KB << 4);
	return make_float2(__uint_as_float(__byte_perm(wa, 0x47000000u, sel)), __uint_as_float(__byte_perm(wb, 0x47000000u, sel)));
}

struct DftAcc { float2 a, b, p, q; };            /* re = a - b, im = p + q; each packed (row A, row B) */

/* acc += y * t for the lane's two rows; t = (Tr, Ti) is warp-uniform.
 * Four independent accumulators keep the dependent FFMA chains short. */
__device__ __forceinline__ void dft_mac(DftAcc &acc, float2 yr, float2 yi, float2 t)
{
	const float2 tr = make_float2(t.x, t.x), ti = make_float2(t.y, t.y);
	acc.a = ffma2(yr, tr, acc.a);
	acc.b = ffma2(yi, ti, acc.b);
	acc.p = ffma2(yr, ti, acc.p);
	acc.q = ffma2(yi, tr, acc.q);
}

/* mbarrier + bulk-copy (TMA 1-D) plumbing */
__device__ __forceinline__ unsigned smem_u32(const void *p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long *bar, unsigned count)
{
	asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long *bar, unsigned bytes)
{
	asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long *bar, unsigned parity)
{
	asm volatile("{\n\t.reg .pred p;\n\tWAIT_%=:\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t@p bra DONE_%=;\n\tbra WAIT_%=;\n\tDONE_%=:\n\t}"
	             ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, unsigned bytes, unsigned long long *bar)
{
	asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
	             ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

/* one lane of a converged warp, chosen by the hardware: the compiler then knows the guarded block runs once per
 * warp and keeps warp-uniform operands (addresses built from a shuffled warp index) in uniform registers */
__device__ __forceinline__ bool elect_one()
{
	unsigned p;
	asm volatile("{\n\t.reg .pred q;\n\telect.sync _|q, 0xffffffff;\n\tselp.u32 %0, 1, 0, q;\n\t}" : "=r"(p));
	return p != 0;
}

/* Shared-memory plan of one CTA: WARPS warps, each with STAGES private tile buffers of 64 rows. */
template <int UNITS, int WARPS, int STAGES> struct DftPlan {
	static constexpr int ROWBYTES = UNITS * 16;
	/* rows per bulk copy, each copy followed by 16 bytes of padding.  The eight lanes of an LDS.128
	 * phase read eight consecutive rows at the same offset: they hit eight different 16-byte bank groups
	 * when the row stride is an odd number of units (UNITS odd after padding every row), or — UNITS = 20,
	 * stride = 4 mod 8 — when every second row is shifted by one more unit (pad after every two rows). */
	static constexpr int RPC = (UNITS % 8 == 4) ? 2 : 1;
	static constexpr int GROUP = RPC * ROWBYTES + 16;
	static constexpr int TILE_BYTES = DFT_ROWS / RPC * GROUP;
	static __device__ __forceinline__ int row_off(int r) { return (r / RPC) * GROUP + (r % RPC) * ROWBYTES; }
	static constexpr int N2 = UNITS * 2;                                     /* K/4 */
	static constexpr int TW_BYTES = N2 * CH_GROUP * 8;
	static constexpr int BAR_OFF = WARPS * STAGES * TILE_BYTES + TW_BYTES;
	static constexpr int SMEM = BAR_OFF + WARPS * STAGES * 8;
};

template <int UNITS, int WARPS, int STAGES, int MINB, bool FOLD8>
__global__ void __launch_bounds__(32 * WARPS, MINB)
k_channelize_dft(const uint8_t *__restrict__ in, size_t stream_stride, const float2 *__restrict__ tw,
                 const unsigned *__restrict__ meta, float *__restrict__ dm, int nch, int ngrp, size_t nsamp)
{
	using P = DftPlan<UNITS, WARPS, STAGES>;
	constexpr int CU = UNITS / 4;                 /* 16-byte units per quarter row */
	constexpr int N2 = P::N2;
	constexpr int NTILE = OUTBLK / DFT_ROWS;
	extern __shared__ __align__(16) unsigned char smem[];
	const int l = threadIdx.x & 31, w = threadIdx.x >> 5;
	const int blk = blockIdx.x, s = blockIdx.y, g = blockIdx.z;
	unsigned char *mytiles = smem + (size_t)w * STAGES * P::TILE_BYTES;
	const float4 *stw = reinterpret_cast<const float4 *>(smem + (size_t)WARPS * STAGES * P::TILE_BYTES);   /* [ch][n2] (Tr, Ti) */
	unsigned long long *bars = reinterpret_cast<unsigned long long *>(smem + P::BAR_OFF) + w * STAGES;
	const uint8_t *src_blk = in + (size_t)s * stream_stride + (size_t)blk * OUTBLK * P::ROWBYTES;
	const unsigned m = meta[(size_t)s * ngrp + g];    /* residue k_c mod 4 (0 or 2) of channel slot c in bits 2c, 2c+1 */

	if (l == 0)
		for (int i = 0; i < STAGES; i++) mbar_init(bars + i, 1);
	asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
	{
		const uint4 *tsrc = reinterpret_cast<const uint4 *>(tw + ((size_t)s * ngrp + g) * N2 * CH_GROUP);
		uint4 *tdst = reinterpret_cast<uint4 *>(smem + (size_t)WARPS * STAGES * P::TILE_BYTES);
		for (int q = threadIdx.x; q < P::TW_BYTES / 16; q += 32 * WARPS) cp_async16(tdst + q, tsrc + q);
		cp_async_commit();
		cp_async_wait_all();
	}
	__syncthreads();

	/* this warp's tiles: w, w + WARPS, ...; tile n of the warp uses stage n % STAGES */
	const int ntile = (NTILE - w + WARPS - 1) / WARPS;
	auto issue = [&](int n) {
		const int tile = w + n * WARPS;
		unsigned char *st = mytiles + (size_t)(n % STAGES) * P::TILE_BYTES;
		unsigned long long *bar = bars + n % STAGES;
		if (l == 0) {
			mbar_expect_tx(bar, DFT_ROWS * P::ROWBYTES);
			const uint8_t *src = src_blk + (size_t)tile * DFT_ROWS * P::ROWBYTES;
#pragma unroll 4
			for (int i = 0; i < DFT_ROWS / P::RPC; i++)
				bulk_g2s(st + (size_t)i * P::GROUP, src + (size_t)i * P::RPC * P::ROWBYTES, P::RPC * P::ROWBYTES, bar);
		}
	};
	for (int n = 0; n < STAGES && n < ntile; n++) issue(n);
	const int nc = min(CH_GROUP, nch - g * CH_GROUP);

	for (int n = 0; n < ntile; n++) {
		const int tile = w + n * WARPS;
		mbar_wait(bars + n % STAGES, (unsigned)((n / STAGES) & 1));
		const unsigned char *st = mytiles + (size_t)(n % STAGES) * P::TILE_BYTES;
		const uint4 *rowA = reinterpret_cast<const uint4 *>(st + P::row_off(l));
		const uint4 *rowB = reinterpret_cast<const uint4 *>(st + P::row_off(l + 32));
		DftAcc acc[CH_GROUP];
#pragma unroll
		for (int c = 0; c < CH_GROUP; c++) acc[c].a = acc[c].b = acc[c].p = acc[c].q = make_float2(0.f, 0.f);

		if constexpr (!FOLD8) {
			/* unit j covers samples 8j..8j+7 of each quarter: one LDS.128 per quarter and row (their latency
			 * is left to the other warps of the SM to cover) */
	#pragma unroll 1
			for (int j = 0; j < CU; j++) {
				uint4 qa[4], qb[4];
	#pragma unroll
				for (int n1 = 0; n1 < 4; n1++) { qa[n1] = rowA[n1 * CU + j]; qb[n1] = rowB[n1 * CU + j]; }
	#pragma unroll
				for (int eh = 0; eh < 2; eh++) {      /* four samples of each quarter at a time */
					float2 y0r[4], y0i[4], y2r[4], y2i[4];
	#pragma unroll
					for (int k = 0; k < 4; k++) {
						float2 xi[4], xq[4];
	#pragma unroll
						for (int n1 = 0; n1 < 4; n1++) {
							const unsigned wa = eh ? (k < 2 ? qa[n1].z : qa[n1].w) : (k < 2 ? qa[n1].x : qa[n1].y);
							const unsigned wb = eh ? (k < 2 ? qb[n1].z : qb[n1].w) : (k < 2 ? qb[n1].x : qb[n1].y);
							if (k & 1) { xi[n1] = dft_cvt<2>(wa, wb); xq[n1] = dft_cvt<3>(wa, wb); }
							else       { xi[n1] = dft_cvt<0>(wa, wb); xq[n1] = dft_cvt<1>(wa, wb); }
						}
						/* sums carry the 2 x 32768 planted by dft_cvt (exact: < 2^24); differences do not.  Y_0
						 * also sheds the converter's mid-scale 4 x 127.5 here: any constant is invisible to a
						 * channel (its twiddles sum to zero) but a large one costs accumulate precision */
						const float2 sI02 = fadd2_rn(xi[0], xi[2]), sI13 = fadd2_rn(xi[1], xi[3]);
						const float2 sQ02 = fadd2_rn(xq[0], xq[2]), sQ13 = fadd2_rn(xq[1], xq[3]);
						const float2 bias = make_float2(-131582.0f, -131582.0f);
						y0r[k] = fadd2_rn(fadd2_rn(sI02, sI13), bias);
						y0i[k] = fadd2_rn(fadd2_rn(sQ02, sQ13), bias);
						y2r[k] = fsub2(sI02, sI13);
						y2i[k] = fsub2(sQ02, sQ13);
					}
					/* channel c's four twiddles: two LDS.128, fetched one channel ahead of their use so the
					 * load latency hides under the previous channel's FFMAs (the residue dispatch below is a
					 * uniform branch the scheduler does not move loads across) */
					const float4 *tj = stw + (j * 2 + eh) * 2;
					float4 t0 = tj[0], t1 = tj[1];
	#pragma unroll
					for (int c = 0; c < CH_GROUP; c++) {
						const float4 u0 = t0, u1 = t1;
						if (c + 1 < CH_GROUP) { t0 = tj[(c + 1) * (N2 / 2)]; t1 = tj[(c + 1) * (N2 / 2) + 1]; }
						const float2 tt[4] = { make_float2(u0.x, u0.y), make_float2(u0.z, u0.w), make_float2(u1.x, u1.y), make_float2(u1.z, u1.w) };
						if (((m >> (2 * c)) & 3u) == 0) {             /* warp-uniform: k_c mod 4 is 0 or 2 */
	#pragma unroll
							for (int k = 0; k < 4; k++) dft_mac(acc[c], y0r[k], y0i[k], tt[k]);
						} else {
	#pragma unroll
							for (int k = 0; k < 4; k++) dft_mac(acc[c], y2r[k], y2i[k], tt[k]);
						}
					}
				}
			}
		} else {
			/* Bins are even (k = 2k'), so the row folds in half first: z[n] = x[n] + x[n + K/2] and D is bin
			 * k' of the K/2-point DFT of z; the same four-way split of THAT gives
			 *   D = sum_{n2 < K/8} T[n2] * Y'_{k' mod 4}[n2],   Y'_r[n2] = sum_{n1<4} z[(K/8)*n1 + n2] * (-j)^(r*n1)
			 * with the same twiddles T[n2] = exp(-j*2*pi*k*n2/K)/K/127.5 and all four residues in play:
			 * 26 packed additions per n2 (exact) and K/8 complex MACs per channel.  Group g4 covers samples
			 * 4*g4..4*g4+3 of each eighth of the row: one LDS.64 per eighth and row. */
			const unsigned char *ra = st + P::row_off(l), *rb = st + P::row_off(l + 32);
#pragma unroll 1
			for (int g4 = 0; g4 < CU; g4++) {
				uint2 ea[8], eb[8];
#pragma unroll
				for (int e = 0; e < 8; e++) {
					ea[e] = *reinterpret_cast<const uint2 *>(ra + e * (UNITS * 2) + g4 * 8);
					eb[e] = *reinterpret_cast<const uint2 *>(rb + e * (UNITS * 2) + g4 * 8);
				}
				float2 yr[4][4], yi[4][4];            /* [residue][sample of the group] */
#pragma unroll
				for (int k = 0; k < 4; k++) {
					float2 zi[4], zq[4];
#pragma unroll
					for (int n1 = 0; n1 < 4; n1++) {
						const unsigned wa0 = k < 2 ? ea[n1].x : ea[n1].y, wb0 = k < 2 ? eb[n1].x : eb[n1].y;
						const unsigned wa1 = k < 2 ? ea[n1 + 4].x : ea[n1 + 4].y, wb1 = k < 2 ? eb[n1 + 4].x : eb[n1 + 4].y;
						if (k & 1) {
							zi[n1] = fadd2_rn(dft_cvt<2>(wa0, wb0), dft_cvt<2>(wa1, wb1));
							zq[n1] = fadd2_rn(dft_cvt<3>(wa0, wb0), dft_cvt<3>(wa1, wb1));
						} else {
							zi[n1] = fadd2_rn(dft_cvt<0>(wa0, wb0), dft_cvt<0>(wa1, wb1));
							zq[n1] = fadd2_rn(dft_cvt<1>(wa0, wb0), dft_cvt<1>(wa1, wb1));
						}
					}
					/* every z carries 2 x 32768 from dft_cvt: sums of four carry 262144 (exact, < 2^24) and Y'_0
					 * also sheds the converter's mid-scale 8 x 127.5; differences carry nothing */
					const float2 sI02 = fadd2_rn(zi[0], zi[2]), sI13 = fadd2_rn(zi[1], zi[3]);
					const float2 sQ02 = fadd2_rn(zq[0], zq[2]), sQ13 = fadd2_rn(zq[1], zq[3]);
					const float2 dI02 = fsub2(zi[0], zi[2]), dI13 = fsub2(zi[1], zi[3]);
					const float2 dQ02 = fsub2(zq[0], zq[2]), dQ13 = fsub2(zq[1], zq[3]);
					const float2 bias = make_float2(-263164.0f, -263164.0f);
					yr[0][k] = fadd2_rn(fadd2_rn(sI02, sI13), bias);
					yi[0][k] = fadd2_rn(fadd2_rn(sQ02, sQ13), bias);
					yr[2][k] = fsub2(sI02, sI13);
					yi[2][k] = fsub2(sQ02, sQ13);
					yr[1][k] = fadd2_rn(dI02, dQ13); yi[1][k] = fsub2(dQ02, dI13);      /* (z0-z2) - j(z1-z3) */
					yr[3][k] = fsub2(dI02, dQ13);      yi[3][k] = fadd2_rn(dQ02, dI13); /* (z0-z2) + j(z1-z3) */
				}
				const float4 *tj = stw + g4 * 2;
				float4 t0 = tj[0], t1 = tj[1];
#pragma unroll
				for (int c = 0; c < CH_GROUP; c++) {
					const float4 u0 = t0, u1 = t1;
					if (c + 1 < CH_GROUP) { t0 = tj[(c + 1) * (N2 / 2)]; t1 = tj[(c + 1) * (N2 / 2) + 1]; }
					const float2 tt[4] = { make_float2(u0.x, u0.y), make_float2(u0.z, u0.w), make_float2(u1.x, u1.y), make_float2(u1.z, u1.w) };
					const unsigned r8 = (m >> (16 + 2 * c)) & 3u;     /* warp-uniform: (k_c / 2) mod 4 */
					if (r8 == 0) {
#pragma unroll
						for (int k = 0; k < 4; k++) dft_mac(acc[c], yr[0][k], yi[0][k], tt[k]);
					} else if (r8 == 1) {
#pragma unroll
						for (int k = 0; k < 4; k++) dft_mac(acc[c], yr[1][k], yi[1][k], tt[k]);
					} else if (r8 == 2) {
#pragma unroll
						for (int k = 0; k < 4; k++) dft_mac(acc[c], yr[2][k], yi[2][k], tt[k]);
					} else {
#pragma unroll
						for (int k = 0; k < 4; k++) dft_mac(acc[c], yr[3][k], yi[3][k], tt[k]);
					}
				}
			}
		}
		/* every lane has its rows in registers: the stage can take the warp's tile n + STAGES */
		__syncwarp();
		if (n + STAGES < ntile) issue(n + STAGES);
		/* |D| out (rtl.c:353) for the lane's two rows */
#pragma unroll
		for (int half = 0; half < 2; half++) {
			float e[CH_GROUP];
#pragma unroll
			for (int c = 0; c < CH_GROUP; c++) {
				const float re = half ? __fadd_rn(acc[c].a.y, -acc[c].b.y) : __fadd_rn(acc[c].a.x, -acc[c].b.x);
				const float im = half ? __fadd_rn(acc[c].p.y, acc[c].q.y) : __fadd_rn(acc[c].p.x, acc[c].q.x);
				/* |D| in float: half an ulp, this form's tolerance is 1e-5.  u8 input bounds it: |x - 127.5| <= 127.5 and
				 * |tw| = 1/(127.5 K), so |D| <= ~1.5 (no overflow); where re*re goes denormal the absolute error is < 3e-23,
				 * against 1e-6 of a row total that is >= 0.5/127.5/K (every sample is >= 0.5 from 127.5) */
				e[c] = __fsqrt_rn(__fmaf_rn(re, re, __fmul_rn(im, im)));
			}
			const size_t mrow = (size_t)blk * OUTBLK + (size_t)tile * DFT_ROWS + l + half * 32;
			float *o = dm + ((size_t)s * nsamp + mrow) * nch + g * CH_GROUP;
			if (nc == CH_GROUP && (nch & 3) == 0) {
				reinterpret_cast<float4 *>(o)[0] = make_float4(e[0], e[1], e[2], e[3]);
				reinterpret_cast<float4 *>(o)[1] = make_float4(e[4], e[5], e[6], e[7]);
			} else {
#pragma unroll
				for (int c = 0; c < CH_GROUP; c++)
					if (c < nc) o[c] = e[c];
			}
		}
	}
}

template <int UNITS, int WARPS, int STAGES, int MINB, bool FOLD8>
static int launch_dft_t(const uint8_t *in, size_t stream_stride, const float2 *tw, const unsigned *meta, float *dm,
                        int nch, int nstreams, int nblk, size_t nsamp, cudaStream_t stream)
{
	const int ngrp = (nch + CH_GROUP - 1) / CH_GROUP;
	constexpr int smem = DftPlan<UNITS, WARPS, STAGES>::SMEM;
	auto kern = k_channelize_dft<UNITS, WARPS, STAGES, MINB, FOLD8>;
	if (cudaError_t e = smem_max_carveout(kern, smem)) return (int)e;
	dim3 grid(nblk, nstreams, ngrp);
	kern<<<grid, 32 * WARPS, smem, stream>>>(in, stream_stride, tw, meta, dm, nch, ngrp, nsamp);
	return (int)cudaGetLastError();
}

/* The folded fast form with ONE row per lane and the pair packing moved from "two rows" to "(re, im)": a lane's
 * accumulators for channel c are A = (a, p) and B = (q, b), fed by two float2 FMAs per complex MAC —
 *     A += (yr, yr) * (Tr, Ti)        B += (yi, yi) * (Tr, Ti)          re = A.x - B.y, im = A.y + B.x
 * — the very same four sums, term for term and in the same order, that the two-rows-per-lane kernel above keeps in
 * a, b, p, q: the envelope is BIT-IDENTICAL to that kernel's (and to the CPU restatement orc_channelize_dft8).  The
 * shared 4-point DFTs run on (I, Q) pairs, exact in float like before.  What changes is the footprint: a warp's tile
 * is 32 rows (10.5 KB instead of 21 KB) and a thread holds one row's worth of state (~100 registers instead of 162),
 * so 16-20 warps fit an SM instead of 10 — the two-row kernel is latency bound at 2.5 warps per scheduler — and the
 * demod warps that share the SMs displace smaller pieces. */
constexpr int DFT1_ROWS = 32;

/* KIND: IN_U8IQ (2 bytes per complex sample, UNITS = K/8 sixteen-byte units per row) or IN_CS16IQ (4 bytes per complex
 * sample: the same kernel with rows twice as long, another converter, and rows padded one by one — 16·UNITS·2 bytes is a
 * multiple of 128, so every row needs its own 16-byte shift to spread the lanes over the bank groups) */
template <int KIND, int UNITS, int WARPS> struct Dft1Plan {
	static constexpr int BPS = KIND == IN_CS16IQ ? 4 : 2;                     /* bytes per complex sample */
	static constexpr int ROWBYTES = UNITS * 8 * BPS;
	static constexpr int RPC = (KIND != IN_CS16IQ && UNITS % 8 == 4) ? 2 : 1; /* rows per bulk copy, see DftPlan */
	static constexpr int GROUP = RPC * ROWBYTES + 16;
	static constexpr int TILE_BYTES = DFT1_ROWS / RPC * GROUP;
	static __device__ __forceinline__ int row_off(int r) { return (r / RPC) * GROUP + (r % RPC) * ROWBYTES; }
	static constexpr int N2 = UNITS * 2;                                      /* K/4: twiddles are stored for the 4-way split */
	static constexpr int TW_BYTES = N2 * CH_GROUP * 8;
	static constexpr int BAR_OFF = WARPS * TILE_BYTES + TW_BYTES;
	static constexpr int SMEM = BAR_OFF + WARPS * 8;
};

/* bytes `KB`, `KB+1` (I, Q of one sample) of word w as (32768 + I, 32768 + Q) */
template <int KB> __device__ __forceinline__ float2 dft1_cvt(unsigned w)
{
	constexpr unsigned si = 0x7404u | (KB << 4), sq = 0x7404u | ((KB + 1) << 4);
	return make_float2(__uint_as_float(__byte_perm(w, 0x47000000u, si)), __uint_as_float(__byte_perm(w, 0x47000000u, sq)));
}
/* CS16: the two 16-bit halves of w (already XORed, see the kernel) planted in the mantissa of 2^23: (2^23 + lo, 2^23 + hi) */
__device__ __forceinline__ float2 dft1_cvt16(unsigned w)
{
	return make_float2(__uint_as_float(__byte_perm(w, 0x4B000000u, 0x7410)), __uint_as_float(__byte_perm(w, 0x4B000000u, 0x7432)));
}

template <int KIND, int UNITS, int WARPS, int MINB, bool PF>
__global__ void __launch_bounds__(32 * WARPS, MINB)
k_channelize_dft1(const uint8_t *__restrict__ in, size_t stream_stride, const float2 *__restrict__ tw,
                  const unsigned *__restrict__ meta, float *__restrict__ dm, int nch, int ngrp, size_t nsamp)
{
	using P = Dft1Plan<KIND, UNITS, WARPS>;
	constexpr int CU = UNITS / 4;                 /* groups of 4 samples per eighth of a row */
	constexpr int N2 = P::N2;
	constexpr int NTILE = OUTBLK / DFT1_ROWS;
	extern __shared__ __align__(16) unsigned char smem[];
	const int l = threadIdx.x & 31;
	const int w = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0);     /* warp-uniform for the compiler too: the bulk-copy operands stay in uniform registers */
	const int blk = blockIdx.x, s = blockIdx.y, g = blockIdx.z;
	unsigned char *mytile = smem + (size_t)w * P::TILE_BYTES;
	const float4 *stw = reinterpret_cast<const float4 *>(smem + (size_t)WARPS * P::TILE_BYTES);   /* [ch][n2] (Tr, Ti) */
	unsigned long long *bar = reinterpret_cast<unsigned long long *>(smem + P::BAR_OFF) + w;
	const uint8_t *src_blk = in + (size_t)s * stream_stride + (size_t)blk * OUTBLK * P::ROWBYTES;
	const unsigned m = __shfl_sync(0xffffffffu, meta[(size_t)s * ngrp + g], 0);    /* (k_c / 2) mod 4 of channel slot c in bits 16 + 2c, 17 + 2c */

	if (l == 0) mbar_init(bar, 1);
	asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
	/* Which Y a channel multiplies is its bin's residue (k_c / 2) mod 4 — warp-uniform, so a branch, not selects.  To
	 * make that branch cheap the CTA works on its channel slots SORTED by residue (a stable counting sort of the eight
	 * 2-bit fields, once per CTA): slot j holds channel perm[j], the twiddles are staged in slot order, the envelope is
	 * stored through perm[], and the MAC section below is four straight-line columns (one per residue) that a warp walks
	 * left to right, moving one column over where the next slot's residue is larger: one compare + branch per slot
	 * instead of a compare-and-branch chain per channel. */
	unsigned pw = 0;                             /* perm[j] in bits 3j .. 3j+2 */
	int bnd0, bnd1, bnd2;                        /* first slot whose residue is > 0, > 1, > 2 */
	{
		int cnt[4] = { 0, 0, 0, 0 };
#pragma unroll
		for (int c = 0; c < CH_GROUP; c++) {
			const unsigned r = (m >> (16 + 2 * c)) & 3u;
#pragma unroll
			for (int q = 0; q < 4; q++) cnt[q] += (r == (unsigned)q);
		}
		bnd0 = cnt[0]; bnd1 = bnd0 + cnt[1]; bnd2 = bnd1 + cnt[2];
		int pos[4] = { 0, bnd0, bnd1, bnd2 };
#pragma unroll
		for (int c = 0; c < CH_GROUP; c++) {
			const unsigned r = (m >> (16 + 2 * c)) & 3u;
			int at = 0;
#pragma unroll
			for (int q = 0; q < 4; q++) { at = (r == (unsigned)q) ? pos[q] : at; pos[q] += (r == (unsigned)q); }
			pw |= (unsigned)c << (3 * at);
		}
	}
	{
		const uint4 *tsrc = reinterpret_cast<const uint4 *>(tw + ((size_t)s * ngrp + g) * N2 * CH_GROUP);
		uint4 *tdst = reinterpret_cast<uint4 *>(smem + (size_t)WARPS * P::TILE_BYTES);
		constexpr int PER = N2 * 8 / 16;         /* 16-byte pieces per channel */
		for (int q = threadIdx.x; q < P::TW_BYTES / 16; q += 32 * WARPS) {
			const int j = q / PER, off = q - j * PER;
			cp_async16(tdst + q, tsrc + ((pw >> (3 * j)) & 7u) * PER + off);
		}
		cp_async_commit();
		cp_async_wait_all();
	}
	__syncthreads();

	/* this warp's tiles: w, w + WARPS, ...; the streaming inputs (CS16) may end inside a block: tiles that start past
	 * the last row are not touched, the last one reads up to 31 rows of slack behind the input (context.cu allocates it) */
	const size_t rows_left = nsamp - (size_t)blk * OUTBLK;
	const int tiles_here = rows_left >= (size_t)OUTBLK ? NTILE : (int)((rows_left + DFT1_ROWS - 1) / DFT1_ROWS);
	const int ntile = (tiles_here - w + WARPS - 1) / WARPS;
	auto issue = [&](int n) {
		if (elect_one()) {
			mbar_expect_tx(bar, DFT1_ROWS * P::ROWBYTES);
			const uint8_t *src = src_blk + (size_t)(w + n * WARPS) * DFT1_ROWS * P::ROWBYTES;
#pragma unroll
			for (int i = 0; i < DFT1_ROWS / P::RPC; i++)
				bulk_g2s(mytile + (size_t)i * P::GROUP, src + (size_t)i * P::RPC * P::ROWBYTES, P::RPC * P::ROWBYTES, bar);
		}
	};
	if (ntile > 0) issue(0);
	const int nc = min(CH_GROUP, nch - g * CH_GROUP);

	for (int n = 0; n < ntile; n++) {
		const int tile = w + n * WARPS;
		mbar_wait(bar, (unsigned)(n & 1));
		const unsigned char *ra = mytile + P::row_off(l);
		float2 A[CH_GROUP], B[CH_GROUP];
#pragma unroll
		for (int c = 0; c < CH_GROUP; c++) A[c] = B[c] = make_float2(0.f, 0.f);

#pragma unroll 1
		for (int g4 = 0; g4 < CU; g4++) {
			uint2 e8[8];
			uint4 e16[8];
#pragma unroll
			for (int e = 0; e < 8; e++) {
				if (KIND == IN_CS16IQ) e16[e] = *reinterpret_cast<const uint4 *>(ra + e * (UNITS * 4) + g4 * 16);
				else e8[e] = *reinterpret_cast<const uint2 *>(ra + e * (UNITS * 2) + g4 * 8);
			}
			float2 Y[4][4];                       /* [residue][sample of the group] = (re, im) */
#pragma unroll
			for (int k = 0; k < 4; k++) {
				float2 z[4];
#pragma unroll
				for (int n1 = 0; n1 < 4; n1++) {
					if (KIND == IN_CS16IQ) {
						/* int16 v as the unsigned v + 32768 (XOR 0x8000) in the first half of the row, as 32767 - v (XOR 0x7fff) in
						 * the second: both planted in the mantissa of 2^23, their DIFFERENCE is v0 + v1 + 1, exact (operands in
						 * [2^23, 2^24)) — one XOR per word, two PRMT, one packed subtraction per folded sample */
						const uint4 a = e16[n1], b = e16[n1 + 4];
						const unsigned w0 = (k == 0 ? a.x : k == 1 ? a.y : k == 2 ? a.z : a.w) ^ 0x80008000u;
						const unsigned w1 = (k == 0 ? b.x : k == 1 ? b.y : k == 2 ? b.z : b.w) ^ 0x7fff7fffu;
						z[n1] = fsub2(dft1_cvt16(w0), dft1_cvt16(w1));
					} else {
						const unsigned w0 = k < 2 ? e8[n1].x : e8[n1].y, w1 = k < 2 ? e8[n1 + 4].x : e8[n1 + 4].y;
						z[n1] = (k & 1) ? fadd2_rn(dft1_cvt<2>(w0), dft1_cvt<2>(w1)) : fadd2_rn(dft1_cvt<0>(w0), dft1_cvt<0>(w1));
					}
				}
				/* u8: every z carries 2 x 32768 from the converter: sums of four carry 262144 (exact, < 2^24) and Y'_0 also
				 * sheds the converter's mid-scale 8 x 127.5; CS16: every z carries + 1, |z| < 2^17; differences carry nothing */
				const float2 s02 = fadd2_rn(z[0], z[2]), s13 = fadd2_rn(z[1], z[3]);
				const float2 d02 = fsub2(z[0], z[2]);
				const float2 wj = make_float2(__fadd_rn(z[1].y, -z[3].y), __fadd_rn(z[3].x, -z[1].x));   /* -j (z1 - z3) */
				const float y0bias = KIND == IN_CS16IQ ? -4.0f : -263164.0f;
				Y[0][k] = fadd2_rn(fadd2_rn(s02, s13), make_float2(y0bias, y0bias));
				Y[2][k] = fsub2(s02, s13);
				Y[1][k] = fadd2_rn(d02, wj);    /* (z0 - z2) - j (z1 - z3) */
				Y[3][k] = fsub2(d02, wj);         /* (z0 - z2) + j (z1 - z3) */
			}
			const float4 *tj = stw + g4 * 2;
			float4 nu0 = make_float4(0.f, 0.f, 0.f, 0.f), nu1 = nu0;
			if (PF) { nu0 = tj[0]; nu1 = tj[1]; }
#define ACB_DFT1_MAC(J, R)                                                                 \
			{                                                                                      \
				const float4 u0 = PF ? nu0 : tj[(J) * (N2 / 2)], u1 = PF ? nu1 : tj[(J) * (N2 / 2) + 1];   \
				/* PF: loaded one slot ahead, whichever column that was */                             \
				if (PF && (J) + 1 < CH_GROUP) { nu0 = tj[((J) + 1) * (N2 / 2)]; nu1 = tj[((J) + 1) * (N2 / 2) + 1]; } \
				const float2 tt[4] = { make_float2(u0.x, u0.y), make_float2(u0.z, u0.w),               \
				                       make_float2(u1.x, u1.y), make_float2(u1.z, u1.w) };             \
				_Pragma("unroll") for (int k = 0; k < 4; k++) {                                        \
					A[J] = ffma2(make_float2(Y[R][k].x, Y[R][k].x), tt[k], A[J]);                          \
					B[J] = ffma2(make_float2(Y[R][k].y, Y[R][k].y), tt[k], B[J]);                          \
				}                                                                                      \
			}
#define ACB_DFT1_C0(J) if ((J) >= bnd0) goto c1_##J; ACB_DFT1_MAC(J, 0)
#define ACB_DFT1_C1(J) c1_##J: if ((J) >= bnd1) goto c2_##J; ACB_DFT1_MAC(J, 1)
#define ACB_DFT1_C2(J) c2_##J: if ((J) >= bnd2) goto c3_##J; ACB_DFT1_MAC(J, 2)
#define ACB_DFT1_C3(J) c3_##J: ACB_DFT1_MAC(J, 3)
#define ACB_DFT1_COL(C) C(0) C(1) C(2) C(3) C(4) C(5) C(6) C(7)
			ACB_DFT1_COL(ACB_DFT1_C0) goto macs_done;
			ACB_DFT1_COL(ACB_DFT1_C1) goto macs_done;
			ACB_DFT1_COL(ACB_DFT1_C2) goto macs_done;
			ACB_DFT1_COL(ACB_DFT1_C3)
			macs_done:;
#undef ACB_DFT1_COL
#undef ACB_DFT1_C3
#undef ACB_DFT1_C2
#undef ACB_DFT1_C1
#undef ACB_DFT1_C0
#undef ACB_DFT1_MAC
		}
		/* every lane has its row in registers: the buffer can take the warp's next tile */
		__syncwarp();
		if (n + 1 < ntile) issue(n + 1);
		float e[CH_GROUP];
#pragma unroll
		for (int c = 0; c < CH_GROUP; c++) {
			const float re = __fadd_rn(A[c].x, -B[c].y), im = __fadd_rn(A[c].y, B[c].x);
			/* |D| in float.  Integer input bounds it: u8 as in k_channelize_dft; CS16 |x| <= 32768 scaled by 1/32768
			 * or 1/4, so |D| <= ~1.2e4 (no overflow), and a row that is not all zeros has a total >= 2^-15/K, far above
			 * the < 3e-23 absolute error of a denormal re*re */
			e[c] = __fsqrt_rn(__fmaf_rn(re, re, __fmul_rn(im, im)));
		}
		const size_t mrow = (size_t)blk * OUTBLK + (size_t)tile * DFT1_ROWS + l;
		float *o = dm + ((size_t)s * nsamp + mrow) * nch + g * CH_GROUP;
		/* slot j is channel perm[j]: eight 4-byte stores into the lane's own 32-byte sector */
#pragma unroll
		for (int j = 0; j < CH_GROUP; j++) {
			const int c = (int)((pw >> (3 * j)) & 7u);
			if (c < nc && mrow < nsamp) o[c] = e[j];
		}
	}
}

template <int KIND, int UNITS, int WARPS, int MINB, bool PF>
static int launch_dft1_t(const uint8_t *in, size_t stream_stride, const float2 *tw, const unsigned *meta, float *dm,
                         int nch, int nstreams, int nblk, size_t nsamp, cudaStream_t stream)
{
	const int ngrp = (nch + CH_GROUP - 1) / CH_GROUP;
	constexpr int smem = Dft1Plan<KIND, UNITS, WARPS>::SMEM;
	auto kern = k_channelize_dft1<KIND, UNITS, WARPS, MINB, PF>;
	if (cudaError_t e = smem_max_carveout(kern, smem)) return (int)e;
	dim3 grid(nblk, nstreams, ngrp);
	kern<<<grid, 32 * WARPS, smem, stream>>>(in, stream_stride, tw, meta, dm, nch, ngrp, nsamp);
	return (int)cudaGetLastError();
}

/* ------------------------------------------------------------------------------------------
 * K1, overlapping window, polyphase fast form (ACB_FLAG_FAST_FILTER; DESIGN.md §4).  With every channel on the 12.5 kHz
 * raster the low-pass table of a taps > K context is w[i] = h[i] * exp(-j*2*pi*k*(i - H)/K) * scale: one real prototype
 * times a DFT exponential of period K.  Split the window of row m by the phase n = (i - H) mod K:
 *
 *     D = sum_{n < K} T[n] * z_m[n],   z_m[n] = sum_r p[n + H + r*K] * x[m*K + n + r*K],   p = fl(K * h),
 *     T[n] = exp(-j*2*pi*k*n/K)/K * scale   (the twiddles of the boxcar fast form)
 *
 * z_m (the polyphase pre-sum) is shared by every channel of the stream; each channel then needs the bin of a K-point
 * DFT of one row, which is k_channelize_dft1's fold / shared 4-point DFT / residue-sorted MAC columns unchanged.
 *
 * Shape: k_channelize_dft1's, with the window.  A warp's tile is its 32 rows plus the hpad samples in front of them (the
 * halo, HR = ceil(hpad/K) more rows, the first one partial), staged by one bulk copy per row; rows before the submit come
 * from the stream's history (u8: the context's buffer; CS16: the samples in front of the input), the same address rule as
 * k_channelize<MODE, true>.  Lane l builds z of its row l from the staged window — for each 4-sample group of an eighth
 * of the row, the terms r = rlo .. 0 in ascending tap order, one FFMA per component — folds and splits it in registers
 * and hands it to the MAC columns: z never leaves the SM.  p (taps_pad floats, zero weights in front like the exact
 * table) is read through L1 with a warp-uniform address.  Terms whose row lies before the stream start (absolute row
 * pos0 + m + r < 0) are skipped, so the rows after acb_create / acb_reset need no second kernel: for u8 the zero bytes of
 * a cleared history would convert to -127.37, not to 0.
 *
 * Zero-weight terms (the front padding of p) leave z exactly as it was: z starts at +0, fma(+0, x, +0) = +0, and once a
 * real term has arrived, z + (+-0) = z.  So this kernel's z equals the restatement's sum over the valid terms only
 * (tests/host/ovl_fast_oracle.c: orc_channelize_ovl_fast), bit for bit.
 * ---------------------------------------------------------------------------------------- */
template <int KIND, int UNITS, int WARPS>
__global__ void __launch_bounds__(32 * WARPS)
k_channelize_ovl_fast(const uint8_t *__restrict__ in, size_t stream_stride, const uint8_t *__restrict__ hist, size_t hist_stride,
                      int hpad, unsigned long long pos0, const float *__restrict__ pw, const float2 *__restrict__ tw,
                      const unsigned *__restrict__ meta, float *__restrict__ dm, int nch, int ngrp, size_t nsamp)
{
	using P = Dft1Plan<KIND, UNITS, WARPS>;
	constexpr int K = UNITS * 8, BPS = P::BPS;
	constexpr int CU = UNITS / 4;                 /* groups of 4 samples per eighth of a row */
	constexpr int N2 = P::N2;
	constexpr int NTILE = OUTBLK / DFT1_ROWS;
	extern __shared__ __align__(16) unsigned char smem[];
	const int l = threadIdx.x & 31;
	const int w = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0);
	const int blk = blockIdx.x, s = blockIdx.y, g = blockIdx.z;
	const int HR = (hpad + K - 1) / K;            /* halo rows in front of the tile, the first one from sample n0 on */
	const int n0 = HR * K - hpad;
	/* rows one by one, each shifted by 16 more bytes (a lane's terms r, r+1 are one stride apart: one add per term) */
	constexpr int STRIDE = P::ROWBYTES + 16;
	const size_t tile_bytes = (size_t)(DFT1_ROWS + HR) * STRIDE;
	unsigned char *mytile = smem + (size_t)w * tile_bytes;
	const float4 *stw = reinterpret_cast<const float4 *>(smem + (size_t)WARPS * tile_bytes);     /* [slot][n2] (Tr, Ti) */
	unsigned long long *bar = reinterpret_cast<unsigned long long *>(smem + (size_t)WARPS * tile_bytes + P::TW_BYTES) + w;
	const uint8_t *src_s = in + (size_t)s * stream_stride;
	const uint8_t *hist_s = hist + (size_t)s * hist_stride + (size_t)hpad * BPS;      /* where sample 0 of the submit would sit */
	const unsigned m = __shfl_sync(0xffffffffu, meta[(size_t)s * ngrp + g], 0);

	if (l == 0) mbar_init(bar, 1);
	asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
	/* channel slots sorted by residue (k_c / 2) mod 4, as in k_channelize_dft1 */
	unsigned pperm = 0;
	int bnd0, bnd1, bnd2;
	{
		int cnt[4] = { 0, 0, 0, 0 };
#pragma unroll
		for (int c = 0; c < CH_GROUP; c++) {
			const unsigned r = (m >> (16 + 2 * c)) & 3u;
#pragma unroll
			for (int q = 0; q < 4; q++) cnt[q] += (r == (unsigned)q);
		}
		bnd0 = cnt[0]; bnd1 = bnd0 + cnt[1]; bnd2 = bnd1 + cnt[2];
		int pos[4] = { 0, bnd0, bnd1, bnd2 };
#pragma unroll
		for (int c = 0; c < CH_GROUP; c++) {
			const unsigned r = (m >> (16 + 2 * c)) & 3u;
			int at = 0;
#pragma unroll
			for (int q = 0; q < 4; q++) { at = (r == (unsigned)q) ? pos[q] : at; pos[q] += (r == (unsigned)q); }
			pperm |= (unsigned)c << (3 * at);
		}
	}
	{
		const uint4 *tsrc = reinterpret_cast<const uint4 *>(tw + ((size_t)s * ngrp + g) * N2 * CH_GROUP);
		uint4 *tdst = reinterpret_cast<uint4 *>(smem + (size_t)WARPS * tile_bytes);
		constexpr int PER = N2 * 8 / 16;
		for (int q = threadIdx.x; q < P::TW_BYTES / 16; q += 32 * WARPS) {
			const int j = q / PER, off = q - j * PER;
			cp_async16(tdst + q, tsrc + ((pperm >> (3 * j)) & 7u) * PER + off);
		}
		cp_async_commit();
		cp_async_wait_all();
	}
	__syncthreads();

	const size_t rows_left = nsamp - (size_t)blk * OUTBLK;
	const int tiles_here = rows_left >= (size_t)OUTBLK ? NTILE : (int)((rows_left + DFT1_ROWS - 1) / DFT1_ROWS);
	const int ntile = (tiles_here - w + WARPS - 1) / WARPS;
	auto issue = [&](int n) {
		if (elect_one()) {
			mbar_expect_tx(bar, (unsigned)((hpad + DFT1_ROWS * K) * BPS));
			const long long row0 = (long long)blk * OUTBLK + (long long)(w + n * WARPS) * DFT1_ROWS - HR;
			for (int b = 0; b < DFT1_ROWS + HR; b++) {
				const int s0 = b == 0 ? n0 : 0;
				const long long smp = (row0 + b) * K + s0;           /* >= -hpad: before the submit means in the history */
				const uint8_t *src = smp < 0 ? hist_s + smp * BPS : src_s + smp * BPS;
				bulk_g2s(mytile + (size_t)b * STRIDE + s0 * BPS, src, (unsigned)((K - s0) * BPS), bar);
			}
		}
	};
	if (ntile > 0) issue(0);
	const int nc = min(CH_GROUP, nch - g * CH_GROUP);

	for (int n = 0; n < ntile; n++) {
		const int tile = w + n * WARPS;
		mbar_wait(bar, (unsigned)(n & 1));
		const size_t mrow = (size_t)blk * OUTBLK + (size_t)tile * DFT1_ROWS + l;
		const unsigned long long mabs = pos0 + mrow;                  /* row counted from the stream start */
		float2 A[CH_GROUP], B[CH_GROUP];
#pragma unroll
		for (int c = 0; c < CH_GROUP; c++) A[c] = B[c] = make_float2(0.f, 0.f);

#pragma unroll 1
		for (int g4 = 0; g4 < CU; g4++) {
			/* the pre-sum z of samples n .. n+3 of eighth e, in ascending tap order */
			auto presum = [&](int e, float2 (&z)[4]) {
				const int nn = e * (K / 8) + 4 * g4;
				int rlo = -((nn + hpad) / K);                            /* warp-uniform: the same for the 4 samples */
				if ((unsigned long long)(-rlo) > mabs) rlo = -(int)mabs;  /* rows before the stream start: omitted */
#pragma unroll
				for (int k = 0; k < 4; k++) z[k] = make_float2(0.f, 0.f);
				const float *pr = pw + nn + hpad;
				const unsigned char *myrow = mytile + (size_t)(l + HR) * STRIDE + nn * BPS;
#pragma unroll 2
				for (int r = rlo; r <= 0; r++) {
					const unsigned char *q = myrow + r * STRIDE;
					const float4 pv = __ldg(reinterpret_cast<const float4 *>(pr + r * K));
					const float pk[4] = { pv.x, pv.y, pv.z, pv.w };
					float2 x[4];
					if (KIND == IN_CS16IQ) {
						const uint4 u = *reinterpret_cast<const uint4 *>(q);
						x[0] = cvt_cs16(u.x); x[1] = cvt_cs16(u.y); x[2] = cvt_cs16(u.z); x[3] = cvt_cs16(u.w);
					} else {
						const uint2 u = *reinterpret_cast<const uint2 *>(q);
						x[0] = cvt_iq(u.x, 0); x[1] = cvt_iq(u.x, 1); x[2] = cvt_iq(u.y, 0); x[3] = cvt_iq(u.y, 1);
					}
#pragma unroll
					for (int k = 0; k < 4; k++) z[k] = ffma2(x[k], make_float2(pk[k], pk[k]), z[k]);
				}
			};
			float2 Y[4][4];                       /* [residue][sample of the group] = (re, im) */
#pragma unroll
			for (int n1 = 0; n1 < 4; n1++) {      /* fold: z'[n] = z[n] + z[n + K/2], eighths n1 and n1 + 4 */
				float2 za[4], zb[4];
				presum(n1, za);
				presum(n1 + 4, zb);
#pragma unroll
				for (int k = 0; k < 4; k++) Y[n1][k] = fadd2_rn(za[k], zb[k]);
			}
#pragma unroll
			for (int k = 0; k < 4; k++) {
				const float2 z0 = Y[0][k], z1 = Y[1][k], z2 = Y[2][k], z3 = Y[3][k];
				const float2 s02 = fadd2_rn(z0, z2), s13 = fadd2_rn(z1, z3);
				const float2 d02 = fsub2(z0, z2);
				const float2 wj = make_float2(__fadd_rn(z1.y, -z3.y), __fadd_rn(z3.x, -z1.x));   /* -j (z1 - z3) */
				Y[0][k] = fadd2_rn(s02, s13);
				Y[2][k] = fsub2(s02, s13);
				Y[1][k] = fadd2_rn(d02, wj);      /* (z0 - z2) - j (z1 - z3) */
				Y[3][k] = fsub2(d02, wj);         /* (z0 - z2) + j (z1 - z3) */
			}
			const float4 *tj = stw + g4 * 2;
			float4 nu0 = tj[0], nu1 = tj[1];
#define ACB_OVF_MAC(J, R)                                                                  \
			{                                                                                      \
				const float4 u0 = nu0, u1 = nu1;                                                       \
				if ((J) + 1 < CH_GROUP) { nu0 = tj[((J) + 1) * (N2 / 2)]; nu1 = tj[((J) + 1) * (N2 / 2) + 1]; } \
				const float2 tt[4] = { make_float2(u0.x, u0.y), make_float2(u0.z, u0.w),               \
				                       make_float2(u1.x, u1.y), make_float2(u1.z, u1.w) };             \
				_Pragma("unroll") for (int k = 0; k < 4; k++) {                                        \
					A[J] = ffma2(make_float2(Y[R][k].x, Y[R][k].x), tt[k], A[J]);                          \
					B[J] = ffma2(make_float2(Y[R][k].y, Y[R][k].y), tt[k], B[J]);                          \
				}                                                                                      \
			}
#define ACB_OVF_C0(J) if ((J) >= bnd0) goto c1_##J; ACB_OVF_MAC(J, 0)
#define ACB_OVF_C1(J) c1_##J: if ((J) >= bnd1) goto c2_##J; ACB_OVF_MAC(J, 1)
#define ACB_OVF_C2(J) c2_##J: if ((J) >= bnd2) goto c3_##J; ACB_OVF_MAC(J, 2)
#define ACB_OVF_C3(J) c3_##J: ACB_OVF_MAC(J, 3)
#define ACB_OVF_COL(C) C(0) C(1) C(2) C(3) C(4) C(5) C(6) C(7)
			ACB_OVF_COL(ACB_OVF_C0) goto macs_done;
			ACB_OVF_COL(ACB_OVF_C1) goto macs_done;
			ACB_OVF_COL(ACB_OVF_C2) goto macs_done;
			ACB_OVF_COL(ACB_OVF_C3)
			macs_done:;
#undef ACB_OVF_COL
#undef ACB_OVF_C3
#undef ACB_OVF_C2
#undef ACB_OVF_C1
#undef ACB_OVF_C0
#undef ACB_OVF_MAC
		}
		/* every lane is done with the staged window: the buffer can take the warp's next tile */
		__syncwarp();
		if (n + 1 < ntile) issue(n + 1);
		float e[CH_GROUP];
#pragma unroll
		for (int c = 0; c < CH_GROUP; c++) {
			const float re = __fadd_rn(A[c].x, -B[c].y), im = __fadd_rn(A[c].y, B[c].x);
			/* |D| in float, as k_channelize_dft1: integer input and a prototype of sum 1 bound it (u8: |D| <= ~1.5, CS16:
			 * <= ~1.2e4 times the filter's peak gain, no overflow); the < 3e-23 absolute error of a denormal re*re is far
			 * below 1e-6 of the row total sum |x| |w| of any row that is not all zeros */
			e[c] = __fsqrt_rn(__fmaf_rn(re, re, __fmul_rn(im, im)));
		}
		float *o = dm + ((size_t)s * nsamp + mrow) * nch + g * CH_GROUP;
#pragma unroll
		for (int j = 0; j < CH_GROUP; j++) {
			const int c = (int)((pperm >> (3 * j)) & 7u);
			if (c < nc && mrow < nsamp) o[c] = e[j];
		}
	}
}

template <int KIND, int UNITS, int WARPS>
static int launch_ovl_fast_t(const uint8_t *in, size_t stream_stride, const Hist &h, const float *p, const float2 *tw,
                             const unsigned *meta, float *dm, int nch, int nstreams, int nblk, size_t nsamp, cudaStream_t stream)
{
	using P = Dft1Plan<KIND, UNITS, WARPS>;
	const int ngrp = (nch + CH_GROUP - 1) / CH_GROUP;
	const int HR = (h.hpad + UNITS * 8 - 1) / (UNITS * 8);
	/* shared memory grows with the halo only: (32 + HR) rows per warp */
	const int smem = WARPS * (DFT1_ROWS + HR) * (P::ROWBYTES + 16) + P::TW_BYTES + WARPS * 8;
	auto kern = k_channelize_ovl_fast<KIND, UNITS, WARPS>;
	if (cudaError_t e = smem_max_carveout(kern, smem)) return (int)e;
	dim3 grid(nblk, nstreams, ngrp);
	kern<<<grid, 32 * WARPS, smem, stream>>>(in, stream_stride, reinterpret_cast<const uint8_t *>(h.base), h.stride, h.hpad, h.pos0,
	                                         p, tw, meta, dm, nch, ngrp, nsamp);
	return (int)cudaGetLastError();
}

/* u8 IQ or CS16 IQ, taps > K, K in {160, 192}, every channel on the 12.5 kHz raster; `nsamp` output rows per stream, any
 * count (CS16: the input buffer carries 32 rows of slack); `p` = taps_pad floats, fl(K*h) behind hpad - H zeros */
static int launch_channelize_ovl_fast(int mode, const void *in, size_t stream_stride, const Hist &h, const float *p, const float *tw,
                                      const unsigned *meta, float *dm, int K, int nch, int nstreams, size_t nsamp, cudaStream_t stream)
{
	if (nsamp == 0) return 0;
	const uint8_t *i8 = reinterpret_cast<const uint8_t *>(in);
	const float2 *t4 = reinterpret_cast<const float2 *>(tw);
	const int nblk = (int)((nsamp + OUTBLK - 1) / OUTBLK);
#define ACB_OVF_GO(M, U) launch_ovl_fast_t<M, U, 2>(i8, stream_stride, h, p, t4, meta, dm, nch, nstreams, nblk, nsamp, stream)
	if (mode == IN_CS16IQ) {
		if (K == 160) return ACB_OVF_GO(IN_CS16IQ, 20);
		if (K == 192) return ACB_OVF_GO(IN_CS16IQ, 24);
	} else if (mode == IN_U8IQ) {
		if (K == 160) return ACB_OVF_GO(IN_U8IQ, 20);
		if (K == 192) return ACB_OVF_GO(IN_U8IQ, 24);
	}
#undef ACB_OVF_GO
	return (int)cudaErrorInvalidValue;
}

/* ------------------------------------------------------------------------------------------
 * K1, wideband fast form (ACB_FLAG_FAST_WIDEBAND; DESIGN.md §4): the boxcar fast form (taps = K, orc_channelize_dft8*) and
 * the polyphase form (taps > K, orc_channelize_ovl_fast*) for any K % 8 == 0 up to ACB_MAXK and any channel count.  The
 * narrow kernels above put one group of 8 channels in a CTA and redo the row's shared work for every group; here one CTA
 * takes rows_per_cta rows (tiles of T = 4*RB) of one stream and up to WB_CTILE channels:
 *
 *   front half (once per row for all channels): the integer fold and 4-point split of the row (boxcar), or the pre-sum
 *     z_m[n] = sum_r p[n + H + r*K] * x[m*K + n + r*K] in ascending tap order followed by the float fold and split
 *     (polyphase), into Y'[residue][row][n2] in shared memory.  Samples and weights are read through L1/L2 with the
 *     columns n2 owned by consecutive threads; every fetch lies in [-hpad, nsamp*K) samples of the stream, the samples
 *     before the submit coming from the history (u8: the context's buffer; CS16: in front of the rows), and terms
 *     whose row lies before the stream start are omitted (as k_channelize_ovl_fast; for u8 the zero bytes of a cleared
 *     history would convert to -127.37, not to 0).
 *   back half (one SIMT complex GEMM per residue class): a thread owns RB rows x WB_CB channel slots of one residue and
 *     walks n2 upwards with the restatements' four fmaf chains per output.  The twiddles come from ONE table E of
 *     2K - 1 entries in shared memory, E[r] = the planner's T for (k*n2) % K = r (hostmath.cpp: acb_wb_twiddles): a
 *     channel's index moves by k modulo K in C-remainder form, so T_c[n2] = E[(k_c*n2) % K] bit for bit.  The slots are
 *     sorted by residue and padded per residue to whole groups of WB_CB (context.cu: upload_wb_plan), so a thread's Y'
 *     loads are one address for the whole group and mostly for the whole warp.
 *
 * meta per (stream, channel tile): [0] groups of WB_CB slots, [1] which E table (CS16: the variant), then (k, channel)
 * per slot, channel -1 for padding.
 * ---------------------------------------------------------------------------------------- */
template <int KIND, bool OVL, int RB>
__global__ void __launch_bounds__(WB_THREADS, 2)
k_channelize_wb(const uint8_t *__restrict__ in, size_t stream_stride, const uint8_t *__restrict__ hist, size_t hist_stride,
                int hpad, unsigned long long pos0, const float *__restrict__ pw, const float2 *__restrict__ E,
                const int *__restrict__ meta, float *__restrict__ dm, int K, int nch, int nctile, size_t nsamp, int rows_per_cta)
{
	constexpr int T = 4 * RB, BPS = KIND == IN_CS16IQ ? 4 : 2;
	const int N8 = K >> 3;
	extern __shared__ __align__(16) unsigned char smem[];
	float2 *Ys = reinterpret_cast<float2 *>(smem);                 /* [residue][row][n2] */
	float2 *Es = Ys + (size_t)4 * T * N8;                           /* E[r], r in (-K, K), at Es[r + K - 1] */
	const int s = blockIdx.y;
	const int *ms = meta + ((size_t)s * nctile + blockIdx.z) * WB_META;
	const int ng = ms[0];
	const float2 *Eg = E + (size_t)ms[1] * (2 * K - 1);
	for (int i = threadIdx.x; i < 2 * K - 1; i += WB_THREADS) Es[i] = Eg[i];

	/* back-half work item: row group rg (rows rg*RB ..), channel group cg */
	const int rg = (int)threadIdx.x / ng, cg = (int)threadIdx.x - rg * ng;
	int kk[WB_CB];                                /* the slots' channels are read again at the store: fewer live registers */
#pragma unroll
	for (int c = 0; c < WB_CB; c++) kk[c] = rg < 4 ? ms[2 + 2 * (cg * WB_CB + c)] : 0;
	const int res = (((kk[0] / 2) % 4) + 4) % 4;                      /* slot 0 of a group is always a channel */

	/* the CTA's rows in tiles of T; the bounds and stream pointers are recomputed from the parameters where they are used
	 * rather than held across the back half, whose accumulators need the registers */
	for (int t0 = 0; t0 < rows_per_cta; t0 += T) {
		const size_t r0 = (size_t)blockIdx.x * rows_per_cta + t0;
		if (r0 >= nsamp) break;
		__syncthreads();                          /* E staged / the previous tile's Y' consumed */
		const uint8_t *src_s = in + (size_t)s * stream_stride;
		const uint8_t *hist_s = OVL ? hist + (size_t)s * hist_stride + (size_t)hpad * BPS : nullptr;   /* where sample 0 of the submit would sit */
		for (int it = threadIdx.x; it < T * N8; it += WB_THREADS) {
			const int j = it / N8, n2 = it - j * N8;
			const size_t row = r0 + j;
			float2 y[4] = { make_float2(0.f, 0.f), make_float2(0.f, 0.f), make_float2(0.f, 0.f), make_float2(0.f, 0.f) };
			if (row < nsamp) {
				if (!OVL) {
					/* boxcar: the fold and split in integers, exact (orc_channelize_dft8*) */
					const uint8_t *rp = src_s + row * (size_t)K * BPS;
					int zi[4], zq[4];
#pragma unroll
					for (int n1 = 0; n1 < 4; n1++) {
						const int ia = N8 * n1 + n2, ib = N8 * (n1 + 4) + n2;
						if (KIND == IN_CS16IQ) {
							const unsigned a = __ldg(reinterpret_cast<const unsigned *>(rp) + ia);
							const unsigned b = __ldg(reinterpret_cast<const unsigned *>(rp) + ib);
							zi[n1] = (int)(short)(a & 0xffffu) + (int)(short)(b & 0xffffu);
							zq[n1] = (int)(short)(a >> 16) + (int)(short)(b >> 16);
						} else {
							const unsigned a = __ldg(reinterpret_cast<const unsigned short *>(rp) + ia);
							const unsigned b = __ldg(reinterpret_cast<const unsigned short *>(rp) + ib);
							zi[n1] = (int)(a & 0xffu) + (int)(b & 0xffu);
							zq[n1] = (int)(a >> 8) + (int)(b >> 8);
						}
					}
					const int bias = KIND == IN_CS16IQ ? 0 : 1020;
					y[0] = make_float2((float)(zi[0] + zi[1] + zi[2] + zi[3] - bias), (float)(zq[0] + zq[1] + zq[2] + zq[3] - bias));
					y[2] = make_float2((float)(zi[0] - zi[1] + zi[2] - zi[3]), (float)(zq[0] - zq[1] + zq[2] - zq[3]));
					y[1] = make_float2((float)((zi[0] - zi[2]) + (zq[1] - zq[3])), (float)((zq[0] - zq[2]) - (zi[1] - zi[3])));
					y[3] = make_float2((float)((zi[0] - zi[2]) - (zq[1] - zq[3])), (float)((zq[0] - zq[2]) + (zi[1] - zi[3])));
				} else {
					/* polyphase: the pre-sum of the eight samples n2 + e*K/8, then fold and split (orc_channelize_ovl_fast*) */
					const unsigned long long mabs = pos0 + row;          /* row counted from the stream start */
					float2 zz[8];
#pragma unroll
					for (int e = 0; e < 8; e++) {
						const int nn = e * N8 + n2;
						int rlo = -((nn + hpad) / K);
						if ((unsigned long long)(-rlo) > mabs) rlo = -(int)mabs;   /* rows before the stream start: omitted */
						const float *pr = pw + nn + hpad;
						const long long smp0 = (long long)row * K + nn;
						float a = 0.f, b = 0.f;
						for (int r = rlo; r <= 0; r++) {
							const long long smp = smp0 + (long long)r * K;   /* >= -hpad */
							const uint8_t *q = smp < 0 ? hist_s + smp * BPS : src_s + smp * BPS;
							float xr, xi;
							if (KIND == IN_CS16IQ) {
								const unsigned u = __ldg(reinterpret_cast<const unsigned *>(q));
								xr = (float)(short)(u & 0xffffu);
								xi = (float)(short)(u >> 16);
							} else {
								const unsigned u = __ldg(reinterpret_cast<const unsigned short *>(q));
								xr = __fadd_rn((float)(u & 0xffu), -127.37f);
								xi = __fadd_rn((float)(u >> 8), -127.37f);
							}
							const float pk = __ldg(pr + r * K);
							a = __fmaf_rn(pk, xr, a);
							b = __fmaf_rn(pk, xi, b);
						}
						zz[e] = make_float2(a, b);
					}
					float2 z[4];
#pragma unroll
					for (int n1 = 0; n1 < 4; n1++) z[n1] = fadd2_rn(zz[n1], zz[n1 + 4]);
					const float2 s02 = fadd2_rn(z[0], z[2]), s13 = fadd2_rn(z[1], z[3]);
					const float2 d02 = fsub2(z[0], z[2]);
					const float2 wj = make_float2(__fadd_rn(z[1].y, -z[3].y), __fadd_rn(z[3].x, -z[1].x));   /* -j (z1 - z3) */
					y[0] = fadd2_rn(s02, s13);
					y[2] = fsub2(s02, s13);
					y[1] = fadd2_rn(d02, wj);
					y[3] = fsub2(d02, wj);
				}
			}
#pragma unroll
			for (int q = 0; q < 4; q++) Ys[((size_t)q * T + j) * N8 + n2] = y[q];
		}
		__syncthreads();
		if (rg >= 4) continue;

		float acc[RB][WB_CB][4];                  /* ax, ay, bx, by: re = ax - by, im = ay + bx */
#pragma unroll
		for (int j = 0; j < RB; j++)
#pragma unroll
			for (int c = 0; c < WB_CB; c++) acc[j][c][0] = acc[j][c][1] = acc[j][c][2] = acc[j][c][3] = 0.f;
		int idx[WB_CB];
#pragma unroll
		for (int c = 0; c < WB_CB; c++) idx[c] = 0;
		const float2 *Yr = Ys + ((size_t)res * T + rg * RB) * N8;
		const float2 *Ec = Es + (K - 1);
#pragma unroll 1
		for (int n2 = 0; n2 < N8; n2++) {
			float2 t[WB_CB];
#pragma unroll
			for (int c = 0; c < WB_CB; c++) {
				t[c] = Ec[idx[c]];
				int v = idx[c] + kk[c];           /* (k*(n2+1)) % K from (k*n2) % K, |k| < K/2 */
				v = v >= K ? v - K : v;
				idx[c] = v <= -K ? v + K : v;
			}
#pragma unroll
			for (int j = 0; j < RB; j++) {
				const float2 yv = Yr[j * N8 + n2];
#pragma unroll
				for (int c = 0; c < WB_CB; c++) {
					acc[j][c][0] = __fmaf_rn(yv.x, t[c].x, acc[j][c][0]);
					acc[j][c][1] = __fmaf_rn(yv.x, t[c].y, acc[j][c][1]);
					acc[j][c][2] = __fmaf_rn(yv.y, t[c].x, acc[j][c][2]);
					acc[j][c][3] = __fmaf_rn(yv.y, t[c].y, acc[j][c][3]);
				}
			}
		}
#pragma unroll
		for (int j = 0; j < RB; j++) {
			const size_t row = r0 + rg * RB + j;
			if (row >= nsamp) continue;
			float *o = dm + ((size_t)s * nsamp + row) * nch;
#pragma unroll
			for (int c = 0; c < WB_CB; c++) {
				const int chc = __ldg(meta + ((size_t)s * nctile + blockIdx.z) * WB_META + 3 + 2 * (cg * WB_CB + c));
				if (chc < 0) continue;
				const float re = __fadd_rn(acc[j][c][0], -acc[j][c][3]), im = __fadd_rn(acc[j][c][1], acc[j][c][2]);
				/* |D| in float, bounded as in k_channelize_dft1 / k_channelize_ovl_fast */
				o[chc] = __fsqrt_rn(__fmaf_rn(re, re, __fmul_rn(im, im)));
			}
		}
	}
}

/* rows per tile: 12 where two CTAs per SM still fit, Y' (4*K bytes per row) + E ((2K - 1) * 8 bytes) <= 113 KB (K <= 1808),
 * else 8.  16-row tiles (RB = 4) would not fit their 64 accumulators in the 96 registers two 288-thread CTAs leave. */
static int wb_rb(int K)
{
	return 16 * 3 * K + (2 * K - 1) * 8 <= 113 * 1024 ? 3 : 2;
}

/* tiles per CTA of the wideband kernels (k_channelize_wb, k_channelize_wb_real): up to 8 (E is staged once per CTA), fewer
 * where that would leave less than four waves of two CTAs per SM — a CTA runs its tiles in series, so a grid short of
 * the SMs leaves them idle */
static int wb_tiles_per_cta(size_t nsamp, int T, int nstreams, int nctile)
{
	int dev = 0, nsm = 132;
	if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, dev);
	const size_t tiles = (nsamp + T - 1) / T * (size_t)nstreams * nctile;
	return (int)std::max<size_t>(1, std::min<size_t>(8, tiles / ((size_t)8 * nsm)));
}

template <int KIND, bool OVL, int RB>
static int launch_wb_t(const uint8_t *in, size_t stream_stride, const Hist &h, const float *p, const float2 *E, const int *meta,
                       float *dm, int K, int nch, int nstreams, size_t nsamp, cudaStream_t stream)
{
	constexpr int T = 4 * RB;
	const int smem = 4 * T * (K / 8) * 8 + (2 * K - 1) * 8;
	const int nctile = (nch + WB_CTILE - 1) / WB_CTILE;
	auto kern = k_channelize_wb<KIND, OVL, RB>;
	if (cudaError_t e = smem_max_carveout(kern, smem)) return (int)e;
	const int rows_per_cta = wb_tiles_per_cta(nsamp, T, nstreams, nctile) * T;
	dim3 grid((unsigned)((nsamp + rows_per_cta - 1) / rows_per_cta), nstreams, nctile);
	kern<<<grid, WB_THREADS, smem, stream>>>(in, stream_stride, reinterpret_cast<const uint8_t *>(h.base), h.stride, h.hpad, h.pos0,
	                                         p, E, meta, dm, K, nch, nctile, nsamp, rows_per_cta);
	return (int)cudaGetLastError();
}

/* u8 IQ or CS16 IQ, K % 8 == 0, K <= ACB_MAXK, any nch, every channel on the 12.5 kHz raster; taps = K (h.hpad = 0) or
 * taps > K (`p` = taps_pad floats, fl(K*h) behind hpad - H zeros); `nsamp` output rows per stream, any count */
static int launch_channelize_wb(int mode, const void *in, size_t stream_stride, const Hist &h, const float *p, const float *E,
                                const int *meta, float *dm, int K, int nch, int nstreams, size_t nsamp, cudaStream_t stream)
{
	if (nsamp == 0) return 0;
	if ((K & 7) || K > 2048 || (mode != IN_U8IQ && mode != IN_CS16IQ)) return (int)cudaErrorInvalidValue;
	const uint8_t *i8 = reinterpret_cast<const uint8_t *>(in);
	const float2 *E2 = reinterpret_cast<const float2 *>(E);
	const int rb = wb_rb(K);
#define ACB_WB_GO(M, O, R) launch_wb_t<M, O, R>(i8, stream_stride, h, p, E2, meta, dm, K, nch, nstreams, nsamp, stream)
#define ACB_WB_RB(M, O) return rb == 3 ? ACB_WB_GO(M, O, 3) : ACB_WB_GO(M, O, 2)
	if (mode == IN_CS16IQ) {
		if (h.hpad) ACB_WB_RB(IN_CS16IQ, true);
		ACB_WB_RB(IN_CS16IQ, false);
	}
	if (h.hpad) ACB_WB_RB(IN_U8IQ, true);
	ACB_WB_RB(IN_U8IQ, false);
#undef ACB_WB_RB
#undef ACB_WB_GO
}

/* ------------------------------------------------------------------------------------------
 * Fast form of the REAL-input channelizer (air.c:291-341 with the table of air.c:278-285): wf[i] = exp(-j*2*pi*k*i/K)/K is
 * a sampled exponential with k = (Fc - Fr + rate/4) / 12.5 kHz a whole number whenever the channels and the tuner
 * centre sit on the 12.5 kHz raster (air.c:66 puts Fc there), so D is bin k of the K-point DFT of a REAL row:
 *   D = sum_{n2 < K/4} T[n2] * Y_r[n2],  r = k mod 4,  T[n2] = exp(-j*2*pi*k*n2/K)/K,
 *   Y_0 = (x0 + x2) + (x1 + x3)   Y_2 = (x0 + x2) - (x1 + x3)          real
 *   Y_1 = (x0 - x2) - j (x1 - x3) Y_3 = (x0 - x2) + j (x1 - x3)        x_q = x[(K/4) q + n2]
 * 6 additions per n2 shared by all channels, then K/4 real x complex (r even: one float2 FMA per n2) or complex x complex
 * (r odd: two) MACs per channel instead of K: 8 channels cost ~10 FP32 lane-ops per input sample where the reference's
 * order costs 32 — the kernel becomes a memory streamer.  Same shape as k_channelize_dft1: one row per lane, whole rows
 * by cp.async.bulk into a private 32-row tile per warp, channel slots sorted so that the MAC section is straight-line
 * columns (r = 0 | r = 2 | r odd; residues 1 and 3 accumulate the same two sums and differ in one sign at the end).
 * NOT the reference's operation order (tolerance: include/acars_b200.h); bit-identical to oracle's orc_channelize_rdft.
 * ---------------------------------------------------------------------------------------- */
/* LPR lanes share a row: lane l works on row l % ROWS of the warp's tile and takes the h-th contiguous range of n2 pairs,
 * h = l / ROWS; the LPR partial sums are added pairwise (h ^ 1, then h ^ 2, ...) at the end.  A row of K floats is 800 bytes
 * and more: with one lane per row a warp's tile is 26-103 KB, 8 warps or fewer fit an SM and the kernel sits at 29 % issue
 * utilisation waiting for its own dependent FMA chains; LPR = K/100 keeps the tile at 13 KB. */
template <int K8, int LPR, int WARPS> struct RdftPlan {
	static constexpr int K = K8 * 8;
	static constexpr int ROWS = 32 / LPR;                             /* rows per warp tile */
	static constexpr int ROWBYTES = K * 4;
	static constexpr int GROUP = ROWBYTES + 16;                       /* every row shifted by one more 16-byte unit */
	static constexpr int TILE_BYTES = ROWS * GROUP;
	static constexpr int N2 = K / 4;
	static constexpr int TW_BYTES = N2 * CH_GROUP * 8;
	static constexpr int BAR_OFF = WARPS * TILE_BYTES + TW_BYTES;
	static constexpr int SMEM = BAR_OFF + WARPS * 8;
	static constexpr int PER = (K8 + LPR - 1) / LPR;                  /* n2 pairs per lane */
};

template <int K8, int LPR, int WARPS, int MINB>
__global__ void __launch_bounds__(32 * WARPS, MINB)
k_channelize_rdft(const uint8_t *__restrict__ in, size_t stream_stride, const float2 *__restrict__ tw,
                  const unsigned *__restrict__ meta, float *__restrict__ dm, int nch, int ngrp, size_t nsamp)
{
	using P = RdftPlan<K8, LPR, WARPS>;
	constexpr int N2 = P::N2, ROWS = P::ROWS;
	constexpr int NTILE = OUTBLK / ROWS;
	extern __shared__ __align__(16) unsigned char smem[];
	const int l = threadIdx.x & 31;
	const int w = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0);
	const int blk = blockIdx.x, s = blockIdx.y, g = blockIdx.z;
	unsigned char *mytile = smem + (size_t)w * P::TILE_BYTES;
	const float4 *stw = reinterpret_cast<const float4 *>(smem + (size_t)WARPS * P::TILE_BYTES);   /* [slot][n2] (Tr, Ti) */
	unsigned long long *bar = reinterpret_cast<unsigned long long *>(smem + P::BAR_OFF) + w;
	const uint8_t *src_blk = in + (size_t)s * stream_stride + (size_t)blk * OUTBLK * P::ROWBYTES;
	const unsigned m = __shfl_sync(0xffffffffu, meta[(size_t)s * ngrp + g], 0);    /* k_c mod 4 of channel c in bits 2c, 2c + 1 */

	if (l == 0) mbar_init(bar, 1);
	asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
	/* slots sorted by column: residue 0, residue 2, odd residues (stable); perm[j] in bits 3j.., sign of slot j in bit j */
	unsigned pw = 0, neg = 0;
	int bnd0, bnd1;
	{
		int cnt[3] = { 0, 0, 0 };
#pragma unroll
		for (int c = 0; c < CH_GROUP; c++) {
			const unsigned r = (m >> (2 * c)) & 3u;
			const int cls = r == 0 ? 0 : r == 2 ? 1 : 2;
#pragma unroll
			for (int q = 0; q < 3; q++) cnt[q] += (cls == q);
		}
		bnd0 = cnt[0]; bnd1 = bnd0 + cnt[1];
		int pos[3] = { 0, bnd0, bnd1 };
#pragma unroll
		for (int c = 0; c < CH_GROUP; c++) {
			const unsigned r = (m >> (2 * c)) & 3u;
			const int cls = r == 0 ? 0 : r == 2 ? 1 : 2;
			int at = 0;
#pragma unroll
			for (int q = 0; q < 3; q++) { at = (cls == q) ? pos[q] : at; pos[q] += (cls == q); }
			pw |= (unsigned)c << (3 * at);
			neg |= (unsigned)(r == 3) << at;
		}
	}
	{
		const uint4 *tsrc = reinterpret_cast<const uint4 *>(tw + ((size_t)s * ngrp + g) * N2 * CH_GROUP);
		uint4 *tdst = reinterpret_cast<uint4 *>(smem + (size_t)WARPS * P::TILE_BYTES);
		constexpr int PER16 = N2 * 8 / 16;
		for (int q = threadIdx.x; q < P::TW_BYTES / 16; q += 32 * WARPS) {
			const int j = q / PER16, off = q - j * PER16;
			cp_async16(tdst + q, tsrc + ((pw >> (3 * j)) & 7u) * PER16 + off);
		}
		cp_async_commit();
		cp_async_wait_all();
	}
	__syncthreads();

	const size_t rows_left = nsamp - (size_t)blk * OUTBLK;
	const int tiles_here = rows_left >= (size_t)OUTBLK ? NTILE : (int)((rows_left + ROWS - 1) / ROWS);
	const int ntile = (tiles_here - w + WARPS - 1) / WARPS;
	auto issue = [&](int n) {
		if (elect_one()) {
			mbar_expect_tx(bar, ROWS * P::ROWBYTES);
			const uint8_t *src = src_blk + (size_t)(w + n * WARPS) * ROWS * P::ROWBYTES;
#pragma unroll
			for (int i = 0; i < ROWS; i++)
				bulk_g2s(mytile + (size_t)i * P::GROUP, src + (size_t)i * P::ROWBYTES, P::ROWBYTES, bar);
		}
	};
	if (ntile > 0) issue(0);
	const int nc = min(CH_GROUP, nch - g * CH_GROUP);
	const int row = l % ROWS, h = l / ROWS;
	const int gp0 = h * P::PER, gp1 = min(K8, gp0 + P::PER);

	for (int n = 0; n < ntile; n++) {
		const int tile = w + n * WARPS;
		mbar_wait(bar, (unsigned)(n & 1));
		const unsigned char *ra = mytile + (size_t)row * P::GROUP;
		float2 A[CH_GROUP], B[CH_GROUP];
#pragma unroll
		for (int c = 0; c < CH_GROUP; c++) A[c] = B[c] = make_float2(0.f, 0.f);

#pragma unroll 1
		for (int gp = gp0; gp < gp1; gp++) {              /* n2 = 2 gp, 2 gp + 1 */
			const float2 x0 = *reinterpret_cast<const float2 *>(ra + 0 * P::K + gp * 8);
			const float2 x1 = *reinterpret_cast<const float2 *>(ra + 1 * P::K + gp * 8);
			const float2 x2 = *reinterpret_cast<const float2 *>(ra + 2 * P::K + gp * 8);
			const float2 x3 = *reinterpret_cast<const float2 *>(ra + 3 * P::K + gp * 8);
			const float2 s02 = fadd2_rn(x0, x2), s13 = fadd2_rn(x1, x3);
			const float2 y0 = fadd2_rn(s02, s13), y2 = fsub2(s02, s13);
			const float2 d02 = fsub2(x0, x2), d13 = fsub2(x1, x3);
			const float4 *tj = stw + gp;
#define ACB_RDFT_E(J, Y)                                                                   \
			{                                                                                      \
				const float4 u = tj[(J) * (N2 / 2)];                                                   \
				A[J] = ffma2(make_float2(Y.x, Y.x), make_float2(u.x, u.y), A[J]);                      \
				A[J] = ffma2(make_float2(Y.y, Y.y), make_float2(u.z, u.w), A[J]);                      \
			}
#define ACB_RDFT_O(J)                                                                      \
			{                                                                                      \
				const float4 u = tj[(J) * (N2 / 2)];                                                   \
				A[J] = ffma2(make_float2(d02.x, d02.x), make_float2(u.x, u.y), A[J]);                  \
				B[J] = ffma2(make_float2(d13.x, d13.x), make_float2(u.x, u.y), B[J]);                  \
				A[J] = ffma2(make_float2(d02.y, d02.y), make_float2(u.z, u.w), A[J]);                  \
				B[J] = ffma2(make_float2(d13.y, d13.y), make_float2(u.z, u.w), B[J]);                  \
			}
#define ACB_RDFT_C0(J) if ((J) >= bnd0) goto r1_##J; ACB_RDFT_E(J, y0)
#define ACB_RDFT_C1(J) r1_##J: if ((J) >= bnd1) goto r2_##J; ACB_RDFT_E(J, y2)
#define ACB_RDFT_C2(J) r2_##J: ACB_RDFT_O(J)
#define ACB_RDFT_COL(C) C(0) C(1) C(2) C(3) C(4) C(5) C(6) C(7)
			ACB_RDFT_COL(ACB_RDFT_C0) goto rmacs_done;
			ACB_RDFT_COL(ACB_RDFT_C1) goto rmacs_done;
			ACB_RDFT_COL(ACB_RDFT_C2)
			rmacs_done:;
#undef ACB_RDFT_COL
#undef ACB_RDFT_C2
#undef ACB_RDFT_C1
#undef ACB_RDFT_C0
#undef ACB_RDFT_O
#undef ACB_RDFT_E
		}
		__syncwarp();
		if (n + 1 < ntile) issue(n + 1);
		/* the row's LPR partial sums, pairwise: (p0 + p1) + (p2 + p3) ... — both partners compute the same sum */
#pragma unroll
		for (int step = ROWS; step < 32; step *= 2) {
#pragma unroll
			for (int j = 0; j < CH_GROUP; j++) {
				A[j].x = __fadd_rn(A[j].x, __shfl_xor_sync(0xffffffffu, A[j].x, step));
				A[j].y = __fadd_rn(A[j].y, __shfl_xor_sync(0xffffffffu, A[j].y, step));
				B[j].x = __fadd_rn(B[j].x, __shfl_xor_sync(0xffffffffu, B[j].x, step));
				B[j].y = __fadd_rn(B[j].y, __shfl_xor_sync(0xffffffffu, B[j].y, step));
			}
		}
		const size_t mrow = (size_t)blk * OUTBLK + (size_t)tile * ROWS + row;
		if (h == 0 && mrow < nsamp) {
			float *o = dm + ((size_t)s * nsamp + mrow) * nch + g * CH_GROUP;
#pragma unroll
			for (int j = 0; j < CH_GROUP; j++) {
				/* r = 1: D = (A.x + B.y) + j (A.y - B.x); r = 3: the other signs; r even: B is zero */
				const float sg = ((neg >> j) & 1u) ? -1.0f : 1.0f;
				const float re = __fadd_rn(A[j].x, __fmul_rn(sg, B[j].y)), im = __fadd_rn(A[j].y, -__fmul_rn(sg, B[j].x));
				/* |D| in double, as envelope() does: float input has no bound, and in float re*re overflows for
				 * |D| > ~1.8e19 and goes denormal below ~1e-19 (tests/test_gpu_air.py runs 2^-70 .. 2^70) */
				const float e = envelope(make_float2(re, im));
				const int c = (int)((pw >> (3 * j)) & 7u);
				if (c < nc) o[c] = e;
			}
		}
	}
}

template <int K8, int LPR, int WARPS, int MINB>
static int launch_rdft_t(const uint8_t *in, size_t stream_stride, const float2 *tw, const unsigned *meta, float *dm,
                         int nch, int nstreams, int nblk, size_t nsamp, cudaStream_t stream)
{
	const int ngrp = (nch + CH_GROUP - 1) / CH_GROUP;
	constexpr int smem = RdftPlan<K8, LPR, WARPS>::SMEM;
	auto kern = k_channelize_rdft<K8, LPR, WARPS, MINB>;
	if (cudaError_t e = smem_max_carveout(kern, smem)) return (int)e;
	dim3 grid(nblk, nstreams, ngrp);
	kern<<<grid, 32 * WARPS, smem, stream>>>(in, stream_stride, tw, meta, dm, nch, ngrp, nsamp);
	return (int)cudaGetLastError();
}

/* the Airspy rates: 2.5 MS/s (K = 200), 3 (240), 5 (400), 6 (480), 10 (800) */
static bool channelize_rdft_supports(int K) { return K == 200 || K == 240 || K == 400 || K == 480 || K == 800; }
/* lanes per row of k_channelize_rdft (the CPU restatement needs it: it fixes the order of the partial sums) */
int channelize_rdft_lanes_per_row(int K) { return K >= 800 ? 8 : K >= 400 ? 4 : 2; }

/* float32 real input (air.c), taps == K, every channel on the 12.5 kHz raster around Fc; `nsamp` output rows per stream,
 * any count (the input buffer carries 32 rows of slack).  stream_stride in bytes. */
static int launch_channelize_rdft(const void *in, size_t stream_stride, const float *tw, const unsigned *meta, float *dm,
                                  int K, int nch, int nstreams, size_t nsamp, cudaStream_t stream)
{
	if (nsamp == 0) return 0;
	const uint8_t *i8 = reinterpret_cast<const uint8_t *>(in);
	const float2 *t4 = reinterpret_cast<const float2 *>(tw);
	const int nblk = (int)((nsamp + OUTBLK - 1) / OUTBLK);
	const int w2 = getenv("ACB_FAST_WARPS") ? atoi(getenv("ACB_FAST_WARPS")) : 4;
#define ACB_RDFT_GO(K8, LPR, W, M) launch_rdft_t<K8, LPR, W, M>(i8, stream_stride, t4, meta, dm, nch, nstreams, nblk, nsamp, stream)
	/* 13-16 KB of tile per warp everywhere; 4 warps per CTA: 16 warps per SM at K = 200, 12 at the other rates */
	if (K == 200) return w2 == 2 ? ACB_RDFT_GO(25, 2, 2, 7) : ACB_RDFT_GO(25, 2, 4, 4);
	if (K == 240) return ACB_RDFT_GO(30, 2, 4, 3);
	if (K == 400) return ACB_RDFT_GO(50, 4, 4, 3);
	if (K == 480) return ACB_RDFT_GO(60, 4, 4, 3);
	if (K == 800) return ACB_RDFT_GO(100, 8, 4, 3);
#undef ACB_RDFT_GO
	return (int)cudaErrorInvalidValue;
}

/* ------------------------------------------------------------------------------------------
 * Polyphase fast form of the overlapping window for REAL input (ACB_FLAG_FAST_FILTER_REAL, taps > K): with every channel on
 * the raster, w[i] = h[i] * exp(-j*2*pi*k*(i - H)/K), so D is bin k of the K-sample real row
 *   z_m[n] = sum_r p[n + H + r*K] * x[m*K + n + r*K],   p = fl(K*h), r <= 0 ascending (ascending tap order), one FMA per term
 * and that bin is taken exactly as k_channelize_rdft takes it from a row of input (the same lanes per row, n2-pair ranges,
 * MAC columns and pairwise tree; twiddles from acb_fast_plan_air, which carry the 1/K).
 *
 * Shape: one CTA per (1024-row block, stream, channel group), as k_channelize_rdft.  The CTA walks its block in steps of
 * T = WARPS * ROWS rows through a ring of HR + T staged rows (HR = ceil(hpad/K)): each input row is staged once per CTA
 * and the halo once per block, so shared memory is (HR + T) rows, not a private (ROWS + HR)-row window per warp.  A step:
 *  1. the next T rows arrive by bulk copies (the first step also brings the HR rows in front of the block, the first one
 *     from sample n0 on: rows before the submit are the history right in front of the input in d_real);
 *  2. the pre-sum: thread u owns the CW columns u*CW .. of every row, walks the step's rows four at a time (each staged
 *     sample is read once for four rows; p is read through L1 once per term) and writes z_m over the slot of input row
 *     m - HR, which no later row of this step reads: a thread only overwrites its own columns, and rows <= m are done;
 *  3. the rdft's DFT half on the z rows, then the envelope in double;
 *  4. the z slots are where the next step's rows land.
 * Terms before the stream start READ the history, which acb_create / acb_reset zero: z starts at +0 and is never -0 (an
 * exact zero sum rounds to +0), so fma(p, +0, z) = z, and the table's zero front padding gives fma(+0, x, +0) = +0 for
 * the finite samples there.  The result is the sum over the valid terms only (tests/host/ovl_fast_real_oracle.c:
 * orc_ovl_presum_real, then orc_channelize_rdft), bit for bit.  Every fetch lies in [-hpad, nsamp*K) samples of its
 * stream: no slack rows are read.
 * ---------------------------------------------------------------------------------------- */
template <int CW> struct ColsF;
template <> struct ColsF<2> {
	static __device__ __forceinline__ void ld(const float *a, float (&v)[2]) { const float2 u = *reinterpret_cast<const float2 *>(a); v[0] = u.x; v[1] = u.y; }
	static __device__ __forceinline__ void ldg(const float *a, float (&v)[2]) { const float2 u = __ldg(reinterpret_cast<const float2 *>(a)); v[0] = u.x; v[1] = u.y; }
	static __device__ __forceinline__ void st(float *a, const float (&v)[2]) { *reinterpret_cast<float2 *>(a) = make_float2(v[0], v[1]); }
};
template <> struct ColsF<4> {
	static __device__ __forceinline__ void ld(const float *a, float (&v)[4]) { const float4 u = *reinterpret_cast<const float4 *>(a); v[0] = u.x; v[1] = u.y; v[2] = u.z; v[3] = u.w; }
	static __device__ __forceinline__ void ldg(const float *a, float (&v)[4]) { const float4 u = __ldg(reinterpret_cast<const float4 *>(a)); v[0] = u.x; v[1] = u.y; v[2] = u.z; v[3] = u.w; }
	static __device__ __forceinline__ void st(float *a, const float (&v)[4]) { *reinterpret_cast<float4 *>(a) = make_float4(v[0], v[1], v[2], v[3]); }
};

template <int K8, int LPR, int WARPS, int CW>
__global__ void __launch_bounds__(32 * WARPS)
k_channelize_ovl_rdft(const uint8_t *__restrict__ in, size_t stream_stride, int hpad, const float *__restrict__ ptab,
                      const float2 *__restrict__ tw, const unsigned *__restrict__ meta, float *__restrict__ dm, int nch, int ngrp,
                      size_t nsamp)
{
	using P = RdftPlan<K8, LPR, WARPS>;
	constexpr int K = P::K, N2 = P::N2, ROWS = P::ROWS, T = ROWS * WARPS, NU = K / CW;
	constexpr int GF = P::GROUP / 4;                  /* ring row pitch in floats (a row plus 16 bytes, as the rdft tile) */
	static_assert(T % 4 == 0 && K % 4 == 0, "rows go four at a time; columns in 16-byte units");
	extern __shared__ __align__(16) unsigned char smem[];
	const int l = threadIdx.x & 31;
	const int w = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0);
	const int blk = blockIdx.x, s = blockIdx.y, g = blockIdx.z;
	const int HR = (hpad + K - 1) / K, NR = HR + T, n0 = HR * K - hpad;
	float *ring = reinterpret_cast<float *>(smem);
	const float4 *stw = reinterpret_cast<const float4 *>(smem + (size_t)NR * P::GROUP);             /* [slot][n2] (Tr, Ti) */
	unsigned long long *bar = reinterpret_cast<unsigned long long *>(smem + (size_t)NR * P::GROUP + P::TW_BYTES);
	const uint8_t *src_s = in + (size_t)s * stream_stride;          /* sample 0 of the submit; the history sits in front */
	const unsigned m = __shfl_sync(0xffffffffu, meta[(size_t)s * ngrp + g], 0);

	if (threadIdx.x == 0) mbar_init(bar, 1);
	asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
	/* slots sorted by column as in k_channelize_rdft */
	unsigned pw = 0, neg = 0;
	int bnd0, bnd1;
	{
		int cnt[3] = { 0, 0, 0 };
#pragma unroll
		for (int c = 0; c < CH_GROUP; c++) {
			const unsigned r = (m >> (2 * c)) & 3u;
			const int cls = r == 0 ? 0 : r == 2 ? 1 : 2;
#pragma unroll
			for (int q = 0; q < 3; q++) cnt[q] += (cls == q);
		}
		bnd0 = cnt[0]; bnd1 = bnd0 + cnt[1];
		int pos[3] = { 0, bnd0, bnd1 };
#pragma unroll
		for (int c = 0; c < CH_GROUP; c++) {
			const unsigned r = (m >> (2 * c)) & 3u;
			const int cls = r == 0 ? 0 : r == 2 ? 1 : 2;
			int at = 0;
#pragma unroll
			for (int q = 0; q < 3; q++) { at = (cls == q) ? pos[q] : at; pos[q] += (cls == q); }
			pw |= (unsigned)c << (3 * at);
			neg |= (unsigned)(r == 3) << at;
		}
	}
	{
		const uint4 *tsrc = reinterpret_cast<const uint4 *>(tw + ((size_t)s * ngrp + g) * N2 * CH_GROUP);
		uint4 *tdst = reinterpret_cast<uint4 *>(smem + (size_t)NR * P::GROUP);
		constexpr int PER16 = N2 * 8 / 16;
		for (int q = threadIdx.x; q < P::TW_BYTES / 16; q += 32 * WARPS) {
			const int j = q / PER16, off = q - j * PER16;
			cp_async16(tdst + q, tsrc + ((pw >> (3 * j)) & 7u) * PER16 + off);
		}
		cp_async_commit();
		cp_async_wait_all();
	}
	__syncthreads();

	const long long row_base = (long long)blk * OUTBLK;
	const int rows_here = (int)min((size_t)OUTBLK, nsamp - (size_t)row_base);
	const int nstep = (rows_here + T - 1) / T;
	/* rows q (relative to the block) live in slot (q + HR) mod NR */
	auto issue = [&](int i) {
		if (elect_one()) {
			const int q0 = i == 0 ? -HR : i * T, q1 = min((i + 1) * T, rows_here);
			mbar_expect_tx(bar, (unsigned)(((q1 - q0) * K - (i == 0 ? n0 : 0)) * 4));
			int sl = (q0 + HR) % NR;
			for (int q = q0; q < q1; q++) {
				const int s0 = q == -HR ? n0 : 0;
				const long long smp = (row_base + q) * K + s0;           /* >= -hpad: before the submit means in the history */
				bulk_g2s(ring + (size_t)sl * GF + s0, src_s + smp * 4, (unsigned)((K - s0) * 4), bar);
				sl = sl + 1 == NR ? 0 : sl + 1;
			}
		}
	};
	if (w == 0) issue(0);
	const int nc = min(CH_GROUP, nch - g * CH_GROUP);
	const int row = l % ROWS, h = l / ROWS;
	const int gp0 = h * P::PER, gp1 = min(K8, gp0 + P::PER);

	for (int i = 0; i < nstep; i++) {
		const int j0 = i * T, nrows = min(T, rows_here - j0);
		mbar_wait(bar, (unsigned)(i & 1));

		/* 2. the pre-sum of rows j0 .. j0 + nrows - 1 (a last partial group of four runs on stale slots and is not stored) */
		for (int u = threadIdx.x; u < NU; u += 32 * WARPS) {
			const int nn = u * CW;
			const int rlo = -((nn + hpad) / K);            /* terms r = rlo .. 0, the same for the CW columns */
			const float *pr = ptab + nn + hpad;             /* p of term r at pr + r*K */
#pragma unroll 1
			for (int jb = 0; jb < nrows; jb += 4) {
				float acc[4][CW], pp[4][CW];
#pragma unroll
				for (int b = 0; b < 4; b++)
#pragma unroll
					for (int c = 0; c < CW; c++) acc[b][c] = pp[b][c] = 0.0f;
				/* input row j0 + jb + t for t = rlo .. 3 feeds row j0 + jb + b as its term r = t - b; pp[(t - rlo) mod 4]
				 * holds p of term t, which rows b = 0 .. 3 use at t .. t + 3 */
				int sl = (j0 + jb + rlo + HR) % NR;
#pragma unroll 1
				for (int t0 = rlo; t0 <= 3; t0 += 4) {
#pragma unroll
					for (int k = 0; k < 4; k++) {
						const int t = t0 + k;
						if (t <= 3) {
							float x[CW];
							ColsF<CW>::ld(ring + (size_t)sl * GF + nn, x);
							sl = sl + 1 == NR ? 0 : sl + 1;
							if (t <= 0) ColsF<CW>::ldg(pr + t * K, pp[k]);
#pragma unroll
							for (int b = 0; b < 4; b++) {
								if (t - b >= rlo && t - b <= 0) {
#pragma unroll
									for (int c = 0; c < CW; c++) acc[b][c] = __fmaf_rn(pp[(k - b) & 3][c], x[c], acc[b][c]);
								}
							}
						}
					}
				}
#pragma unroll
				for (int b = 0; b < 4; b++) ColsF<CW>::st(ring + (size_t)((j0 + jb + b) % NR) * GF + nn, acc[b]);
			}
		}
		__syncthreads();

		/* 3. the DFT half, k_channelize_rdft's operations on the z row of step row w*ROWS + row */
		const int j = w * ROWS + row;
		const unsigned char *ra = reinterpret_cast<const unsigned char *>(ring + (size_t)((j0 + j) % NR) * GF);
		float2 A[CH_GROUP], B[CH_GROUP];
#pragma unroll
		for (int c = 0; c < CH_GROUP; c++) A[c] = B[c] = make_float2(0.f, 0.f);

#pragma unroll 1
		for (int gp = gp0; gp < gp1; gp++) {              /* n2 = 2 gp, 2 gp + 1 */
			const float2 x0 = *reinterpret_cast<const float2 *>(ra + 0 * P::K + gp * 8);
			const float2 x1 = *reinterpret_cast<const float2 *>(ra + 1 * P::K + gp * 8);
			const float2 x2 = *reinterpret_cast<const float2 *>(ra + 2 * P::K + gp * 8);
			const float2 x3 = *reinterpret_cast<const float2 *>(ra + 3 * P::K + gp * 8);
			const float2 s02 = fadd2_rn(x0, x2), s13 = fadd2_rn(x1, x3);
			const float2 y0 = fadd2_rn(s02, s13), y2 = fsub2(s02, s13);
			const float2 d02 = fsub2(x0, x2), d13 = fsub2(x1, x3);
			const float4 *tj = stw + gp;
#define ACB_ORD_E(J, Y)                                                                    \
			{                                                                                      \
				const float4 u = tj[(J) * (N2 / 2)];                                                   \
				A[J] = ffma2(make_float2(Y.x, Y.x), make_float2(u.x, u.y), A[J]);                      \
				A[J] = ffma2(make_float2(Y.y, Y.y), make_float2(u.z, u.w), A[J]);                      \
			}
#define ACB_ORD_O(J)                                                                       \
			{                                                                                      \
				const float4 u = tj[(J) * (N2 / 2)];                                                   \
				A[J] = ffma2(make_float2(d02.x, d02.x), make_float2(u.x, u.y), A[J]);                  \
				B[J] = ffma2(make_float2(d13.x, d13.x), make_float2(u.x, u.y), B[J]);                  \
				A[J] = ffma2(make_float2(d02.y, d02.y), make_float2(u.z, u.w), A[J]);                  \
				B[J] = ffma2(make_float2(d13.y, d13.y), make_float2(u.z, u.w), B[J]);                  \
			}
#define ACB_ORD_C0(J) if ((J) >= bnd0) goto o1_##J; ACB_ORD_E(J, y0)
#define ACB_ORD_C1(J) o1_##J: if ((J) >= bnd1) goto o2_##J; ACB_ORD_E(J, y2)
#define ACB_ORD_C2(J) o2_##J: ACB_ORD_O(J)
#define ACB_ORD_COL(C) C(0) C(1) C(2) C(3) C(4) C(5) C(6) C(7)
			ACB_ORD_COL(ACB_ORD_C0) goto omacs_done;
			ACB_ORD_COL(ACB_ORD_C1) goto omacs_done;
			ACB_ORD_COL(ACB_ORD_C2)
			omacs_done:;
#undef ACB_ORD_COL
#undef ACB_ORD_C2
#undef ACB_ORD_C1
#undef ACB_ORD_C0
#undef ACB_ORD_O
#undef ACB_ORD_E
		}
		/* 4. every thread is done with the z rows: their slots take the next step's input (the async proxy writes where the
		 * generic proxy wrote and read) */
		asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
		__syncthreads();
		if (w == 0 && i + 1 < nstep) issue(i + 1);
#pragma unroll
		for (int step = ROWS; step < 32; step *= 2) {
#pragma unroll
			for (int jj = 0; jj < CH_GROUP; jj++) {
				A[jj].x = __fadd_rn(A[jj].x, __shfl_xor_sync(0xffffffffu, A[jj].x, step));
				A[jj].y = __fadd_rn(A[jj].y, __shfl_xor_sync(0xffffffffu, A[jj].y, step));
				B[jj].x = __fadd_rn(B[jj].x, __shfl_xor_sync(0xffffffffu, B[jj].x, step));
				B[jj].y = __fadd_rn(B[jj].y, __shfl_xor_sync(0xffffffffu, B[jj].y, step));
			}
		}
		const size_t mrow = (size_t)row_base + j0 + j;
		if (h == 0 && j < nrows) {
			float *o = dm + ((size_t)s * nsamp + mrow) * nch + g * CH_GROUP;
#pragma unroll
			for (int jj = 0; jj < CH_GROUP; jj++) {
				const float sg = ((neg >> jj) & 1u) ? -1.0f : 1.0f;
				const float re = __fadd_rn(A[jj].x, __fmul_rn(sg, B[jj].y)), im = __fadd_rn(A[jj].y, -__fmul_rn(sg, B[jj].x));
				const float e = envelope(make_float2(re, im));           /* in double: float input has no bound */
				const int c = (int)((pw >> (3 * jj)) & 7u);
				if (c < nc) o[c] = e;
			}
		}
	}
}

/* shared memory of k_channelize_ovl_rdft: the (HR + T)-row ring, the twiddles and the barrier */
template <int K8, int LPR, int WARPS>
static int ovl_rdft_smem(int hpad)
{
	using P = RdftPlan<K8, LPR, WARPS>;
	const int HR = (hpad + P::K - 1) / P::K;
	return (HR + P::ROWS * WARPS) * P::GROUP + P::TW_BYTES + 8;
}

template <int K8, int LPR, int WARPS, int CW>
static int launch_ovl_rdft_t(const uint8_t *in, size_t stream_stride, int hpad, const float *p, const float2 *tw,
                             const unsigned *meta, float *dm, int nch, int nstreams, int nblk, size_t nsamp, cudaStream_t stream)
{
	const int ngrp = (nch + CH_GROUP - 1) / CH_GROUP;
	const int smem = ovl_rdft_smem<K8, LPR, WARPS>(hpad);
	auto kern = k_channelize_ovl_rdft<K8, LPR, WARPS, CW>;
	if (cudaError_t e = smem_max_carveout(kern, smem)) return (int)e;
	dim3 grid(nblk, nstreams, ngrp);
	kern<<<grid, 32 * WARPS, smem, stream>>>(in, stream_stride, hpad, p, tw, meta, dm, nch, ngrp, nsamp);
	return (int)cudaGetLastError();
}

/* float32 real input, taps > K (hpad > 0), K in the rdft's five rates, every channel on the 12.5 kHz raster; `in` = sample 0
 * of stream 0's submit with each stream's hpad-sample history right in front of it (d_real); `nsamp` output rows per
 * stream, any count; `p` = taps_pad floats, fl(K*h) behind hpad - H zeros */
static int launch_channelize_ovl_rdft(const void *in, size_t stream_stride, int hpad, const float *p, const float *tw,
                                      const unsigned *meta, float *dm, int K, int nch, int nstreams, size_t nsamp, cudaStream_t stream)
{
	if (nsamp == 0) return 0;
	if (hpad <= 0 || hpad % 4) return (int)cudaErrorInvalidValue;           /* 16-byte copies; taps <= K has no history */
	const uint8_t *i8 = reinterpret_cast<const uint8_t *>(in);
	const float2 *t4 = reinterpret_cast<const float2 *>(tw);
	const int nblk = (int)((nsamp + OUTBLK - 1) / OUTBLK);
	/* 4 warps; T = 64 rows per step at K = 200 / 240, 32 at 400 / 480, 16 at 800.  Columns per pre-sum thread: 2 where K/4
	 * units would leave most of the 128 threads idle */
#define ACB_ORD_GO(K8, LPR, CW) launch_ovl_rdft_t<K8, LPR, 4, CW>(i8, stream_stride, hpad, p, t4, meta, dm, nch, nstreams, nblk, nsamp, stream)
	if (K == 200) return ACB_ORD_GO(25, 2, 2);
	if (K == 240) return ACB_ORD_GO(30, 2, 2);
	if (K == 400) return ACB_ORD_GO(50, 4, 4);
	if (K == 480) return ACB_ORD_GO(60, 4, 4);
	if (K == 800) return ACB_ORD_GO(100, 8, 4);
#undef ACB_ORD_GO
	return (int)cudaErrorInvalidValue;
}

/* ------------------------------------------------------------------------------------------
 * K1, wideband fast form for REAL input (ACB_FLAG_FAST_WIDEBAND_REAL; DESIGN.md §4): k_channelize_rdft's definition at
 * taps = K (orc_channelize_rdft) and k_channelize_ovl_rdft's at taps > K (orc_ovl_presum_real, then orc_channelize_rdft)
 * for any K % 8 == 0 up to ACB_MAXK and any channel count.  The narrow kernels put 8 channels in a CTA and redo the row's
 * quarter split (and at taps > K the whole pre-sum) for every group of 8; here, as in k_channelize_wb, one CTA takes
 * rows_per_cta rows (tiles of T rows) of one stream and up to WB_CTILE channels:
 *
 *   front half (once per row for all channels): at taps > K the pre-sum z_m[n] = sum_r p[n + H + r*K] * x[m*K + n + r*K]
 *     in ascending tap order, one fmaf per term; then the quarter split per n2 < K/4: s02, s13, y0 = s02 + s13,
 *     y2 = s02 - s13, d02, d13, the rounded additions orc_channelize_rdft makes for every channel, made once.  Into shared
 *     memory as three columns [row][n2]: y0, y2 and (d02, d13), 4*K bytes per row.  Terms before the stream start READ
 *     the history in front of the rows in d_real, which acb_create / acb_reset zero: as in k_channelize_ovl_rdft, z starts
 *     at +0, those terms and the zero front padding of p come first, and fma(p, +-0, +0) = +0 leaves it there, so the sum
 *     is that of the valid terms only.  Every fetch lies in [-hpad, nsamp*K) samples of the stream.
 *   back half: a work item is WBR_RB rows x WB_CB channel slots of one column (k mod 4 = 0: y0; 2: y2; odd: d02 and d13
 *     with two sums, residues 1 and 3 differing in one sign at the end).  LPR consecutive lanes share an item, lane h
 *     summing the h-th range of ceil(K/8 / LPR) n2 pairs in n2 order; the LPR partial sums are then added by xor shuffles
 *     in the definition's pairwise tree (h ^ 1, then h ^ 2, ...): k_channelize_rdft's ranges and tree, LPR = 2 / 4 / 8 for
 *     K < 400 / < 800 / >= 800 (channelize_rdft_lanes_per_row), at any K.  The twiddles come from ONE table staged in
 *     shared memory, E[r] = acb_fast_plan_air's T for (k*n2) % K = r in [0, K) (acb_wb_twiddles' real variant).  The
 *     item's outputs are spread over its LPR lanes, which all hold the same sums.  |D| in double (envelope()): float
 *     input has no bound.
 *
 * meta per (stream, channel tile) as k_channelize_wb's; the slots are sorted by column (context.cu: upload_wb_plan).
 * ---------------------------------------------------------------------------------------- */
constexpr int WBR_THREADS = 256;
constexpr int WBR_RB = 4;                     /* rows per back-half item */

template <int LPR, bool OVL>
__global__ void __launch_bounds__(WBR_THREADS, 2)
k_channelize_wb_real(const uint8_t *__restrict__ in, size_t stream_stride, int hpad, const float *__restrict__ pw,
                     const float2 *__restrict__ E, const int *__restrict__ meta, float *__restrict__ dm, int K, int nch,
                     int nctile, size_t nsamp, int T, int rows_per_cta)
{
	constexpr int RB = WBR_RB, CB = WB_CB;
	const int N2 = K >> 2, K8 = K >> 3, PER = (K8 + LPR - 1) / LPR;
	extern __shared__ __align__(16) unsigned char smem[];
	float *Y0 = reinterpret_cast<float *>(smem);                         /* [row][n2] */
	float *Y2 = Y0 + (size_t)T * N2;
	float2 *DD = reinterpret_cast<float2 *>(Y2 + (size_t)T * N2);        /* (d02, d13) */
	float2 *Es = DD + (size_t)T * N2;                                     /* E[r], r in [0, K) */
	const int s = blockIdx.y;
	const int *ms = meta + ((size_t)s * nctile + blockIdx.z) * WB_META;
	const int ng = ms[0];
	for (int i = threadIdx.x; i < K; i += WBR_THREADS) Es[i] = E[K - 1 + i];
	const int nitem = (T / RB) * ng;

	for (int t0 = 0; t0 < rows_per_cta; t0 += T) {
		const size_t r0 = (size_t)blockIdx.x * rows_per_cta + t0;
		if (r0 >= nsamp) break;
		__syncthreads();                          /* E staged / the previous tile's Y' consumed */
		const float *src = reinterpret_cast<const float *>(in + (size_t)s * stream_stride);   /* sample 0 of the submit */
		for (int it = threadIdx.x; it < T * N2; it += WBR_THREADS) {
			const int j = it / N2, n2 = it - j * N2;
			const size_t row = r0 + j;
			float y0 = 0.f, y2 = 0.f, d02 = 0.f, d13 = 0.f;
			if (row < nsamp) {
				float x[4];
#pragma unroll
				for (int q = 0; q < 4; q++) {
					const int nn = q * N2 + n2;
					const float *xs = src + (long long)row * K + nn;
					if (!OVL) {
						x[q] = __ldg(xs);
					} else {
						const int rlo = -((nn + hpad) / K);            /* >= -hpad samples: the history */
						const float *pr = pw + nn + hpad;
						float a = 0.f;
						for (int r = rlo; r <= 0; r++) a = __fmaf_rn(__ldg(pr + r * K), __ldg(xs + (long long)r * K), a);
						x[q] = a;
					}
				}
				const float s02 = __fadd_rn(x[0], x[2]), s13 = __fadd_rn(x[1], x[3]);
				y0 = __fadd_rn(s02, s13);
				y2 = __fsub_rn(s02, s13);
				d02 = __fsub_rn(x[0], x[2]);
				d13 = __fsub_rn(x[1], x[3]);
			}
			Y0[it] = y0;
			Y2[it] = y2;
			DD[it] = make_float2(d02, d13);
		}
		__syncthreads();

		/* items (row group, channel group), channel group fastest; a warp holds 32 / LPR whole items, so the shuffles
		 * stay inside one; lanes past the last item run an empty range */
		for (int u0 = 0; u0 < nitem * LPR; u0 += WBR_THREADS) {
			const int u = u0 + (int)threadIdx.x, item = u / LPR, h = u & (LPR - 1);
			const bool valid = item < nitem;
			const int rg = valid ? item / ng : 0, cg = valid ? item - rg * ng : 0;
			const int *sl = ms + 2 + 2 * cg * CB;
			int kk[CB], idx[CB];
			const int g0 = h * PER, g1 = valid ? min(K8, g0 + PER) : g0;
#pragma unroll
			for (int c = 0; c < CB; c++) {
				kk[c] = sl[2 * c];
				idx[c] = (kk[c] * 2 * g0) % K;        /* (k*n2) % K at the range's first n2, 0 <= k < K */
			}
			float acc[RB][CB][4];                     /* ax, ay, bx, by (orc_channelize_rdft) */
#pragma unroll
			for (int j = 0; j < RB; j++)
#pragma unroll
				for (int c = 0; c < CB; c++) acc[j][c][0] = acc[j][c][1] = acc[j][c][2] = acc[j][c][3] = 0.f;
			const int col = kk[0] & 3;                /* slot 0 of a group is always a channel */
			const int roff = rg * RB * N2;
			if (col & 1) {
				const float2 *Yr = DD + roff;
#pragma unroll 1
				for (int n2 = 2 * g0; n2 < 2 * g1; n2++) {
					float2 t[CB];
#pragma unroll
					for (int c = 0; c < CB; c++) {
						t[c] = Es[idx[c]];
						const int v = idx[c] + kk[c];
						idx[c] = v >= K ? v - K : v;
					}
#pragma unroll
					for (int j = 0; j < RB; j++) {
						const float2 d = Yr[j * N2 + n2];
#pragma unroll
						for (int c = 0; c < CB; c++) {
							acc[j][c][0] = __fmaf_rn(d.x, t[c].x, acc[j][c][0]);
							acc[j][c][1] = __fmaf_rn(d.x, t[c].y, acc[j][c][1]);
							acc[j][c][2] = __fmaf_rn(d.y, t[c].x, acc[j][c][2]);
							acc[j][c][3] = __fmaf_rn(d.y, t[c].y, acc[j][c][3]);
						}
					}
				}
			} else {
				const float *Yr = (col == 0 ? Y0 : Y2) + roff;
#pragma unroll 1
				for (int n2 = 2 * g0; n2 < 2 * g1; n2++) {
					float2 t[CB];
#pragma unroll
					for (int c = 0; c < CB; c++) {
						t[c] = Es[idx[c]];
						const int v = idx[c] + kk[c];
						idx[c] = v >= K ? v - K : v;
					}
#pragma unroll
					for (int j = 0; j < RB; j++) {
						const float y = Yr[j * N2 + n2];
#pragma unroll
						for (int c = 0; c < CB; c++) {
							acc[j][c][0] = __fmaf_rn(y, t[c].x, acc[j][c][0]);
							acc[j][c][1] = __fmaf_rn(y, t[c].y, acc[j][c][1]);
						}
					}
				}
			}
			/* the LPR partial sums, pairwise: (p0 + p1) + (p2 + p3) ... — every lane of the item computes the same sum */
#pragma unroll
			for (int step = 1; step < LPR; step *= 2)
#pragma unroll
				for (int j = 0; j < RB; j++)
#pragma unroll
					for (int c = 0; c < CB; c++)
#pragma unroll
						for (int q = 0; q < 4; q++)
							acc[j][c][q] = __fadd_rn(acc[j][c][q], __shfl_xor_sync(0xffffffffu, acc[j][c][q], step));
			if (!valid) continue;
#pragma unroll
			for (int j = 0; j < RB; j++) {
				const size_t row = r0 + rg * RB + j;
#pragma unroll
				for (int c = 0; c < CB; c++) {
					if (((j * CB + c) & (LPR - 1)) != h) continue;
					const int chc = sl[2 * c + 1];
					if (row >= nsamp || chc < 0) continue;
					/* r = 1: D = (ax + by) + j (ay - bx); r = 3: the other signs; r even: b is zero */
					const float sg = (kk[c] & 3) == 3 ? -1.0f : 1.0f;
					const float re = __fadd_rn(acc[j][c][0], __fmul_rn(sg, acc[j][c][3]));
					const float im = __fadd_rn(acc[j][c][1], -__fmul_rn(sg, acc[j][c][2]));
					dm[((size_t)s * nsamp + row) * nch + chc] = envelope(make_float2(re, im));
				}
			}
		}
	}
}

/* rows per tile of k_channelize_wb_real: the most, a multiple of WBR_RB and at most 32, whose Y' (4*K bytes per row) and
 * E (8*K bytes) leave room for two CTAs per SM (113 KB each): 32 rows up to K = 848, 12 at K = 2048; the most shared
 * memory is 115 648 bytes (K = 1112, 24 rows) */
static int wbr_rows(int K)
{
	return std::min(32, (113 * 1024 - 8 * K) / (4 * K) / WBR_RB * WBR_RB);
}

template <int LPR, bool OVL>
static int launch_wbr_t(const uint8_t *in, size_t stream_stride, int hpad, const float *p, const float2 *E, const int *meta,
                        float *dm, int K, int nch, int nstreams, size_t nsamp, cudaStream_t stream)
{
	const int T = wbr_rows(K);
	const int smem = 4 * T * K + 8 * K;
	const int nctile = (nch + WB_CTILE - 1) / WB_CTILE;
	auto kern = k_channelize_wb_real<LPR, OVL>;
	if (cudaError_t e = smem_max_carveout(kern, smem)) return (int)e;
	const int rows_per_cta = wb_tiles_per_cta(nsamp, T, nstreams, nctile) * T;
	dim3 grid((unsigned)((nsamp + rows_per_cta - 1) / rows_per_cta), nstreams, nctile);
	kern<<<grid, WBR_THREADS, smem, stream>>>(in, stream_stride, hpad, p, E, meta, dm, K, nch, nctile, nsamp, T, rows_per_cta);
	return (int)cudaGetLastError();
}

/* float32 real input, K % 8 == 0, K <= ACB_MAXK, any nch, every channel on the 12.5 kHz raster; taps = K (hpad = 0) or
 * taps > K (`p` = taps_pad floats, fl(K*h) behind hpad - H zeros); `in` = sample 0 of stream 0's submit with each
 * stream's hpad-sample history right in front of it (d_real); `nsamp` output rows per stream, any count */
static int launch_channelize_wb_real(const void *in, size_t stream_stride, int hpad, const float *p, const float *E, const int *meta,
                                     float *dm, int K, int nch, int nstreams, size_t nsamp, cudaStream_t stream)
{
	if (nsamp == 0) return 0;
	if ((K & 7) || K > 2048 || hpad < 0) return (int)cudaErrorInvalidValue;
	const uint8_t *i8 = reinterpret_cast<const uint8_t *>(in);
	const float2 *E2 = reinterpret_cast<const float2 *>(E);
	const int lpr = channelize_rdft_lanes_per_row(K);
#define ACB_WBR_GO(L, O) launch_wbr_t<L, O>(i8, stream_stride, hpad, p, E2, meta, dm, K, nch, nstreams, nsamp, stream)
	if (hpad) return lpr == 8 ? ACB_WBR_GO(8, true) : lpr == 4 ? ACB_WBR_GO(4, true) : ACB_WBR_GO(2, true);
	return lpr == 8 ? ACB_WBR_GO(8, false) : lpr == 4 ? ACB_WBR_GO(4, false) : ACB_WBR_GO(2, false);
#undef ACB_WBR_GO
}

static bool channelize_dft_supports(int K) { return K == 160 || K == 192; }

/* u8 IQ, K in {160, 192} (the reference's two rates), taps == K, every channel on the 12.5 kHz raster
 * around Fc (context.cu checks and builds tw/meta) */
static int launch_channelize_dft(const void *in, size_t stream_stride, const float *tw, const unsigned *meta, float *dm,
                                 int K, int nch, int nstreams, int nblk, size_t nsamp, bool fold8, cudaStream_t stream)
{
	if (nblk == 0) return 0;
	const uint8_t *i8 = reinterpret_cast<const uint8_t *>(in);
	const float2 *t4 = reinterpret_cast<const float2 *>(tw);
	/* the two-rows-per-lane kernel: 2 warps per CTA, one tile buffer per warp; K=160: 44.5 KB of shared memory and <= 200
	 * registers -> 5 CTAs = 10 warps per SM */
	const int minb = getenv("ACB_DFT_MINB") ? atoi(getenv("ACB_DFT_MINB")) : 0;     /* experiment switch: register cap */
	/* default: the folded form with one row per lane, 2 warps per CTA (about half the registers and shared memory of the
	 * two-rows-per-lane kernel, so twice the warps per SM).  ACB_FAST_ROWS=2 selects the two-row kernel, ACB_FAST_WARPS=4
	 * four warps per CTA, ACB_FAST_PF=0 twiddle loads in place instead of one slot ahead: comparison switches, all
	 * bit-identical and tested. */
	const int rows1 = getenv("ACB_FAST_ROWS") ? atoi(getenv("ACB_FAST_ROWS")) : 1;
	if (fold8 && rows1 == 1) {
		const int w2 = getenv("ACB_FAST_WARPS") ? atoi(getenv("ACB_FAST_WARPS")) : 2;
		const bool pf = getenv("ACB_FAST_PF") ? atoi(getenv("ACB_FAST_PF")) != 0 : true;   /* experiment switch: twiddles one slot ahead */
#define ACB_DFT1_GO(U, W, M, F) launch_dft1_t<IN_U8IQ, U, W, M, F>(i8, stream_stride, t4, meta, dm, nch, nstreams, nblk, nsamp, stream)
		if (K == 160) return w2 != 2 ? ACB_DFT1_GO(20, 4, 4, true) : pf ? ACB_DFT1_GO(20, 2, 8, true) : ACB_DFT1_GO(20, 2, 8, false);
		if (K == 192) return w2 != 2 ? ACB_DFT1_GO(24, 4, 4, true) : pf ? ACB_DFT1_GO(24, 2, 8, true) : ACB_DFT1_GO(24, 2, 8, false);
#undef ACB_DFT1_GO
	}
	if (K == 160 && fold8 && minb == 8) return launch_dft_t<20, 2, 1, 8, true>(i8, stream_stride, t4, meta, dm, nch, nstreams, nblk, nsamp, stream);
	if (K == 160 && fold8 && minb == 6) return launch_dft_t<20, 2, 1, 6, true>(i8, stream_stride, t4, meta, dm, nch, nstreams, nblk, nsamp, stream);
	if (K == 160) return fold8 ? launch_dft_t<20, 2, 1, 5, true>(i8, stream_stride, t4, meta, dm, nch, nstreams, nblk, nsamp, stream)
	                           : launch_dft_t<20, 2, 1, 5, false>(i8, stream_stride, t4, meta, dm, nch, nstreams, nblk, nsamp, stream);
	if (K == 192) return fold8 ? launch_dft_t<24, 2, 1, 4, true>(i8, stream_stride, t4, meta, dm, nch, nstreams, nblk, nsamp, stream)
	                           : launch_dft_t<24, 2, 1, 4, false>(i8, stream_stride, t4, meta, dm, nch, nstreams, nblk, nsamp, stream);
	return (int)cudaErrorInvalidValue;
}

/* CS16 IQ (soapy.c / sdrplay.c), same conditions as above; `nsamp` output rows per stream, any count: the last block may be
 * partial (the input buffer carries 32 rows of slack).  stream_stride in bytes. */
static int launch_channelize_dft_cs16(const void *in, size_t stream_stride, const float *tw, const unsigned *meta, float *dm,
                                      int K, int nch, int nstreams, size_t nsamp, cudaStream_t stream)
{
	if (nsamp == 0) return 0;
	const uint8_t *i8 = reinterpret_cast<const uint8_t *>(in);
	const float2 *t4 = reinterpret_cast<const float2 *>(tw);
	const int nblk = (int)((nsamp + OUTBLK - 1) / OUTBLK);
	/* a warp's tile is 32 rows x (4K + 16) bytes = 20.5 KB at K = 160: 2 warps per CTA -> 5 CTAs = 10 warps per SM */
	const int w2 = getenv("ACB_FAST_WARPS") ? atoi(getenv("ACB_FAST_WARPS")) : 2;
#define ACB_DFT1_GO(U, W, M) launch_dft1_t<IN_CS16IQ, U, W, M, true>(i8, stream_stride, t4, meta, dm, nch, nstreams, nblk, nsamp, stream)
	if (K == 160) return w2 == 1 ? ACB_DFT1_GO(20, 1, 8) : ACB_DFT1_GO(20, 2, 5);
	if (K == 192) return w2 == 1 ? ACB_DFT1_GO(24, 1, 8) : ACB_DFT1_GO(24, 2, 4);
#undef ACB_DFT1_GO
	return (int)cudaErrorInvalidValue;
}

/* SDRplay's stream callback delivers I and Q as separate int16 arrays (sdrplay.c:196-205): out[s][i] = (xi[s][i], xq[s][i])
 * as the interleaved CS16 sample the channelizer reads.  Pure data movement, 8 bytes per sample. */
__global__ void __launch_bounds__(256)
k_interleave_cs16(const int16_t *__restrict__ xi, const int16_t *__restrict__ xq, size_t plane_stride,
                  uint32_t *__restrict__ out, size_t out_stride, size_t nsamples)
{
	const int s = blockIdx.y;
	const uint16_t *pi = reinterpret_cast<const uint16_t *>(xi) + (size_t)s * plane_stride;
	const uint16_t *pq = reinterpret_cast<const uint16_t *>(xq) + (size_t)s * plane_stride;
	uint32_t *o = out + (size_t)s * out_stride;
	for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < nsamples; i += (size_t)gridDim.x * blockDim.x)
		o[i] = (uint32_t)pi[i] | ((uint32_t)pq[i] << 16);
}

int launch_interleave_cs16(const int16_t *xi, const int16_t *xq, size_t plane_stride, uint32_t *out, size_t out_stride,
                           size_t nsamples, int nstreams, cudaStream_t stream)
{
	if (nsamples == 0) return 0;
	const unsigned gx = (unsigned)std::min<size_t>((nsamples + 255) / 256, 1184);
	k_interleave_cs16<<<dim3(gx, nstreams), 256, 0, stream>>>(xi, xq, plane_stride, out, out_stride, nsamples);
	return (int)cudaGetLastError();
}

/* The device submits of the streaming kinds: stream s's `nsamples` new 4-byte samples land behind its history and carried
 * remainder, out[s][i] = a[s][i] (float32 real or interleaved CS16), or out[s][i] = (a[s][i], b[s][i]) from the caller's
 * separate I and Q planes (PLANAR).  The source has any 4-byte (planes: 2-byte) alignment and stride; the destination
 * row starts at hpad + carry samples, generally not on 16 bytes, so a head of up to 3 samples and a tail of up to 3 go
 * singly and every whole 16-byte unit between them is one vector store.  Pure data movement, read once, written once. */
template <bool PLANAR>
__device__ __forceinline__ void append4_row(const void *__restrict__ a, const void *__restrict__ b, size_t src_stride,
                                            uint32_t *__restrict__ out, size_t out_stride, size_t nsamples)
{
	const int s = blockIdx.y;
	const uint32_t *x = reinterpret_cast<const uint32_t *>(a) + (size_t)s * src_stride;
	const uint16_t *pi = reinterpret_cast<const uint16_t *>(a) + (size_t)s * src_stride;
	const uint16_t *pq = reinterpret_cast<const uint16_t *>(b) + (size_t)s * src_stride;
	uint32_t *o = out + (size_t)s * out_stride;
	auto at = [&](size_t i) -> uint32_t {
		if constexpr (PLANAR) return (uint32_t)pi[i] | ((uint32_t)pq[i] << 16);
		else return x[i];
	};
	const size_t head = min(nsamples, (size_t)(((16 - ((uintptr_t)o & 15)) & 15) / 4));
	const size_t nvec = (nsamples - head) / 4, tail0 = head + 4 * nvec;
	const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x, nth = (size_t)gridDim.x * blockDim.x;
	uint4 *ov = reinterpret_cast<uint4 *>(o + head);
	for (size_t v = tid; v < nvec; v += nth) {
		const size_t i = head + 4 * v;
		ov[v] = make_uint4(at(i), at(i + 1), at(i + 2), at(i + 3));
	}
	if (tid < head) o[tid] = at(tid);
	if (tid < nsamples - tail0) o[tail0 + tid] = at(tail0 + tid);
}

template <bool PLANAR>
__global__ void __launch_bounds__(256)
k_append4(const void *__restrict__ a, const void *__restrict__ b, size_t src_stride, uint32_t *__restrict__ out,
          size_t out_stride, size_t nsamples)
{
	append4_row<PLANAR>(a, b, src_stride, out, out_stride, nsamples);
}

/* The ragged form: stream s's count[s] samples land at out + s*out_stride + off[s] (its history and own carry) */
template <bool PLANAR>
__global__ void __launch_bounds__(256)
k_append4_ragged(const void *__restrict__ a, const void *__restrict__ b, size_t src_stride, uint32_t *__restrict__ out,
                 size_t out_stride, const int *__restrict__ off, const int *__restrict__ count)
{
	const int s = blockIdx.y;
	append4_row<PLANAR>(a, b, src_stride, out + off[s], out_stride, (size_t)count[s]);
}

int launch_append4_ragged(const void *a, const void *b, size_t src_stride, uint32_t *out, size_t out_stride, const int *off,
                          const int *count, size_t max_count, int nstreams, cudaStream_t stream)
{
	if (max_count == 0) return 0;
	const unsigned gx = (unsigned)std::min<size_t>((max_count / 4 + 255) / 256 + 1, 1184);
	if (b) k_append4_ragged<true><<<dim3(gx, nstreams), 256, 0, stream>>>(a, b, src_stride, out, out_stride, off, count);
	else k_append4_ragged<false><<<dim3(gx, nstreams), 256, 0, stream>>>(a, nullptr, src_stride, out, out_stride, off, count);
	return (int)cudaGetLastError();
}

/* Ragged streaming submits: stream s's unconsumed tail (its last `hpad` samples before it, the next submit's history, and
 * rem[s] samples no row took) moves from src + s*stride + nrows[s]*K to the front of the other buffer, dst + s*stride */
__global__ void __launch_bounds__(256)
k_move_tail(const uint32_t *__restrict__ src, uint32_t *__restrict__ dst, size_t stride, int K, int hpad,
            const int *__restrict__ nrows, const int *__restrict__ rem)
{
	const int s = blockIdx.y;
	const uint32_t *p = src + (size_t)s * stride + (size_t)nrows[s] * K;
	uint32_t *o = dst + (size_t)s * stride;
	const int n = hpad + rem[s];
	for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) o[i] = p[i];
}

int launch_move_tail(const uint32_t *src, uint32_t *dst, size_t stride, int K, int hpad, const int *nrows, const int *rem,
                     int nstreams, cudaStream_t stream)
{
	const unsigned gx = (unsigned)((hpad + K + 255) / 256);      /* rem < K */
	k_move_tail<<<dim3(gx, nstreams), 256, 0, stream>>>(src, dst, stride, K, hpad, nrows, rem);
	return (int)cudaGetLastError();
}

/* Ragged u8 submits at taps > K: stream s's last `hb` bytes of input, at in + s*stride + nblk[s]*blk_bytes - hb, become its
 * history; a stream that brought no block keeps the history it had */
__global__ void __launch_bounds__(256)
k_hist_gather(const uint8_t *__restrict__ in, size_t stride, size_t blk_bytes, const int *__restrict__ nblk,
              uint8_t *__restrict__ hist, int hb)
{
	const int s = blockIdx.y;
	if (nblk[s] == 0) return;
	const uint8_t *p = in + (size_t)s * stride + (size_t)nblk[s] * blk_bytes - hb;
	uint8_t *o = hist + (size_t)s * hb;
	for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < hb; i += gridDim.x * blockDim.x) o[i] = p[i];
}

int launch_hist_gather(const uint8_t *in, size_t stride, size_t blk_bytes, const int *nblk, uint8_t *hist, int hb, int nstreams,
                       cudaStream_t stream)
{
	k_hist_gather<<<dim3((unsigned)((hb + 255) / 256), nstreams), 256, 0, stream>>>(in, stride, blk_bytes, nblk, hist, hb);
	return (int)cudaGetLastError();
}

int launch_append4(const void *a, const void *b, size_t src_stride, uint32_t *out, size_t out_stride, size_t nsamples, int nstreams,
                   cudaStream_t stream)
{
	if (nsamples == 0) return 0;
	const unsigned gx = (unsigned)std::min<size_t>((nsamples / 4 + 255) / 256 + 1, 1184);
	if (b) k_append4<true><<<dim3(gx, nstreams), 256, 0, stream>>>(a, b, src_stride, out, out_stride, nsamples);
	else k_append4<false><<<dim3(gx, nstreams), 256, 0, stream>>>(a, nullptr, src_stride, out, out_stride, nsamples);
	return (int)cudaGetLastError();
}

/* Rows the pipeline kernel does not take (K that breaks 16-byte row alignment; the < 1024 rows
 * left over by a real-input submit of arbitrary length): one thread per (output, channel),
 * straight from global memory, same arithmetic.  Correctness path, not tuned. */
template <int MODE>
__global__ void __launch_bounds__(128)
k_channelize_generic(const uint8_t *__restrict__ in, size_t stream_stride, const uint8_t *__restrict__ wf,
                     float *__restrict__ dm, int K, int taps, int nch, int ngrp, size_t row0, size_t nrows, size_t nsamp)
{
	const size_t gid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
	const int s = blockIdx.y;
	if (gid >= nrows * nch) return;
	const size_t m = row0 + gid / nch;
	const int ch = (int)(gid % nch);
	float dr = 0.f, di = 0.f;
	if (MODE == IN_F32REAL) {
		const float *p = reinterpret_cast<const float *>(in + (size_t)s * stream_stride) + m * K;
		const float2 *w = reinterpret_cast<const float2 *>(wf) + ((size_t)s * ngrp + ch / CH_GROUP) * taps * CH_GROUP + (ch % CH_GROUP);
		for (int i = 0; i < taps; i++) {
			const float2 ww = w[(size_t)i * CH_GROUP];
			dr = __fadd_rn(dr, __fmul_rn(ww.x, p[i]));
			di = __fadd_rn(di, __fmul_rn(ww.y, p[i]));
		}
	} else if (MODE == IN_CS16IQ) {
		const short *p = reinterpret_cast<const short *>(in + (size_t)s * stream_stride) + m * K * 2;
		const float2 *w = reinterpret_cast<const float2 *>(wf) + ((size_t)s * ngrp + ch / CH_GROUP) * taps * CH_GROUP + (ch % CH_GROUP);
		for (int ind = 0; ind < taps; ind++) {
			const float a = (float)p[2 * ind], b = (float)p[2 * ind + 1];
			const float2 ww = w[(size_t)ind * CH_GROUP];
			dr = __fadd_rn(dr, __fadd_rn(__fmul_rn(a, ww.x), __fmul_rn(b, -ww.y)));
			di = __fadd_rn(di, __fadd_rn(__fmul_rn(a, ww.y), __fmul_rn(b, ww.x)));
		}
	} else {
		const uint8_t *p = in + (size_t)s * stream_stride + m * K * 2;
		const float2 *w = reinterpret_cast<const float2 *>(wf) + ((size_t)s * ngrp + ch / CH_GROUP) * taps * CH_GROUP + (ch % CH_GROUP);
		for (int ind = 0; ind < taps; ind++) {
			float a = __fadd_rn((float)p[2 * ind], -127.37f), b = __fadd_rn((float)p[2 * ind + 1], -127.37f);
			float2 ww = w[(size_t)ind * CH_GROUP];
			float pr = __fadd_rn(__fmul_rn(a, ww.x), __fmul_rn(b, -ww.y));
			float pi = __fadd_rn(__fmul_rn(a, ww.y), __fmul_rn(b, ww.x));
			dr = __fadd_rn(dr, pr);
			di = __fadd_rn(di, pi);
		}
	}
	dm[((size_t)s * nsamp + m) * nch + ch] = envelope(make_float2(dr, di));
}

static int launch_channelize_generic(int mode, const void *in, size_t stream_stride, const void *wf, float *dm,
                                     int K, int taps, int nch, int nstreams, size_t row0, size_t nrows, size_t nsamp, cudaStream_t stream)
{
	if (nrows == 0) return 0;
	const int ngrp = (nch + CH_GROUP - 1) / CH_GROUP;
	const size_t total = nrows * nch;
	dim3 grid((unsigned)((total + 127) / 128), nstreams);
	const uint8_t *i8 = (const uint8_t *)in, *w8 = (const uint8_t *)wf;
	if (mode == IN_F32REAL) k_channelize_generic<IN_F32REAL><<<grid, 128, 0, stream>>>(i8, stream_stride, w8, dm, K, taps, nch, ngrp, row0, nrows, nsamp);
	else if (mode == IN_CS16IQ) k_channelize_generic<IN_CS16IQ><<<grid, 128, 0, stream>>>(i8, stream_stride, w8, dm, K, taps, nch, ngrp, row0, nrows, nsamp);
	else k_channelize_generic<IN_U8IQ><<<grid, 128, 0, stream>>>(i8, stream_stride, w8, dm, K, taps, nch, ngrp, row0, nrows, nsamp);
	return (int)cudaGetLastError();
}

/* The generic kernel's overlapping-window form (taps = K + hpad > K): tap i of row m reads sample m*K - hpad + i of the
 * submit, from the stream's history when that index is negative.  Taps whose sample precedes the start of the stream
 * (absolute row pos0 + m, counted from acb_create / acb_reset) are omitted, as the definition says; this is also the
 * path that gives the u8 pipeline kernel's first rows after a reset their exact value (a raw zero byte of u8 history
 * would convert to -127.37, not to 0). */
template <int MODE>
__global__ void __launch_bounds__(128)
k_channelize_generic_ovl(const uint8_t *__restrict__ in, size_t stream_stride, const uint8_t *__restrict__ wf,
                         float *__restrict__ dm, int K, int taps, int nch, int ngrp, size_t row0, size_t nrows, size_t nsamp,
                         const uint8_t *__restrict__ hist, size_t hist_stride, int hpad, unsigned long long pos0)
{
	constexpr int TB = MODE == IN_U8IQ ? 2 : 4;                      /* input bytes per sample */
	const size_t gid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
	const int s = blockIdx.y;
	if (gid >= nrows * nch) return;
	const size_t m = row0 + gid / nch;
	const int ch = (int)(gid % nch);
	const uint8_t *p = in + (size_t)s * stream_stride, *hp = hist + (size_t)s * hist_stride + (size_t)hpad * TB;
	const long long o0 = (long long)m * K - hpad;                    /* sample of tap 0, relative to the submit */
	const long long a0 = (long long)(pos0 + m) * K - hpad;           /* the same, counted from the stream start */
	const int first = a0 < 0 ? (int)-a0 : 0;
	float dr = 0.f, di = 0.f;
	if (MODE == IN_F32REAL) {
		const float2 *w = reinterpret_cast<const float2 *>(wf) + ((size_t)s * ngrp + ch / CH_GROUP) * taps * CH_GROUP + (ch % CH_GROUP);
		for (int i = first; i < taps; i++) {
			const long long o = o0 + i;
			const float x = *reinterpret_cast<const float *>(o < 0 ? hp + o * TB : p + o * TB);
			const float2 ww = w[(size_t)i * CH_GROUP];
			dr = __fadd_rn(dr, __fmul_rn(ww.x, x));
			di = __fadd_rn(di, __fmul_rn(ww.y, x));
		}
	} else {
		const float2 *w = reinterpret_cast<const float2 *>(wf) + ((size_t)s * ngrp + ch / CH_GROUP) * taps * CH_GROUP + (ch % CH_GROUP);
		for (int i = first; i < taps; i++) {
			const long long o = o0 + i;
			const uint8_t *q = o < 0 ? hp + o * TB : p + o * TB;
			float a, b;
			if (MODE == IN_CS16IQ) {
				a = (float)reinterpret_cast<const short *>(q)[0];
				b = (float)reinterpret_cast<const short *>(q)[1];
			} else {
				a = __fadd_rn((float)q[0], -127.37f);
				b = __fadd_rn((float)q[1], -127.37f);
			}
			const float2 ww = w[(size_t)i * CH_GROUP];
			dr = __fadd_rn(dr, __fadd_rn(__fmul_rn(a, ww.x), __fmul_rn(b, -ww.y)));
			di = __fadd_rn(di, __fadd_rn(__fmul_rn(a, ww.y), __fmul_rn(b, ww.x)));
		}
	}
	dm[((size_t)s * nsamp + m) * nch + ch] = envelope(make_float2(dr, di));
}

static int launch_channelize_generic_ovl(int mode, const void *in, size_t stream_stride, const void *wf, float *dm,
                                         int K, int taps, int nch, int nstreams, size_t row0, size_t nrows, size_t nsamp,
                                         const Hist &h, cudaStream_t stream)
{
	if (nrows == 0) return 0;
	const int ngrp = (nch + CH_GROUP - 1) / CH_GROUP;
	const size_t total = nrows * nch;
	dim3 grid((unsigned)((total + 127) / 128), nstreams);
	const uint8_t *i8 = (const uint8_t *)in, *w8 = (const uint8_t *)wf, *h8 = (const uint8_t *)h.base;
#define ACB_GEN_OVL(M) k_channelize_generic_ovl<M><<<grid, 128, 0, stream>>>(i8, stream_stride, w8, dm, K, taps, nch, ngrp, row0, nrows, nsamp, \
	                                                                         h8, h.stride, h.hpad, h.pos0)
	if (mode == IN_F32REAL) ACB_GEN_OVL(IN_F32REAL);
	else if (mode == IN_CS16IQ) ACB_GEN_OVL(IN_CS16IQ);
	else ACB_GEN_OVL(IN_U8IQ);
#undef ACB_GEN_OVL
	return (int)cudaGetLastError();
}

/* K1's forms, tried in this order (chan_form):
 *
 *   input       condition                                                      form
 *   u8 / CS16   ACB_FLAG_FAST_CHANNELIZER, taps == K, K in {160, 192}          CHAN_DFT       k_channelize_dft(1)
 *               ACB_FLAG_FAST_FILTER, taps > K, K in {160, 192}                CHAN_OVL_FAST  k_channelize_ovl_fast
 *               ACB_FLAG_FAST_WIDEBAND, taps >= K, K % 8 == 0                  CHAN_WB        k_channelize_wb
 *               K % 8 != 0 (u8), K % 4 != 0 (CS16)                             CHAN_GENERIC   k_channelize_generic(_ovl)
 *               otherwise                                                      CHAN_EXACT     k_channelize_iq4
 *   real        ACB_FLAG_FAST_CHANNELIZER, taps == K, channelize_rdft_supports  CHAN_RDFT      k_channelize_rdft
 *               ACB_FLAG_FAST_FILTER_REAL, taps > K, channelize_rdft_supports  CHAN_OVL_RDFT  k_channelize_ovl_rdft
 *               ACB_FLAG_FAST_WIDEBAND_REAL, taps >= K, K % 8 == 0             CHAN_WB_REAL   k_channelize_wb_real
 *               K % 4 != 0                                                     CHAN_GENERIC   k_channelize_generic(_ovl)
 *               otherwise                                                      CHAN_EXACT     k_channelize_real4
 *
 * A fast form (all but EXACT and GENERIC) runs only while every stream is planned on the 12.5 kHz raster; a submit runs
 * EXACT otherwise (context.cu). */
ChanForm chan_form(int in_kind, int K, int taps, int f)
{
	if (in_kind == IN_KIND_F32REAL) {
		if ((f & ACB_FLAG_FAST_CHANNELIZER) && taps == K && channelize_rdft_supports(K)) return CHAN_RDFT;
		if ((f & ACB_FLAG_FAST_FILTER_REAL) && taps > K && channelize_rdft_supports(K)) return CHAN_OVL_RDFT;
		if ((f & ACB_FLAG_FAST_WIDEBAND_REAL) && taps >= K && K % 8 == 0) return CHAN_WB_REAL;
		return K % 4 ? CHAN_GENERIC : CHAN_EXACT;
	}
	if ((f & ACB_FLAG_FAST_CHANNELIZER) && taps == K && channelize_dft_supports(K)) return CHAN_DFT;
	if ((f & ACB_FLAG_FAST_FILTER) && taps > K && channelize_dft_supports(K)) return CHAN_OVL_FAST;
	if ((f & ACB_FLAG_FAST_WIDEBAND) && taps >= K && K % 8 == 0) return CHAN_WB;
	return K % (in_kind == IN_KIND_U8IQ ? 8 : 4) ? CHAN_GENERIC : CHAN_EXACT;
}

int launch_chan(const ChanLaunch &L, size_t nrows, cudaStream_t stream, int &launched)
{
	const int K = L.K, nch = L.nch, ns = L.nstreams;
	const size_t nsamp = L.nsamp;
	if (L.form != CHAN_EXACT && L.form != CHAN_GENERIC) {
		if (nrows != nsamp) return (int)cudaErrorInvalidValue;
		launched++;
	}
	switch (L.form) {
	case CHAN_DFT:
		return L.in_kind == IN_KIND_CS16IQ
		           ? launch_channelize_dft_cs16(L.in, L.stride, L.tw, L.twmeta, L.dm, K, nch, ns, nsamp, stream)
		           : launch_channelize_dft(L.in, L.stride, L.tw, L.twmeta, L.dm, K, nch, ns, (int)(nsamp / OUTBLK), nsamp, L.fold8, stream);
	case CHAN_RDFT: return launch_channelize_rdft(L.in, L.stride, L.tw, L.twmeta, L.dm, K, nch, ns, nsamp, stream);
	case CHAN_OVL_FAST:
		return launch_channelize_ovl_fast(L.in_kind, L.in, L.stride, L.hist, L.p, L.tw, L.twmeta, L.dm, K, nch, ns, nsamp, stream);
	case CHAN_OVL_RDFT:
		return launch_channelize_ovl_rdft(L.in, L.stride, L.hist.hpad, L.p, L.tw, L.twmeta, L.dm, K, nch, ns, nsamp, stream);
	case CHAN_WB: return launch_channelize_wb(L.in_kind, L.in, L.stride, L.hist, L.p, L.wbE, L.wbmeta, L.dm, K, nch, ns, nsamp, stream);
	case CHAN_WB_REAL: return launch_channelize_wb_real(L.in, L.stride, L.hist.hpad, L.p, L.wbE, L.wbmeta, L.dm, K, nch, ns, nsamp, stream);
	case CHAN_EXACT:
	case CHAN_GENERIC: break;
	}
	const int blocks = L.form == CHAN_EXACT ? (int)(nrows / OUTBLK) : 0;
	if (blocks) {
		launched++;
		if (int e = launch_channelize(L.in_kind, L.in, L.stride, L.wf, L.dm, K, L.taps_pad, nch, ns, blocks, nsamp, L.hist, stream)) return e;
	}
	const size_t row0 = (size_t)blocks * OUTBLK;
	if (nrows == row0) return 0;
	launched++;
	return L.hist.hpad ? launch_channelize_generic_ovl(L.in_kind, L.in, L.stride, L.wf, L.dm, K, L.taps_pad, nch, ns, row0, nrows - row0,
	                                                   nsamp, L.hist, stream)
	                   : launch_channelize_generic(L.in_kind, L.in, L.stride, L.wf, L.dm, K, L.taps_pad, nch, ns, row0, nrows - row0, nsamp,
	                                               stream);
}

/* Per stream the tables are wf [grp][taps_pad][8] (c, d), tw [grp][8][K/4] (Tr, Ti), twmeta [grp] and wbmeta [channel
 * tile][WB_META], as the kernels above read them; p and the E tables serve every stream. */
ChanLaunch chan_stream(const ChanLaunch &L, int s, unsigned long long pos0)
{
	const size_t ngrp = (L.nch + CH_GROUP - 1) / CH_GROUP, nctile = (L.nch + WB_CTILE - 1) / WB_CTILE;
	ChanLaunch o = L;
	o.in += s * L.stride;
	o.hist.base = (const uint8_t *)L.hist.base + s * L.hist.stride;
	o.hist.pos0 = pos0;
	o.dm += s * L.nsamp * L.nch;
	o.wf += s * ngrp * L.taps_pad * CH_GROUP * 2;
	if (L.tw) o.tw += s * ngrp * CH_GROUP * (L.K / 4) * 2;
	if (L.twmeta) o.twmeta += s * ngrp;
	if (L.wbmeta) o.wbmeta += s * nctile * WB_META;
	o.nstreams = 1;
	return o;
}

/* ------------------------------------------------------------------------------------------
 * K2: MSK demodulator + bit/byte framing, one channel per lane
 *
 * The recurrence is serial per channel (VCO phase -> ring -> matched filter -> PLL -> VCO step,
 * with the frame synchroniser resetting the PLL), so the kernel is latency bound; what it can
 * do is (a) never diverge: every lane runs "up to 6 samples, then one bit" per outer iteration
 * (the bit clock fires every 5.2 samples), (b) expose the 6 independent sincos evaluations of an
 * iteration to the scheduler at once, (c) use a branch-free table sincos (20 FP64 ops) instead
 * of the library one (~45 + slow path), (d) prefetch the 6 envelope samples.
 * ---------------------------------------------------------------------------------------- */

/* acars.c:350-366: queue the finished block.  lvl = 10*log10(lvlsum/bitcount) is left to the host
 * (glibc log10) so the float matches the reference bit for bit.  Returns where the frame went: EV_SHORT, EV_LOST, or
 * -1 = into the ring. */
static __device__ __forceinline__ int emit_frame_at(const ChainState *st, RawFrame *ring, RingCtl *ctl, unsigned cap,
                                                    int stream, int chn, int len, int err, double lvlsum, int bitcount,
                                                    unsigned long long pos, unsigned long long soh_pos)
{
	/* blk_thread drops blocks shorter than 13 bytes unseen (acars.c:124-129): they never take a slot, so a
	 * ring sized for the shortest deliverable frame (19 bytes on air = 792 samples) cannot be overrun by a
	 * transmitter sending degenerate frames; the host adds the count to raw_frames / fec_dropped */
	if (len < 13) { atomicAdd(&ctl->short_frames, 1u); return EV_SHORT; }
	const unsigned slot = atomicAdd(&ctl->count, 1u);
	if (slot >= cap) return EV_LOST;               /* overflow: counted by the host (frames_lost), decoding goes on */
	RawFrame *f = ring + slot;
	f->stream = stream; f->chn = chn;
	f->len = len; f->err = err;
	f->lvlsum = lvlsum; f->bitcount = bitcount; f->pad0 = 0;          /* pad0: FEC status, set by k_block_fec */
	f->pos = pos; f->soh_pos = soh_pos;
	f->crc[0] = st->crc[0]; f->crc[1] = st->crc[1];
	for (int i = 0; i < 6; i++) f->pad1[i] = 0;            /* the record goes to the host as a whole */
	const uint2 *src = reinterpret_cast<const uint2 *>(st->txt);
	uint2 *dst = reinterpret_cast<uint2 *>(f->txt);
	for (int i = 0; i < TXTCAP / 8; i++) dst[i] = src[i];
	return -1;
}

/* Out of line and by value: it runs once per frame, and keeping it away from the loop keeps the loop's state in
 * registers. */
static __device__ __noinline__ void emit_frame(const ChainState *st, RawFrame *ring, RingCtl *ctl, unsigned cap,
                                               int stream, int chn, int len, int err, double lvlsum, int bitcount,
                                               unsigned long long pos, unsigned long long soh_pos)
{
	emit_frame_at(st, ring, ctl, cap, stream, chn, len, err, lvlsum, bitcount, pos, soh_pos);
}

/* the counting kernels' form: the same, and where the frame went */
static __device__ __noinline__ int emit_frame_counted(const ChainState *st, RawFrame *ring, RingCtl *ctl, unsigned cap,
                                                      int stream, int chn, int len, int err, double lvlsum, int bitcount,
                                                      unsigned long long pos, unsigned long long soh_pos)
{
	return emit_frame_at(st, ring, ctl, cap, stream, chn, len, err, lvlsum, bitcount, pos, soh_pos);
}

/* accessor for frame_sm.h: state in registers, text in the chain's HBM record */
struct DevFrameAcc {
	DemodRegs &r;
	ChainState *st;
	RawFrame *ring;
	RingCtl *ctl;
	unsigned cap;
	int stream, chn;
	bool leader;             /* the lane of the channel's group that owns the HBM side effects */

	__device__ __forceinline__ int &state() { return r.state; }
	__device__ __forceinline__ int &nbits() { return r.nbits; }
	__device__ __forceinline__ int &bitcount() { return r.bitcount; }
	__device__ __forceinline__ int &blk_len() { return r.blk_len; }
	__device__ __forceinline__ int &blk_err() { return r.blk_err; }
	__device__ __forceinline__ unsigned &msk_s() { return r.S; }
	__device__ __forceinline__ double &msk_df() { return r.df; }
	__device__ __forceinline__ double &lvlsum() { return r.lvlsum; }
	__device__ __forceinline__ void txt_put(int i, unsigned char c) { if (leader) st->txt[i] = c; }
	/* only the leader's value is ever stored (crc_put); the shadows' reads are don't-cares */
	__device__ __forceinline__ unsigned char txt_get(int i) { return leader ? st->txt[i] : (unsigned char)0; }
	__device__ __forceinline__ void crc_put(int i, unsigned char c) { if (leader) st->crc[i] = c; }
	bool v2;                 /* demod_core.h's loop: the bit's sample position is pos0 + fire_n (r.pos is only set at the end) */
	__device__ __forceinline__ unsigned long long bit_pos() const { return v2 ? r.pos0 + (unsigned long long)(long long)r.fire_n : r.pos; }
	__device__ __forceinline__ bool frame_begin() { r.soh_pos = bit_pos(); return true; }   /* acars.c:283-292 */
	__device__ __forceinline__ void frame_emit()
	{
		if (leader) emit_frame(st, ring, ctl, cap, stream, chn, r.blk_len, r.blk_err, r.lvlsum, r.bitcount, bit_pos(), r.soh_pos);
	}
};

/* The counting kernels' accessor (ACB_FLAG_DECODE_STATS): DevFrameAcc plus the event hook.  Only the leader lane writes,
 * only on the rare events of frame_sm.h (no SYN-hunting bit raises one), into its chain's counters of this submit; no
 * other lane shares them, so plain increments do. */
struct DevFrameAccStats : DevFrameAcc {
	unsigned *cnt;           /* EV_COUNT counters of this chain */

	__device__ __forceinline__ void event(int e) { if (leader) cnt[e]++; }
	__device__ __forceinline__ void frame_emit()
	{
		if (!leader) return;
		const int where = emit_frame_counted(st, ring, ctl, cap, stream, chn, r.blk_len, r.blk_err, r.lvlsum, r.bitcount, bit_pos(),
		                                     r.soh_pos);
		if (where >= 0) cnt[where]++;
	}
};

/* cos/sin of k*pi/32 as double-double (hi, lo), built on the host in long double */
__device__ double2 g_sc_cos[64], g_sc_sin[64];

int upload_sincos_table(const double *cos_hi_lo, const double *sin_hi_lo, cudaStream_t stream)
{
	cudaError_t e = cudaMemcpyToSymbolAsync(g_sc_cos, cos_hi_lo, sizeof(double) * 128, 0, cudaMemcpyHostToDevice, stream);
	if (e != cudaSuccess) return (int)e;
	e = cudaMemcpyToSymbolAsync(g_sc_sin, sin_hi_lo, sizeof(double) * 128, 0, cudaMemcpyHostToDevice, stream);
	if (e != cudaSuccess) return (int)e;
	return (int)cudaStreamSynchronize(stream);      /* the sources are the caller's stack arrays */
}

/* cos(p), sin(p) for p in [0, 2*pi] — the VCO phase after msk.c:82-83.  p = k*pi/32 + r with
 * |r| <= pi/64 (three-part pi/32, so r keeps full relative accuracy next to the zeros of sin and
 * cos, which are table points with exact entries); short Taylor polynomials for sin r and
 * cos r - 1; angle addition against the double-double table.  Max error measured against 80-bit
 * references: 1.7 ulp (typ. < 0.6), i.e. the class of CUDA's own sincos; see DESIGN.md for why
 * ~1 ulp here is invisible after the (float) rounding of in*cexp(-j p) (msk.c:90). */
constexpr double SC_MAGIC = 6755399441055744.0;     /* 1.5 * 2^52 */
__device__ __forceinline__ void sincos_vco(double p, const double2 *tcos, const double2 *tsin, double &sn, double &cs)
{
	const double t = fma(p, 0x1.45f306dc9c883p+3, SC_MAGIC);               /* p * 32/pi, rounded to integer */
	const int k = __double2loint(t) & 63;
	const double kd = t - SC_MAGIC;
	double r = fma(-kd, 0x1.921fb54442d18p-4, p);
	r = fma(-kd, 0x1.1a62633145c07p-58, r);
	r = fma(-kd, -0x1.f1976b7ed8fbcp-114, r);
	const double r2 = r * r;
	double sp = fma(r2, (1.0 / 362880), (-1.0 / 5040));
	sp = fma(sp, r2, (1.0 / 120));
	sp = fma(sp, r2, (-1.0 / 6));
	const double sr = fma(r * r2, sp, r);                    /* sin r */
	double cp = fma(r2, (1.0 / 40320), (-1.0 / 720));
	cp = fma(cp, r2, (1.0 / 24));
	cp = fma(cp, r2, (-0.5));
	const double cm = r2 * cp;                               /* cos r - 1 */
	const double2 C = tcos[k], S = tsin[k];
	cs = C.x + fma(-S.x, sr, fma(C.x, cm, C.y));
	sn = S.x + fma(C.x, sr, fma(S.x, cm, S.y));
}

/* lanes per channel: 4 (8 channels per warp), or 8 (4 channels per warp, one mixer evaluation per lane
 * instead of two) for contexts small enough that the doubled warp count still fits one warp per SM
 * sub-partition (context.cu decides) */

/* One warp = 8 channels of one stream x 4 lanes per channel.  The 4 lanes of a channel run the
 * SAME recurrence on the same inputs (identical registers, no communication needed) except for
 * the mixer: lane `sub` evaluates in*cexp(-j phi) for candidate samples sub and 4+sub and drops
 * the result into the channel's ring in shared memory.  SIMT lanes are the one way to get the
 * independent sincos evaluations of a bit period executed side by side: as straight-line code of
 * one lane, ptxas schedules them back to back (6 x 16 dependent FP64 ops x 8 cycles).  Only the
 * group leader touches HBM state (frame text, frame ring, state write-back). */
template <int DEMOD_GROUP>
__global__ void __launch_bounds__(32)
k_demod(ChainState *__restrict__ states, const float *__restrict__ dm, int nsamp, int nch, int nstreams,
        int wps, RawFrame *__restrict__ ring, RingCtl *__restrict__ ctl, unsigned cap)
{
	constexpr int DEMOD_CPW = 32 / DEMOD_GROUP;      /* channels per warp */
	__shared__ float s_h[FLENO + 3];
	/* rows FLEN.. : one scratch row per lane of the group, for mixer outputs past the bit instant */
	__shared__ float s_re[FLEN + DEMOD_GROUP][DEMOD_CPW], s_im[FLEN + DEMOD_GROUP][DEMOD_CPW];
	__shared__ double2 s_cos[64], s_sin[64];

	for (int i = threadIdx.x; i < FLENO; i += 32) s_h[i] = c_h[i];
	for (int i = threadIdx.x; i < 64; i += 32) { s_cos[i] = g_sc_cos[i]; s_sin[i] = g_sc_sin[i]; }

	const int lane = threadIdx.x;
	const int grp = lane / DEMOD_GROUP, sub = lane % DEMOD_GROUP;
	const int warp = blockIdx.x;
	const int s = warp / wps;
	const int ch_raw = (warp - s * wps) * DEMOD_CPW + grp;
	const bool valid = ch_raw < nch;                 /* surplus groups shadow the last channel, silently */
	const int ch = valid ? ch_raw : nch - 1;
	const bool leader = valid && sub == 0;

	ChainState *st = states + (size_t)s * nch + ch;
	DemodRegs r;
	r.phi = st->phi; r.df = st->df; r.lvlsum = st->lvlsum; r.clk = st->clk; r.bitcount = st->bitcount;
	r.S = st->S; r.idx = st->idx; r.nbits = st->nbits; r.state = st->state; r.outbits = st->outbits;
	r.blk_len = st->blk_len; r.blk_err = st->blk_err; r.pos = st->pos; r.soh_pos = st->soh_pos;
	for (int k = sub; k < FLEN; k += DEMOD_GROUP) { s_re[k][grp] = st->inb_re[k]; s_im[k][grp] = st->inb_im[k]; }
	__syncwarp();

	DevFrameAcc acc{ r, st, ring, ctl, cap, s, ch, leader, false };

	const double TWO_PI = 2.0 * M_PI;
	const double S0 = 1800.0 / 12500 * 2.0 * M_PI;             /* msk.c:81 */
	const double THR = 3 * M_PI / 2.0;                         /* msk.c:96,100 */
	const double INV_S0 = 1.0 / (1800.0 / 12500 * 2.0 * M_PI);
	const double PLLC = (double)0.52f;                         /* msk.c:66 (float constant) */
	const double PLLK = (1.0 - (double)0.52f) * (double)38e-4f;/* msk.c:130 (1.0-PLLC)*PLLG */

	const float *in = dm + (size_t)s * nsamp * nch + ch;
	const unsigned long long pos0 = r.pos;
	double clkd = (double)r.clk;             /* MskClk: a float value carried in a double register */
	/* which of the six candidate phases this lane mixes: 4 lanes -> samples sub and 4 + sub (the latter
	 * only for sub < 2; lanes 2, 3 get phase 4 or 5 for their discarded second evaluation, as before);
	 * 8 lanes -> sample sub (lanes 6, 7 idle on phase 5) */
	long long pick[DEMOD_LOOK];
#pragma unroll
	for (int k = 0; k < DEMOD_LOOK; k++) {
		bool mine;
		if (DEMOD_GROUP == 4) mine = k < 4 ? (sub == k) : ((sub & 1) == (k - 4));
		else mine = k < DEMOD_LOOK - 1 ? (sub == k) : (sub >= k);
		pick[k] = mine ? -1LL : 0LL;
	}
	int n = 0;
	/* channels of a warp consume 5 or 6 samples per iteration each, so they finish a few
	 * iterations apart: finished groups idle through empty iterations (m = 0) */
	while (__any_sync(0xffffffffu, n < nsamp)) {
		const int m = max(0, min(DEMOD_LOOK, nsamp - n));
		/* this lane's two candidate samples */
		const int k1 = sub, k2 = DEMOD_GROUP + sub;
		const float x1 = in[(size_t)min(n + k1, nsamp - 1) * nch];
		const float x2 = DEMOD_GROUP == 4 ? in[(size_t)min(n + k2, nsamp - 1) * nch] : 0.f;
		if (n + 2 * DEMOD_LOOK < nsamp) asm volatile("prefetch.global.L1 [%0];" ::"l"(in + (size_t)(n + 2 * DEMOD_LOOK) * nch));

		/* VCO step is constant until the next bit (msk.c:81): MskDf only changes in the bit path */
		const double sv = __dadd_rn(S0, r.df);
		const double fire_at = __dadd_rn(THR, -__dmul_rn(sv, 0.5));
		/* 1/sv for the phase-index fast path below: three Newton steps from 1/S0 (|sv/S0 - 1| < 2e-2),
		 * off the critical path */
		double inv_s = INV_S0;
		inv_s = fma(inv_s, fma(-sv, inv_s, 1.0), inv_s);
		inv_s = fma(inv_s, fma(-sv, inv_s, 1.0), inv_s);
		inv_s = fma(inv_s, fma(-sv, inv_s, 1.0), inv_s);

		/* the two cheap serial chains of the next samples: phase (msk.c:82-83) and bit clock
		 * (msk.c:95-96), each rounded step by step exactly like the reference's loop; straight-line
		 * code (selects, no branches) */
		double pk[DEMOD_LOOK], ck[DEMOD_LOOK];
		{
			double p = r.phi, c = clkd;
#pragma unroll
			for (int k = 0; k < DEMOD_LOOK; k++) {
				p = __dadd_rn(p, sv);
				p = (p >= TWO_PI) ? __dadd_rn(p, -TWO_PI) : p;
				c = round_to_f32<false>(__dadd_rn(c, sv));
				pk[k] = p;
				ck[k] = c;
			}
		}
		/* first of the m available samples at which the clock fires (msk.c:96), if any; the state
		 * after `cnt` samples is picked with bit masks (a select chain on the index would be
		 * turned into a local-memory array by the compiler) */
		int cnt = m;                 /* samples consumed this iteration */
		bool fired = false;
#pragma unroll
		for (int k = DEMOD_LOOK - 1; k >= 0; k--) {
			const bool f = (k < m) & (ck[k] >= fire_at);
			cnt = f ? k + 1 : cnt;
			fired = fired | f;
		}
		double p;
		{
			long long pb = (cnt == 0) ? __double_as_longlong(r.phi) : 0, cb = (cnt == 0) ? __double_as_longlong(clkd) : 0;
#pragma unroll
			for (int k = 0; k < DEMOD_LOOK; k++) {
				const long long mk = -(long long)(cnt == k + 1);
				pb |= __double_as_longlong(pk[k]) & mk;
				cb |= __double_as_longlong(ck[k]) & mk;
			}
			p = __longlong_as_double(pb);
			clkd = __longlong_as_double(cb);
		}
		/* mixer (msk.c:86-91): in * cexp(-j phi), this lane's share */
		if (DEMOD_GROUP == 4) {
			/* lane-dependent picks as mask selects: written as a ?: chain on `sub` the compiler branches,
			 * and the lanes of a group then run the arms one after the other */
			const double p1 = __longlong_as_double((__double_as_longlong(pk[0]) & pick[0]) | (__double_as_longlong(pk[1]) & pick[1]) |
			                                       (__double_as_longlong(pk[2]) & pick[2]) | (__double_as_longlong(pk[3]) & pick[3]));
			const double p2 = __longlong_as_double((__double_as_longlong(pk[4]) & pick[4]) | (__double_as_longlong(pk[5]) & pick[5]));
			double sn1, cs1, sn2, cs2;
			sincos_vco(p1, s_cos, s_sin, sn1, cs1);
			sincos_vco(p2, s_cos, s_sin, sn2, cs2);
			const double xd1 = (double)x1, xd2 = (double)x2;
			const float re1 = __double2float_rn(__dmul_rn(xd1, cs1)), im1 = __double2float_rn(__dmul_rn(xd1, -sn1));
			const float re2 = __double2float_rn(__dmul_rn(xd2, cs2)), im2 = __double2float_rn(__dmul_rn(xd2, -sn2));
			unsigned row1 = r.idx + k1, row2 = r.idx + k2;
			row1 = (row1 >= FLEN) ? row1 - FLEN : row1;
			row2 = (row2 >= FLEN) ? row2 - FLEN : row2;
			row1 = (k1 < cnt) ? row1 : FLEN + sub;                 /* past the bit instant: scratch row */
			row2 = (k2 < cnt && k2 < DEMOD_LOOK) ? row2 : FLEN + sub;
			__syncwarp();          /* the previous bit's matched filter has read the rows being replaced */
			s_re[row1][grp] = re1; s_im[row1][grp] = im1;
			s_re[row2][grp] = re2; s_im[row2][grp] = im2;
			__syncwarp();
		} else {                   /* one candidate sample per lane (lanes 6, 7 of the group idle here) */
			const double p1 = __longlong_as_double((__double_as_longlong(pk[0]) & pick[0]) | (__double_as_longlong(pk[1]) & pick[1]) |
			                                       (__double_as_longlong(pk[2]) & pick[2]) | (__double_as_longlong(pk[3]) & pick[3]) |
			                                       (__double_as_longlong(pk[4]) & pick[4]) | (__double_as_longlong(pk[5]) & pick[5]));
			double sn1, cs1;
			sincos_vco(p1, s_cos, s_sin, sn1, cs1);
			const double xd1 = (double)x1;
			const float re1 = __double2float_rn(__dmul_rn(xd1, cs1)), im1 = __double2float_rn(__dmul_rn(xd1, -sn1));
			unsigned row1 = r.idx + k1;
			row1 = (row1 >= FLEN) ? row1 - FLEN : row1;
			row1 = (k1 < cnt && k1 < DEMOD_LOOK) ? row1 : FLEN + sub;
			__syncwarp();
			s_re[row1][grp] = re1; s_im[row1][grp] = im1;
			__syncwarp();
		}
		r.idx = (r.idx + cnt) % FLEN;
		r.phi = p;
		r.pos = pos0 + (unsigned long long)(n + cnt - 1);       /* the sample that fired the bit */

		if (fired) {
			clkd = round_to_f32<false>(__dadd_rn(clkd, -THR));

			/* matched filter (msk.c:103-107): 11 taps out of the x12 oversampled half cosine.
			 * Phase index o = (int)(12*(MskClk/s + 0.5)): with inv_s good to 1e-15 the product gives
			 * the value to ~1e-14; only when that lands within 1e-9 of an integer (where the
			 * truncation could differ) is the reference's exact division sequence replayed. */
			double u = fma(__dmul_rn(clkd, inv_s), 12.0, 6.0);
			if (fabs(u - rint(u)) < 1e-9) u = __dmul_rn(12.0, __dadd_rn(__ddiv_rn(clkd, sv), 0.5));
			int o = __double2int_rz(u);
			o = min(max(o, 0), MFLTOVER);
			float vr = 0.f, vi = 0.f;
			const float *hp = s_h + o;
			int kk = r.idx;
#pragma unroll
			for (int j = 0; j < FLEN; j++) {
				const float hh = hp[MFLTOVER * j];
				vr = __fadd_rn(vr, __fmul_rn(hh, s_re[kk][grp]));
				vi = __fadd_rn(vi, __fmul_rn(hh, s_im[kk][grp]));
				kk = (kk + 1 == FLEN) ? 0 : kk + 1;
			}
			/* normalise (msk.c:110-113) */
			const float lvl = envelope(make_float2(vr, vi));
			const double d = __dadd_rn((double)lvl, 1e-8);
			vr = __double2float_rn(__ddiv_rn((double)vr, d));
			vi = __double2float_rn(__ddiv_rn((double)vi, d));
			r.lvlsum = __dadd_rn(r.lvlsum, (double)__fmul_rn(__fmul_rn(lvl, lvl), 0.25f));
			r.bitcount++;

			/* decision + phase error (msk.c:115-127) */
			float vo;
			double dphi;
			if (r.S & 1u) { vo = vi; dphi = (vo >= 0.f) ? (double)(-vr) : (double)vr; }
			else          { vo = vr; dphi = (vo >= 0.f) ? (double)vi : (double)(-vi); }
			const float bitv = (r.S & 2u) ? -vo : vo;

			/* putbit (msk.c:53-63) */
			r.outbits >>= 1;
			if (bitv > 0.f) r.outbits |= 0x80u;
			if (--r.nbits <= 0) frame_byte(acc, (unsigned char)r.outbits);
			r.S++;

			/* PLL filter (msk.c:130) — after putbit, so a frame resync's MskDf=0 is filtered too */
			r.df = __dadd_rn(__dmul_rn(PLLC, r.df), __dmul_rn(PLLK, dphi));
		}
		n += cnt;
	}
	if (!leader) return;
	r.pos = pos0 + (unsigned long long)nsamp;
	r.clk = (float)clkd;

	st->phi = r.phi; st->df = r.df; st->lvlsum = r.lvlsum; st->clk = r.clk; st->bitcount = r.bitcount;
	st->S = r.S; st->idx = r.idx; st->nbits = r.nbits; st->state = r.state; st->outbits = r.outbits;
	st->blk_len = r.blk_len; st->blk_err = r.blk_err; st->pos = r.pos; st->soh_pos = r.soh_pos;
#pragma unroll
	for (int k = 0; k < FLEN; k++) { st->inb_re[k] = s_re[k][grp]; st->inb_im[k] = s_im[k][grp]; }
}

/* K2, current form: the loop lives in demod_core.h (shared with the CPU tests' single-lane emulation).
 * One warp per CTA so chains spread over all SMs; L lanes per channel, 32/L channels per warp; state in
 * registers across the whole launch, ring and tables in shared memory, state written back at the end
 * (channel_t's role between demodMSK calls, msk.c:71-72, 134-135). */
struct WarpEnv {
	static __device__ __forceinline__ bool any(bool x) { return __any_sync(0xffffffffu, x) != 0; }
	static __device__ __forceinline__ bool all(bool x) { return __all_sync(0xffffffffu, x) != 0; }
	static __device__ __forceinline__ void sync() { __syncwarp(); }
	static __device__ __forceinline__ int max(int x) { return __reduce_max_sync(0xffffffffu, x); }
};

__device__ DcF4 g_h2[MFLTOVER + 1][3];           /* matched filter, transposed: g_h2[o] = h[o + 12 j] (msk.c:104-107) */

int upload_matched_filter(const float *h, cudaStream_t stream)
{
	float t[MFLTOVER + 1][12];
	for (int o = 0; o <= MFLTOVER; o++)
		for (int j = 0; j < 12; j++) t[o][j] = j < FLEN ? h[o + MFLTOVER * j] : 0.f;
	cudaError_t e = cudaMemcpyToSymbolAsync(c_h, h, sizeof(float) * FLENO, 0, cudaMemcpyHostToDevice, stream);
	if (e != cudaSuccess) return (int)e;
	e = cudaMemcpyToSymbolAsync(g_h2, t, sizeof(t), 0, cudaMemcpyHostToDevice, stream);
	if (e != cudaSuccess) return (int)e;
	return (int)cudaStreamSynchronize(stream);
}

/* K2's body, shared by k_demod2 and its counting form k_demod2_stats (STATS: the frame synchroniser's events go to
 * counts[chain * EV_COUNT + e]; k_demod2 passes none and never sees the hook) */
template <int L, bool F2F, bool PIN, bool STATS, bool RAGGED = false>
__device__ __forceinline__ void demod2_body(DemodShared<32 / L> &sm, ChainState *__restrict__ states, const float *__restrict__ dm,
                                            int nsamp, int nch, int nstreams, RawFrame *__restrict__ ring,
                                            RingCtl *__restrict__ ctl, unsigned cap, unsigned *__restrict__ counts,
                                            const int *__restrict__ nrows = nullptr)
{
	constexpr int CPW = 32 / L;                  /* channels per warp */
	const int lane = threadIdx.x;
	for (int i = lane; i < 64; i += 32) {
		sm.tcos[i].x = g_sc_cos[i].x; sm.tcos[i].y = g_sc_cos[i].y;
		sm.tsin[i].x = g_sc_sin[i].x; sm.tsin[i].y = g_sc_sin[i].y;
	}
	for (int i = lane; i < (MFLTOVER + 1) * 3; i += 32) (&sm.h2[0][0])[i] = (&g_h2[0][0])[i];

	const int grp = lane / L, sub = lane % L;
	/* chains (stream, channel) are numbered stream-major and dealt CPW to a warp, across stream boundaries: a
	 * warp of 32 single-lane chains serves four 8-channel streams */
	const long long nchain = (long long)nstreams * nch;
	const long long g_raw = (long long)blockIdx.x * CPW + grp;
	const bool valid = g_raw < nchain;               /* surplus groups of the last warp shadow the last chain, silently */
	const long long g = valid ? g_raw : nchain - 1;
	const int s = (int)(g / nch), ch = (int)(g - (long long)s * nch);
	const bool leader = valid && sub == 0;

	ChainState *st = states + (size_t)s * nch + ch;
	DemodRegs r;
	r.phi = st->phi; r.df = st->df; r.lvlsum = st->lvlsum; r.clk = st->clk; r.bitcount = st->bitcount;
	r.S = st->S; r.idx = st->idx; r.nbits = st->nbits; r.state = st->state; r.outbits = st->outbits;
	r.blk_len = st->blk_len; r.blk_err = st->blk_err; r.pos = st->pos; r.soh_pos = st->soh_pos;
	for (int k = sub; k < FLEN; k += L) {
		DcF2 v;
		v.x = st->inb_re[k]; v.y = st->inb_im[k];
		sm.ring[k][grp] = v;
		sm.ring[k + FLEN][grp] = v;
	}
	__syncwarp();

	/* RAGGED: stream s has nrows[s] rows of its own; the envelope keeps the launch's nsamp rows per stream */
	const int n_s = RAGGED ? nrows[s] : nsamp;
	if constexpr (STATS) {
		DevFrameAccStats acc{ { r, st, ring, ctl, cap, s, ch, leader, true }, counts + (size_t)g * EV_COUNT };
		demod_run<L, F2F, PIN, WarpEnv, RAGGED>(r, sm, dm + (size_t)s * nsamp * nch + ch, nch, n_s, sub, grp, acc);
	} else {
		DevFrameAcc acc{ r, st, ring, ctl, cap, s, ch, leader, true };
		demod_run<L, F2F, PIN, WarpEnv, RAGGED>(r, sm, dm + (size_t)s * nsamp * nch + ch, nch, n_s, sub, grp, acc);
	}

	if (!leader) return;
	st->phi = r.phi; st->df = r.df; st->lvlsum = r.lvlsum; st->clk = r.clk; st->bitcount = r.bitcount;
	st->S = r.S; st->idx = r.idx; st->nbits = r.nbits; st->state = r.state; st->outbits = r.outbits;
	st->blk_len = r.blk_len; st->blk_err = r.blk_err; st->pos = r.pos; st->soh_pos = r.soh_pos;
#pragma unroll
	for (int k = 0; k < FLEN; k++) { st->inb_re[k] = sm.ring[k][grp].x; st->inb_im[k] = sm.ring[k][grp].y; }
}

template <int L, bool F2F, bool PIN, int MINB = 1>     /* MINB = 0: no occupancy request */
__global__ void __launch_bounds__(32, MINB)
k_demod2(ChainState *__restrict__ states, const float *__restrict__ dm, int nsamp, int nch, int nstreams,
         int wps, RawFrame *__restrict__ ring, RingCtl *__restrict__ ctl, unsigned cap)
{
	__shared__ DemodShared<32 / L> sm;
	(void)wps;
	demod2_body<L, F2F, PIN, false>(sm, states, dm, nsamp, nch, nstreams, ring, ctl, cap, nullptr);
}

/* the counting form (ACB_FLAG_DECODE_STATS): the same launch geometry, launch bounds and shared memory */
template <int L, bool F2F, bool PIN, int MINB = 1>
__global__ void __launch_bounds__(32, MINB)
k_demod2_stats(ChainState *__restrict__ states, const float *__restrict__ dm, int nsamp, int nch, int nstreams,
               RawFrame *__restrict__ ring, RingCtl *__restrict__ ctl, unsigned cap, unsigned *__restrict__ counts)
{
	__shared__ DemodShared<32 / L> sm;
	demod2_body<L, F2F, PIN, true>(sm, states, dm, nsamp, nch, nstreams, ring, ctl, cap, counts);
}

/* The ragged forms (submits whose streams carry different row counts): stream s demodulates nrows[s] of the nsamp rows
 * each stream has in the envelope; the same launch geometry, launch bounds and shared memory as the even forms */
template <int L, bool F2F, bool PIN, int MINB = 1>
__global__ void __launch_bounds__(32, MINB)
k_demod2_ragged(ChainState *__restrict__ states, const float *__restrict__ dm, int nsamp, int nch, int nstreams,
                RawFrame *__restrict__ ring, RingCtl *__restrict__ ctl, unsigned cap, const int *__restrict__ nrows)
{
	__shared__ DemodShared<32 / L> sm;
	demod2_body<L, F2F, PIN, false, true>(sm, states, dm, nsamp, nch, nstreams, ring, ctl, cap, nullptr, nrows);
}

template <int L, bool F2F, bool PIN, int MINB = 1>
__global__ void __launch_bounds__(32, MINB)
k_demod2_stats_ragged(ChainState *__restrict__ states, const float *__restrict__ dm, int nsamp, int nch, int nstreams,
                      RawFrame *__restrict__ ring, RingCtl *__restrict__ ctl, unsigned cap, unsigned *__restrict__ counts,
                      const int *__restrict__ nrows)
{
	__shared__ DemodShared<32 / L> sm;
	demod2_body<L, F2F, PIN, true, true>(sm, states, dm, nsamp, nch, nstreams, ring, ctl, cap, counts, nrows);
}

/* SM count and shared memory per SM of the current device, asked per launch: contexts of one process may sit on
 * different devices */
static void demod_sm_limits(int &sm_count, int &smem_per_sm)
{
	int dev = 0;
	sm_count = smem_per_sm = 0;
	if (cudaGetDevice(&dev) == cudaSuccess) {
		cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, dev);
		cudaDeviceGetAttribute(&smem_per_sm, cudaDevAttrMaxSharedMemoryPerMultiprocessor, dev);
	}
	if (sm_count <= 0) sm_count = 132;
	if (smem_per_sm <= 0) smem_per_sm = 228 * 1024;
}

/* Residency budget of K2 beside the exact IQ channelizer (tools/residency_budget.py prints it from the built library,
 * tests/test_residency_budget.py holds it).  The demod of submit i runs underneath the channelizer of submit i+1, on a
 * stream of greater priority (context.cu): a K2 CTA that fits is dispatched before the next K1 CTA.
 *   registers: k_channelize_iq4 allocates 160 x 128 = 20 480 per CTA, three CTAs leave 4 096 of the SM's 65 536.  One
 *              retired K1 CTA plus that spare is 24 576: six one-warp K2 CTAs at 128 registers per thread, eight (the
 *              share of an SM at 4224 streams x 8 channels) at 96 — hence launch_demod_one_lane's capped form.
 *   shared:    K2 8 304 B (one lane per chain) + 1 KB reserved per CTA; K1 4 KB + 1 KB.
 * K2 asks for the smallest shared-memory configuration that holds its CTAs of one SM (at most 16: the registers allow
 * no more) beside three K1 CTAs — 100 KB for eight — and leaves the rest to L1, as K1 does (launch_channelize_iq4).  The
 * envelope K2 reads comes through L1: asking for the largest carve-out (28 KB of L1) made it 1.1x slower alone (2.58
 * against 2.33 ms, H100 SXM 700 W, 4224 streams x 8 blocks) and the pipelined step 3 % slower (15.9 against 15.5 ms); a
 * configuration too small for its CTAs (64 KB: six fit) made it 1.6x slower alone.
 * Launches of fewer than four warps per SM (not one per scheduler) keep the largest carve-out: there K2's serial chain is
 * the whole step and K1 is small, and a K1 that runs faster beside it only takes issue slots from it (one stream of 256
 * channels, K = 1600, 513 taps: K1 0.21 instead of 0.28 ms, K2 0.67 instead of 0.58 ms, the step 15 % slower). */
constexpr int DEMOD_SMEM_RESERVED = 1024;                       /* per CTA, the system's */
constexpr int DEMOD_SMEM_BESIDE = 3 * (4096 + DEMOD_SMEM_RESERVED);   /* three k_channelize_iq4<u8> CTAs */
constexpr int DEMOD_MAX_WARPS_PER_SM = 16;
constexpr int DEMOD_MIN_WARPS_SHARING = 4;                      /* per SM: below, K2 is the step and keeps the largest carve-out */

template <int LANES, bool F2F, bool PIN, int MINB = 1, bool STATS = false, bool RAGGED = false>
static int launch_demod_t(ChainState *st, const float *dm, int nsamp, int nch, int nstreams,
                          RawFrame *ring, RingCtl *ctl, unsigned cap, cudaStream_t stream, unsigned *counts = nullptr,
                          const int *nrows = nullptr)
{
	constexpr int CPW = 32 / LANES;
	const int wps = (nch + CPW - 1) / CPW;
	const long long nchain = (long long)nstreams * nch;
	const int grid = (int)((nchain + CPW - 1) / CPW);    /* one warp per CTA so that chains spread over all SMs */
	int sm_count, smem_per_sm;
	demod_sm_limits(sm_count, smem_per_sm);
	const long long per_sm = std::min<long long>((grid + sm_count - 1) / sm_count, DEMOD_MAX_WARPS_PER_SM);
	const long long need = per_sm * ((long long)sizeof(DemodShared<CPW>) + DEMOD_SMEM_RESERVED) + DEMOD_SMEM_BESIDE;
	const int carve = per_sm < DEMOD_MIN_WARPS_SHARING ? (int)cudaSharedmemCarveoutMaxShared
	                                                   : (int)std::min<long long>(100, (need * 100 + smem_per_sm - 1) / smem_per_sm);
	if constexpr (RAGGED && STATS) {
		cudaError_t e = cudaFuncSetAttribute(k_demod2_stats_ragged<LANES, F2F, PIN, MINB>, cudaFuncAttributePreferredSharedMemoryCarveout, carve);
		if (e != cudaSuccess) return (int)e;
		k_demod2_stats_ragged<LANES, F2F, PIN, MINB><<<grid, 32, 0, stream>>>(st, dm, nsamp, nch, nstreams, ring, ctl, cap, counts, nrows);
		return (int)cudaGetLastError();
	} else if constexpr (RAGGED) {
		cudaError_t e = cudaFuncSetAttribute(k_demod2_ragged<LANES, F2F, PIN, MINB>, cudaFuncAttributePreferredSharedMemoryCarveout, carve);
		if (e != cudaSuccess) return (int)e;
		k_demod2_ragged<LANES, F2F, PIN, MINB><<<grid, 32, 0, stream>>>(st, dm, nsamp, nch, nstreams, ring, ctl, cap, nrows);
		return (int)cudaGetLastError();
	}
	if constexpr (STATS) {
		cudaError_t e = cudaFuncSetAttribute(k_demod2_stats<LANES, F2F, PIN, MINB>, cudaFuncAttributePreferredSharedMemoryCarveout, carve);
		if (e != cudaSuccess) return (int)e;
		k_demod2_stats<LANES, F2F, PIN, MINB><<<grid, 32, 0, stream>>>(st, dm, nsamp, nch, nstreams, ring, ctl, cap, counts);
		return (int)cudaGetLastError();
	}
	cudaError_t e = cudaFuncSetAttribute(k_demod2<LANES, F2F, PIN, MINB>, cudaFuncAttributePreferredSharedMemoryCarveout, carve);
	if (e != cudaSuccess) return (int)e;
	k_demod2<LANES, F2F, PIN, MINB><<<grid, 32, 0, stream>>>(st, dm, nsamp, nch, nstreams, wps, ring, ctl, cap);
	return (int)cudaGetLastError();
}

/* The pinned forms (2, 4, 8 lanes) in two register budgets.  Told that one CTA per SM is all it asks for
 * (__launch_bounds__(32, 1)), ptxas spends more registers on a wider schedule: fewer instructions where the kernel is
 * latency bound, but fewer warps per SM where it is not.  So: the wide schedule while there are at most 8 warps per SM,
 * the lean one beyond. */
template <int LANES, bool F2F, bool STATS = false, bool RAGGED = false>
static int launch_demod_pinned(ChainState *st, const float *dm, int nsamp, int nch, int nstreams,
                               RawFrame *ring, RingCtl *ctl, unsigned cap, cudaStream_t stream, unsigned *counts = nullptr,
                               const int *nrows = nullptr)
{
	int sm_count, smem_per_sm;
	demod_sm_limits(sm_count, smem_per_sm);
	const long long warps = ((long long)nstreams * nch * LANES + 31) / 32;
	return warps <= 8LL * sm_count
	           ? launch_demod_t<LANES, F2F, true, 1, STATS, RAGGED>(st, dm, nsamp, nch, nstreams, ring, ctl, cap, stream, counts, nrows)
	           : launch_demod_t<LANES, F2F, true, 0, STATS, RAGGED>(st, dm, nsamp, nch, nstreams, ring, ctl, cap, stream, counts, nrows);
}

/* The one-lane form in two register budgets.  Left alone ptxas takes 128 registers per thread; of those CTAs six fit
 * into the registers one retired K1 CTA frees (launch_demod_t), so with more than six warps per SM the rest wait for a
 * second K1 CTA to retire and K1 is left with one CTA of its three on that SM meanwhile.  __launch_bounds__(32, 20)
 * caps the kernel at 96 registers (no spills): eight fit.  Alone it is 4 % slower (2.43 against 2.33 ms), under K1 the
 * step is 1 % faster (15.31 against 15.48-15.60 ms, three alternated runs each, same card and shape as above). */
constexpr int DEMOD_MINB_96REG = 20;
constexpr int DEMOD_WARPS_PER_K1_CTA = 6;

template <bool STATS = false, bool RAGGED = false>
static int launch_demod_one_lane(ChainState *st, const float *dm, int nsamp, int nch, int nstreams,
                                 RawFrame *ring, RingCtl *ctl, unsigned cap, cudaStream_t stream, unsigned *counts = nullptr,
                                 const int *nrows = nullptr)
{
	int sm_count, smem_per_sm;
	demod_sm_limits(sm_count, smem_per_sm);
	const long long warps = ((long long)nstreams * nch + 31) / 32;
	return warps <= (long long)DEMOD_WARPS_PER_K1_CTA * sm_count
	           ? launch_demod_t<1, false, false, 1, STATS, RAGGED>(st, dm, nsamp, nch, nstreams, ring, ctl, cap, stream, counts, nrows)
	           : launch_demod_t<1, false, false, DEMOD_MINB_96REG, STATS, RAGGED>(st, dm, nsamp, nch, nstreams, ring, ctl, cap, stream, counts,
	                                                                              nrows);
}

template <int LANES>
static int launch_demod_v1(ChainState *st, const float *dm, int nsamp, int nch, int nstreams,
                           RawFrame *ring, RingCtl *ctl, unsigned cap, cudaStream_t stream)
{
	constexpr int CPW = 32 / LANES;
	const int wps = (nch + CPW - 1) / CPW;
	cudaError_t e = cudaFuncSetAttribute(k_demod<LANES>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
	if (e != cudaSuccess) return (int)e;
	k_demod<LANES><<<nstreams * wps, 32, 0, stream>>>(st, dm, nsamp, nch, nstreams, wps, ring, ctl, cap);
	return (int)cudaGetLastError();
}

/* Lanes per channel.  Every lane of a channel's group repeats the serial part of a bit period and the group
 * only splits the six mixer evaluations, so fewer lanes = fewer instructions per channel; more lanes = a
 * shorter chain per bit.  The kernel is latency bound until there are several warps per scheduler, so: the
 * most lanes that still leave about one warp per SM sub-partition, the fewest once the chains alone fill
 * the machine. */
int demod_pick_lanes(long long nchains, int sm_count)
{
	/* the fewest lanes that still put a warp on every scheduler (tools/ab_demod.py sweeps the alternatives) */
	const long long slots = 4LL * sm_count;      /* one warp per scheduler */
	for (int lanes = 1; lanes < 8; lanes *= 2)
		if (nchains * lanes >= 32 * slots) return lanes;
	return 8;
}

/* lanes: 1, 2, 4 or 8 lanes per channel, each in its A/B-chosen form: loop constants pinned in registers for 2, 4, 8
 * lanes, not pinned for 1 lane; + 32 = the other choice; + 16 = bit clock rounded
 * with the F2F conversion pair instead of integer ops (round_to_f32); negative (-4, -8) = the round-1 kernel, kept for
 * A/B runs */
int launch_demod(ChainState *st, const float *dm, int nsamp, int nch, int nstreams,
                 RawFrame *ring, RingCtl *ctl, unsigned cap, int lanes, cudaStream_t stream, const int *nrows)
{
	if (nrows) {                 /* the ragged forms of the default widths only */
#define ACB_DEMOD_ARGS st, dm, nsamp, nch, nstreams, ring, ctl, cap, stream, nullptr, nrows
		switch (lanes) {
		case 8: return launch_demod_pinned<8, false, false, true>(ACB_DEMOD_ARGS);
		case 4: return launch_demod_pinned<4, false, false, true>(ACB_DEMOD_ARGS);
		case 2: return launch_demod_pinned<2, false, false, true>(ACB_DEMOD_ARGS);
		case 1: return launch_demod_one_lane<false, true>(ACB_DEMOD_ARGS);
		default: return (int)cudaErrorInvalidValue;
		}
#undef ACB_DEMOD_ARGS
	}
#define ACB_DEMOD_ARGS st, dm, nsamp, nch, nstreams, ring, ctl, cap, stream
	switch (lanes) {
	case -8: return launch_demod_v1<8>(ACB_DEMOD_ARGS);
	case -4: return launch_demod_v1<4>(ACB_DEMOD_ARGS);
	case 8: return launch_demod_pinned<8, false>(ACB_DEMOD_ARGS);
	case 2: return launch_demod_pinned<2, false>(ACB_DEMOD_ARGS);
	case 1: return launch_demod_one_lane<>(ACB_DEMOD_ARGS);
	case 17: return launch_demod_t<1, true, false>(ACB_DEMOD_ARGS);          /* F2F bit clock at one lane */
	case 24: return launch_demod_pinned<8, true>(ACB_DEMOD_ARGS);
	case 20: return launch_demod_pinned<4, true>(ACB_DEMOD_ARGS);
	case 40: return launch_demod_t<8, false, false>(ACB_DEMOD_ARGS);
	case 36: return launch_demod_t<4, false, false>(ACB_DEMOD_ARGS);
	case 34: return launch_demod_t<2, false, false>(ACB_DEMOD_ARGS);
	case 33: return launch_demod_t<1, false, true>(ACB_DEMOD_ARGS);
	default: return launch_demod_pinned<4, false>(ACB_DEMOD_ARGS);
	}
#undef ACB_DEMOD_ARGS
}

/* the counting forms of the default widths (what launch_demod runs for lanes 1, 2, 4, 8), each in the same register
 * budgets and under the same carve-out rules */
int launch_demod_stats(ChainState *st, const float *dm, int nsamp, int nch, int nstreams,
                       RawFrame *ring, RingCtl *ctl, unsigned cap, int lanes, unsigned *counts, cudaStream_t stream, const int *nrows)
{
	if (nrows) {
#define ACB_DEMOD_ARGS st, dm, nsamp, nch, nstreams, ring, ctl, cap, stream, counts, nrows
		switch (lanes) {
		case 8: return launch_demod_pinned<8, false, true, true>(ACB_DEMOD_ARGS);
		case 4: return launch_demod_pinned<4, false, true, true>(ACB_DEMOD_ARGS);
		case 2: return launch_demod_pinned<2, false, true, true>(ACB_DEMOD_ARGS);
		case 1: return launch_demod_one_lane<true, true>(ACB_DEMOD_ARGS);
		default: return (int)cudaErrorInvalidValue;
		}
#undef ACB_DEMOD_ARGS
	}
#define ACB_DEMOD_ARGS st, dm, nsamp, nch, nstreams, ring, ctl, cap, stream, counts
	switch (lanes) {
	case 8: return launch_demod_pinned<8, false, true>(ACB_DEMOD_ARGS);
	case 4: return launch_demod_pinned<4, false, true>(ACB_DEMOD_ARGS);
	case 2: return launch_demod_pinned<2, false, true>(ACB_DEMOD_ARGS);
	case 1: return launch_demod_one_lane<true>(ACB_DEMOD_ARGS);
	default: return (int)cudaErrorInvalidValue;
	}
#undef ACB_DEMOD_ARGS
}

/* ------------------------------------------------------------------------------------------
 * K3: block FEC, one thread per finished frame (blk_thread, acars.c:123-207; fixprerr acars.c:39-64;
 * fixdberr acars.c:66-90).  Integer only.  Works in place on the frame ring right behind the demod:
 * status in RawFrame::pad0 (1 = deliver, 2 = drop), err = parity errors found, txt repaired and
 * parity-stripped.  CRC and syndrome tables are generated in shared memory per CTA (syndrom.h:15-48,
 * 52-295) rather than stored.
 * ---------------------------------------------------------------------------------------- */

constexpr int FEC_SYN_BYTES = 252;      /* covers len <= 250 (the reference table has 242 rows; a
                                           241-byte block indexes past it there, see hostmath.cpp) */

__device__ __forceinline__ unsigned fec_crc_step(const unsigned short *tab, unsigned crc, unsigned c)
{
	return ((crc >> 8) ^ tab[(crc ^ c) & 0xffu]) & 0xffffu;               /* update_crc, syndrom.h:49 */
}

__device__ __forceinline__ bool fec_crc_bytes_hit(const unsigned short *syn, unsigned crc)
{
	bool hit = false;
#pragma unroll
	for (int i = 0; i < 16; i++) hit |= (syn[i] == crc);                  /* acars.c:57-62, 70-74 */
	return hit;
}

/* K3's body, shared by k_block_fec and its counting form k_block_fec_stats (STATS: each frame's FEC_WHY_* also goes to
 * RawFrame::pad1[0], following blk_thread's control flow) */
template <bool STATS>
__device__ __forceinline__ void block_fec_body(unsigned short *s_crc, unsigned short *s_syn, RawFrame *__restrict__ ring,
                                               const RingCtl *__restrict__ ctl, unsigned cap)
{
	/* the grid is sized for the busiest step (one thread per frame up to 4 * SMs * 128 frames, 67 584 on a 132-SM H100,
	 * then a stride loop; tests/test_gpu_scale.py runs more than two passes); CTAs
	 * with no frame leave before building the tables */
	if (blockIdx.x * blockDim.x >= min(ctl->count, cap)) return;
	for (int b = threadIdx.x; b < 256; b += blockDim.x) {
		unsigned r = b;
		for (int k = 0; k < 8; k++) r = (r & 1u) ? (r >> 1) ^ 0x8408u : r >> 1;
		s_crc[b] = (unsigned short)r;
	}
	__syncthreads();
	if (threadIdx.x < 8) {                                                /* one bit position per thread */
		unsigned r = s_crc[1u << threadIdx.x];
		for (int p = 0; p < FEC_SYN_BYTES; p++) {
			s_syn[threadIdx.x + 8 * p] = (unsigned short)r;
			r = fec_crc_step(s_crc, r, 0);
		}
	}
	__syncthreads();

	const unsigned count = min(ctl->count, cap);
	for (unsigned f = blockIdx.x * blockDim.x + threadIdx.x; f < count; f += gridDim.x * blockDim.x) {
		RawFrame *fr = ring + f;
		unsigned char *txt = fr->txt;
		const int len = fr->len;
		int status = 2;
		unsigned why = 0;
		do {
			if (len < 13 || len > 250) { why = FEC_WHY_SHORT; break; }        /* acars.c:124-129 */
			txt[12] = (unsigned char)((txt[12] & 0x83u) | 0x02u);             /* force STX/ETX, acars.c:132-133 */
			int bad[3], nbad = 0;
			unsigned crc = 0;
			for (int i = 0; i < len; i++) {
				const unsigned c = txt[i];
				if ((__popc(c) & 1) == 0) { if (nbad < 3) bad[nbad] = i; nbad++; }
				crc = fec_crc_step(s_crc, crc, c);
			}
			if (nbad > 3) { why = FEC_WHY_PARITY_EXCESS; break; }             /* acars.c:145-152 */
			crc = fec_crc_step(s_crc, crc, fr->crc[0]);
			crc = fec_crc_step(s_crc, crc, fr->crc[1]);
			fr->err = nbad;
			why = (nbad ? FEC_WHY_PARITY : 0u) | (crc ? FEC_WHY_CRC : 0u);      /* acars.c:153-155, 166-167 */
			bool ok = true;
			if (nbad) {
				/* fixprerr, depth first in the reference's order: bit of the first bad byte outermost */
				ok = false;
				const int p0 = 8 * (len - bad[0] + 1), p1 = nbad > 1 ? 8 * (len - bad[1] + 1) : 0, p2 = nbad > 2 ? 8 * (len - bad[2] + 1) : 0;
				for (int i0 = 0; i0 < 8 && !ok; i0++) {
					const unsigned c0 = crc ^ s_syn[i0 + p0];
					if (nbad == 1) {
						if (c0 == 0 || fec_crc_bytes_hit(s_syn, c0)) { txt[bad[0]] ^= (unsigned char)(1u << i0); ok = true; }
						continue;
					}
					for (int i1 = 0; i1 < 8 && !ok; i1++) {
						const unsigned c1 = c0 ^ s_syn[i1 + p1];
						if (nbad == 2) {
							if (c1 == 0 || fec_crc_bytes_hit(s_syn, c1)) {
								txt[bad[1]] ^= (unsigned char)(1u << i1); txt[bad[0]] ^= (unsigned char)(1u << i0); ok = true;
							}
							continue;
						}
						for (int i2 = 0; i2 < 8 && !ok; i2++) {
							const unsigned c2 = c1 ^ s_syn[i2 + p2];
							if (c2 == 0 || fec_crc_bytes_hit(s_syn, c2)) {
								txt[bad[2]] ^= (unsigned char)(1u << i2); txt[bad[1]] ^= (unsigned char)(1u << i1);
								txt[bad[0]] ^= (unsigned char)(1u << i0); ok = true;
							}
						}
					}
				}
			} else if (crc) {
				/* fixdberr: single wrong bit in the BCS, else two wrong bits in one byte */
				ok = fec_crc_bytes_hit(s_syn, crc);
				for (int k = 0; k < len && !ok; k++) {
					const int base = 8 * (len - k + 1);
					for (int i = 0; i < 8 && !ok; i++)
						for (int j = 0; j < 8 && !ok; j++)
							if (i != j && (crc ^ s_syn[i + base] ^ s_syn[j + base]) == 0) {
								txt[k] ^= (unsigned char)((1u << i) | (1u << j));
								ok = true;
							}
				}
			}
			if (!ok) { why |= FEC_WHY_UNFIXABLE; break; }                     /* acars.c:171-175, 183-187 */
			if (nbad || crc) why |= FEC_WHY_FIXED;                            /* acars.c:177-178, 189-190 */
			int still = 0;                                                    /* acars.c:194-207 */
			for (int i = 0; i < len; i++) {
				const unsigned c = txt[i];
				still += ((__popc(c) & 1) == 0);
				txt[i] = (unsigned char)(c & 0x7fu);
			}
			status = still ? 2 : 1;
			if (still) why |= FEC_WHY_PARITY_PROBLEM;
		} while (0);
		fr->pad0 = status;
		if (STATS) fr->pad1[0] = (unsigned char)why;
	}
}

__global__ void __launch_bounds__(128)
k_block_fec(RawFrame *__restrict__ ring, const RingCtl *__restrict__ ctl, unsigned cap)
{
	__shared__ unsigned short s_crc[256];
	__shared__ unsigned short s_syn[8 * FEC_SYN_BYTES];
	block_fec_body<false>(s_crc, s_syn, ring, ctl, cap);
}

__global__ void __launch_bounds__(128)
k_block_fec_stats(RawFrame *__restrict__ ring, const RingCtl *__restrict__ ctl, unsigned cap)
{
	__shared__ unsigned short s_crc[256];
	__shared__ unsigned short s_syn[8 * FEC_SYN_BYTES];
	block_fec_body<true>(s_crc, s_syn, ring, ctl, cap);
}

int launch_block_fec(RawFrame *ring, const RingCtl *ctl, unsigned cap, cudaStream_t stream)
{
	int dev = 0, sm_count = 0;               /* grid-stride over the frames: 4 CTAs per SM of the device it runs on */
	if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sm_count <= 0)
		sm_count = 132;
	k_block_fec<<<4 * sm_count, 128, 0, stream>>>(ring, ctl, cap);
	return (int)cudaGetLastError();
}

int launch_block_fec_stats(RawFrame *ring, const RingCtl *ctl, unsigned cap, cudaStream_t stream)
{
	int dev = 0, sm_count = 0;
	if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sm_count <= 0)
		sm_count = 132;
	k_block_fec_stats<<<4 * sm_count, 128, 0, stream>>>(ring, ctl, cap);
	return (int)cudaGetLastError();
}

/* ---- ACB_FLAG_LEVEL_STATS: input and envelope levels (launch_level_input, launch_level_dm) ----
 * Memory-bound reductions over what a submit already holds.  Integer counts and sums are exact in any order; the float64
 * sums are made in a fixed order (each thread in address order, then fixed trees, then the partials in chunk / window
 * order), so the same input with the same cuts gives the same bits.  No floating-point atomics. */
constexpr int LVL_THREADS = 256;

/* one thread's share of a chunk of input words (4 bytes: two u8 samples, one CS16 sample or one real sample) */
template <int KIND> struct LevelAcc {
	unsigned clip = 0;
	unsigned long long m1 = 0, m2 = 0;            /* u8: sum of the bytes, of their squares; CS16: -, sum of I^2 + Q^2 */
	double p = 0.0;                               /* real: sum of x^2 */
	unsigned hi = 0, lo = 0xffffffffu;            /* u8: per-byte max / min; CS16: hi = largest |component| */
	float pk = 0.0f;                              /* real: largest |x| */
	__device__ __forceinline__ void add(unsigned w)
	{
		if (KIND == IN_U8IQ) {
			/* a thread sees at most 8 * 4 words per chunk: the byte sums stay far below 2^32 */
			m1 = __dp4a(w, 0x01010101u, (unsigned)m1);
			m2 = __dp4a(w, w, (unsigned)m2);
			/* a byte is 0 or 255 exactly when its 8 bits are equal: b ^ (b >> 1) has no bit set in 0..6 */
			const unsigned u = (w ^ (w >> 1)) & 0x7f7f7f7fu, z = ~((u + 0x7f7f7f7fu) | u) & 0x80808080u;
			clip += ((z & 0x00008080u) != 0) + ((z & 0x80800000u) != 0);
			hi = __vmaxu4(hi, w);
			lo = __vminu4(lo, w);
		} else if (KIND == IN_CS16IQ) {
			const int i = (int)(short)(w & 0xffffu), q = (int)w >> 16;
			m2 += (unsigned)(i * i) + (unsigned)(q * q);
			clip += (i == -32768) | (i == 32767) | (q == -32768) | (q == 32767);
			hi = max(hi, (unsigned)max(abs(i), abs(q)));
		} else {
			const float x = __uint_as_float(w);
			const double xd = (double)x;
			p = __dadd_rn(p, __dmul_rn(xd, xd));
			clip += (x <= -1.0f) | (x >= 2047.0f / 2048.0f);
			pk = fmaxf(pk, fabsf(x));
		}
	}
	__device__ __forceinline__ LevelPart part() const
	{
		LevelPart r;
		r.clipped = clip;
		r.m1 = m1;
		r.m2 = KIND == IN_F32REAL ? (unsigned long long)__double_as_longlong(p) : m2;
		if (KIND == IN_U8IQ) {
			unsigned bmax = 0, bmin = 255;
			for (int k = 0; k < 4; k++) bmax = max(bmax, (hi >> (8 * k)) & 0xffu), bmin = min(bmin, (lo >> (8 * k)) & 0xffu);
			/* |(float)b - 127.37f| is exact: the difference of the two floats has at most 24 significant bits */
			r.peak = fmaxf(0.0f, fmaxf((float)bmax - 127.37f, 127.37f - (float)bmin));
		} else {
			r.peak = KIND == IN_CS16IQ ? (float)hi : pk;
		}
		r.pad = 0;
		return r;
	}
};

/* partials a, b into a (integers add exactly; the real kind's float64 sum in m2's bits) */
template <int KIND> __device__ __forceinline__ void level_merge(LevelPart &a, const LevelPart &b)
{
	a.clipped += b.clipped;
	a.m1 += b.m1;
	a.m2 = KIND == IN_F32REAL ? (unsigned long long)__double_as_longlong(__dadd_rn(__longlong_as_double((long long)a.m2),
	                                                                               __longlong_as_double((long long)b.m2)))
	                          : a.m2 + b.m2;
	a.peak = fmaxf(a.peak, b.peak);
}

template <int KIND> __device__ __forceinline__ void level_shfl_merge(LevelPart &v, int lane_mask)
{
	LevelPart o;
	o.clipped = __shfl_xor_sync(0xffffffffu, v.clipped, lane_mask);
	o.m1 = __shfl_xor_sync(0xffffffffu, v.m1, lane_mask);
	o.m2 = __shfl_xor_sync(0xffffffffu, v.m2, lane_mask);
	o.peak = __shfl_xor_sync(0xffffffffu, v.peak, lane_mask);
	level_merge<KIND>(v, o);                      /* the butterfly adds the same two values in every lane: a + b == b + a */
}

/* bytes of input per sample (u8: I, Q bytes; CS16: I, Q int16; real: one float) */
template <int KIND> __host__ __device__ constexpr int level_sample_bytes() { return KIND == IN_U8IQ ? 2 : 4; }

/* grid (chunk, stream): stream s's rows*K samples at in + s*stride, LVL_CHUNK bytes per CTA, 16-byte loads (the rows start
 * 16-byte aligned; a streaming kind's last few words, when rows*K is not a multiple of 4, go one by one) */
template <int KIND>
__global__ void __launch_bounds__(LVL_THREADS)
k_level_in(const uint8_t *__restrict__ in, size_t stride, int K, int nrows, const int *__restrict__ rows, LevelPart *__restrict__ part,
           size_t part_stride)
{
	const int s = blockIdx.y;
	const size_t bytes = (size_t)(rows ? rows[s] : nrows) * K * level_sample_bytes<KIND>();
	const size_t c0 = (size_t)blockIdx.x * LVL_CHUNK;
	if (c0 >= bytes) return;
	const size_t c1 = min(bytes, c0 + LVL_CHUNK);
	const uint8_t *base = in + (size_t)s * stride;
	LevelAcc<KIND> a;
	const size_t v1 = c0 + (c1 - c0) / 16 * 16;
#pragma unroll 4
	for (size_t o = c0 + 16 * (size_t)threadIdx.x; o < v1; o += 16 * LVL_THREADS) {
		const uint4 w = __ldcs(reinterpret_cast<const uint4 *>(base + o));       /* read once: do not keep it in L2 */
		a.add(w.x); a.add(w.y); a.add(w.z); a.add(w.w);
	}
	for (size_t o = v1 + 4 * (size_t)threadIdx.x; o < c1; o += 4 * LVL_THREADS) a.add(*reinterpret_cast<const unsigned *>(base + o));
	LevelPart v = a.part();
	for (int m = 16; m; m >>= 1) level_shfl_merge<KIND>(v, m);
	__shared__ LevelPart s_w[LVL_THREADS / 32];
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	if (lane == 0) s_w[warp] = v;
	__syncthreads();
	if (warp == 0) {
		v = s_w[lane < LVL_THREADS / 32 ? lane : 0];
		if (lane >= LVL_THREADS / 32) v = LevelPart{ 0, 0, 0, 0.0f, 0 };   /* the real kind's +0.0 has all bits zero */
		for (int m = 16; m; m >>= 1) level_shfl_merge<KIND>(v, m);
		if (lane == 0) part[(size_t)s * part_stride + blockIdx.x] = v;
	}
}

/* one warp per stream: its chunks' partials in a fixed order (lane l takes chunks l, l + 32, ..., then a butterfly) */
template <int KIND>
__global__ void __launch_bounds__(256)
k_level_in_fin(int K, int nrows, const int *__restrict__ rows, int nstreams, const LevelPart *__restrict__ part, size_t part_stride,
               LevelIn *__restrict__ out)
{
	const int s = (int)((blockIdx.x * (size_t)blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
	if (s >= nstreams) return;
	const unsigned long long samples = (unsigned long long)(rows ? rows[s] : nrows) * (unsigned long long)K;
	const size_t nchunk = (samples * level_sample_bytes<KIND>() + LVL_CHUNK - 1) / LVL_CHUNK;
	LevelPart v{ 0, 0, 0, 0.0f, 0 };
	for (size_t j = lane; j < nchunk; j += 32) level_merge<KIND>(v, part[(size_t)s * part_stride + j]);
	for (int m = 16; m; m >>= 1) level_shfl_merge<KIND>(v, m);
	if (lane) return;
	double p;
	if (KIND == IN_U8IQ) {
		/* components v = (b - 127) - d with d = 127.37f - 127 (exact, 16 significant bits):
		 * sum v^2 = sum (b-127)^2 - 2 d sum (b-127) + N d^2, the two sums exact integers */
		const unsigned long long n = 2 * samples;
		const long long s1 = (long long)v.m1 - 127 * (long long)n;
		const unsigned long long s2 = v.m2 + 16129ull * n - 254ull * v.m1;
		const double d = (double)(127.37f - 127.0f);
		p = __dadd_rn(__dsub_rn((double)s2, __dmul_rn(2.0 * d, (double)s1)), __dmul_rn((double)n, __dmul_rn(d, d)));
	} else {
		p = KIND == IN_CS16IQ ? (double)v.m2 : __longlong_as_double((long long)v.m2);
	}
	out[s] = LevelIn{ samples, v.clipped, p, v.peak, 0.0f };
}

template <int KIND>
static int launch_level_input_t(const uint8_t *in, size_t stride, int K, int nrows, const int *rows, int nstreams, LevelPart *part,
                                size_t part_stride, LevelIn *out, cudaStream_t stream, int &launched)
{
	const size_t nchunk = ((size_t)nrows * K * level_sample_bytes<KIND>() + LVL_CHUNK - 1) / LVL_CHUNK;
	if (nchunk == 0) return (int)cudaErrorInvalidValue;
	k_level_in<KIND><<<dim3((unsigned)nchunk, nstreams), LVL_THREADS, 0, stream>>>(in, stride, K, nrows, rows, part, part_stride);
	k_level_in_fin<KIND><<<(unsigned)((nstreams * 32 + 255) / 256), 256, 0, stream>>>(K, nrows, rows, nstreams, part, part_stride, out);
	launched += 2;
	return (int)cudaGetLastError();
}

int launch_level_input(int in_kind, const uint8_t *in, size_t stride, int K, int nrows, const int *rows, int nstreams, LevelPart *part,
                       size_t part_stride, LevelIn *out, cudaStream_t stream, int &launched)
{
	if (in_kind == IN_KIND_U8IQ) return launch_level_input_t<IN_U8IQ>(in, stride, K, nrows, rows, nstreams, part, part_stride, out, stream, launched);
	if (in_kind == IN_KIND_CS16IQ) return launch_level_input_t<IN_CS16IQ>(in, stride, K, nrows, rows, nstreams, part, part_stride, out, stream, launched);
	return launch_level_input_t<IN_F32REAL>(in, stride, K, nrows, rows, nstreams, part, part_stride, out, stream, launched);
}

/* Window j of stream s in this submit: rows [lo, hi) with the stream's open window holding n0 rows, so that
 * j * 1024 - n0 starts window j (the first one closes the open window) */
__device__ __forceinline__ void level_window(int j, int n0, int rows, int &lo, int &hi)
{
	lo = max(0, j * OUTBLK - n0);
	hi = min(rows, (j + 1) * OUTBLK - n0);
}

/* grid (window, stream, channel tile), LVL_THREADS threads as LVL_THREADS / ct row lanes x ct channels: each warp reads
 * whole runs of dm[s][n][c] (channels contiguous), each thread its channel's rows in order, then a fixed tree over the
 * row lanes */
__global__ void __launch_bounds__(LVL_THREADS)
k_level_dm(const float *__restrict__ dm, int nrows, const int *__restrict__ rows, int nch, int ct, const LevelCarry *__restrict__ carry,
           double *__restrict__ seg_sum, float *__restrict__ seg_peak, int seg_stride)
{
	const int s = blockIdx.y, j = blockIdx.x;
	int lo, hi;
	level_window(j, carry[(size_t)s * nch].rows, rows ? rows[s] : nrows, lo, hi);
	if (lo >= hi) return;
	const int nl = LVL_THREADS / ct, r0 = threadIdx.x / ct, cc = threadIdx.x % ct, c = blockIdx.z * ct + cc;
	double sum = 0.0;
	float pk = 0.0f;
	if (c < nch) {
		const float *p = dm + (size_t)s * nrows * nch + c;
#pragma unroll 4
		for (int n = lo + r0; n < hi; n += nl) {
			const float x = __ldcs(p + (size_t)n * nch);
			const double xd = (double)x;
			sum = __dadd_rn(sum, __dmul_rn(xd, xd));
			pk = fmaxf(pk, x);
		}
	}
	__shared__ double s_sum[LVL_THREADS];
	__shared__ float s_pk[LVL_THREADS];
	s_sum[threadIdx.x] = sum;
	s_pk[threadIdx.x] = pk;
	__syncthreads();
	for (int h = nl / 2; h; h >>= 1) {
		if (r0 < h) {
			s_sum[threadIdx.x] = __dadd_rn(s_sum[threadIdx.x], s_sum[threadIdx.x + h * ct]);
			s_pk[threadIdx.x] = fmaxf(s_pk[threadIdx.x], s_pk[threadIdx.x + h * ct]);
		}
		__syncthreads();
	}
	if (r0 == 0 && c < nch) {
		const size_t o = ((size_t)s * seg_stride + j) * nch + c;
		seg_sum[o] = s_sum[threadIdx.x];
		seg_peak[o] = s_pk[threadIdx.x];
	}
}

/* one thread per chain: its windows' partials in order; closed windows give their mean, the last open one becomes the
 * carry */
__global__ void __launch_bounds__(256)
k_level_dm_fin(int nrows, const int *__restrict__ rows, int nch, int nstreams, LevelCarry *__restrict__ carry,
               const double *__restrict__ seg_sum, const float *__restrict__ seg_peak, int seg_stride, LevelChan *__restrict__ out)
{
	const size_t g = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
	if (g >= (size_t)nstreams * nch) return;
	const int s = (int)(g / nch), c = (int)(g % nch), n = rows ? rows[s] : nrows;
	LevelCarry cr = carry[g];
	const int n0 = cr.rows;                       /* the windows of this submit are placed by the carry it started with */
	LevelChan r{ (unsigned long long)n, 0.0, 0.0f, 0.0f, 0, 0.0 };
	const int nwin = n ? (n0 + n + OUTBLK - 1) / OUTBLK : 0;
	for (int j = 0; j < nwin; j++) {
		int lo, hi;
		level_window(j, n0, n, lo, hi);
		const size_t o = ((size_t)s * seg_stride + j) * nch + c;
		const double x = seg_sum[o];
		r.power_sum = __dadd_rn(r.power_sum, x);
		r.peak = fmaxf(r.peak, seg_peak[o]);
		const double w = j ? x : __dadd_rn(cr.sum, x);
		const int wr = (j ? 0 : n0) + (hi - lo);
		if (wr == OUTBLK) {
			const double mean = w / OUTBLK;
			r.floor = r.windows ? fmin(r.floor, mean) : mean;
			r.windows++;
			cr.sum = 0.0;
			cr.rows = 0;
		} else {
			cr.sum = w;
			cr.rows = wr;
		}
	}
	carry[g] = cr;
	out[g] = r;
}

int launch_level_dm(const float *dm, int nrows, const int *rows, int nch, int nstreams, double *seg_sum, float *seg_peak, int seg_stride,
                    LevelCarry *carry, LevelChan *out, cudaStream_t stream, int &launched)
{
	/* channels per tile: the channel count rounded up to a power of two, at most a warp's worth */
	int ct = 1;
	while (ct < nch && ct < 32) ct *= 2;
	const unsigned nwin = (unsigned)(nrows / OUTBLK + 2);                     /* an open window, whole ones, a new open one */
	if (nwin > (unsigned)seg_stride) return (int)cudaErrorInvalidValue;
	k_level_dm<<<dim3(nwin, nstreams, (nch + ct - 1) / ct), LVL_THREADS, 0, stream>>>(dm, nrows, rows, nch, ct, carry, seg_sum, seg_peak,
	                                                                                  seg_stride);
	const size_t nchain = (size_t)nstreams * nch;
	k_level_dm_fin<<<(unsigned)((nchain + 255) / 256), 256, 0, stream>>>(nrows, rows, nch, nstreams, carry, seg_sum, seg_peak, seg_stride, out);
	launched += 2;
	return (int)cudaGetLastError();
}

/* ---- ACB_FLAG_FREQ_STATS: each chain's carrier rotation between the two halves of a row (launch_freq_input) ----
 * A row's half sums a = sum_{n<h} x[n] w[n] and b = sum_{n<h} x[h+n] w[h+n] (h = K/2, w the chain's NCO table) are a
 * complex matrix product of the staged rows and the tables, in float with FMA; the row's terms b conj(a), |a||b| and
 * |a|^2 + |b|^2 are formed in double.  Each warp owns one chain of a FQ_CT-chain tile and every row of a FQ_ROWS-row
 * chunk (lane l: rows l, l + 32, l + 64, l + 96): the lane adds its rows in order, a butterfly adds the lanes, and the
 * final pass adds the chunks in order.  That order depends on the row index alone, not on nch or on where a chain sits
 * in its context, so a channel split gives a single context's bits. */
constexpr int FQ_CT = 8;                         /* chains per CTA: one per warp */
constexpr int FQ_RPL = FREQ_ROWS / 32;           /* rows per lane */
constexpr int FQ_KT = 16;                        /* half-row samples staged per step */

template <int KIND> struct FreqX { using T = float2; };
template <> struct FreqX<IN_F32REAL> { using T = float; };

/* sample n of a row, converted as the channelizer converts it */
template <int KIND> __device__ __forceinline__ typename FreqX<KIND>::T freq_load(const uint8_t *row, int n)
{
	if constexpr (KIND == IN_U8IQ) {
		const unsigned short v = *reinterpret_cast<const unsigned short *>(row + 2 * (size_t)n);
		return make_float2((float)(v & 0xffu) - 127.37f, (float)(v >> 8) - 127.37f);
	} else if constexpr (KIND == IN_CS16IQ) {
		const unsigned v = *reinterpret_cast<const unsigned *>(row + 4 * (size_t)n);
		return make_float2((float)(short)(v & 0xffffu), (float)((int)v >> 16));
	} else {
		return *reinterpret_cast<const float *>(row + 4 * (size_t)n);
	}
}

__device__ __forceinline__ void freq_mac(float2 &acc, float2 x, float2 w)
{
	acc.x = fmaf(x.x, w.x, acc.x);
	acc.x = fmaf(-x.y, w.y, acc.x);
	acc.y = fmaf(x.x, w.y, acc.y);
	acc.y = fmaf(x.y, w.x, acc.y);
}
__device__ __forceinline__ void freq_mac(float2 &acc, float x, float2 w)
{
	acc.x = fmaf(x, w.x, acc.x);
	acc.y = fmaf(x, w.y, acc.y);
}

__device__ __forceinline__ void freq_shfl_add(FreqPart &v, int m)
{
	v.re = __dadd_rn(v.re, __shfl_xor_sync(0xffffffffu, v.re, m));
	v.im = __dadd_rn(v.im, __shfl_xor_sync(0xffffffffu, v.im, m));
	v.mag = __dadd_rn(v.mag, __shfl_xor_sync(0xffffffffu, v.mag, m));
	v.pow = __dadd_rn(v.pow, __shfl_xor_sync(0xffffffffu, v.pow, m));
}

/* grid (row chunk, stream, chain tile), FQ_CT warps */
template <int KIND>
__global__ void __launch_bounds__(FQ_CT * 32)
k_freq_in(const uint8_t *__restrict__ in, size_t stride, int K, int nrows, const int *__restrict__ rows, int nch,
          const float2 *__restrict__ nco, FreqPart *__restrict__ part, size_t part_stride)
{
	using X = typename FreqX<KIND>::T;
	constexpr int SB = KIND == IN_U8IQ ? 2 : 4;
	const int s = blockIdx.y, j = blockIdx.x, nr = rows ? rows[s] : nrows, r0 = j * FREQ_ROWS;
	if (r0 >= nr) return;
	const int h = K / 2, lane = threadIdx.x & 31, warp = threadIdx.x >> 5, c0 = blockIdx.z * FQ_CT, c = c0 + warp;
	__shared__ X s_x[2][FQ_KT][FREQ_ROWS + 1];          /* + 1: the staging stores (kk fastest) fall in different banks */
	__shared__ float2 s_w[2][FQ_KT][FQ_CT];
	const uint8_t *base = in + (size_t)s * stride;
	float2 a[FQ_RPL], b[FQ_RPL];
#pragma unroll
	for (int i = 0; i < FQ_RPL; i++) a[i] = b[i] = make_float2(0.0f, 0.0f);
	for (int n0 = 0; n0 < h; n0 += FQ_KT) {
		__syncthreads();
		for (int e = threadIdx.x; e < 2 * FQ_KT * FREQ_ROWS; e += FQ_CT * 32) {
			const int kk = e % FQ_KT, hr = e / FQ_KT, half = hr & 1, r = hr >> 1;
			X v{};
			if (n0 + kk < h && r0 + r < nr) v = freq_load<KIND>(base + (size_t)(r0 + r) * K * SB, half * h + n0 + kk);
			s_x[half][kk][r] = v;
		}
		if (threadIdx.x < 2 * FQ_KT * FQ_CT) {
			const int kk = threadIdx.x % FQ_KT, half = (threadIdx.x / FQ_KT) & 1, cc = threadIdx.x / (2 * FQ_KT);
			float2 w = make_float2(0.0f, 0.0f);
			if (n0 + kk < h && c0 + cc < nch) w = nco[((size_t)s * nch + c0 + cc) * K + half * h + n0 + kk];
			s_w[half][kk][cc] = w;
		}
		__syncthreads();
#pragma unroll 4
		for (int kk = 0; kk < FQ_KT; kk++) {
			const float2 wa = s_w[0][kk][warp], wb = s_w[1][kk][warp];
#pragma unroll
			for (int i = 0; i < FQ_RPL; i++) {
				freq_mac(a[i], s_x[0][kk][lane + 32 * i], wa);
				freq_mac(b[i], s_x[1][kk][lane + 32 * i], wb);
			}
		}
	}
	FreqPart v{ 0.0, 0.0, 0.0, 0.0 };
#pragma unroll
	for (int i = 0; i < FQ_RPL; i++) {
		if (r0 + lane + 32 * i >= nr) continue;
		const double ar = a[i].x, ai = a[i].y, br = b[i].x, bi = b[i].y;
		const double pa = __dadd_rn(__dmul_rn(ar, ar), __dmul_rn(ai, ai)), pb = __dadd_rn(__dmul_rn(br, br), __dmul_rn(bi, bi));
		v.re = __dadd_rn(v.re, __dadd_rn(__dmul_rn(br, ar), __dmul_rn(bi, ai)));
		v.im = __dadd_rn(v.im, __dsub_rn(__dmul_rn(bi, ar), __dmul_rn(br, ai)));
		v.mag = __dadd_rn(v.mag, __dmul_rn(__dsqrt_rn(pa), __dsqrt_rn(pb)));
		v.pow = __dadd_rn(v.pow, __dadd_rn(pa, pb));
	}
	for (int m = 16; m; m >>= 1) freq_shfl_add(v, m);
	if (lane == 0 && c < nch) part[((size_t)s * part_stride + j) * nch + c] = v;
}

/* one thread per chain: its chunks in order; chains not measured (on[g] == 0) report nothing */
__global__ void __launch_bounds__(256)
k_freq_fin(int nrows, const int *__restrict__ rows, int nch, int nstreams, const int *__restrict__ on, const FreqPart *__restrict__ part,
           size_t part_stride, FreqChan *__restrict__ out)
{
	const size_t g = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
	if (g >= (size_t)nstreams * nch) return;
	const int s = (int)(g / nch), c = (int)(g % nch), n = rows ? rows[s] : nrows;
	FreqChan r{ 0, 0.0, 0.0, 0.0, 0.0 };
	if (on[g]) {
		r.pairs = (unsigned long long)n;
		for (int j = 0; j < (n + FREQ_ROWS - 1) / FREQ_ROWS; j++) {
			const FreqPart p = part[((size_t)s * part_stride + j) * nch + c];
			r.s_re = __dadd_rn(r.s_re, p.re);
			r.s_im = __dadd_rn(r.s_im, p.im);
			r.mag_sum = __dadd_rn(r.mag_sum, p.mag);
			r.power_sum = __dadd_rn(r.power_sum, p.pow);
		}
	}
	out[g] = r;
}

template <int KIND>
static int launch_freq_input_t(const uint8_t *in, size_t stride, int K, int nrows, const int *rows, int nch, int nstreams, const float2 *nco,
                               const int *on, FreqPart *part, size_t part_stride, FreqChan *out, cudaStream_t stream, int &launched)
{
	const unsigned nchunk = (unsigned)((nrows + FREQ_ROWS - 1) / FREQ_ROWS);
	if (nchunk == 0 || nchunk > part_stride) return (int)cudaErrorInvalidValue;
	k_freq_in<KIND><<<dim3(nchunk, nstreams, (nch + FQ_CT - 1) / FQ_CT), FQ_CT * 32, 0, stream>>>(in, stride, K, nrows, rows, nch, nco, part,
	                                                                                              part_stride);
	const size_t nchain = (size_t)nstreams * nch;
	k_freq_fin<<<(unsigned)((nchain + 255) / 256), 256, 0, stream>>>(nrows, rows, nch, nstreams, on, part, part_stride, out);
	launched += 2;
	return (int)cudaGetLastError();
}

int launch_freq_input(int in_kind, const uint8_t *in, size_t stride, int K, int nrows, const int *rows, int nch, int nstreams, const float *nco,
                      const int *on, FreqPart *part, size_t part_stride, FreqChan *out, cudaStream_t stream, int &launched)
{
	const float2 *nco2 = reinterpret_cast<const float2 *>(nco);
	if (in_kind == IN_KIND_U8IQ)
		return launch_freq_input_t<IN_U8IQ>(in, stride, K, nrows, rows, nch, nstreams, nco2, on, part, part_stride, out, stream, launched);
	if (in_kind == IN_KIND_CS16IQ)
		return launch_freq_input_t<IN_CS16IQ>(in, stride, K, nrows, rows, nch, nstreams, nco2, on, part, part_stride, out, stream, launched);
	return launch_freq_input_t<IN_F32REAL>(in, stride, K, nrows, rows, nch, nstreams, nco2, on, part, part_stride, out, stream, launched);
}

/* Moving streams (acb_save_streams / acb_load_streams): stream list[i]'s device regions to and from record i of a staging
 * buffer.  blockIdx.y is the record; blockIdx.x walks the regions in SP_CHUNK pieces (R.chunk0[k] is region k's first).
 * A piece whose two addresses and ends are all 16-byte aligned moves in 16-byte vectors, any other in 4-byte words (the
 * fast plans' per-stream metadata has 4-byte strides). */
constexpr int SP_THREADS = 256;
constexpr unsigned SP_CHUNK = SP_THREADS * 16 * 4;

template <bool UNPACK>
__device__ __forceinline__ void stream_copy(const StreamRegions &R, const int *__restrict__ list, uint8_t *rec, size_t rec_bytes)
{
	const unsigned x = blockIdx.x;
	int k = 0;
	while (k + 1 < R.nreg && x >= R.chunk0[k + 1]) k++;
	const StreamRegion &g = R.r[k];
	uint8_t *dev = g.base + (size_t)list[blockIdx.y] * g.stride;
	uint8_t *blob = rec + (size_t)blockIdx.y * rec_bytes + g.off;
	const size_t lo = (size_t)(x - R.chunk0[k]) * SP_CHUNK, hi = min(lo + SP_CHUNK, g.bytes);
	uint8_t *dst = UNPACK ? dev : blob;
	const uint8_t *src = UNPACK ? blob : dev;
	if ((((uintptr_t)dev | (uintptr_t)blob | lo | hi) & 15) == 0) {
		for (size_t b = lo + threadIdx.x * 16; b < hi; b += SP_THREADS * 16)
			*reinterpret_cast<uint4 *>(dst + b) = *reinterpret_cast<const uint4 *>(src + b);
	} else {
		for (size_t b = lo + threadIdx.x * 4; b < hi; b += SP_THREADS * 4)
			*reinterpret_cast<uint32_t *>(dst + b) = *reinterpret_cast<const uint32_t *>(src + b);
	}
}

__global__ void __launch_bounds__(SP_THREADS)
k_stream_pack(const __grid_constant__ StreamRegions R, const int *__restrict__ list, uint8_t *rec, size_t rec_bytes)
{
	stream_copy<false>(R, list, rec, rec_bytes);
}

__global__ void __launch_bounds__(SP_THREADS)
k_stream_unpack(const __grid_constant__ StreamRegions R, const int *__restrict__ list, uint8_t *rec, size_t rec_bytes)
{
	stream_copy<true>(R, list, rec, rec_bytes);
}

int launch_stream_move(StreamRegions R, const int *list, int n, uint8_t *rec, size_t rec_bytes, bool unpack, cudaStream_t stream,
                       int &launched)
{
	if (R.nreg < 1 || R.nreg > SP_MAXREG || n < 1 || n > 65535) return (int)cudaErrorInvalidValue;
	R.chunk0[0] = 0;
	for (int k = 0; k < R.nreg; k++) {
		if (R.r[k].bytes % 4 || R.r[k].off % 16 || R.r[k].off + R.r[k].bytes > rec_bytes) return (int)cudaErrorInvalidValue;
		R.chunk0[k + 1] = R.chunk0[k] + (unsigned)((R.r[k].bytes + SP_CHUNK - 1) / SP_CHUNK);
	}
	const dim3 grid(R.chunk0[R.nreg], (unsigned)n);
	if (grid.x == 0) return 0;
	if (unpack) k_stream_unpack<<<grid, SP_THREADS, 0, stream>>>(R, list, rec, rec_bytes);
	else k_stream_pack<<<grid, SP_THREADS, 0, stream>>>(R, list, rec, rec_bytes);
	launched++;
	return (int)cudaGetLastError();
}

} // namespace acb

