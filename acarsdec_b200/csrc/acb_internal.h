/* Internal device/host shared layouts of libacars_b200 (not part of the C ABI). */
#ifndef ACB_INTERNAL_H
#define ACB_INTERNAL_H

#include <stddef.h>
#include <stdint.h>

#include <vector>

namespace acb {

constexpr int FLEN = 11;        /* msk.c:25  INTRATE/1200 + 1 */
constexpr int MFLTOVER = 12;    /* msk.c:26 */
constexpr int FLENO = 133;      /* msk.c:27 */
constexpr int OUTBLK = 1024;    /* rtl.c:49 */
constexpr int TXTCAP = 256;     /* >= acarsdec.h:55's 250, padded */

/* Persistent per-(stream,channel) demodulator + framing state in HBM: what channel_t carries
 * between demodMSK calls (acarsdec.h:76-89; msk.c:71-72,134-135), plus the frame being
 * assembled (msgblk_t, acarsdec.h:48-57).  8-byte aligned, 448 bytes. */
struct ChainState {
	double phi, df, lvlsum;           /* MskPhi, MskDf, MskLvlSum */
	float clk;                        /* MskClk (float state!) */
	int bitcount;                     /* MskBitCount */
	unsigned S, idx;                  /* MskS, idx */
	int nbits, state;                 /* nbits, Acarsstate */
	unsigned outbits;
	int blk_len;
	int blk_err;
	int pad0;
	unsigned long long pos;           /* envelope samples consumed so far */
	unsigned long long soh_pos;       /* pos at the SOH of the frame in progress */
	float inb_re[FLEN], inb_im[FLEN]; /* msk.c:40 ring */
	unsigned char crc[2];
	unsigned char pad1[6];
	unsigned char txt[TXTCAP];
};

/* A completed (pre-FEC) frame, device -> host. */
struct RawFrame {
	int stream, chn, len, err;
	double lvlsum;
	int bitcount;
	int pad0;                         /* block-FEC status: 0 = not processed, 1 = deliver, 2 = drop */
	unsigned long long pos, soh_pos;
	unsigned char crc[2];
	unsigned char pad1[6];            /* pad1[0]: why the block FEC ended as it did, FEC_WHY_* (k_block_fec_stats only) */
	unsigned char txt[TXTCAP];
};

/* blk_thread's verdicts (acars.c:124-206) as k_block_fec_stats records them: a frame in the ring ends in exactly one of
 * PARITY_EXCESS, UNFIXABLE, PARITY_PROBLEM or delivery (status 1); PARITY, CRC and FIXED are on the way there */
enum FecWhy {
	FEC_WHY_PARITY = 1,               /* 1..MAXPERR parity errors (acars.c:153-155) */
	FEC_WHY_CRC = 2,                  /* CRC non-zero (acars.c:166-167) */
	FEC_WHY_FIXED = 4,                /* "errors fixed" (acars.c:177-178, 189-190) */
	FEC_WHY_UNFIXABLE = 8,            /* "not able to fix errors" (acars.c:172-173, 184-185) */
	FEC_WHY_PARITY_EXCESS = 16,       /* more than MAXPERR parity errors (acars.c:145-152) */
	FEC_WHY_PARITY_PROBLEM = 32,      /* the final parity re-check failed (acars.c:202-206) */
	FEC_WHY_SHORT = 64                /* under 13 or over 250 bytes (acars.c:124-129; the ring holds none) */
};

struct RingCtl {
	unsigned count;                   /* frames appended (may exceed capacity: overflow) */
	unsigned short_frames;            /* frames of fewer than 13 bytes, dropped before taking a slot (acars.c:124-129) */
	unsigned pad[2];
};

/* channelizer tile geometry */
constexpr int CH_TILE = 128;          /* threads per two-row channelizer CTA (2 output rows each) */
constexpr int CH_GROUP = 8;           /* channels accumulated per pass */

/* wideband fast form (k_channelize_wb): channels per CTA, channel slots per thread, slot capacity per channel tile (every
 * residue class padded to whole groups of WB_CB), the per-(stream, tile) plan in ints: groups, E table, (k, channel) per slot */
constexpr int WB_THREADS = 288;
constexpr int WB_CTILE = 256;
constexpr int WB_CB = 4;
constexpr int WB_SLOTS = WB_CTILE + 4 * (WB_CB - 1) + 4;
constexpr int WB_META = 2 + 2 * WB_SLOTS;

} // namespace acb

/* hostmath.cpp: the wideband form's twiddle table E[r + K - 1], r in (-K, K), with the fast planners' expression for the
 * exponent r = (k*n2) % K; variant -1: u8 (acb_fast_plan), ACB_WB_TW_REAL: real input (acb_fast_plan_air, K % 8 == 0),
 * else a CS16 variant (acb_fast_plan_cs16).  1 on success. */
#define ACB_WB_TW_REAL 2
extern "C" int acb_wb_twiddles(int variant, int K, float *E);

/* kernels.cu entry points (host-callable launchers) */
struct CUstream_st;
namespace acb {
enum InputKind { IN_KIND_U8IQ = 0, IN_KIND_F32REAL = 1, IN_KIND_CS16IQ = 2 };
/* Input history of a context with taps > K (the overlapping window): stream s's last `hpad` samples before the submit
 * start at (const char *)base + s*stride.  hpad = 0: taps <= K, no history.  pos0 = the submit's first output row,
 * counted from acb_create / acb_reset (rows whose window reaches before the stream start omit those terms). */
struct Hist {
	const void *base;
	size_t stride;
	int hpad;
	unsigned long long pos0;
};
int launch_channelize(int mode, const void *in, size_t stream_stride_bytes, const float *wf, float *dm,
                      int K, int taps, int nch, int nstreams, int nblk, size_t nsamp, const Hist &h, CUstream_st *stream);
int launch_channelize_generic(int mode, const void *in, size_t stream_stride, const void *wf, float *dm,
                              int K, int taps, int nch, int nstreams, size_t row0, size_t nrows, size_t nsamp, CUstream_st *stream);
int launch_channelize_generic_ovl(int mode, const void *in, size_t stream_stride, const void *wf, float *dm,
                                  int K, int taps, int nch, int nstreams, size_t row0, size_t nrows, size_t nsamp,
                                  const Hist &h, CUstream_st *stream);
int launch_demod(ChainState *st, const float *dm, int nsamp, int nch, int nstreams,
                 RawFrame *ring, RingCtl *ctl, unsigned cap, int lanes_per_channel, CUstream_st *stream);
/* The counting form (ACB_FLAG_DECODE_STATS): the same demodulator, and chain g adds its frame synchroniser's events to
 * counts[g * EV_COUNT + e] (frame_sm.h; the caller clears them).  Lanes 1, 2, 4 or 8 only (the default forms): anything
 * else returns cudaErrorInvalidValue and launches nothing. */
int launch_demod_stats(ChainState *st, const float *dm, int nsamp, int nch, int nstreams,
                       RawFrame *ring, RingCtl *ctl, unsigned cap, int lanes_per_channel, unsigned *counts, CUstream_st *stream);
int demod_pick_lanes(long long nchains, int sm_count);
bool channelize_dft_supports(int K);
int launch_channelize_dft(const void *in, size_t stream_stride, const float *tw, const unsigned *meta, float *dm,
                          int K, int nch, int nstreams, int nblk, size_t nsamp, bool fold8, CUstream_st *stream);
int launch_channelize_dft_cs16(const void *in, size_t stream_stride, const float *tw, const unsigned *meta, float *dm,
                               int K, int nch, int nstreams, size_t nsamp, CUstream_st *stream);
int launch_channelize_ovl_fast(int mode, const void *in, size_t stream_stride, const Hist &h, const float *p, const float *tw,
                               const unsigned *meta, float *dm, int K, int nch, int nstreams, size_t nsamp, CUstream_st *stream);
int launch_channelize_wb(int mode, const void *in, size_t stream_stride, const Hist &h, const float *p, const float *E,
                         const int *meta, float *dm, int K, int nch, int nstreams, size_t nsamp, CUstream_st *stream);
bool channelize_rdft_supports(int K);
int launch_channelize_rdft(const void *in, size_t stream_stride, const float *tw, const unsigned *meta, float *dm,
                           int K, int nch, int nstreams, size_t nsamp, CUstream_st *stream);
int launch_channelize_ovl_rdft(const void *in, size_t stream_stride, int hpad, const float *p, const float *tw,
                               const unsigned *meta, float *dm, int K, int nch, int nstreams, size_t nsamp, CUstream_st *stream);
int launch_channelize_wb_real(const void *in, size_t stream_stride, int hpad, const float *p, const float *E, const int *meta,
                              float *dm, int K, int nch, int nstreams, size_t nsamp, CUstream_st *stream);
int launch_block_fec(RawFrame *ring, const RingCtl *ctl, unsigned cap, CUstream_st *stream);
/* the same repair, and each frame's FEC_WHY_* in RawFrame::pad1[0] */
int launch_block_fec_stats(RawFrame *ring, const RingCtl *ctl, unsigned cap, CUstream_st *stream);
int launch_interleave_cs16(const int16_t *xi, const int16_t *xq, size_t plane_stride, uint32_t *out, size_t out_stride,
                           size_t nsamples, int nstreams, CUstream_st *stream);
/* device submits of the streaming kinds: `nsamples` 4-byte samples per stream from a (b = NULL) or from the int16 planes a, b
 * (interleaved on the way), source rows `src_stride` samples apart, to out + s*out_stride (any 4-byte alignment) */
int launch_append4(const void *a, const void *b, size_t src_stride, uint32_t *out, size_t out_stride, size_t nsamples, int nstreams,
                   CUstream_st *stream);
int upload_matched_filter(const float *h, CUstream_st *stream);
int upload_sincos_table(const double *cos_hi_lo, const double *sin_hi_lo, CUstream_st *stream);

/* context.cu, host side, shared with multi.cpp */
/* sets the message acb_last_error() returns (of the calling thread); returns `code` */
int fail(int code, const char *fmt, ...);
/* Emission-group starts of a streaming submit that covers envelope samples [pos, pos + nout): the first is pos, then
 * one per `period` outputs (ACB_GROUP_OUTPUTS) or per transfer of `period` input samples (ACB_GROUP_INPUT) */
std::vector<unsigned long long> stream_groups(int unit, unsigned long long period, int K, unsigned long long pos, size_t nout);
} // namespace acb

#endif
