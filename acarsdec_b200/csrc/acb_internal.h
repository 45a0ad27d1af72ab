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
 * assembled (msgblk_t, acarsdec.h:48-57).  8-byte aligned, 432 bytes. */
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
struct acb_ctx;
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
/* K1, the channelizer: the form a context runs (chan_form, kernels.cu, holds the table of which form applies when) */
enum ChanForm { CHAN_EXACT, CHAN_GENERIC, CHAN_DFT, CHAN_RDFT, CHAN_OVL_FAST, CHAN_OVL_RDFT, CHAN_WB, CHAN_WB_REAL };
ChanForm chan_form(int in_kind, int K, int taps, int flags);
/* One channelizer launch: `form` over `nstreams` streams of input `in` (stream s at in + s*stride bytes) into
 * dm[stream][nsamp][nch], with the context's tables (each stream's own rows of them, see chan_stream).  The streaming
 * kinds' history sits right in front of the rows (hist.base = in - hpad samples, hist.stride = stride). */
struct ChanLaunch {
	ChanForm form;
	int in_kind;                 /* IN_KIND_* */
	const uint8_t *in;
	size_t stride;
	Hist hist;
	const float *wf, *p, *tw;
	const unsigned *twmeta;
	const float *wbE;
	const int *wbmeta;
	float *dm;
	int K, taps_pad, nch, nstreams;
	size_t nsamp;                /* rows per stream of dm */
	bool fold8;
};
/* Rows [0, nrows) of every stream of L: EXACT through the block kernel over whole 1024-row blocks and the generic kernel
 * over the rest, GENERIC through the generic kernel; the fast forms take every row (nrows == nsamp).  Adds the kernels it
 * launches to `launched`; returns a cudaError_t. */
int launch_chan(const ChanLaunch &L, size_t nrows, CUstream_st *stream, int &launched);
/* stream s of L alone, its window's terms before the stream start omitted from position pos0 */
ChanLaunch chan_stream(const ChanLaunch &L, int s, unsigned long long pos0);
/* nrows != NULL (device array): the ragged form, stream s demodulates its first nrows[s] <= nsamp rows (lanes 1, 2, 4 or 8
 * only: anything else returns cudaErrorInvalidValue) */
int launch_demod(ChainState *st, const float *dm, int nsamp, int nch, int nstreams,
                 RawFrame *ring, RingCtl *ctl, unsigned cap, int lanes_per_channel, CUstream_st *stream, const int *nrows = nullptr);
/* The counting form (ACB_FLAG_DECODE_STATS): the same demodulator, and chain g adds its frame synchroniser's events to
 * counts[g * EV_COUNT + e] (frame_sm.h; the caller clears them).  Lanes 1, 2, 4 or 8 only (the default forms): anything
 * else returns cudaErrorInvalidValue and launches nothing. */
int launch_demod_stats(ChainState *st, const float *dm, int nsamp, int nch, int nstreams,
                       RawFrame *ring, RingCtl *ctl, unsigned cap, int lanes_per_channel, unsigned *counts, CUstream_st *stream,
                       const int *nrows = nullptr);
int demod_pick_lanes(long long nchains, int sm_count);
int launch_block_fec(RawFrame *ring, const RingCtl *ctl, unsigned cap, CUstream_st *stream);
/* the same repair, and each frame's FEC_WHY_* in RawFrame::pad1[0] */
int launch_block_fec_stats(RawFrame *ring, const RingCtl *ctl, unsigned cap, CUstream_st *stream);
int launch_interleave_cs16(const int16_t *xi, const int16_t *xq, size_t plane_stride, uint32_t *out, size_t out_stride,
                           size_t nsamples, int nstreams, CUstream_st *stream);
/* device submits of the streaming kinds: `nsamples` 4-byte samples per stream from a (b = NULL) or from the int16 planes a, b
 * (interleaved on the way), source rows `src_stride` samples apart, to out + s*out_stride (any 4-byte alignment) */
int launch_append4(const void *a, const void *b, size_t src_stride, uint32_t *out, size_t out_stride, size_t nsamples, int nstreams,
                   CUstream_st *stream);
/* Ragged submits (device arrays, one entry per stream): the append lands count[s] samples at out + s*out_stride + off[s];
 * the tail move copies stream s's hpad + rem[s] samples from row nrows[s] to the front of the other buffer; the history
 * gather takes each u8 stream's last hb bytes at nblk[s] blocks (a stream with none keeps its history) */
int launch_append4_ragged(const void *a, const void *b, size_t src_stride, uint32_t *out, size_t out_stride, const int *off,
                          const int *count, size_t max_count, int nstreams, CUstream_st *stream);
int launch_move_tail(const uint32_t *src, uint32_t *dst, size_t stride, int K, int hpad, const int *nrows, const int *rem,
                     int nstreams, CUstream_st *stream);
int launch_hist_gather(const uint8_t *in, size_t stride, size_t blk_bytes, const int *nblk, uint8_t *hist, int hb, int nstreams,
                       CUstream_st *stream);
/* ACB_FLAG_LEVEL_STATS.  k_level_in: one CTA per LVL_CHUNK input bytes of a stream, its partial (u8: clipped, sum of the
 * bytes, sum of their squares; CS16: clipped, -, sum of I^2 + Q^2; real: clipped, -, the float64 sum of x^2 in m2's bits)
 * to part[s * part_stride + chunk]; a final pass adds each stream's partials in chunk order into out[s].  k_level_dm: one
 * CTA per (stream, 1024-row window, channel tile), each window's partial sum and peak per channel to
 * seg_sum / seg_peak[(s * seg_stride + j) * nch + c]; a final pass per chain adds them in window order, closes the windows
 * with the chain's open-window carry and writes out[s * nch + c].  `rows` != NULL (device array): the ragged form, stream
 * s counts its first rows[s] <= nrows rows.  Both add the kernels they launch to `launched`; they return a cudaError_t. */
constexpr int LVL_CHUNK = 256 * 16 * 8;
struct LevelPart { unsigned long long clipped, m1, m2; float peak; unsigned pad; };
struct LevelCarry { double sum; int rows; int pad; };    /* a chain's open window: its rows so far and their sum of dm^2 */
/* one submit's results, laid out as acb_input_level_t and acb_chan_level_t (context.cu checks it) */
struct LevelIn { unsigned long long samples, clipped; double power_sum; float peak, pad; };
struct LevelChan { unsigned long long rows; double power_sum; float peak, pad; unsigned long long windows; double floor; };
int launch_level_input(int in_kind, const uint8_t *in, size_t stride, int K, int nrows, const int *rows, int nstreams,
                       LevelPart *part, size_t part_stride, LevelIn *out, CUstream_st *stream, int &launched);
int launch_level_dm(const float *dm, int nrows, const int *rows, int nch, int nstreams, double *seg_sum, float *seg_peak,
                    int seg_stride, LevelCarry *carry, LevelChan *out, CUstream_st *stream, int &launched);
/* ACB_FLAG_FREQ_STATS.  k_freq_in: one CTA per (FREQ_ROWS-row chunk, stream, 8-chain tile); each row's own K samples
 * (the same `in`, `stride`, `rows` as launch_level_input) against nco[(s * nch + c) * K + n] ((re, im) float pairs,
 * the chain's cos - j sin table), each chunk's sums per chain to part[(s * part_stride + chunk) * nch + c]; a final pass adds each
 * chain's chunks in order into out[s * nch + c], zero for chains with on[g] == 0.  Returns a cudaError_t. */
constexpr int FREQ_ROWS = 128;
struct FreqPart { double re, im, mag, pow; };
/* one submit's sums, laid out as the head of acb_chan_freq_t (context.cu checks it) */
struct FreqChan { unsigned long long pairs; double s_re, s_im, mag_sum, power_sum; };
int launch_freq_input(int in_kind, const uint8_t *in, size_t stride, int K, int nrows, const int *rows, int nch, int nstreams,
                      const float *nco, const int *on, FreqPart *part, size_t part_stride, FreqChan *out, CUstream_st *stream,
                      int &launched);
/* Moving streams: each stream's device state is up to SP_MAXREG regions, stream s's `bytes` (a multiple of 4) at
 * base + s*stride, placed at `off` (a multiple of 16) in its record.  launch_stream_move copies list[i]'s regions to
 * (unpack = false: k_stream_pack) or from (true: k_stream_unpack) record i at rec + i*rec_bytes, in one launch; it fills
 * chunk0 itself, adds the kernel to `launched` and returns a cudaError_t. */
constexpr int SP_MAXREG = 8;
struct StreamRegion { uint8_t *base; size_t stride, bytes, off; };
struct StreamRegions { StreamRegion r[SP_MAXREG]; unsigned chunk0[SP_MAXREG + 1]; int nreg; };
int launch_stream_move(StreamRegions R, const int *list, int n, uint8_t *rec, size_t rec_bytes, bool unpack, CUstream_st *stream,
                       int &launched);
int upload_matched_filter(const float *h, CUstream_st *stream);
int upload_sincos_table(const double *cos_hi_lo, const double *sin_hi_lo, CUstream_st *stream);

/* context.cu, host side, shared with multi.cpp */
/* stream blobs (acb_save_streams): the header's size; mv_seal sets a blob's record count and CRC; mv_validate is every
 * refusal of acb_load_streams(c, ..., n, blob, size) that does not depend on the stream list */
constexpr size_t MV_HEAD_BYTES = 64;
void mv_seal(void *blob, size_t size, int count);
int mv_validate(::acb_ctx *c, const void *blob, size_t size, int n);
struct MvHead {
	char magic[8];
	uint32_t version, crc;
	int32_t in_kind, K, taps, nch, form, flags, group_unit, count;
	uint64_t group_period, record_bytes;
};
static_assert(sizeof(MvHead) == 64, "the blob header is 64 bytes");
struct MvRecHead { uint64_t pos, carry; uint32_t fast_ok, pad; uint64_t pad2; };
static_assert(sizeof(MvRecHead) == 32, "the record's host part is 32 bytes");
constexpr int MV_FLAGS = 256 | 512 | 1024;     /* ACB_FLAG_DECODE_STATS | ACB_FLAG_LEVEL_STATS | ACB_FLAG_FREQ_STATS */
enum MvRegion { R_STATE, R_IN, R_WF, R_TW, R_TWMETA, R_WBMETA, R_LCARRY };
/* A record of a configuration: its device regions (tag, offset, bytes) in order, then the statistics' offsets */
struct MvLayout {
	int nreg;
	int tag[SP_MAXREG];
	size_t off[SP_MAXREG], bytes[SP_MAXREG];
	size_t off_dstats, off_lin, off_lch, off_fch, rec_bytes;
};
MvLayout mv_layout(int in_kind, int K, int taps, int nch, int form, int flags);
/* a blob header of this context's configuration: magic, version and fingerprint (count and CRC left 0) */
void mv_fingerprint(::acb_ctx *c, MvHead &h);
/* the wideband plan of one stream (nct = ceil(nch / WB_CTILE) blocks of WB_META ints) from its channels' bins */
void wb_meta(int in_kind, int nch, const int *kbin, int etab, int *meta);
/* sets the message acb_last_error() returns (of the calling thread); returns `code` */
int fail(int code, const char *fmt, ...);
/* Emission-group starts of a streaming submit that covers envelope samples [pos, pos + nout): the first is pos, then
 * one per `period` outputs (ACB_GROUP_OUTPUTS) or per transfer of `period` input samples (ACB_GROUP_INPUT) */
std::vector<unsigned long long> stream_groups(int unit, unsigned long long period, int K, unsigned long long pos, size_t nout);
/* The number, counted from the stream's start, of the emission group that holds envelope sample `pos` (u8: its 1024-row
 * block; the streaming kinds: the group of stream_groups, none for ACB_GROUP_SUBMIT) */
unsigned long long group_number(bool u8, int unit, unsigned long long period, int K, unsigned long long pos);
} // namespace acb

#endif
