/*
 * libacars_b200 context: device memory, streams, submit/sync/drain (C ABI in include/acars_b200.h).
 *
 * Replaces, for N streams x C channels at once, what the reference does per RTL block on its
 * input thread (in_callback rtl.c:314-361 -> demodMSK msk.c:67 -> decodeAcars acars.c:246) and
 * on its blk_thread (acars.c:93-215).  Data flow per submit:
 *
 *   host u8 IQ --copy stream--> d_iq[buf] --channelizer stream--> K1 k_channelize -> d_dm[b] (HBM)
 *                                           --demod stream-------> K2 k_demod    -> frame ring[b]
 *                                           --FEC stream---------> K3 k_block_fec on ring[b], frame count -> host
 *   K2 of submit i (latency bound: one serial recurrence per channel) runs concurrently with K1
 *   of submits i+1, i+2; envelope buffers and frame rings come in threes (NPIPE) between them.
 *   acb_collect / acb_sync: D2H of that submit's frames -> consumer thread -> output queue
 *
 * Up to three submits are in flight: input staging is double-buffered, so the H2D copy of submit i+1
 * overlaps the kernels of i, and the read-back of i overlaps the kernels of i+1 and i+2.
 * The frames of a finished submit are sorted into emission order and queued by a CONSUMER THREAD (the role of the
 * reference's blk_thread, acars.c:93-215, minus the FEC, which runs on the device): at a Tsample/s a step carries tens
 * of thousands of messages, and that per-message host work must not sit between two launches.
 */
#include <cuda_runtime.h>
#include <math.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <chrono>
#include <condition_variable>
#include <deque>
#include <memory>
#include <mutex>
#include <system_error>
#include <thread>
#include <vector>

#include "../../include/acars_b200.h"
#include "acb_internal.h"
#include "frame_sm.h"

using namespace acb;

extern "C" void acb_build_sincos_table(double *cos_hi_lo, double *sin_hi_lo);

static thread_local char g_err[512] = "";

int acb::fail(int code, const char *fmt, ...)
{
	va_list ap;
	va_start(ap, fmt);
	vsnprintf(g_err, sizeof(g_err), fmt, ap);
	va_end(ap);
	return code;
}

#define CU(call)                                                                                   \
	do {                                                                                           \
		cudaError_t e_ = (call);                                                                   \
		if (e_ != cudaSuccess)                                                                     \
			return fail(ACB_ERR_CUDA, "%s: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); \
	} while (0)

extern "C" const char *acb_last_error(void) { return g_err; }
extern "C" const char *acb_version(void) { return "acars_b200 0.1 (sm_90a)"; }

struct EvTriple { cudaEvent_t a, b, b2, c; bool chan; };   /* a..b = K1 on s_comp, b2 = K2 starts on s_dem, c = block FEC done on s_fec */

/* Submits in flight = envelope buffers = frame rings.  Three, not two: with two, the host may queue the channelizer of
 * submit N+2 only once the demod of submit N has finished (it reuses that submit's buffers), so every step ended with the
 * demod running alone and began with both kernels starting together; with three the channelizer of N+2 is already queued
 * behind that of N+1 and both kernels run back to back on their streams. */
constexpr int NPIPE = 3;

/* Emission-order groups of one submit (input blocks / chunks).  Even submits (every stream at the same position):
 * `starts` holds the groups every stream shares and `off` is empty.  Otherwise stream s's groups are
 * starts[off[s] .. off[s+1]), and base[s] is the number, counted from the stream's own start, of its first one: frames
 * leave in (that number, stream, channel, time) order. */
struct Groups {
	std::vector<unsigned long long> starts;
	std::vector<unsigned> off;
	std::vector<unsigned long long> base;
};

/* one submit in flight: which frame ring it appends to and how its frames are grouped */
struct Ticket {
	EvTriple ev;                                   /* a..b = channelizer, b..c = demod; c = done */
	int ring;
	Groups groups;
	unsigned long long seq;                        /* the submit's number (acb_ctx::nsubmit when it was made) */
};

/* Ragged submits' per-stream counts on the device: slots of 4 * nstreams ints (rows | a | b | c, see stage_begin), reused
 * round robin once the work that read them is done */
constexpr int NRAG = NPIPE + 1;

struct acb_ctx {
	acb_config_t cfg;
	int ngrp;
	size_t blk_bytes;            /* 1024*K*2 */
	cudaStream_t s_copy, s_comp, s_dem, s_fec;   /* H2D copies | channelizer (K1) | demod (K2) | block FEC (K3) + its count read-back */
	uint8_t *d_iq[2];
	cudaEvent_t ev_copied[2], ev_consumed[2];
	bool buf_used[2];
	int next_buf;
	float *d_wf;                 /* [stream][grp][taps_pad][8] float2 (c, d) */
	ChanForm form;
	float *d_wbE;                /* WB*: the twiddle table(s) E of acb_wb_twiddles, 2K - 1 (Tr, Ti) each; CS16: one per variant */
	int *d_wbmeta;               /* WB*: [stream][channel tile][WB_META] residue-sorted slots (upload_wb_plan) */
	float *d_p;                  /* OVL_*, WB* at taps > K: the pre-sum weights fl(K*h), taps_pad floats, zeros in front */
	bool fold8;                  /* DFT: fold the row in half first (8-way split, K/8 MACs per channel) */
	int demod_lanes;             /* lanes per channel in k_demod: 8 for small contexts, else 4 */
	float *d_tw;                 /* DFT, RDFT, OVL_*: [stream][grp][8 ch][K/4] (Tr, Ti) twiddles */
	unsigned *d_twmeta;          /* DFT, RDFT, OVL_*: [stream][grp] residues k_c mod 4, 2 bits per channel slot */
	std::vector<unsigned char> fast_ok;   /* per stream: planned on the 12.5 kHz raster (0 after acb_set_wf: caller's own table) */
	float *d_dm[NPIPE];          /* [stream][nsamp][nch], one per submit in flight */
	cudaEvent_t ev_k1_done[NPIPE], ev_dm_free[NPIPE], ev_k2_done[NPIPE], ev_ring_read[NPIPE];
	bool ring_read_pending[NPIPE];
	bool dm_used[NPIPE];
	bool k1_pending[NPIPE];      /* ev_k1_done[b] recorded and not yet waited for by the host */
	int last_dm;
	size_t dm_floats;
	ChainState *d_state;
	cudaStream_t s_d2h;
	RawFrame *d_ring[NPIPE];     /* frame rings, one per submit in flight so that one can be read
	                                back while the next submits' demods append to the others */
	RingCtl *d_ctl[NPIPE];
	unsigned ring_cap;
	RawFrame *h_ring[NPIPE];     /* pinned, one per frame ring: the consumer may still read one while the next lands in another */
	RingCtl *h_ctl[NPIPE];       /* pinned */
	int last_nsamp;
	unsigned long long nsubmit;
	std::vector<unsigned long long> pos;   /* per stream: envelope samples submitted since create / reset */
	std::deque<Ticket> inflight; /* oldest first; at most NPIPE */
	/* output queue: one batch per harvested submit, already in emission order; drained by bulk copies (at a
	 * Tsample/s a step carries tens of thousands of messages: per-message queue operations were the host's
	 * largest cost) */
	struct Batch { std::unique_ptr<acb_msg_t[]> v; size_t n, rd; };
	std::deque<Batch> outq;
	size_t outq_count;
	/* consumer thread: everything from `outq` to `jobs_done`, plus stats.raw_frames / fec_dropped, is guarded by mtx */
	struct Job { Groups groups; int ring; unsigned count; unsigned long long seq; bool chan; };
	std::thread consumer;
	std::mutex mtx;
	std::condition_variable cv_job, cv_done;
	std::deque<Job> jobs;
	bool stop;
	unsigned long long jobs_queued, jobs_done, ring_job[NPIPE];   /* ring_job[b]: sequence number of the last job reading h_ring[b] */
	char consumer_err[256];
	std::vector<EvTriple> ev_free;
	cudaEvent_t mark[2], ev_join;
	bool overflowed;
	acb_stats_t stats;
	int taps;                    /* FIR length per output row (<= ACB_MAXTAPS_PER_K * K) */
	int taps_pad;                /* taps <= K: taps rounded up to whole 16-byte units of input (zero weights behind);
	                                taps > K: K + hpad (zero weights in front) */
	int hpad;                    /* taps > K: H = taps - K rounded up to whole 16-byte units of input; else 0 */
	uint8_t *d_hist;             /* u8 IQ, taps > K: per stream, the last hpad samples of its input so far */
	int in_kind;                 /* IN_KIND_*: u8 IQ blocks | float32 real (air.c) | CS16 IQ (soapy.c, sdrplay.c) */
	bool real_input;             /* in_kind != u8: 4-byte input elements, arbitrary submit lengths, carried remainder */
	float *d_real[2];            /* per stream: [hpad history + carry + new samples], alternating per submit */
	size_t real_cap;             /* floats per stream in d_real */
	std::vector<size_t> carry;   /* per stream: samples not yet consumed (< K) */
	int real_buf;
	cudaEvent_t ev_real_copied, ev_real_free[2];   /* H2D of a streaming submit landed | d_real[b] may be overwritten */
	bool real_used[2];
	int16_t *d_planar;           /* CS16 planar input: both planes of one submit, interleaved on the device */
	size_t planar_cap;           /* int16 elements per plane and stream */
	cudaStream_t s_order;        /* streaming kinds: collects the acb_wait_event waits for the next device submit's append */
	cudaEvent_t ev_order;        /* recorded on s_order behind the last of those waits */
	bool order_pending;          /* ev_order has a wait the copy stream has not yet been ordered behind */
	int group_unit;              /* ACB_GROUP_*: how the streaming front-ends' frames are grouped for emission */
	unsigned long long group_period;
	/* ACB_FLAG_DECODE_STATS: per frame ring (submit in flight), the counting demod's EV_COUNT counters per chain, cleared
	 * before its launch and read back with that submit's frames; the consumer adds them and each frame's FEC verdict to
	 * dstats */
	bool decode_stats;
	std::mutex dstats_mtx;       /* guards dstats: the consumer adds to it without holding up acb_drain on mtx */
	unsigned *d_evcnt[NPIPE];
	unsigned *h_evcnt[NPIPE];    /* pinned */
	std::vector<acb_decode_stats_t> dstats;      /* guarded by dstats_mtx */
	std::vector<unsigned long long> dstats_from; /* per stream: the first submit its counts cover (acb_reset_stream); dstats_mtx */
	/* ACB_FLAG_LEVEL_STATS: per frame ring (submit in flight), the submit's input and envelope levels, written whole by the
	 * level kernels on the channelizer stream (behind K1) and read back with that submit's frames; the consumer adds them to
	 * lin / lch.  The open windows' carry (d_lcarry) is device state in submit order, on the channelizer stream. */
	bool level_stats;
	std::mutex lstats_mtx;       /* guards lin, lch, lstats_from, fch */
	LevelIn *d_lin[NPIPE], *h_lin[NPIPE];         /* [stream] (h_* pinned) */
	LevelChan *d_lch[NPIPE], *h_lch[NPIPE];       /* [chain] */
	cudaEvent_t ev_lvl_done[NPIPE];               /* behind the level kernels of the submit using ring b */
	LevelPart *d_lpart;                           /* k_level_in's per-chunk partials, [stream][lpart_stride] */
	size_t lpart_stride;
	double *d_lseg_sum;                           /* k_level_dm's per-window partials, [stream][max_blocks + 2][nch] */
	float *d_lseg_peak;
	LevelCarry *d_lcarry;                         /* [chain] */
	std::vector<acb_input_level_t> lin;           /* guarded by lstats_mtx */
	std::vector<acb_chan_level_t> lch;
	std::vector<unsigned long long> lstats_from;  /* per stream: the first submit its levels and frequency sums cover */
	/* ACB_FLAG_FREQ_STATS: the same rings, event, read-back and consumer as the level statistics (dev_stats: either flag);
	 * the sums are added to fch under lstats_mtx.  fch also holds each chain's plan (freq_hz, step), and d_fnco / d_fon
	 * its NCO table and whether it is measured. */
	bool freq_stats;
	bool dev_stats;                               /* level_stats || freq_stats: the kernels behind K1 and their read-back */
	float *d_fnco;                                /* [stream][nch][K] (re, im) */
	int *d_fon;                                   /* [chain] */
	FreqPart *d_fpart;                            /* [stream][fpart_stride][nch] */
	size_t fpart_stride;
	FreqChan *d_fch[NPIPE], *h_fch[NPIPE];        /* [chain] (h_* pinned) */
	std::vector<acb_chan_freq_t> fch;             /* guarded by lstats_mtx */
	int *d_rag[NRAG], *h_rag[NRAG];               /* ragged submits' counts (h_rag pinned) */
	cudaEvent_t ev_rag_used[NRAG][3];             /* behind the last reads of slot i on the copy, channelizer and demod streams */
	bool rag_used[NRAG];
	unsigned long long rag_seq;
	/* acb_save_streams / acb_load_streams: [stream list | records] staging, grown on demand; ev_mv follows the last load's
	 * unpack, which reads d_mv */
	uint8_t *d_mv, *h_mv;                         /* h_mv pinned */
	size_t mv_cap;
	cudaEvent_t ev_mv;
	bool mv_pending;
};

static void consumer_main(acb_ctx *c);
static void wait_consumer(acb_ctx *c, unsigned long long seq);

static int ctx_use(acb_ctx *c)
{
	CU(cudaSetDevice(c->cfg.device));
	return ACB_OK;
}

/* Host -> device upload that is complete when it returns.  A plain cudaMemcpy from pageable memory may
 * return once the data is staged, before the DMA has landed, and the context's streams are non-blocking
 * (not ordered behind the legacy stream): a kernel launched right after could read the old contents. */
static int upload(acb_ctx *c, void *dst, const void *src, size_t bytes)
{
	CU(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, c->s_copy));
	CU(cudaStreamSynchronize(c->s_copy));
	return ACB_OK;
}

extern "C" void *acb_host_alloc(size_t bytes)
{
	void *p = nullptr;
	if (cudaHostAlloc(&p, bytes, cudaHostAllocDefault) != cudaSuccess) {
		fail(ACB_ERR_CUDA, "cudaHostAlloc(%zu) failed", bytes);
		return nullptr;
	}
	return p;
}
extern "C" void acb_host_free(void *p) { if (p) cudaFreeHost(p); }

extern "C" void *acb_device_alloc(acb_ctx_t *c, size_t bytes)
{
	void *p = nullptr;
	if (!c || ctx_use(c)) return nullptr;
	if (cudaMalloc(&p, bytes) != cudaSuccess) {
		fail(ACB_ERR_NOMEM, "cudaMalloc(%zu) failed", bytes);
		return nullptr;
	}
	return p;
}
extern "C" void acb_device_free(acb_ctx_t *c, void *p) { if (c && p && !ctx_use(c)) cudaFree(p); }

extern "C" int acb_copy_to_device(acb_ctx_t *c, void *dst, const void *src, size_t bytes)
{
	if (!c) return fail(ACB_ERR_ARG, "null context");
	if (int r = ctx_use(c)) return r;
	return upload(c, dst, src, bytes);
}

static int sync_streams(acb_ctx *c)
{
	CU(cudaStreamSynchronize(c->s_comp));
	CU(cudaStreamSynchronize(c->s_dem));
	CU(cudaStreamSynchronize(c->s_fec));
	return ACB_OK;
}

/* the sums of n chains; their plan (freq_hz, step) stays */
static void clear_freq_sums(acb_chan_freq_t *t, size_t n)
{
	for (size_t i = 0; i < n; i++) t[i] = acb_chan_freq_t{ 0, 0.0, 0.0, 0.0, 0.0, t[i].freq_hz, t[i].step };
}

static int reset_states(acb_ctx *c)
{
	const size_t n = (size_t)c->cfg.nstreams * c->cfg.nch;
	std::vector<ChainState> init(n);
	memset(init.data(), 0, n * sizeof(ChainState));
	for (auto &s : init) {       /* initMsk msk.c:34-40 zeroes; initAcars acars.c:230-234 */
		s.nbits = 8;
		s.state = 0;             /* WSYN */
	}
	/* everything stream-ordered on s_copy and complete on return: the context's streams are non-blocking,
	 * so nothing on the legacy stream (plain cudaMemset/cudaMemcpy) is ordered against them */
	if (int r = upload(c, c->d_state, init.data(), n * sizeof(ChainState))) return r;
	for (int i = 0; i < NPIPE; i++) CU(cudaMemsetAsync(c->d_ctl[i], 0, sizeof(RingCtl), c->s_copy));
	/* taps > K: the history restarts.  int16 and float32 zero convert to 0, so zero history is the definition's
	 * omitted terms exactly (the same +-0 argument as for the front padding, acb_create).  A zero u8 byte converts to
	 * -127.37: the first rows after a reset are recomputed with the omitted terms (run_kernels), the zeros here only
	 * keep the pipeline kernel's discarded values finite. */
	if (c->d_hist) CU(cudaMemsetAsync(c->d_hist, 0, (size_t)c->cfg.nstreams * c->hpad * 2, c->s_copy));
	if (c->hpad && c->real_input)
		for (int i = 0; i < 2; i++)
			CU(cudaMemset2DAsync(c->d_real[i], c->real_cap * sizeof(float), 0, (size_t)c->hpad * sizeof(float), c->cfg.nstreams, c->s_copy));
	CU(cudaStreamSynchronize(c->s_copy));
	c->pos.assign(c->cfg.nstreams, 0);
	c->carry.assign(c->cfg.nstreams, 0);
	{
		std::lock_guard<std::mutex> lk(c->mtx);
		c->outq.clear();
		c->outq_count = 0;
	}
	if (c->decode_stats) {       /* the counts go with the undrained messages: those of a reset context restart from nothing */
		std::lock_guard<std::mutex> lk(c->dstats_mtx);
		memset(c->dstats.data(), 0, c->dstats.size() * sizeof(acb_decode_stats_t));
	}
	if (c->level_stats) {        /* the windows restart with the streams */
		CU(cudaMemsetAsync(c->d_lcarry, 0, c->lch.size() * sizeof(LevelCarry), c->s_copy));
		CU(cudaStreamSynchronize(c->s_copy));
		std::lock_guard<std::mutex> lk(c->lstats_mtx);
		memset(c->lin.data(), 0, c->lin.size() * sizeof(acb_input_level_t));
		memset(c->lch.data(), 0, c->lch.size() * sizeof(acb_chan_level_t));
	}
	if (c->freq_stats) {
		std::lock_guard<std::mutex> lk(c->lstats_mtx);
		clear_freq_sums(c->fch.data(), c->fch.size());
	}
	c->overflowed = false;
	return ACB_OK;
}

/* The history (hpad samples) and padded table length (taps_pad) of a context of this kind, K, taps and form */
static void taps_geometry(int in_kind, int K, int taps, ChanForm form, int &hpad, int &taps_pad)
{
	const int per_unit = in_kind != IN_KIND_U8IQ ? 4 : 8;   /* taps per 16 bytes of input (4-byte vs 2-byte taps) */
	hpad = 0;
	if (taps > K) {
		/* overlapping window: H = taps - K samples of the previous rows, rounded up to whole units and padded in
		 * FRONT with zero weights (acb_set_wf).  Leading zero-weight terms leave the sum unchanged: the accumulator
		 * starts at +0, each such term is a product with a zero weight, i.e. +-0 (finite input), and +0 + (+-0) = +0
		 * in round-to-nearest, so the accumulator is still exactly +0 when the first real term p arrives, and
		 * +0 + p = p is what the unpadded sum starts with.  That holds for any K, so the generic kernel uses the same
		 * layout. */
		hpad = (taps - K + per_unit - 1) / per_unit * per_unit;
		taps_pad = K + hpad;
	} else {
		taps_pad = form == CHAN_GENERIC ? taps : (taps + per_unit - 1) / per_unit * per_unit;
		if (taps_pad > K) taps_pad = K;      /* K itself is a multiple of per_unit here */
	}
}

extern "C" int acb_create(const acb_config_t *cfg, acb_ctx_t **out)
{
	if (!cfg || !out) return fail(ACB_ERR_ARG, "null argument");
	if (cfg->K < 1 || cfg->K > ACB_MAXK) return fail(ACB_ERR_ARG, "K=%d out of range 1..%d", cfg->K, ACB_MAXK);
	if (cfg->nstreams < 1 || cfg->nch < 1 || cfg->max_blocks < 1) return fail(ACB_ERR_ARG, "nstreams/nch/max_blocks must be >= 1");
	/* streams are grid.y of the channelizer launches (and of k_interleave_cs16), which CUDA caps at 65535 */
	if (cfg->nstreams > ACB_MAXSTREAMS) return fail(ACB_ERR_ARG, "nstreams=%d exceeds %d", cfg->nstreams, ACB_MAXSTREAMS);
	if (cfg->taps < 0 || cfg->taps > ACB_MAXTAPS_PER_K * cfg->K)
		return fail(ACB_ERR_ARG, "taps=%d must be 0 (= K) or 1..%d*K=%d", cfg->taps, ACB_MAXTAPS_PER_K, ACB_MAXTAPS_PER_K * cfg->K);
	if ((cfg->flags & ACB_FLAG_REAL_INPUT) && (cfg->flags & ACB_FLAG_CS16_INPUT)) return fail(ACB_ERR_ARG, "REAL_INPUT and CS16_INPUT are exclusive");
	int ndev = 0;
	if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
		return fail(ACB_ERR_CUDA, "no CUDA device: libacars_b200 has no CPU fallback");
	if (cfg->device < 0 || cfg->device >= ndev) return fail(ACB_ERR_ARG, "device %d of %d", cfg->device, ndev);
	CU(cudaSetDevice(cfg->device));
	cudaDeviceProp prop;
	CU(cudaGetDeviceProperties(&prop, cfg->device));
	if (prop.major != 9 || prop.minor != 0)
		return fail(ACB_ERR_CUDA, "device %d is sm_%d%d; this library carries sm_90a code only", cfg->device, prop.major, prop.minor);

	acb_ctx *c = new acb_ctx();
	c->cfg = *cfg;
	c->ngrp = (cfg->nch + CH_GROUP - 1) / CH_GROUP;
	c->blk_bytes = (size_t)OUTBLK * cfg->K * 2;
	c->in_kind = (cfg->flags & ACB_FLAG_REAL_INPUT) ? IN_KIND_F32REAL : (cfg->flags & ACB_FLAG_CS16_INPUT) ? IN_KIND_CS16IQ : IN_KIND_U8IQ;
	c->real_input = c->in_kind != IN_KIND_U8IQ;
	c->taps = cfg->taps ? cfg->taps : cfg->K;
	c->form = chan_form(c->in_kind, cfg->K, c->taps, cfg->flags);
	taps_geometry(c->in_kind, cfg->K, c->taps, c->form, c->hpad, c->taps_pad);
	c->d_hist = nullptr;
	c->d_real[0] = c->d_real[1] = nullptr;
	c->d_planar = nullptr;
	c->planar_cap = 0;
	c->ev_real_copied = nullptr;
	c->ev_real_free[0] = c->ev_real_free[1] = nullptr;
	c->s_order = nullptr;
	c->ev_order = nullptr;
	c->order_pending = false;
	c->real_buf = 0;
	c->group_unit = ACB_GROUP_SUBMIT;
	c->group_period = 0;
	c->next_buf = 0;
	c->last_nsamp = 0;
	c->nsubmit = 0;
	c->outq_count = 0;
	c->stop = false;
	c->jobs_queued = c->jobs_done = 0;
	c->ring_job[0] = c->ring_job[1] = 0;
	c->consumer_err[0] = 0;
	c->h_ring[0] = c->h_ring[1] = nullptr;
	c->overflowed = false;
	memset(&c->stats, 0, sizeof(c->stats));
	for (int i = 0; i < NRAG; i++) c->d_rag[i] = nullptr, c->h_rag[i] = nullptr;
	c->decode_stats = (cfg->flags & ACB_FLAG_DECODE_STATS) != 0;
	for (int i = 0; i < NPIPE; i++) c->d_evcnt[i] = nullptr, c->h_evcnt[i] = nullptr;
	c->level_stats = (cfg->flags & ACB_FLAG_LEVEL_STATS) != 0;
	for (int i = 0; i < NPIPE; i++) c->d_lin[i] = c->h_lin[i] = nullptr, c->d_lch[i] = c->h_lch[i] = nullptr, c->ev_lvl_done[i] = nullptr;
	c->d_lpart = nullptr;
	c->d_lseg_sum = nullptr;
	c->d_lseg_peak = nullptr;
	c->d_lcarry = nullptr;
	c->freq_stats = (cfg->flags & ACB_FLAG_FREQ_STATS) != 0;
	c->dev_stats = c->level_stats || c->freq_stats;
	c->d_fnco = nullptr;
	c->d_fon = nullptr;
	c->d_fpart = nullptr;
	for (int i = 0; i < NPIPE; i++) c->d_fch[i] = c->h_fch[i] = nullptr;
	c->d_mv = c->h_mv = nullptr;
	c->mv_cap = 0;
	c->ev_mv = nullptr;
	c->mv_pending = false;
	*out = c;

	{
		/* K2 and K3 are small, latency bound and on the serial chain of the pipeline (K2(i+1) waits for K2(i), K1(i+NPIPE)
		 * for K2(i)'s envelope buffer); K1 is the throughput kernel that fills whatever is left.  So the demod, FEC and
		 * read-back streams get the greatest priority and the channelizer and input-copy streams the least: when an SM
		 * has room, a waiting K2 CTA is dispatched before the next K1 CTA.  Priority only orders the dispatch of CTAs;
		 * it pre-empts nothing. */
		int least = 0, greatest = 0;
		CU(cudaDeviceGetStreamPriorityRange(&least, &greatest));
		CU(cudaStreamCreateWithPriority(&c->s_copy, cudaStreamNonBlocking, least));
		CU(cudaStreamCreateWithPriority(&c->s_comp, cudaStreamNonBlocking, least));
		CU(cudaStreamCreateWithPriority(&c->s_dem, cudaStreamNonBlocking, greatest));
		CU(cudaStreamCreateWithPriority(&c->s_fec, cudaStreamNonBlocking, greatest));
		CU(cudaStreamCreateWithPriority(&c->s_d2h, cudaStreamNonBlocking, greatest));
	}
	CU(cudaEventCreateWithFlags(&c->ev_join, cudaEventDisableTiming));
	CU(cudaEventCreateWithFlags(&c->ev_mv, cudaEventDisableTiming));
	CU(cudaEventCreate(&c->mark[0]));
	CU(cudaEventCreate(&c->mark[1]));
	const size_t in_bytes = (size_t)cfg->nstreams * cfg->max_blocks * c->blk_bytes;
	for (int i = 0; i < 2; i++) {
		c->d_iq[i] = nullptr;
		c->buf_used[i] = false;
		if (!(cfg->flags & ACB_FLAG_NO_INPUT_STAGING) && !c->real_input) CU(cudaMalloc(&c->d_iq[i], in_bytes));
		if (c->real_input) {
			/* room for the history (taps > K), the carried remainder (< K) plus one submit, rounded so streams stay
			 * 32-B aligned */
			c->real_cap = (((size_t)cfg->max_blocks * OUTBLK + 1) * cfg->K + c->hpad + 7) & ~(size_t)7;     /* streams 32-B aligned: whole sectors per chunk */
			/* + 32 rows: the fast CS16 / real-input kernels fetch whole tiles of up to 32 rows, the last one may reach past the last row */
			CU(cudaMalloc(&c->d_real[i], ((size_t)cfg->nstreams * c->real_cap + 32 * (size_t)cfg->K) * sizeof(float)));
			CU(cudaEventCreateWithFlags(&c->ev_real_free[i], cudaEventDisableTiming));
			c->real_used[i] = false;
		}
		CU(cudaEventCreateWithFlags(&c->ev_copied[i], cudaEventDisableTiming));
		CU(cudaEventCreateWithFlags(&c->ev_consumed[i], cudaEventDisableTiming));
	}
	if (c->real_input) {
		CU(cudaEventCreateWithFlags(&c->ev_real_copied, cudaEventDisableTiming));
		CU(cudaStreamCreateWithFlags(&c->s_order, cudaStreamNonBlocking));
		CU(cudaEventCreateWithFlags(&c->ev_order, cudaEventDisableTiming));
	}
	/* u8 IQ history: its own buffer (acb_submit_device copies no input).  The streaming kinds keep theirs in front of
	 * the carried remainder in d_real. */
	if (c->hpad && !c->real_input) CU(cudaMalloc(&c->d_hist, (size_t)cfg->nstreams * c->hpad * 2));
	const size_t wf_floats = (size_t)cfg->nstreams * c->ngrp * c->taps_pad * CH_GROUP * 2;
	CU(cudaMalloc(&c->d_wf, wf_floats * sizeof(float)));
	CU(cudaMemsetAsync(c->d_wf, 0, wf_floats * sizeof(float), c->s_copy));
	CU(cudaStreamSynchronize(c->s_copy));
	c->d_wbE = nullptr;
	c->d_wbmeta = nullptr;
	c->d_p = nullptr;
	c->fast_ok.assign(cfg->nstreams, 0);
	c->fold8 = true;             /* K/8 instead of K/4 MACs per channel than the plain 4-way split */
	if (const char *e = getenv("ACB_FAST_FOLD8")) c->fold8 = atoi(e) != 0;          /* comparison switch; both are tested */
	{
		/* 8 lanes per channel halve the mixer's share of the serial chain but double the warps: a gain only while
		 * there is still at most one demod warp per SM sub-partition; beyond that the extra warps cost more than
		 * they hide */
		c->demod_lanes = demod_pick_lanes((long long)cfg->nstreams * cfg->nch, prop.multiProcessorCount);
		/* comparison switch (tests force every width; tools/ab_demod.py sweeps it): 1, 2, 4, 8 lanes per channel,
		 * +16 = F2F bit-clock rounding, +32 = constants not pinned, -4 / -8 = the round-1 kernel (launch_demod) */
		if (const char *e = getenv("ACB_DEMOD_LANES")) {
			const int v = atoi(e), l = v & 15;
			/* ACB_FLAG_DECODE_STATS: the plain widths only, the forms with a counting kernel (the others keep the pick) */
			const bool counted = v == 1 || v == 2 || v == 4 || v == 8;
			if (c->decode_stats ? counted : (v == -4 || v == -8 || (v > 0 && v < 64 && (l == 1 || l == 2 || l == 4 || l == 8))))
				c->demod_lanes = v;
		}
	}
	const bool wb = c->form == CHAN_WB || c->form == CHAN_WB_REAL, ovl = c->form == CHAN_OVL_FAST || c->form == CHAN_OVL_RDFT;
	if (ovl || c->form == CHAN_DFT || c->form == CHAN_RDFT) {
		CU(cudaMalloc(&c->d_tw, (size_t)cfg->nstreams * c->ngrp * CH_GROUP * (cfg->K / 4) * 2 * sizeof(float)));
		CU(cudaMalloc(&c->d_twmeta, (size_t)cfg->nstreams * c->ngrp * sizeof(unsigned)));
	}
	if (wb) {
		const int ntab = c->in_kind == IN_KIND_CS16IQ ? 2 : 1;
		const size_t per = (size_t)(2 * cfg->K - 1) * 2;
		std::vector<float> E(ntab * per);
		for (int t = 0; t < ntab; t++)
			acb_wb_twiddles(c->in_kind == IN_KIND_CS16IQ ? t : c->in_kind == IN_KIND_F32REAL ? ACB_WB_TW_REAL : -1, cfg->K, &E[t * per]);
		CU(cudaMalloc(&c->d_wbE, E.size() * sizeof(float)));
		if (int r = upload(c, c->d_wbE, E.data(), E.size() * sizeof(float))) return r;
		const size_t nct = (size_t)(cfg->nch + WB_CTILE - 1) / WB_CTILE;
		CU(cudaMalloc(&c->d_wbmeta, (size_t)cfg->nstreams * nct * WB_META * sizeof(int)));
	}
	if (ovl || (wb && c->hpad)) {
		/* the polyphase weights p[i] = fl(K * h[i]), laid out like the exact table (taps_pad entries, the hpad - H in front
		 * zero): the same for every channel and stream; with the twiddles' 1/K the pre-sum's bin carries h[i] * scale */
		std::vector<float> h(c->taps), p(c->taps_pad, 0.0f);
		acb_build_lowpass(cfg->K, c->taps, h.data());
		for (int i = 0; i < c->taps; i++) p[c->taps_pad - c->taps + i] = (float)cfg->K * h[i];
		CU(cudaMalloc(&c->d_p, p.size() * sizeof(float)));
		if (int r = upload(c, c->d_p, p.data(), p.size() * sizeof(float))) return r;
	}
	c->dm_floats = (size_t)cfg->nstreams * cfg->max_blocks * OUTBLK * cfg->nch;
	for (int i = 0; i < NPIPE; i++) {
		CU(cudaMalloc(&c->d_dm[i], c->dm_floats * sizeof(float)));
		CU(cudaEventCreateWithFlags(&c->ev_k1_done[i], cudaEventDisableTiming));
		CU(cudaEventCreateWithFlags(&c->ev_dm_free[i], cudaEventDisableTiming));
		CU(cudaEventCreateWithFlags(&c->ev_k2_done[i], cudaEventDisableTiming));
		CU(cudaEventCreateWithFlags(&c->ev_ring_read[i], cudaEventDisableTiming));
		c->ring_read_pending[i] = false;
		c->dm_used[i] = false;
		c->k1_pending[i] = false;
	}
	c->last_dm = 0;
	const size_t nchain = (size_t)cfg->nstreams * cfg->nch;
	CU(cudaMalloc(&c->d_state, nchain * sizeof(ChainState)));
	/* Frames of fewer than 13 text bytes never take a slot (emit_frame drops them like blk_thread does,
	 * acars.c:124-129).  The shortest frame that does is SYN SYN SOH + 13 + BCS(2) + the byte the END
	 * state swallows = 19 bytes = 152 bits = 791 envelope samples (frame_sm.h), so a chain finishes
	 * < 1.3 per 1024-sample block: 2 per block (+4 for the ends of the submit) cannot be overrun */
	size_t cap = nchain * (2 * (size_t)cfg->max_blocks + 4);
	if (cap > (1u << 22)) cap = 1u << 22;
	c->ring_cap = (unsigned)cap;
	for (int i = 0; i < NPIPE; i++) {
		CU(cudaMalloc(&c->d_ring[i], cap * sizeof(RawFrame)));
		CU(cudaMalloc(&c->d_ctl[i], sizeof(RingCtl)));
		CU(cudaHostAlloc(&c->h_ctl[i], sizeof(RingCtl), cudaHostAllocDefault));
	}
	for (int i = 0; i < NPIPE; i++) CU(cudaHostAlloc(&c->h_ring[i], cap * sizeof(RawFrame), cudaHostAllocDefault));
	if (c->decode_stats) {
		c->dstats.assign(nchain, acb_decode_stats_t{});
		c->dstats_from.assign(cfg->nstreams, 0);
		for (int i = 0; i < NPIPE; i++) {
			CU(cudaMalloc(&c->d_evcnt[i], nchain * EV_COUNT * sizeof(unsigned)));
			CU(cudaHostAlloc(&c->h_evcnt[i], nchain * EV_COUNT * sizeof(unsigned), cudaHostAllocDefault));
		}
	}
	if (c->level_stats) {
		static_assert(sizeof(LevelIn) == sizeof(acb_input_level_t) && offsetof(LevelIn, peak) == offsetof(acb_input_level_t, peak),
		              "LevelIn is acb_input_level_t");
		static_assert(sizeof(LevelChan) == sizeof(acb_chan_level_t) && offsetof(LevelChan, floor) == offsetof(acb_chan_level_t, floor),
		              "LevelChan is acb_chan_level_t");
		const int ns = cfg->nstreams;
		c->lin.assign(ns, acb_input_level_t{});
		c->lch.assign(nchain, acb_chan_level_t{});
		for (int i = 0; i < NPIPE; i++) {
			CU(cudaMalloc(&c->d_lin[i], ns * sizeof(LevelIn)));
			CU(cudaHostAlloc(&c->h_lin[i], ns * sizeof(LevelIn), cudaHostAllocDefault));
			CU(cudaMalloc(&c->d_lch[i], nchain * sizeof(LevelChan)));
			CU(cudaHostAlloc(&c->h_lch[i], nchain * sizeof(LevelChan), cudaHostAllocDefault));
		}
		/* a stream's rows of one submit: at most max_blocks * 1024 rows of K samples */
		const size_t in_bytes_max = (size_t)cfg->max_blocks * OUTBLK * cfg->K * (c->in_kind == IN_KIND_U8IQ ? 2 : 4);
		c->lpart_stride = (in_bytes_max + LVL_CHUNK - 1) / LVL_CHUNK;
		CU(cudaMalloc(&c->d_lpart, (size_t)ns * c->lpart_stride * sizeof(LevelPart)));
		const size_t nseg = (size_t)ns * (cfg->max_blocks + 2) * cfg->nch;
		CU(cudaMalloc(&c->d_lseg_sum, nseg * sizeof(double)));
		CU(cudaMalloc(&c->d_lseg_peak, nseg * sizeof(float)));
		CU(cudaMalloc(&c->d_lcarry, nchain * sizeof(LevelCarry)));
	}
	if (c->freq_stats) {
		static_assert(sizeof(FreqChan) == offsetof(acb_chan_freq_t, freq_hz) && offsetof(FreqChan, power_sum) == offsetof(acb_chan_freq_t, power_sum),
		              "FreqChan is the head of acb_chan_freq_t");
		c->fch.assign(nchain, acb_chan_freq_t{});
		for (int i = 0; i < NPIPE; i++) {
			CU(cudaMalloc(&c->d_fch[i], nchain * sizeof(FreqChan)));
			CU(cudaHostAlloc(&c->h_fch[i], nchain * sizeof(FreqChan), cudaHostAllocDefault));
		}
		c->fpart_stride = ((size_t)cfg->max_blocks * OUTBLK + FREQ_ROWS - 1) / FREQ_ROWS;
		CU(cudaMalloc(&c->d_fpart, (size_t)cfg->nstreams * c->fpart_stride * cfg->nch * sizeof(FreqPart)));
		CU(cudaMalloc(&c->d_fnco, nchain * cfg->K * 2 * sizeof(float)));
		CU(cudaMalloc(&c->d_fon, nchain * sizeof(int)));
		CU(cudaMemsetAsync(c->d_fnco, 0, nchain * cfg->K * 2 * sizeof(float), c->s_copy));
		CU(cudaMemsetAsync(c->d_fon, 0, nchain * sizeof(int), c->s_copy));
		CU(cudaStreamSynchronize(c->s_copy));
	}
	if (c->dev_stats) {
		c->lstats_from.assign(cfg->nstreams, 0);
		for (int i = 0; i < NPIPE; i++) CU(cudaEventCreateWithFlags(&c->ev_lvl_done[i], cudaEventDisableTiming));
	}
	c->rag_seq = 0;
	for (int i = 0; i < NRAG; i++) {
		CU(cudaMalloc(&c->d_rag[i], 4 * (size_t)cfg->nstreams * sizeof(int)));
		CU(cudaHostAlloc(&c->h_rag[i], 4 * (size_t)cfg->nstreams * sizeof(int), cudaHostAllocDefault));
		for (auto &e : c->ev_rag_used[i]) CU(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
		c->rag_used[i] = false;
	}
	c->consumer = std::thread(consumer_main, c);

	float h[FLENO];
	acb_build_h(h);
	CU((cudaError_t)upload_matched_filter(h, c->s_copy));
	{
		double tc[128], ts[128];
		acb_build_sincos_table(tc, ts);             /* hostmath.cpp */
		CU((cudaError_t)upload_sincos_table(tc, ts, c->s_copy));
	}
	if (int r = reset_states(c)) return r;
	return ACB_OK;
}

extern "C" void acb_destroy(acb_ctx_t *c)
{
	if (!c) return;
	if (c->consumer.joinable()) {
		{
			std::lock_guard<std::mutex> lk(c->mtx);
			c->stop = true;
		}
		c->cv_job.notify_all();
		c->consumer.join();
	}
	if (ctx_use(c) == ACB_OK) {
		cudaDeviceSynchronize();
		for (int i = 0; i < 2; i++) {
			if (c->d_iq[i]) cudaFree(c->d_iq[i]);
			if (c->d_real[i]) cudaFree(c->d_real[i]);
			if (c->ev_real_free[i]) cudaEventDestroy(c->ev_real_free[i]);
			cudaEventDestroy(c->ev_copied[i]);
			cudaEventDestroy(c->ev_consumed[i]);
		}
		for (auto &t : c->inflight) { cudaEventDestroy(t.ev.a); cudaEventDestroy(t.ev.b); cudaEventDestroy(t.ev.b2); cudaEventDestroy(t.ev.c); }
		for (auto &e : c->ev_free) { cudaEventDestroy(e.a); cudaEventDestroy(e.b); cudaEventDestroy(e.b2); cudaEventDestroy(e.c); }
		if (c->ev_real_copied) cudaEventDestroy(c->ev_real_copied);
		if (c->ev_order) cudaEventDestroy(c->ev_order);
		if (c->s_order) cudaStreamDestroy(c->s_order);
		cudaFree(c->d_planar);
		cudaFree(c->d_hist);
		cudaFree(c->d_wf); cudaFree(c->d_state);
		cudaFree(c->d_tw); cudaFree(c->d_twmeta); cudaFree(c->d_p);
		cudaFree(c->d_wbE); cudaFree(c->d_wbmeta);
		for (int i = 0; i < NPIPE; i++) {
			cudaFree(c->d_dm[i]); cudaEventDestroy(c->ev_k1_done[i]); cudaEventDestroy(c->ev_dm_free[i]);
			cudaEventDestroy(c->ev_k2_done[i]); cudaEventDestroy(c->ev_ring_read[i]);
			cudaFree(c->d_ring[i]); cudaFree(c->d_ctl[i]); cudaFreeHost(c->h_ctl[i]); cudaFreeHost(c->h_ring[i]);
			cudaFree(c->d_evcnt[i]); cudaFreeHost(c->h_evcnt[i]);
			cudaFree(c->d_lin[i]); cudaFreeHost(c->h_lin[i]); cudaFree(c->d_lch[i]); cudaFreeHost(c->h_lch[i]);
			if (c->ev_lvl_done[i]) cudaEventDestroy(c->ev_lvl_done[i]);
		}
		cudaFree(c->d_lpart); cudaFree(c->d_lseg_sum); cudaFree(c->d_lseg_peak); cudaFree(c->d_lcarry);
		for (int i = 0; i < NPIPE; i++) { cudaFree(c->d_fch[i]); cudaFreeHost(c->h_fch[i]); }
		cudaFree(c->d_fpart); cudaFree(c->d_fnco); cudaFree(c->d_fon);
		cudaFree(c->d_mv); cudaFreeHost(c->h_mv);
		if (c->ev_mv) cudaEventDestroy(c->ev_mv);
		for (int i = 0; i < NRAG; i++) {
			if (!c->d_rag[i]) continue;
			cudaFree(c->d_rag[i]); cudaFreeHost(c->h_rag[i]);
			for (auto &e : c->ev_rag_used[i]) cudaEventDestroy(e);
		}
		cudaEventDestroy(c->mark[0]); cudaEventDestroy(c->mark[1]); cudaEventDestroy(c->ev_join);
		cudaStreamDestroy(c->s_copy); cudaStreamDestroy(c->s_comp); cudaStreamDestroy(c->s_dem); cudaStreamDestroy(c->s_fec); cudaStreamDestroy(c->s_d2h);
	}
	delete c;
}

extern "C" int acb_reset(acb_ctx_t *c)
{
	if (!c) return fail(ACB_ERR_ARG, "null context");
	if (int r = ctx_use(c)) return r;
	CU(cudaDeviceSynchronize());
	wait_consumer(c, c->jobs_queued);
	/* submits still in flight are abandoned with their frames: recycle their events, forget pending reads */
	for (auto &t : c->inflight) c->ev_free.push_back(t.ev);
	c->inflight.clear();
	for (int i = 0; i < NPIPE; i++) c->ring_read_pending[i] = false;
	for (int i = 0; i < NPIPE; i++) c->k1_pending[i] = false;
	return reset_states(c);
}

extern "C" int acb_reset_stream(acb_ctx_t *c, int stream)
{
	if (!c) return fail(ACB_ERR_ARG, "null context");
	if (stream < 0 || stream >= c->cfg.nstreams) return fail(ACB_ERR_ARG, "stream %d out of range", stream);
	if (int r = ctx_use(c)) return r;
	/* initMsk + initAcars (reset_states), behind the demods already queued and ahead of the next */
	ChainState *st = c->d_state + (size_t)stream * c->cfg.nch;
	CU(cudaMemsetAsync(st, 0, (size_t)c->cfg.nch * sizeof(ChainState), c->s_dem));
	static_assert(offsetof(ChainState, nbits) % 4 == 0, "nbits: an int whose low byte is set alone (little endian)");
	CU(cudaMemset2DAsync(&st->nbits, sizeof(ChainState), 8, 1, c->cfg.nch, c->s_dem));
	/* the history, behind the channelizer and tail move that wrote it: the next submit's rows of this stream start at row 0 */
	if (c->d_hist) CU(cudaMemsetAsync(c->d_hist + (size_t)stream * c->hpad * 2, 0, (size_t)c->hpad * 2, c->s_comp));
	if (c->hpad && c->real_input)
		CU(cudaMemsetAsync(c->d_real[c->real_buf] + (size_t)stream * c->real_cap, 0, (size_t)c->hpad * sizeof(float), c->s_comp));
	if (c->real_input) {
		/* the next append lands where the tail move put the discarded remainder: it must come after it */
		CU(cudaEventRecord(c->ev_join, c->s_comp));
		CU(cudaStreamWaitEvent(c->s_copy, c->ev_join, 0));
	}
	c->pos[stream] = 0;
	if (c->real_input) c->carry[stream] = 0;
	if (c->decode_stats) {
		std::lock_guard<std::mutex> lk(c->dstats_mtx);
		memset(&c->dstats[(size_t)stream * c->cfg.nch], 0, (size_t)c->cfg.nch * sizeof(acb_decode_stats_t));
		c->dstats_from[stream] = c->nsubmit;
	}
	if (c->level_stats) {
		/* the stream's open windows, behind the level kernels already queued on the channelizer stream */
		CU(cudaMemsetAsync(c->d_lcarry + (size_t)stream * c->cfg.nch, 0, (size_t)c->cfg.nch * sizeof(LevelCarry), c->s_comp));
	}
	if (c->dev_stats) {
		std::lock_guard<std::mutex> lk(c->lstats_mtx);
		if (c->level_stats) {
			c->lin[stream] = acb_input_level_t{};
			memset(&c->lch[(size_t)stream * c->cfg.nch], 0, (size_t)c->cfg.nch * sizeof(acb_chan_level_t));
		}
		if (c->freq_stats) clear_freq_sums(&c->fch[(size_t)stream * c->cfg.nch], c->cfg.nch);
		c->lstats_from[stream] = c->nsubmit;
	}
	return ACB_OK;
}

/* ACB_FLAG_FREQ_STATS: stream s's chains are measured against freq[c] (0: not measured) with NCO step step[c]; the table
 * is built in double and rounded to float once per entry.  Complete on return, like every table upload. */
static int set_freq_plan(acb_ctx *c, int stream, const double *freq, const double *step)
{
	const int nch = c->cfg.nch, K = c->cfg.K;
	std::vector<float> w((size_t)nch * K * 2);
	std::vector<int> on(nch);
	for (int ch = 0; ch < nch; ch++) {
		on[ch] = freq[ch] > 0;
		for (int n = 0; n < K; n++) {
			const double ph = step[ch] * n;
			w[((size_t)ch * K + n) * 2] = (float)cos(ph);
			w[((size_t)ch * K + n) * 2 + 1] = -(float)sin(ph);
		}
	}
	if (int r = upload(c, c->d_fnco + (size_t)stream * w.size(), w.data(), w.size() * sizeof(float))) return r;
	if (int r = upload(c, c->d_fon + (size_t)stream * nch, on.data(), on.size() * sizeof(int))) return r;
	std::lock_guard<std::mutex> lk(c->lstats_mtx);
	for (int ch = 0; ch < nch; ch++) {
		c->fch[(size_t)stream * nch + ch].freq_hz = freq[ch];
		c->fch[(size_t)stream * nch + ch].step = step[ch];
	}
	return ACB_OK;
}

extern "C" int acb_set_wf(acb_ctx_t *c, int stream, const float *wf, int nch)
{
	if (!c || !wf) return fail(ACB_ERR_ARG, "null argument");
	if (stream < 0 || stream >= c->cfg.nstreams || nch != c->cfg.nch) return fail(ACB_ERR_ARG, "stream/nch mismatch");
	if (int r = ctx_use(c)) return r;
	const int T = c->taps, TP = c->taps_pad;      /* taps beyond T keep zero weights: D + (+0) = D */
	const int lead = c->hpad ? TP - T : 0;        /* taps > K: the padding goes in front (acb_create) */
	std::vector<float> t((size_t)c->ngrp * TP * CH_GROUP * 2, 0.0f);     /* (c, d) per (tap, channel), every input kind */
	for (int ch = 0; ch < nch; ch++) {
		const int g = ch / CH_GROUP, cc = ch % CH_GROUP;
		for (int ind = 0; ind < T; ind++) {
			const float re = wf[((size_t)ch * T + ind) * 2], im = wf[((size_t)ch * T + ind) * 2 + 1];
			float *o = &t[(((size_t)g * TP + lead + ind) * CH_GROUP + cc) * 2];
			o[0] = re; o[1] = im;
		}
	}
	if (int r = sync_streams(c)) return r;
	if (int r = upload(c, c->d_wf + (size_t)stream * t.size(), t.data(), t.size() * sizeof(float))) return r;
	c->fast_ok[stream] = 0;                     /* a caller's table has no known structure: exact kernel */
	if (c->freq_stats) {                        /* nor a known frequency: not measured (the planners set it after this) */
		const std::vector<double> zero(nch, 0.0);
		return set_freq_plan(c, stream, zero.data(), zero.data());
	}
	return ACB_OK;
}

/* DFT, RDFT, OVL_*: group the per-channel twiddles and bin residues the way the kernels read them and upload them */
static int upload_fast_plan(acb_ctx *c, int stream, const std::vector<int> &kbin, const std::vector<float> &tw1)
{
	const int nch = c->cfg.nch, N2 = c->cfg.K / 4;
	std::vector<float> tw((size_t)c->ngrp * CH_GROUP * N2 * 2, 0.0f);
	std::vector<unsigned> meta(c->ngrp, 0u);
	for (int ch = 0; ch < nch; ch++) {
		const int g = ch / CH_GROUP, cc = ch % CH_GROUP;
		meta[g] |= (unsigned)(((kbin[ch] % 4) + 4) % 4) << (2 * cc);      /* k mod 4: the 4-way split (u8: 0 or 2; real input: any) */
		meta[g] |= (unsigned)((((kbin[ch] / 2) % 4) + 4) % 4) << (16 + 2 * cc);   /* k even: residue of k/2, for the folded form */
		memcpy(&tw[((size_t)g * CH_GROUP + cc) * N2 * 2], &tw1[(size_t)ch * N2 * 2], (size_t)N2 * 2 * sizeof(float));
	}
	if (int r = upload(c, c->d_tw + (size_t)stream * tw.size(), tw.data(), tw.size() * sizeof(float))) return r;
	if (int r = upload(c, c->d_twmeta + (size_t)stream * meta.size(), meta.data(), meta.size() * sizeof(unsigned))) return r;
	c->fast_ok[stream] = 1;
	return ACB_OK;
}

/* wideband form: per channel tile, the channel slots sorted by bin residue (k/2) mod 4 (real input: by the column the
 * real form reads, k mod 4 = 0, 2 or odd) and each class padded to whole groups of WB_CB (channel -1), so that every
 * thread of k_channelize_wb(_real) multiplies one Y' column; `etab` selects the twiddle table (CS16: the variant) */
void acb::wb_meta(int in_kind, int nch, const int *kbin, int etab, int *meta)
{
	const int nct = (nch + WB_CTILE - 1) / WB_CTILE;
	const bool real = in_kind == IN_KIND_F32REAL;
	auto cls = [real](int k) { return real ? ((k & 3) == 0 ? 0 : (k & 3) == 2 ? 1 : 2) : (((k / 2) % 4) + 4) % 4; };
	std::fill(meta, meta + (size_t)nct * WB_META, 0);
	for (int z = 0; z < nct; z++) {
		int *m = &meta[(size_t)z * WB_META];
		int slot = 0;
		for (int res = 0; res < 4; res++) {
			for (int ch = z * WB_CTILE; ch < std::min(nch, (z + 1) * WB_CTILE); ch++) {
				if (cls(kbin[ch]) != res) continue;
				m[2 + 2 * slot] = kbin[ch];
				m[3 + 2 * slot] = ch;
				slot++;
			}
			for (; slot % WB_CB; slot++) {
				m[2 + 2 * slot] = 0;
				m[3 + 2 * slot] = -1;
			}
		}
		m[0] = slot / WB_CB;
		m[1] = etab;
	}
}

static int upload_wb_plan(acb_ctx *c, int stream, const std::vector<int> &kbin, int etab)
{
	const int nct = (c->cfg.nch + WB_CTILE - 1) / WB_CTILE;
	std::vector<int> meta((size_t)nct * WB_META);
	wb_meta(c->in_kind, c->cfg.nch, kbin.data(), etab, meta.data());
	if (int r = upload(c, c->d_wbmeta + (size_t)stream * meta.size(), meta.data(), meta.size() * sizeof(int))) return r;
	c->fast_ok[stream] = 1;
	return ACB_OK;
}

/* The planners' common tail: the exact tables, `build(ch, wf)` writing channel ch's taps (the low-pass form at taps > K),
 * then the plan the context's form reads.  `plan(kbin, tw1)` is the input kind's acb_fast_plan* (tw1 NULL: the bins
 * only), 1 when every channel sits on the raster: otherwise the stream stays on EXACT.  `etab`: upload_wb_plan's. */
template <class Build, class Plan, class Off>
static int plan_stream(acb_ctx *c, int stream, const Build &build, const Plan &plan, int etab, double f0, const Off &off)
{
	const int nch = c->cfg.nch, T = c->taps;
	std::vector<float> wf((size_t)nch * T * 2);
	for (int ch = 0; ch < nch; ch++) build(ch, &wf[(size_t)ch * T * 2]);
	if (int r = acb_set_wf(c, stream, wf.data(), nch)) return r;
	if (c->freq_stats) {
		/* the measurement mixes with the offset `off(ch)` Hz from f0 (see acb_chan_freq_t) */
		std::vector<double> freq(nch), step(nch);
		for (int ch = 0; ch < nch; ch++) {
			freq[ch] = f0 + off(ch);
			step[ch] = 2.0 * M_PI * off(ch) / ((double)ACB_INTRATE * c->cfg.K);
		}
		if (int r = set_freq_plan(c, stream, freq.data(), step.data())) return r;
	}
	if (c->form == CHAN_EXACT || c->form == CHAN_GENERIC) return ACB_OK;
	std::vector<int> kbin(nch);
	if (c->form == CHAN_WB || c->form == CHAN_WB_REAL) return plan(kbin.data(), nullptr) == 1 ? upload_wb_plan(c, stream, kbin, etab) : ACB_OK;
	std::vector<float> tw1((size_t)nch * (c->cfg.K / 4) * 2);
	return plan(kbin.data(), tw1.data()) == 1 ? upload_fast_plan(c, stream, kbin, tw1) : ACB_OK;
}

extern "C" int acb_set_plan(acb_ctx_t *c, int stream, const unsigned *freqs_hz, int nch, unsigned *fc_out)
{
	if (!c || !freqs_hz) return fail(ACB_ERR_ARG, "null argument");
	const unsigned fc = acb_choose_fc(freqs_hz, nch, c->cfg.K);
	if (fc == 0) return fail(ACB_ERR_PLAN, "Frequencies too far apart");    /* rtl.c:149-152 */
	if (fc_out) *fc_out = fc;
	return acb_set_plan_at(c, stream, freqs_hz, nch, fc);
}

extern "C" int acb_set_plan_at(acb_ctx_t *c, int stream, const unsigned *freqs_hz, int nch, unsigned fc)
{
	if (!c || !freqs_hz) return fail(ACB_ERR_ARG, "null argument");
	if (nch != c->cfg.nch) return fail(ACB_ERR_ARG, "nch mismatch");
	if (c->real_input) return fail(ACB_ERR_ARG, "not a u8-IQ context: use acb_set_plan_air / acb_set_plan_cs16");
	if (c->taps < c->cfg.K) return fail(ACB_ERR_ARG, "taps < K: the planners build K-tap or low-pass tables only; supply yours with acb_set_wf");
	if (fc == 0) return fail(ACB_ERR_PLAN, "centre frequency 0");
	const int K = c->cfg.K, T = c->taps;        /* K, or the low-pass length of an overlapping-window context */
	return plan_stream(c, stream, [&](int ch, float *wf) {
		if (c->hpad) acb_build_wf_lp(acb_stored_fr(freqs_hz[ch]), fc, K, T, wf);
		else acb_build_wf(acb_stored_fr(freqs_hz[ch]), fc, K, wf);
	}, [&](int *kbin, float *tw1) { return acb_fast_plan(freqs_hz, nch, K, fc, kbin, tw1); }, 0,
	(double)fc, [&](int ch) { return (double)((float)acb_stored_fr(freqs_hz[ch]) - (float)fc); });
}

static EvTriple get_events(acb_ctx *c)
{
	EvTriple e;
	if (!c->ev_free.empty()) {
		e = c->ev_free.back();
		c->ev_free.pop_back();
	} else {
		cudaEventCreate(&e.a); cudaEventCreate(&e.b); cudaEventCreate(&e.b2); cudaEventCreate(&e.c);
	}
	return e;
}

/* Collecting a submit has a device half and a host half:
 *   harvest_begin  (submitting thread) waits until its demod kernel is done, reads the frame count, queues the D2H
 *                  copy of its frames (copy stream s_d2h, event ev_ring_read[ring]) and hands the rest to the consumer;
 *   consumer_main  (consumer thread) waits for that copy and queues the frames the device block FEC (k_block_fec, the
 *                  blk_thread role, acars.c:93-215) kept, in the reference's emission order: per input block, channel by
 *                  channel, then time (rtl.c:357-360; soundfile.c:71-77); streams are interleaved as
 *                  if the reference served them in turn.
 * So the host-side sort/copy of submit i-1 never delays the launches of submit i+1; acb_collect / acb_sync wait for the
 * consumer to have caught up with what they collected. */

/* ACB_FLAG_DECODE_STATS: a collected submit's counts into the context's table — the counting demod's per-chain
 * events, and the verdict k_block_fec_stats gave each of its frames in the ring */
static void add_decode_stats(acb_ctx *c, const acb_ctx::Job &job, const RawFrame *ring, const unsigned char *keep)
{
	std::lock_guard<std::mutex> lk(c->dstats_mtx);
	const size_t nchain = c->dstats.size();
	const unsigned *ev = c->h_evcnt[job.ring];
	/* a stream reset after this submit was made (acb_reset_stream) counts from its next submit on */
	auto counted = [c, &job](size_t stream) { return job.seq >= c->dstats_from[stream]; };
	for (size_t g = 0; g < nchain; g++) {
		if (!counted(g / c->cfg.nch)) continue;
		const unsigned *e = ev + g * EV_COUNT;
		acb_decode_stats_t &d = c->dstats[g];
		d.preamble += e[EV_PREAMBLE];
		d.started += e[EV_STARTED];
		d.txt_parity += e[EV_TXT_PARITY];
		d.txt_long += e[EV_TXT_LONG];
		d.txt_missed_end += e[EV_TXT_MISSED_END];
		d.emitted += e[EV_EMITTED];
		d.fec_short += e[EV_SHORT];
		d.lost += e[EV_LOST];
	}
	for (unsigned i = 0; i < job.count; i++) {
		const RawFrame &f = ring[i];
		if (!counted((size_t)f.stream)) continue;
		const unsigned why = f.pad1[0];
		acb_decode_stats_t &d = c->dstats[(size_t)f.stream * c->cfg.nch + f.chn];
		d.fec_parity_excess += (why & FEC_WHY_PARITY_EXCESS) != 0;
		d.fec_parity += (why & FEC_WHY_PARITY) != 0;
		d.fec_crc += (why & FEC_WHY_CRC) != 0;
		d.fec_fixed += (why & FEC_WHY_FIXED) != 0;
		d.fec_unfixable += (why & FEC_WHY_UNFIXABLE) != 0;
		d.fec_parity_problem += (why & FEC_WHY_PARITY_PROBLEM) != 0;
		d.delivered += keep[i];
	}
}

/* ACB_FLAG_LEVEL_STATS: a collected submit's levels into the context's tables (envelope input has no input levels) */
static void add_level_stats(acb_ctx *c, const acb_ctx::Job &job)
{
	std::lock_guard<std::mutex> lk(c->lstats_mtx);
	const int nch = c->cfg.nch;
	const LevelIn *in = c->h_lin[job.ring];
	const LevelChan *ch = c->h_lch[job.ring];
	for (int s = 0; s < c->cfg.nstreams; s++) {
		if (job.seq < c->lstats_from[s]) continue;        /* made before the stream's acb_reset_stream */
		if (job.chan) {
			acb_input_level_t &d = c->lin[s];
			d.samples += in[s].samples;
			d.clipped += in[s].clipped;
			d.power_sum += in[s].power_sum;
			d.peak = std::max(d.peak, in[s].peak);
		}
		for (int k = 0; k < nch; k++) {
			const LevelChan &e = ch[(size_t)s * nch + k];
			acb_chan_level_t &d = c->lch[(size_t)s * nch + k];
			d.rows += e.rows;
			d.power_sum += e.power_sum;
			d.peak = std::max(d.peak, e.peak);
			if (e.windows) d.floor = d.windows ? std::min(d.floor, e.floor) : e.floor;
			d.windows += e.windows;
		}
	}
}

/* ACB_FLAG_FREQ_STATS: a collected submit's sums into the context's table (envelope input measures nothing) */
static void add_freq_stats(acb_ctx *c, const acb_ctx::Job &job)
{
	std::lock_guard<std::mutex> lk(c->lstats_mtx);
	const int nch = c->cfg.nch;
	const FreqChan *e = c->h_fch[job.ring];
	for (int s = 0; s < c->cfg.nstreams; s++) {
		if (job.seq < c->lstats_from[s]) continue;        /* made before the stream's acb_reset_stream */
		for (int k = 0; k < nch; k++) {
			const FreqChan &x = e[(size_t)s * nch + k];
			acb_chan_freq_t &d = c->fch[(size_t)s * nch + k];
			d.pairs += x.pairs;
			d.s_re += x.s_re;
			d.s_im += x.s_im;
			d.mag_sum += x.mag_sum;
			d.power_sum += x.power_sum;
		}
	}
}

static void consume(acb_ctx *c, const acb_ctx::Job &job)
{
	const unsigned count = job.count;
	const auto &gs = job.groups.starts;
	const RawFrame *ring = c->h_ring[job.ring];
	/* emission order = (group, stream, channel, time).  A chain's frames reach the ring in time order (one thread
	 * appends them as it decodes), so a STABLE bucket pass over (group, chain) is the whole sort: O(frames + buckets)
	 * instead of a comparison sort (at a Tsample/s a step carries ~40 000 frames; std::sort on them was half of the
	 * consumer's time, and the consumer, not the GPU, set the step time of the fast pipeline).  Contexts whose
	 * (groups x chains) table would be unreasonable take the comparison sort. */
	const auto t_begin = std::chrono::steady_clock::now();
	const size_t nchain = (size_t)c->cfg.nstreams * c->cfg.nch, nbucket = (gs.size() + 1) * nchain;
	std::vector<unsigned> order(count);
	std::vector<unsigned char> keep(count);             /* 1 = repaired and parity-stripped on the device (k_block_fec) */
	/* test hooks (tests/test_gpu_parity.py): ACB_CONSUMER_SORT=1 forces the comparison sort, ACB_CONSUMER_HELPERS_MIN=n the
	 * helper threads from n frames on */
	const bool force_sort = getenv("ACB_CONSUMER_SORT") && atoi(getenv("ACB_CONSUMER_SORT")) != 0;
	if (!job.groups.off.empty()) {
		/* streams at different positions: each (stream, group) pair of the submit gets its rank in (group number counted
		 * from the stream's start, stream) order; then the bucket pass (or the comparison sort) as below, over
		 * (rank, channel) */
		const auto &off = job.groups.off;
		const auto &base = job.groups.base;
		const unsigned npair = off.back();
		std::vector<unsigned> pair_stream(npair), by_key(npair), rank(npair);
		for (int st = 0; st < c->cfg.nstreams; st++)
			for (unsigned p = off[st]; p < off[st + 1]; p++) pair_stream[p] = (unsigned)st;
		auto gnum = [&](unsigned p) { return base[pair_stream[p]] + (p - off[pair_stream[p]]); };
		for (unsigned p = 0; p < npair; p++) by_key[p] = p;
		std::sort(by_key.begin(), by_key.end(), [&](unsigned a, unsigned b) {
			const unsigned long long ga = gnum(a), gb = gnum(b);
			return ga != gb ? ga < gb : pair_stream[a] < pair_stream[b];
		});
		for (unsigned k = 0; k < npair; k++) rank[by_key[k]] = k;
		/* the pair a frame belongs to: its stream's last group starting at or before it */
		auto pair_of = [&](const RawFrame &f) {
			const auto b = gs.begin() + off[f.stream], e = gs.begin() + off[f.stream + 1];
			const auto it = std::upper_bound(b, e, f.pos);
			return off[f.stream] + (unsigned)(it == b ? 0 : it - b - 1);
		};
		const size_t nb = (size_t)npair * c->cfg.nch;
		if (!force_sort && nb <= ((size_t)1 << 24)) {
			std::vector<unsigned> start(nb + 1, 0u), bucket(count);
			for (unsigned i = 0; i < count; i++) {
				const RawFrame &f = ring[i];
				keep[i] = f.pad0 == 1;
				const size_t bk = (size_t)rank[pair_of(f)] * c->cfg.nch + f.chn;
				bucket[i] = (unsigned)bk;
				start[bk + 1]++;
			}
			for (size_t k = 0; k < nb; k++) start[k + 1] += start[k];
			for (unsigned i = 0; i < count; i++) order[start[bucket[i]]++] = i;
		} else {
			std::vector<unsigned> rk(count);
			for (unsigned i = 0; i < count; i++) { order[i] = i; keep[i] = ring[i].pad0 == 1; rk[i] = rank[pair_of(ring[i])]; }
			std::stable_sort(order.begin(), order.end(), [ring, &rk](unsigned ia, unsigned ib) {
				const RawFrame &x = ring[ia], &y = ring[ib];
				if (rk[ia] != rk[ib]) return rk[ia] < rk[ib];
				if (x.chn != y.chn) return x.chn < y.chn;
				return x.pos < y.pos;
			});
		}
	} else if (!force_sort && nbucket <= ((size_t)1 << 24)) {
		std::vector<unsigned> start(nbucket + 1, 0u), bucket(count);
		for (unsigned i = 0; i < count; i++) {          /* the one pass in ring order: sequential reads */
			const RawFrame &f = ring[i];
			keep[i] = f.pad0 == 1;
			const size_t g = gs.size() == 1 ? (f.pos >= gs[0]) : (size_t)(std::upper_bound(gs.begin(), gs.end(), f.pos) - gs.begin());
			const size_t bk = g * nchain + (size_t)f.stream * c->cfg.nch + f.chn;
			bucket[i] = (unsigned)bk;
			start[bk + 1]++;
		}
		for (size_t k = 0; k < nbucket; k++) start[k + 1] += start[k];
		for (unsigned i = 0; i < count; i++) order[start[bucket[i]]++] = i;
	} else {
		for (unsigned i = 0; i < count; i++) { order[i] = i; keep[i] = ring[i].pad0 == 1; }
		std::stable_sort(order.begin(), order.end(), [ring, &gs](unsigned ia, unsigned ib) {
			const RawFrame &x = ring[ia], &y = ring[ib];
			const size_t gx = (size_t)(std::upper_bound(gs.begin(), gs.end(), x.pos) - gs.begin());
			const size_t gy = (size_t)(std::upper_bound(gs.begin(), gs.end(), y.pos) - gs.begin());
			if (gx != gy) return gx < gy;
			if (x.stream != y.stream) return x.stream < y.stream;
			if (x.chn != y.chn) return x.chn < y.chn;
			return x.pos < y.pos;
		});
	}
	/* The records.  Frames are read in emission order, i.e. at random from an 11 MB ring when a step carries 40 000 of
	 * them: a cache-miss-bound copy (5 ms on one core, more than the GPU needs for the step).  Output slots are fixed
	 * first (a frame the block FEC rejected takes none), then the copy is cut into contiguous ranges of the output,
	 * one helper thread each for large jobs. */
	std::vector<unsigned> slot(count);
	unsigned kept = 0;
	for (unsigned j = 0; j < count; j++) {
		slot[j] = kept;
		kept += keep[order[j]];
	}
	acb_ctx::Batch b;
	b.v.reset(new acb_msg_t[kept ? kept : 1]);
	b.n = kept;
	b.rd = 0;
	const unsigned dropped = count - kept;
	acb_msg_t *out = b.v.get();
	auto fill = [ring, out, &order, &slot, &keep](unsigned j0, unsigned j1) {
		for (unsigned j = j0; j < j1; j++) {
			if (!keep[order[j]]) continue;
			const RawFrame &f = ring[order[j]];
			acb_msg_t &m = out[slot[j]];
			memset(&m, 0, sizeof(m));
			m.stream = f.stream; m.chn = f.chn; m.len = f.len; m.err = f.err;
			m.lvl = (float)(10 * log10(f.lvlsum / f.bitcount));          /* acars.c:351 */
			m.block = f.pos / OUTBLK; m.pos = f.pos; m.soh_pos = f.soh_pos;
			memcpy(m.txt, f.txt, ACB_TXTMAX);
			m.crc[0] = f.crc[0]; m.crc[1] = f.crc[1];
		}
	};
	const unsigned helpers_min = getenv("ACB_CONSUMER_HELPERS_MIN") ? (unsigned)atoi(getenv("ACB_CONSUMER_HELPERS_MIN")) : 8192u;
	const unsigned helpers = count >= helpers_min ? std::min(3u, std::max(1u, std::thread::hardware_concurrency()) - 1u) : 0u;
	if (helpers == 0) {
		fill(0, count);
	} else {
		std::vector<std::thread> pool;
		const unsigned parts = helpers + 1, per = (count + parts - 1) / parts;
		for (unsigned t = 1; t < parts; t++) {
			const unsigned j0 = std::min(count, t * per), j1 = std::min(count, (t + 1) * per);
			try {
				pool.emplace_back(fill, j0, j1);
			} catch (const std::system_error &) {        /* no thread to be had: this one does the range itself */
				fill(j0, j1);
			}
		}
		fill(0, std::min(count, per));
		for (auto &th : pool) th.join();
	}
	if (c->decode_stats) add_decode_stats(c, job, ring, keep.data());     /* before the job counts as done */
	if (c->level_stats) add_level_stats(c, job);
	if (c->freq_stats && job.chan) add_freq_stats(c, job);
	const double ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_begin).count();
	std::lock_guard<std::mutex> lk(c->mtx);
	c->stats.raw_frames += count;
	c->stats.fec_dropped += dropped;
	c->stats.host_ms += ms;
	if (b.n) {
		c->outq_count += b.n;
		c->outq.push_back(std::move(b));
	}
}

static void consumer_main(acb_ctx *c)
{
	cudaSetDevice(c->cfg.device);
	for (;;) {
		acb_ctx::Job job;
		{
			std::unique_lock<std::mutex> lk(c->mtx);
			c->cv_job.wait(lk, [c] { return c->stop || !c->jobs.empty(); });
			if (c->jobs.empty()) return;             /* stop requested and nothing left */
			job = std::move(c->jobs.front());
			c->jobs.pop_front();
		}
		const cudaError_t e = job.count || c->decode_stats || c->dev_stats ? cudaEventSynchronize(c->ev_ring_read[job.ring]) : cudaSuccess;
		if (e == cudaSuccess) consume(c, job);
		{
			std::lock_guard<std::mutex> lk(c->mtx);
			if (e != cudaSuccess && !c->consumer_err[0]) snprintf(c->consumer_err, sizeof(c->consumer_err), "frame read-back: %s", cudaGetErrorString(e));
			c->jobs_done++;
		}
		c->cv_done.notify_all();
	}
}

/* block until the consumer has finished job number `seq` (1-based count of jobs queued so far) */
static void wait_consumer(acb_ctx *c, unsigned long long seq)
{
	std::unique_lock<std::mutex> lk(c->mtx);
	c->cv_done.wait(lk, [c, seq] { return c->jobs_done >= seq; });
}

static int harvest_begin(acb_ctx *c)
{
	if (c->inflight.empty()) return ACB_OK;
	Ticket t = std::move(c->inflight.front());
	c->inflight.pop_front();
	CU(cudaEventSynchronize(t.ev.c));           /* the RingCtl read-back was queued before ev.c */
	float ms = 0;
	if (t.ev.chan && cudaEventElapsedTime(&ms, t.ev.a, t.ev.b) == cudaSuccess) c->stats.chan_ms += ms;
	if (cudaEventElapsedTime(&ms, t.ev.b2, t.ev.c) == cudaSuccess) c->stats.demod_ms += ms;
	c->ev_free.push_back(t.ev);
	unsigned count = c->h_ctl[t.ring]->count;
	const unsigned shortf = c->h_ctl[t.ring]->short_frames;     /* dropped on the device like acars.c:124-129 */
	/* h_ring[ring] was last filled two submits ago: the consumer must be done with it */
	wait_consumer(c, c->ring_job[t.ring]);
	{
		std::lock_guard<std::mutex> lk(c->mtx);
		c->stats.raw_frames += shortf;
		c->stats.fec_dropped += shortf;
		if (count > c->ring_cap) {                   /* reported once by the collecting call; decoding goes on */
			c->overflowed = true;
			c->stats.frames_lost += count - c->ring_cap;
			count = c->ring_cap;
		}
	}
	if (count)
		CU(cudaMemcpyAsync(c->h_ring[t.ring], c->d_ring[t.ring], (size_t)count * sizeof(RawFrame), cudaMemcpyDeviceToHost, c->s_d2h));
	if (c->decode_stats)           /* the submit's demod is done (ev.c follows it): its counters travel with its frames */
		CU(cudaMemcpyAsync(c->h_evcnt[t.ring], c->d_evcnt[t.ring], c->dstats.size() * EV_COUNT * sizeof(unsigned),
		                   cudaMemcpyDeviceToHost, c->s_d2h));
	if (c->dev_stats)              /* the level and frequency kernels run on the channelizer stream: the copies wait for them */
		CU(cudaStreamWaitEvent(c->s_d2h, c->ev_lvl_done[t.ring], 0));
	if (c->level_stats) {
		CU(cudaMemcpyAsync(c->h_lin[t.ring], c->d_lin[t.ring], c->lin.size() * sizeof(LevelIn), cudaMemcpyDeviceToHost, c->s_d2h));
		CU(cudaMemcpyAsync(c->h_lch[t.ring], c->d_lch[t.ring], c->lch.size() * sizeof(LevelChan), cudaMemcpyDeviceToHost, c->s_d2h));
	}
	if (c->freq_stats && t.ev.chan)
		CU(cudaMemcpyAsync(c->h_fch[t.ring], c->d_fch[t.ring], c->fch.size() * sizeof(FreqChan), cudaMemcpyDeviceToHost, c->s_d2h));
	CU(cudaEventRecord(c->ev_ring_read[t.ring], c->s_d2h));
	c->ring_read_pending[t.ring] = true;
	{
		std::lock_guard<std::mutex> lk(c->mtx);
		c->jobs.push_back(acb_ctx::Job{ std::move(t.groups), t.ring, count, t.seq, t.ev.chan });
		c->ring_job[t.ring] = ++c->jobs_queued;
	}
	c->cv_job.notify_one();
	return ACB_OK;
}

/* oldest submit in flight -> output queue, complete on return */
static int collect_oldest(acb_ctx *c)
{
	if (int r = harvest_begin(c)) return r;
	wait_consumer(c, c->jobs_queued);
	if (c->consumer_err[0]) return fail(ACB_ERR_CUDA, "%s", c->consumer_err);
	return ACB_OK;
}

/* ACB_FLAG_LEVEL_STATS / ACB_FLAG_FREQ_STATS: the statistics of the submit using ring b, on the channelizer stream: the
 * input's levels and frequency sums (`in`, NULL for envelope input) and the envelope's levels.  They write that ring's
 * result buffers, so they wait until the read-back of the submit that used it before is done. */
static int run_level(acb_ctx *c, int b, const uint8_t *in, size_t stride, int nsamp, const int *rag)
{
	if (c->ring_read_pending[b]) CU(cudaStreamWaitEvent(c->s_comp, c->ev_ring_read[b], 0));
	int launched = 0, r = 0;
	if (c->level_stats) {
		r = in ? launch_level_input(c->in_kind, in, stride, c->cfg.K, nsamp, rag, c->cfg.nstreams, c->d_lpart, c->lpart_stride, c->d_lin[b],
		                            c->s_comp, launched)
		       : 0;
		if (!r)
			r = launch_level_dm(c->d_dm[b], nsamp, rag, c->cfg.nch, c->cfg.nstreams, c->d_lseg_sum, c->d_lseg_peak, c->cfg.max_blocks + 2,
			                    c->d_lcarry, c->d_lch[b], c->s_comp, launched);
	}
	if (!r && c->freq_stats && in)
		r = launch_freq_input(c->in_kind, in, stride, c->cfg.K, nsamp, rag, c->cfg.nch, c->cfg.nstreams, c->d_fnco, c->d_fon, c->d_fpart,
		                      c->fpart_stride, c->d_fch[b], c->s_comp, launched);
	c->stats.kernel_launches += launched;
	if (r) return fail(ACB_ERR_CUDA, "statistics launch: %s", cudaGetErrorString((cudaError_t)r));
	CU(cudaEventRecord(c->ev_lvl_done[b], c->s_comp));
	return ACB_OK;
}

/* queue K1+K2 (or K2 only) on the compute stream for `nblk` blocks / `nsamp` envelope samples.  Ragged submits (`rag`, a
 * slot of stage_counts, and `h_rows` its host copy): stream s has h_rows[s] <= nsamp rows of its own; K1 computes nsamp
 * rows of every stream, K2 reads each stream's own. */
static int run_kernels(acb_ctx *c, const uint8_t *d_iq, size_t stride, int nblk, int nsamp, const float *dm_host,
                       Groups &&groups, const int *rag = nullptr, const int *h_rows = nullptr)
{
	/* the ring this submit appends to was last used NPIPE submits ago: its frames must be on their
	 * way back before the new demod may clear it — but the host-side work on those frames waits
	 * until the new kernels have been launched */
	while (c->inflight.size() > (size_t)NPIPE)
		if (int r = collect_oldest(c)) return r;
	if (c->inflight.size() == (size_t)NPIPE)
		if (int r = harvest_begin(c)) return r;      /* its frames are the consumer's from here on, whatever happens below */
	/* Input lifetime: when submit N+2 returns, the channelizer of submit N has read its input (host buffer copied,
	 * device buffer consumed) — callers rotating three input buffers, or two with a collect in between, rely on it */
	if (c->nsubmit >= 2) {
		const int b2 = (int)((c->nsubmit - 2) % NPIPE);
		if (c->k1_pending[b2]) {
			CU(cudaEventSynchronize(c->ev_k1_done[b2]));
			c->k1_pending[b2] = false;
		}
	}
	Ticket t;
	t.ring = (int)(c->nsubmit % NPIPE);
	t.groups = std::move(groups);
	t.seq = c->nsubmit;
	t.ev = get_events(c);
	t.ev.chan = d_iq != nullptr;
	const int b = t.ring;                          /* envelope buffer and frame ring of this submit */
	float *dmbuf = c->d_dm[b];
	if (d_iq) {
		/* K1 may overwrite d_dm[b] only after the demod of NPIPE submits ago has read it */
		if (c->dm_used[b]) CU(cudaStreamWaitEvent(c->s_comp, c->ev_dm_free[b], 0));
		CU(cudaEventRecord(t.ev.a, c->s_comp));
		/* the context's form, or EXACT while a stream is not planned on the raster */
		bool fast = c->form != CHAN_EXACT && c->form != CHAN_GENERIC;
		for (int s = 0; fast && s < c->cfg.nstreams; s++) fast = c->fast_ok[s] != 0;
		const ChanForm form = fast || c->form == CHAN_GENERIC ? c->form : CHAN_EXACT;
		/* streams at different positions (acb_reset_stream): the launch takes the furthest one, and the streams near their
		 * start whose window reaches before it are redone below, one by one, at their own position */
		const unsigned long long pos_max = *std::max_element(c->pos.begin(), c->pos.end());
		const bool even_pos = std::all_of(c->pos.begin(), c->pos.end(), [&](unsigned long long p) { return p == pos_max; });
		/* taps > K: where each stream's history sits — the u8 history buffer, or right in front of the input in d_real
		 * for the streaming kinds (submit4), zeros after create / reset */
		const Hist hist = !c->hpad                         ? Hist{ nullptr, 0, 0, pos_max }
		                  : c->in_kind == IN_KIND_U8IQ ? Hist{ c->d_hist, (size_t)c->hpad * 2, c->hpad, pos_max }
		                                               : Hist{ d_iq - (size_t)c->hpad * 4, stride, c->hpad, pos_max };
		ChanLaunch L{ form, c->in_kind, d_iq, stride, hist, c->d_wf, c->d_p, c->d_tw, c->d_twmeta, c->d_wbE, c->d_wbmeta,
		              dmbuf, c->cfg.K, c->taps_pad, c->cfg.nch, c->cfg.nstreams, (size_t)nsamp, c->fold8 };
		int launched = 0;
		int r = launch_chan(L, (size_t)nsamp, c->s_comp, launched);
		/* taps > K, streams near their start.  OVL_FAST and WB omit the window terms before the stream start themselves,
		 * from hist.pos0: at different positions a stream within ceil(hpad / K) rows of its start is redone alone, every
		 * row.  u8 EXACT's block kernel took the zero history bytes (-127.37 after conversion) as terms, and so did
		 * GENERIC's launch at pos_max for the streams behind it: their first ceil(H / K) rows after their start go through
		 * the generic kernel again, which omits those terms — all streams in one launch when they sit at the same position.
		 * The other forms read history that converts to 0, which is the omitted terms exactly. */
		const bool own = form == CHAN_OVL_FAST || form == CHAN_WB;
		if (!r && c->hpad && (own || (c->in_kind == IN_KIND_U8IQ && (form == CHAN_EXACT || form == CHAN_GENERIC)))) {
			const unsigned long long K = (unsigned long long)c->cfg.K, reach = ((own ? c->hpad : c->taps - c->cfg.K) + K - 1) / K;
			L.form = own ? form : CHAN_GENERIC;
			if (even_pos && form == CHAN_EXACT && pos_max < reach)
				r = launch_chan(L, (size_t)std::min<unsigned long long>(reach - pos_max, (unsigned long long)nsamp), c->s_comp, launched);
			for (int s = 0; !r && !even_pos && s < c->cfg.nstreams; s++) {
				const size_t rows = h_rows ? (size_t)h_rows[s] : (size_t)nsamp;
				if (c->pos[s] >= reach || rows == 0) continue;
				r = launch_chan(chan_stream(L, s, c->pos[s]), own ? (size_t)nsamp : std::min<size_t>(reach - c->pos[s], rows), c->s_comp,
				                launched);
			}
		}
		c->stats.kernel_launches += launched;
		if (fast) c->stats.fast_chan_launches++;
		if (c->hpad && c->in_kind == IN_KIND_U8IQ) {
			/* the input's last hpad samples are the next submit's history; the copy follows K1 on the same stream, so
			 * K1 of the next submit sees it and the input-lifetime event below covers it */
			const size_t hb = (size_t)c->hpad * 2, len = (size_t)nblk * c->blk_bytes;
			if (!r && rag) {
				r = launch_hist_gather(d_iq, stride, c->blk_bytes, rag + c->cfg.nstreams, c->d_hist, (int)hb, c->cfg.nstreams, c->s_comp);
				c->stats.kernel_launches++;
			} else if (!r) {
				r = c->cfg.nstreams == 1 ? (int)cudaMemcpyAsync(c->d_hist, d_iq + len - hb, hb, cudaMemcpyDeviceToDevice, c->s_comp)
				                         : (int)cudaMemcpy2DAsync(c->d_hist, hb, d_iq + len - hb, stride, hb, c->cfg.nstreams,
				                                                  cudaMemcpyDeviceToDevice, c->s_comp);
			}
		}
		if (r) return fail(ACB_ERR_CUDA, "channelizer launch: %s", cudaGetErrorString((cudaError_t)r));
		c->stats.chan_launches++;
		CU(cudaEventRecord(t.ev.b, c->s_comp));
		CU(cudaEventRecord(c->ev_k1_done[b], c->s_comp));
		c->k1_pending[b] = true;
		CU(cudaStreamWaitEvent(c->s_dem, c->ev_k1_done[b], 0));
		if (c->dev_stats) {
			/* behind K1, beside the demod; the input-lifetime event moves behind them, as they read the input too */
			if (int r2 = run_level(c, b, d_iq, stride, nsamp, rag)) return r2;
			CU(cudaEventRecord(c->ev_k1_done[b], c->s_comp));
		}
	} else if (dm_host) {
		/* envelope input: the copy is ordered behind the previous demod on the same stream, and
		 * behind any channelizer launch that still targets the other buffer only */
		if (c->level_stats) {      /* and behind the level kernels, which may still read this buffer */
			CU(cudaEventRecord(c->ev_join, c->s_comp));
			CU(cudaStreamWaitEvent(c->s_dem, c->ev_join, 0));
		}
		CU(cudaMemcpyAsync(dmbuf, dm_host, (size_t)c->cfg.nstreams * nsamp * c->cfg.nch * sizeof(float), cudaMemcpyHostToDevice, c->s_dem));
		if (c->level_stats) {
			CU(cudaEventRecord(c->ev_join, c->s_dem));
			CU(cudaStreamWaitEvent(c->s_comp, c->ev_join, 0));
			if (int r2 = run_level(c, b, nullptr, 0, nsamp, nullptr)) return r2;
		}
	}
	if (c->ring_read_pending[b]) {
		CU(cudaStreamWaitEvent(c->s_dem, c->ev_ring_read[b], 0));
		c->ring_read_pending[b] = false;
	}
	CU(cudaMemsetAsync(c->d_ctl[b], 0, sizeof(RingCtl), c->s_dem));
	if (c->decode_stats) CU(cudaMemsetAsync(c->d_evcnt[b], 0, c->dstats.size() * EV_COUNT * sizeof(unsigned), c->s_dem));
	CU(cudaEventRecord(t.ev.b2, c->s_dem));
	int r = c->decode_stats ? launch_demod_stats(c->d_state, dmbuf, nsamp, c->cfg.nch, c->cfg.nstreams, c->d_ring[b], c->d_ctl[b],
	                                             c->ring_cap, c->demod_lanes, c->d_evcnt[b], c->s_dem, rag)
	                        : launch_demod(c->d_state, dmbuf, nsamp, c->cfg.nch, c->cfg.nstreams, c->d_ring[b], c->d_ctl[b], c->ring_cap,
	                                       c->demod_lanes, c->s_dem, rag);
	if (r) return fail(ACB_ERR_CUDA, "demod launch: %s", cudaGetErrorString((cudaError_t)r));
	c->stats.kernel_launches++;
	c->stats.demod_launches++;
	CU(cudaEventRecord(c->ev_dm_free[b], c->s_dem));       /* the envelope buffer is the next-but-two channelizer's from here */
	CU(cudaEventRecord(c->ev_k2_done[b], c->s_dem));
	/* block FEC on the frames this submit appended (blk_thread's job, acars.c:93-215), in place — on its own stream:
	 * it touches this submit's ring only, and the next demod need not wait behind it */
	CU(cudaStreamWaitEvent(c->s_fec, c->ev_k2_done[b], 0));
	r = c->decode_stats ? launch_block_fec_stats(c->d_ring[b], c->d_ctl[b], c->ring_cap, c->s_fec)
	                    : launch_block_fec(c->d_ring[b], c->d_ctl[b], c->ring_cap, c->s_fec);
	if (r) return fail(ACB_ERR_CUDA, "block FEC launch: %s", cudaGetErrorString((cudaError_t)r));
	c->stats.kernel_launches++;
	CU(cudaMemcpyAsync(c->h_ctl[b], c->d_ctl[b], sizeof(RingCtl), cudaMemcpyDeviceToHost, c->s_fec));
	CU(cudaEventRecord(t.ev.c, c->s_fec));
	c->dm_used[b] = true;
	c->last_dm = b;
	c->inflight.push_back(std::move(t));
	c->nsubmit++;
	c->stats.submits++;
	c->last_nsamp = nsamp;
	return ACB_OK;
}

static int check_blocks(acb_ctx *c, const void *p, size_t stride, int nblk)
{
	if (!c || !p) return fail(ACB_ERR_ARG, "null argument");
	if (c->real_input) return fail(ACB_ERR_ARG, "not a u8-IQ context: use acb_submit_real_host / acb_submit_cs16_host");
	if (nblk < 1 || nblk > c->cfg.max_blocks) return fail(ACB_ERR_ARG, "nblk=%d outside 1..%d", nblk, c->cfg.max_blocks);
	if (c->cfg.nstreams > 1 && stride < (size_t)nblk * c->blk_bytes) return fail(ACB_ERR_ARG, "stream_stride smaller than one stream's input");
	if (stride % 16) return fail(ACB_ERR_ARG, "stream_stride must be a multiple of 16 bytes");
	return ACB_OK;
}

/* the ragged calls' counts: each 0..max_blocks, not all 0; `maxb` = the largest, which the stride must hold */
static int check_blocks_ragged(acb_ctx *c, const void *p, size_t stride, const int *nblk, int &maxb)
{
	if (!c || !p || !nblk) return fail(ACB_ERR_ARG, "null argument");
	if (c->real_input) return fail(ACB_ERR_ARG, "not a u8-IQ context: use acb_submit_real_host_ragged / acb_submit_cs16_host_ragged");
	maxb = 0;
	for (int s = 0; s < c->cfg.nstreams; s++) {
		if (nblk[s] < 0 || nblk[s] > c->cfg.max_blocks) return fail(ACB_ERR_ARG, "nblk[%d]=%d outside 0..%d", s, nblk[s], c->cfg.max_blocks);
		maxb = std::max(maxb, nblk[s]);
	}
	if (maxb == 0) return fail(ACB_ERR_ARG, "every stream's nblk is 0");
	if (c->cfg.nstreams > 1 && stride < (size_t)maxb * c->blk_bytes) return fail(ACB_ERR_ARG, "stream_stride smaller than the largest input");
	if (stride % 16) return fail(ACB_ERR_ARG, "stream_stride must be a multiple of 16 bytes");
	return ACB_OK;
}

/* The number, counted from the stream's start, of the emission group that holds envelope sample `pos`: its 1024-row block
 * (u8), or the groups of stream_groups — one per `period` outputs (ACB_GROUP_OUTPUTS), or the first output completed in
 * each transfer of `period` input samples (ACB_GROUP_INPUT: the transfers' first outputs floor(t*T/K), t >= 1, in (0, pos]);
 * ACB_GROUP_SUBMIT has one group per submit and numbers none. */
unsigned long long acb::group_number(bool u8, int unit, unsigned long long period, int Kc, unsigned long long pos)
{
	if (u8) return pos / OUTBLK;
	const unsigned long long T = period, K = (unsigned long long)Kc;
	if (unit == ACB_GROUP_OUTPUTS) return pos / T;
	if (unit == ACB_GROUP_INPUT) return T >= K ? ((pos + 1) * K - 1) / T : pos;
	return 0;
}

/* The emission groups of a submit in which stream s brings rows[s] envelope rows (u8: whole blocks of 1024) */
static Groups submit_groups(const acb_ctx *c, const std::vector<size_t> &rows)
{
	auto of = [c](unsigned long long pos, size_t n) {
		if (c->real_input) return stream_groups(c->group_unit, c->group_period, c->cfg.K, pos, n);
		std::vector<unsigned long long> g(n / OUTBLK);
		for (size_t b = 0; b < g.size(); b++) g[b] = pos + (unsigned long long)b * OUTBLK;
		return g;
	};
	Groups g;
	const int n = c->cfg.nstreams;
	if (std::all_of(c->pos.begin(), c->pos.end(), [c](unsigned long long p) { return p == c->pos[0]; })) {
		g.starts = of(c->pos[0], *std::max_element(rows.begin(), rows.end()));
		return g;
	}
	g.off.assign(n + 1, 0u);
	g.base.assign(n, 0ull);
	for (int s = 0; s < n; s++) {
		if (rows[s]) {
			const auto v = of(c->pos[s], rows[s]);
			g.starts.insert(g.starts.end(), v.begin(), v.end());
			g.base[s] = group_number(!c->real_input, c->group_unit, c->group_period, c->cfg.K, c->pos[s]);
		}
		g.off[s + 1] = (unsigned)g.starts.size();
	}
	return g;
}

/* Ragged submits' counts travel in a slot of 4 * nstreams ints: [rows | a | b | c], where u8 puts its block counts in a
 * and the streaming kinds each stream's carry, new samples and remainder in a, b, c.  stage_begin hands out the next
 * slot once the work that read it last is done; stage_upload copies it on the copy stream and orders the channelizer
 * stream behind it; stage_end marks the streams that read it. */
static int stage_begin(acb_ctx *c, int &slot)
{
	slot = (int)(c->rag_seq++ % NRAG);
	if (c->rag_used[slot])
		for (auto &e : c->ev_rag_used[slot]) CU(cudaEventSynchronize(e));
	c->rag_used[slot] = false;
	return ACB_OK;
}

static int stage_upload(acb_ctx *c, int slot)
{
	CU(cudaMemcpyAsync(c->d_rag[slot], c->h_rag[slot], 4 * (size_t)c->cfg.nstreams * sizeof(int), cudaMemcpyHostToDevice, c->s_copy));
	CU(cudaEventRecord(c->ev_rag_used[slot][0], c->s_copy));
	CU(cudaStreamWaitEvent(c->s_comp, c->ev_rag_used[slot][0], 0));
	return ACB_OK;
}

static int stage_end(acb_ctx *c, int slot)
{
	CU(cudaEventRecord(c->ev_rag_used[slot][0], c->s_copy));
	CU(cudaEventRecord(c->ev_rag_used[slot][1], c->s_comp));
	CU(cudaEventRecord(c->ev_rag_used[slot][2], c->s_dem));
	c->rag_used[slot] = true;
	return ACB_OK;
}

/* Host rows of `elem`-byte samples into a device buffer of row pitch `dpitch`: stream s brings cnt[s].  Even counts are
 * one 2D copy.  Otherwise every stream but the last is copied at the largest count (its row in the caller's buffer is at
 * least that long: the stride holds it) and the last at its own, so nothing past the caller's input is read. */
static int copy_rows(acb_ctx *c, void *dst, size_t dpitch, const void *src, size_t spitch, const std::vector<size_t> &cnt, size_t elem,
                     bool even)
{
	const int n = c->cfg.nstreams;
	if (even) {
		CU(cudaMemcpy2DAsync(dst, dpitch, src, spitch, cnt[0] * elem, n, cudaMemcpyHostToDevice, c->s_copy));
		return ACB_OK;
	}
	const size_t wmax = *std::max_element(cnt.begin(), cnt.end()) * elem;
	CU(cudaMemcpy2DAsync(dst, dpitch, src, spitch, wmax, n - 1, cudaMemcpyHostToDevice, c->s_copy));
	if (cnt[n - 1])
		CU(cudaMemcpyAsync((char *)dst + (size_t)(n - 1) * dpitch, (const char *)src + (size_t)(n - 1) * spitch, cnt[n - 1] * elem,
		                   cudaMemcpyHostToDevice, c->s_copy));
	return ACB_OK;
}

/* u8 IQ submits: `nblk` blocks for every stream, or (nblk_s != NULL, the ragged calls) nblk_s[s] for stream s, nblk the
 * largest.  The channelizer runs nblk blocks of every stream; each stream's demodulator takes its own. */
static int submit_blocks(acb_ctx *c, const uint8_t *iq, size_t stride, int nblk, const int *nblk_s, bool dev)
{
	if (int r = ctx_use(c)) return r;
	if (dev && ((uintptr_t)iq) % 16) return fail(ACB_ERR_ARG, "device input must be 16-byte aligned");
	if (!dev && !c->d_iq[0]) return fail(ACB_ERR_ARG, "context created with ACB_FLAG_NO_INPUT_STAGING");
	const int n = c->cfg.nstreams;
	bool even = true;
	for (int s = 0; nblk_s && s < n; s++) even = even && nblk_s[s] == nblk;
	std::vector<size_t> rows(n, (size_t)nblk * OUTBLK), bytes(n, (size_t)nblk * c->blk_bytes);
	for (int s = 0; !even && s < n; s++) rows[s] = (size_t)nblk_s[s] * OUTBLK, bytes[s] = (size_t)nblk_s[s] * c->blk_bytes;
	int slot = -1;
	if (!even) {
		if (int r = stage_begin(c, slot)) return r;
		for (int s = 0; s < n; s++) c->h_rag[slot][s] = (int)rows[s], c->h_rag[slot][n + s] = nblk_s[s];
		if (int r = stage_upload(c, slot)) return r;
	}
	const int b = c->next_buf;
	const size_t per_stream = (size_t)nblk * c->blk_bytes;
	if (!dev) {
		c->next_buf ^= 1;
		/* the kernels that last read this staging buffer must be done before it is overwritten */
		if (c->buf_used[b]) CU(cudaStreamWaitEvent(c->s_copy, c->ev_consumed[b], 0));
		if (even && (stride == per_stream || n == 1)) {
			CU(cudaMemcpyAsync(c->d_iq[b], iq, per_stream * n, cudaMemcpyHostToDevice, c->s_copy));
		} else if (int r = copy_rows(c, c->d_iq[b], per_stream, iq, stride, bytes, 1, even)) {
			return r;
		}
		CU(cudaEventRecord(c->ev_copied[b], c->s_copy));
		CU(cudaStreamWaitEvent(c->s_comp, c->ev_copied[b], 0));
	}
	if (int r = run_kernels(c, dev ? iq : c->d_iq[b], dev ? stride : per_stream, nblk, nblk * OUTBLK, nullptr, submit_groups(c, rows),
	                        even ? nullptr : c->d_rag[slot], even ? nullptr : c->h_rag[slot]))
		return r;
	if (!dev) {
		CU(cudaEventRecord(c->ev_consumed[b], c->s_comp));      /* staging buffer is free once K1 has read it */
		c->buf_used[b] = true;
	}
	if (!even)
		if (int r = stage_end(c, slot)) return r;
	for (int s = 0; s < n; s++) {
		c->pos[s] += rows[s];
		c->stats.blocks += rows[s] / OUTBLK;
	}
	return ACB_OK;
}

extern "C" int acb_submit_device(acb_ctx_t *c, const uint8_t *iq_dev, size_t stride, int nblk)
{
	if (int r = check_blocks(c, iq_dev, stride, nblk)) return r;
	return submit_blocks(c, iq_dev, stride, nblk, nullptr, true);
}

extern "C" int acb_submit_host(acb_ctx_t *c, const uint8_t *iq, size_t stride, int nblk)
{
	if (int r = check_blocks(c, iq, stride, nblk)) return r;
	return submit_blocks(c, iq, stride, nblk, nullptr, false);
}

extern "C" int acb_submit_device_ragged(acb_ctx_t *c, const uint8_t *iq_dev, size_t stride, const int *nblk)
{
	int maxb = 0;
	if (int r = check_blocks_ragged(c, iq_dev, stride, nblk, maxb)) return r;
	return submit_blocks(c, iq_dev, stride, maxb, nblk, true);
}

extern "C" int acb_submit_host_ragged(acb_ctx_t *c, const uint8_t *iq, size_t stride, const int *nblk)
{
	int maxb = 0;
	if (int r = check_blocks_ragged(c, iq, stride, nblk, maxb)) return r;
	return submit_blocks(c, iq, stride, maxb, nblk, false);
}

extern "C" int acb_set_emission_groups(acb_ctx_t *c, int unit, uint64_t period)
{
	if (!c) return fail(ACB_ERR_ARG, "null context");
	if (unit != ACB_GROUP_SUBMIT && unit != ACB_GROUP_OUTPUTS && unit != ACB_GROUP_INPUT) return fail(ACB_ERR_ARG, "unknown group unit");
	if (unit != ACB_GROUP_SUBMIT && period == 0) return fail(ACB_ERR_ARG, "period must be > 0");
	c->group_unit = unit;
	c->group_period = period;
	return ACB_OK;
}

/* Emission groups of one streaming submit covering envelope samples [pos, pos + nout): the reference hands a
 * channel's new samples to demodMSK per transfer (air.c:336: output m completes with input sample (m+1)K - 1, so
 * transfer g of T samples starts at output floor(g*T/K)) or per full dm_buffer (soapy.c:247 every 1024 outputs,
 * sdrplay.c:229 every 512), channel by channel: frames leave in (group, channel, time) order.  acb_multi_* keys its merge
 * on the same starts. */
std::vector<unsigned long long> acb::stream_groups(int unit, unsigned long long period, int Kc, unsigned long long pos, size_t nout)
{
	std::vector<unsigned long long> g{ pos };
	const unsigned long long lo = pos, hi = pos + nout, K = (unsigned long long)Kc;
	if (unit == ACB_GROUP_OUTPUTS) {
		for (unsigned long long b = (lo / period + 1) * period; b < hi; b += period) g.push_back(b);
	} else if (unit == ACB_GROUP_INPUT) {
		const unsigned long long T = period;
		for (unsigned long long t = (lo * K) / T + 1;; t++) {        /* transfers that start after output `lo` began */
			const unsigned long long b = t * T / K;                  /* first output completed inside transfer t */
			if (b >= hi) break;
			if (b > g.back()) g.push_back(b);
		}
	}
	return g;
}

/* 4-byte samples (float32 real or int16 I,Q) of arbitrary count: appended behind the carried
 * remainder in d_real[b]; `x2` != NULL means planar int16 input (x = I plane, x2 = Q plane), which
 * is interleaved on the way.  `dev`: the input is in device memory (the device calls) and one append
 * kernel moves it; otherwise strided host copies bring it over.  Everything else is the same for both.
 * `ns` != NULL (the ragged calls): stream s brings ns[s] samples and its rows go to nout[s] (may be NULL); streams whose
 * counts and carries all agree take the lockstep path. */
static int submit4(acb_ctx *c, const void *x, const void *x2, bool dev, size_t stride_samples, size_t nsamples,
                   const size_t *ns = nullptr, size_t *nout_s = nullptr)
{
	if (int r = ctx_use(c)) return r;
	const int n = c->cfg.nstreams;
	const size_t K = (size_t)c->cfg.K, hp = (size_t)c->hpad;
	std::vector<size_t> cnt(n), rows(n), rem(n);
	size_t nmax = 0, omax = 0;
	bool even = true;
	for (int s = 0; s < n; s++) {
		cnt[s] = ns ? ns[s] : nsamples;
		const size_t total = c->carry[s] + cnt[s];
		rows[s] = total / K;
		rem[s] = total - rows[s] * K;
		if ((!ns && nsamples == 0) || hp + total > c->real_cap || rows[s] > (size_t)c->cfg.max_blocks * OUTBLK)
			return ns ? fail(ACB_ERR_ARG, "nsamples[%d]=%zu exceeds max_blocks*1024*K", s, cnt[s])
			          : fail(ACB_ERR_ARG, "nsamples=%zu exceeds max_blocks*1024*K", nsamples);
		if (cnt[s] > (size_t)INT32_MAX) return fail(ACB_ERR_ARG, "nsamples[%d]=%zu exceeds 2^31 - 1", s, cnt[s]);
		nmax = std::max(nmax, cnt[s]);
		omax = std::max(omax, rows[s]);
		even = even && cnt[s] == cnt[0] && c->carry[s] == c->carry[0];
	}
	if (nmax == 0) return fail(ACB_ERR_ARG, "every stream's nsamples is 0");
	if (even) nsamples = cnt[0];              /* a ragged call with equal counts and carries is the lockstep call */
	if (n > 1 && stride_samples < nmax) return fail(ACB_ERR_ARG, "stream stride smaller than one stream's input");
	const int b = c->real_buf;
	/* The copy runs on the copy stream, so the H2D of submit i+1 overlaps the channelizer of submit i.
	 * d_real[b] was last read by the channelizer two submits ago and by the copy that moved its tail on.
	 * taps > K: the first hp samples of each stream are its history, rows start behind them. */
	float *const buf0 = c->d_real[b], *const buf = buf0 + hp;
	int slot = -1;
	const int *rag = nullptr;
	if (!even) {
		if (int r = stage_begin(c, slot)) return r;
		int *h = c->h_rag[slot];
		for (int s = 0; s < n; s++) h[s] = (int)rows[s], h[n + s] = (int)c->carry[s], h[2 * n + s] = (int)cnt[s], h[3 * n + s] = (int)rem[s];
		rag = c->d_rag[slot];
	}
	if (c->real_used[b]) CU(cudaStreamWaitEvent(c->s_copy, c->ev_real_free[b], 0));
	if (!even)
		if (int r = stage_upload(c, slot)) return r;
	uint32_t *const dst = reinterpret_cast<uint32_t *>(buf);
	if (dev) {
		/* acb_wait_event: the caller's producer must be done before the append reads the input */
		if (c->order_pending) {
			CU(cudaStreamWaitEvent(c->s_copy, c->ev_order, 0));
			c->order_pending = false;
		}
		int r = even ? launch_append4(x, x2, stride_samples, dst + c->carry[0], c->real_cap, nsamples, n, c->s_copy)
		             : launch_append4_ragged(x, x2, stride_samples, dst, c->real_cap, rag + n, rag + 2 * n, nmax, n, c->s_copy);
		if (r) return fail(ACB_ERR_CUDA, "append launch: %s", cudaGetErrorString((cudaError_t)r));
		c->stats.kernel_launches++;
	} else if (!x2 && even) {
		CU(cudaMemcpy2DAsync(buf + c->carry[0], c->real_cap * sizeof(float), x, stride_samples * sizeof(float),
		                     nsamples * sizeof(float), n, cudaMemcpyHostToDevice, c->s_copy));
	} else {
		/* planar int16 (the SDRplay callback's xi / xq): both planes go over as they are (two dense copies),
		 * a small kernel interleaves them behind the carried remainder.  Ragged interleaved input goes over the same
		 * way, as 4-byte samples, and the ragged append puts each stream behind its own carry. */
		if (nmax > c->planar_cap) {
			CU(cudaStreamSynchronize(c->s_copy));
			cudaFree(c->d_planar);
			c->d_planar = nullptr;
			c->planar_cap = std::max(nmax, (size_t)c->cfg.max_blocks * OUTBLK * K);
			CU(cudaMalloc(&c->d_planar, 2 * (size_t)n * c->planar_cap * sizeof(int16_t)));
		}
		int r = 0;
		if (!x2) {
			uint32_t *stg = reinterpret_cast<uint32_t *>(c->d_planar);
			if (int e = copy_rows(c, stg, c->planar_cap * 4, x, stride_samples * 4, cnt, 4, false)) return e;
			r = launch_append4_ragged(stg, nullptr, c->planar_cap, dst, c->real_cap, rag + n, rag + 2 * n, nmax, n, c->s_copy);
		} else {
			int16_t *pi = c->d_planar, *pq = c->d_planar + (size_t)n * c->planar_cap;
			if (int e = copy_rows(c, pi, c->planar_cap * 2, x, stride_samples * 2, cnt, 2, even)) return e;
			if (int e = copy_rows(c, pq, c->planar_cap * 2, x2, stride_samples * 2, cnt, 2, even)) return e;
			r = even ? launch_interleave_cs16(pi, pq, c->planar_cap, dst + c->carry[0], c->real_cap, nsamples, n, c->s_copy)
			         : launch_append4_ragged(pi, pq, c->planar_cap, dst, c->real_cap, rag + n, rag + 2 * n, nmax, n, c->s_copy);
		}
		if (r) return fail(ACB_ERR_CUDA, "interleave launch: %s", cudaGetErrorString((cudaError_t)r));
		c->stats.kernel_launches++;
	}
	CU(cudaEventRecord(c->ev_real_copied, c->s_copy));
	CU(cudaStreamWaitEvent(c->s_comp, c->ev_real_copied, 0));
	if (omax) {
		if (int r = run_kernels(c, (const uint8_t *)buf, c->real_cap * sizeof(float), 0, (int)omax, nullptr, submit_groups(c, rows), rag,
		                        even ? nullptr : c->h_rag[slot]))
			return r;
		/* the unconsumed tail (air.c:329-334 / soapy.c:238-252 keep a partial sum instead: same
		 * arithmetic order) moves to the front of the other buffer, behind the hp samples before it (the next
		 * submit's history, taps > K) */
		if (even && rem[0] + hp) {
			if (c->real_used[b ^ 1]) CU(cudaStreamWaitEvent(c->s_comp, c->ev_real_free[b ^ 1], 0));
			CU(cudaMemcpy2DAsync(c->d_real[b ^ 1], c->real_cap * sizeof(float), buf + omax * K - hp, c->real_cap * sizeof(float),
			                     (hp + rem[0]) * sizeof(float), n, cudaMemcpyDeviceToDevice, c->s_comp));
		} else if (!even) {
			if (c->real_used[b ^ 1]) CU(cudaStreamWaitEvent(c->s_comp, c->ev_real_free[b ^ 1], 0));
			int r = launch_move_tail(reinterpret_cast<const uint32_t *>(buf0), reinterpret_cast<uint32_t *>(c->d_real[b ^ 1]), c->real_cap,
			                         c->cfg.K, c->hpad, rag, rag + 3 * n, n, c->s_comp);
			if (r) return fail(ACB_ERR_CUDA, "tail move launch: %s", cudaGetErrorString((cudaError_t)r));
			c->stats.kernel_launches++;
		}
		CU(cudaEventRecord(c->ev_real_free[b], c->s_comp));
		c->real_used[b] = true;
		c->real_buf = b ^ 1;
	}
	if (!even)
		if (int r = stage_end(c, slot)) return r;
	for (int s = 0; s < n; s++) {
		c->pos[s] += rows[s];
		c->carry[s] = rem[s];          /* no row: the samples simply stay behind the previous carry */
		if (nout_s) nout_s[s] = rows[s];
	}
	return (int)omax;
}

extern "C" int acb_submit_real_host(acb_ctx_t *c, const float *x, size_t stride_samples, size_t nsamples)
{
	if (!c || !x) return fail(ACB_ERR_ARG, "null argument");
	if (c->in_kind != IN_KIND_F32REAL) return fail(ACB_ERR_ARG, "context was not created with ACB_FLAG_REAL_INPUT");
	return submit4(c, x, nullptr, false, stride_samples, nsamples);
}

extern "C" int acb_submit_cs16_host(acb_ctx_t *c, const int16_t *iq, size_t stride_samples, size_t nsamples)
{
	if (!c || !iq) return fail(ACB_ERR_ARG, "null argument");
	if (c->in_kind != IN_KIND_CS16IQ) return fail(ACB_ERR_ARG, "context was not created with ACB_FLAG_CS16_INPUT");
	return submit4(c, iq, nullptr, false, stride_samples, nsamples);
}

extern "C" int acb_submit_cs16_planar_host(acb_ctx_t *c, const int16_t *xi, const int16_t *xq, size_t stride_samples, size_t nsamples)
{
	if (!c || !xi || !xq) return fail(ACB_ERR_ARG, "null argument");
	if (c->in_kind != IN_KIND_CS16IQ) return fail(ACB_ERR_ARG, "context was not created with ACB_FLAG_CS16_INPUT");
	return submit4(c, xi, xq, false, stride_samples, nsamples);
}

/* The device calls take device memory of the context's device, or managed memory, only: host memory (pinned or
 * pageable) has the host calls, and another device's memory would be read over the peer link if at all. */
static int check_device_input(acb_ctx *c, const void *p, size_t align)
{
	if ((uintptr_t)p % align) return fail(ACB_ERR_ARG, "device input must be %zu-byte aligned", align);
	cudaPointerAttributes a;
	if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
		cudaGetLastError();                         /* not sticky: clear it so the next call does not report it */
		return fail(ACB_ERR_ARG, "input is not memory CUDA knows");
	}
	if (a.type == cudaMemoryTypeManaged || (a.type == cudaMemoryTypeDevice && a.device == c->cfg.device)) return ACB_OK;
	if (a.type == cudaMemoryTypeDevice)
		return fail(ACB_ERR_ARG, "input is on device %d, the context on device %d", a.device, c->cfg.device);
	return fail(ACB_ERR_ARG, "input is host memory: use the host call");
}

extern "C" int acb_submit_real_device(acb_ctx_t *c, const float *x_dev, size_t stride_samples, size_t nsamples)
{
	if (!c || !x_dev) return fail(ACB_ERR_ARG, "null argument");
	if (c->in_kind != IN_KIND_F32REAL) return fail(ACB_ERR_ARG, "context was not created with ACB_FLAG_REAL_INPUT");
	if (int r = check_device_input(c, x_dev, 4)) return r;
	return submit4(c, x_dev, nullptr, true, stride_samples, nsamples);
}

extern "C" int acb_submit_cs16_device(acb_ctx_t *c, const int16_t *iq_dev, size_t stride_samples, size_t nsamples)
{
	if (!c || !iq_dev) return fail(ACB_ERR_ARG, "null argument");
	if (c->in_kind != IN_KIND_CS16IQ) return fail(ACB_ERR_ARG, "context was not created with ACB_FLAG_CS16_INPUT");
	if (int r = check_device_input(c, iq_dev, 4)) return r;
	return submit4(c, iq_dev, nullptr, true, stride_samples, nsamples);
}

extern "C" int acb_submit_cs16_planar_device(acb_ctx_t *c, const int16_t *xi_dev, const int16_t *xq_dev, size_t stride_samples,
                                             size_t nsamples)
{
	if (!c || !xi_dev || !xq_dev) return fail(ACB_ERR_ARG, "null argument");
	if (c->in_kind != IN_KIND_CS16IQ) return fail(ACB_ERR_ARG, "context was not created with ACB_FLAG_CS16_INPUT");
	if (int r = check_device_input(c, xi_dev, 2)) return r;
	if (int r = check_device_input(c, xq_dev, 2)) return r;
	return submit4(c, xi_dev, xq_dev, true, stride_samples, nsamples);
}

/* the ragged forms: the same calls with a count per stream */
extern "C" int acb_submit_real_host_ragged(acb_ctx_t *c, const float *x, size_t stride_samples, const size_t *nsamples, size_t *nout)
{
	if (!c || !x || !nsamples) return fail(ACB_ERR_ARG, "null argument");
	if (c->in_kind != IN_KIND_F32REAL) return fail(ACB_ERR_ARG, "context was not created with ACB_FLAG_REAL_INPUT");
	return submit4(c, x, nullptr, false, stride_samples, 0, nsamples, nout);
}

extern "C" int acb_submit_cs16_host_ragged(acb_ctx_t *c, const int16_t *iq, size_t stride_samples, const size_t *nsamples, size_t *nout)
{
	if (!c || !iq || !nsamples) return fail(ACB_ERR_ARG, "null argument");
	if (c->in_kind != IN_KIND_CS16IQ) return fail(ACB_ERR_ARG, "context was not created with ACB_FLAG_CS16_INPUT");
	return submit4(c, iq, nullptr, false, stride_samples, 0, nsamples, nout);
}

extern "C" int acb_submit_cs16_planar_host_ragged(acb_ctx_t *c, const int16_t *xi, const int16_t *xq, size_t stride_samples,
                                                  const size_t *nsamples, size_t *nout)
{
	if (!c || !xi || !xq || !nsamples) return fail(ACB_ERR_ARG, "null argument");
	if (c->in_kind != IN_KIND_CS16IQ) return fail(ACB_ERR_ARG, "context was not created with ACB_FLAG_CS16_INPUT");
	return submit4(c, xi, xq, false, stride_samples, 0, nsamples, nout);
}

extern "C" int acb_submit_real_device_ragged(acb_ctx_t *c, const float *x_dev, size_t stride_samples, const size_t *nsamples, size_t *nout)
{
	if (!c || !x_dev || !nsamples) return fail(ACB_ERR_ARG, "null argument");
	if (c->in_kind != IN_KIND_F32REAL) return fail(ACB_ERR_ARG, "context was not created with ACB_FLAG_REAL_INPUT");
	if (int r = check_device_input(c, x_dev, 4)) return r;
	return submit4(c, x_dev, nullptr, true, stride_samples, 0, nsamples, nout);
}

extern "C" int acb_submit_cs16_device_ragged(acb_ctx_t *c, const int16_t *iq_dev, size_t stride_samples, const size_t *nsamples,
                                             size_t *nout)
{
	if (!c || !iq_dev || !nsamples) return fail(ACB_ERR_ARG, "null argument");
	if (c->in_kind != IN_KIND_CS16IQ) return fail(ACB_ERR_ARG, "context was not created with ACB_FLAG_CS16_INPUT");
	if (int r = check_device_input(c, iq_dev, 4)) return r;
	return submit4(c, iq_dev, nullptr, true, stride_samples, 0, nsamples, nout);
}

extern "C" int acb_submit_cs16_planar_device_ragged(acb_ctx_t *c, const int16_t *xi_dev, const int16_t *xq_dev, size_t stride_samples,
                                                    const size_t *nsamples, size_t *nout)
{
	if (!c || !xi_dev || !xq_dev || !nsamples) return fail(ACB_ERR_ARG, "null argument");
	if (c->in_kind != IN_KIND_CS16IQ) return fail(ACB_ERR_ARG, "context was not created with ACB_FLAG_CS16_INPUT");
	if (int r = check_device_input(c, xi_dev, 2)) return r;
	if (int r = check_device_input(c, xq_dev, 2)) return r;
	return submit4(c, xi_dev, xq_dev, true, stride_samples, 0, nsamples, nout);
}

extern "C" int acb_set_plan_cs16(acb_ctx_t *c, int stream, const unsigned *freqs_hz, int nch, int variant, unsigned fc_hz, unsigned *fc_out)
{
	if (!c || !freqs_hz) return fail(ACB_ERR_ARG, "null argument");
	if (c->in_kind != IN_KIND_CS16IQ || nch != c->cfg.nch) return fail(ACB_ERR_ARG, "not a CS16 context / nch mismatch");
	if (c->taps < c->cfg.K) return fail(ACB_ERR_ARG, "taps < K: supply the tables with acb_set_wf");
	if (variant != ACB_CS16_SOAPY && variant != ACB_CS16_SDRPLAY) return fail(ACB_ERR_ARG, "unknown CS16 variant");
	const unsigned fc = fc_hz ? fc_hz : acb_choose_fc(freqs_hz, nch, c->cfg.K);      /* soapy.c:132-136, sdrplay.c:124 */
	if (fc == 0) return fail(ACB_ERR_PLAN, "Frequencies too far apart");
	if (fc_out) *fc_out = fc;
	const int K = c->cfg.K, T = c->taps;
	return plan_stream(c, stream, [&](int ch, float *wf) {
		if (c->hpad) acb_cs16_build_wf_lp(variant, freqs_hz[ch], fc, K, T, wf);
		else acb_cs16_build_wf(variant, freqs_hz[ch], fc, K, wf);
	}, [&](int *kbin, float *tw1) { return acb_fast_plan_cs16(variant, freqs_hz, nch, K, fc, kbin, tw1); }, variant,
	(double)fc, [&](int ch) { return (double)((float)freqs_hz[ch] - (float)fc); });
}

static int check_plan_air(acb_ctx *c, const unsigned *freqs_hz, int nch)
{
	if (!c || !freqs_hz) return fail(ACB_ERR_ARG, "null argument");
	if (c->in_kind != IN_KIND_F32REAL || nch != c->cfg.nch) return fail(ACB_ERR_ARG, "not a real-input context / nch mismatch");
	if (c->taps < c->cfg.K) return fail(ACB_ERR_ARG, "taps < K: supply the tables with acb_set_wf");
	return ACB_OK;
}

/* the tables and fast plans of a real-input stream around a given Fc (air.c:263-285) */
static int plan_air(acb_ctx *c, int stream, const unsigned *freqs_hz, int nch, unsigned fc)
{
	const unsigned rate = (unsigned)c->cfg.K * ACB_INTRATE;
	const int T = c->taps;
	return plan_stream(c, stream, [&](int ch, float *wf) {
		if (c->hpad) acb_air_build_wf_lp((int)freqs_hz[ch], (int)fc, rate, T, wf);
		else acb_air_build_wf((int)freqs_hz[ch], (int)fc, rate, wf);
	}, [&](int *kbin, float *tw1) { return acb_fast_plan_air(freqs_hz, nch, c->cfg.K, fc, kbin, tw1); }, 0,
	/* air.c's IF, Fc - Fr + rate/4, is the carrier's mirror image: the measurement mixes with its negative, where the
	 * carrier turns the way its RF offset does */
	(double)fc + rate / 4, [&](int ch) { return -(double)(unsigned)((int)fc - (int)freqs_hz[ch] + (int)(rate / 4)); });
}

extern "C" int acb_set_plan_air(acb_ctx_t *c, int stream, const unsigned *freqs_hz, int nch, unsigned *fc_out)
{
	if (int r = check_plan_air(c, freqs_hz, nch)) return r;
	unsigned lo = freqs_hz[0], hi = freqs_hz[0];
	for (int i = 1; i < nch; i++) { lo = std::min(lo, freqs_hz[i]); hi = std::max(hi, freqs_hz[i]); }
	const unsigned fc = acb_air_choose_fc(lo, hi);
	if (fc_out) *fc_out = fc;
	return plan_air(c, stream, freqs_hz, nch, fc);
}

extern "C" int acb_set_plan_air_at(acb_ctx_t *c, int stream, const unsigned *freqs_hz, int nch, unsigned fc)
{
	if (int r = check_plan_air(c, freqs_hz, nch)) return r;
	if (fc == 0) return fail(ACB_ERR_PLAN, "centre frequency 0");
	return plan_air(c, stream, freqs_hz, nch, fc);
}

extern "C" int acb_submit_dm_host(acb_ctx_t *c, const float *dm, int nsamp)
{
	if (!c || !dm) return fail(ACB_ERR_ARG, "null argument");
	if (int r = ctx_use(c)) return r;
	const size_t n = (size_t)c->cfg.nstreams * nsamp * c->cfg.nch;
	if (nsamp < 1 || n > c->dm_floats) return fail(ACB_ERR_ARG, "nsamp=%d exceeds max_blocks*1024", nsamp);
	/* A pageable source has been staged when the call returns; a pinned one must stay untouched
	 * until the submit is collected. */
	Groups g;
	g.starts.push_back(*std::min_element(c->pos.begin(), c->pos.end()));
	if (int r = run_kernels(c, nullptr, 0, 0, nsamp, dm, std::move(g))) return r;
	for (auto &p : c->pos) p += (unsigned long long)nsamp;
	return ACB_OK;
}

extern "C" int acb_wait_event(acb_ctx_t *c, void *cuda_event)
{
	if (!c || !cuda_event) return fail(ACB_ERR_ARG, "null argument");
	if (int r = ctx_use(c)) return r;
	CU(cudaStreamWaitEvent(c->s_comp, (cudaEvent_t)cuda_event, 0));
	if (c->real_input) {
		/* The streaming device submits read their input on the copy stream.  The wait is taken now, on a stream of its
		 * own, so that it is the event as recorded at this call that counts, and the host submits' copies on the copy
		 * stream are not held up by it; the next device submit orders its append behind ev_order. */
		CU(cudaStreamWaitEvent(c->s_order, (cudaEvent_t)cuda_event, 0));
		CU(cudaEventRecord(c->ev_order, c->s_order));
		c->order_pending = true;
	}
	return ACB_OK;
}

extern "C" int acb_collect(acb_ctx_t *c)
{
	if (!c) return fail(ACB_ERR_ARG, "null context");
	if (int r = ctx_use(c)) return r;
	if (int r = collect_oldest(c)) return r;
	wait_consumer(c, c->jobs_queued);
	if (c->overflowed) {
		c->overflowed = false;
		return fail(ACB_ERR_OVERFLOW, "device frame ring overflowed (%u slots): %llu frames lost so far", c->ring_cap, (unsigned long long)c->stats.frames_lost);
	}
	std::lock_guard<std::mutex> lk(c->mtx);
	return (int)c->outq_count;
}

extern "C" int acb_sync(acb_ctx_t *c)
{
	if (!c) return fail(ACB_ERR_ARG, "null context");
	if (int r = ctx_use(c)) return r;
	while (!c->inflight.empty())
		if (int r = collect_oldest(c)) return r;
	CU(cudaStreamSynchronize(c->s_comp));
	CU(cudaStreamSynchronize(c->s_dem));
	CU(cudaStreamSynchronize(c->s_fec));
	wait_consumer(c, c->jobs_queued);
	if (c->consumer_err[0]) return fail(ACB_ERR_CUDA, "%s", c->consumer_err);
	if (c->overflowed) {
		c->overflowed = false;
		return fail(ACB_ERR_OVERFLOW, "device frame ring overflowed (%u slots): %llu frames lost so far", c->ring_cap, (unsigned long long)c->stats.frames_lost);
	}
	std::lock_guard<std::mutex> lk(c->mtx);
	return (int)c->outq_count;
}

extern "C" int acb_mark(acb_ctx_t *c, int which)
{
	if (!c || which < 0 || which > 1) return fail(ACB_ERR_ARG, "bad argument");
	if (int r = ctx_use(c)) return r;
	/* a timed region starts on the channelizer stream and ends behind the last demod and the last block FEC */
	if (which == 0) {
		CU(cudaEventRecord(c->mark[0], c->s_comp));
	} else {
		CU(cudaEventRecord(c->ev_join, c->s_dem));
		CU(cudaStreamWaitEvent(c->s_fec, c->ev_join, 0));
		CU(cudaEventRecord(c->mark[1], c->s_fec));
	}
	return ACB_OK;
}

extern "C" int acb_elapsed_ms(acb_ctx_t *c, float *ms)
{
	if (!c || !ms) return fail(ACB_ERR_ARG, "null argument");
	if (int r = ctx_use(c)) return r;
	CU(cudaEventSynchronize(c->mark[1]));
	CU(cudaEventElapsedTime(ms, c->mark[0], c->mark[1]));
	return ACB_OK;
}

extern "C" int acb_drain(acb_ctx_t *c, acb_msg_t *out, int max)
{
	if (!c || (!out && max > 0)) return fail(ACB_ERR_ARG, "null argument");
	int n = 0;
	std::lock_guard<std::mutex> lk(c->mtx);
	while (n < max && !c->outq.empty()) {
		acb_ctx::Batch &b = c->outq.front();
		const size_t take = std::min((size_t)(max - n), b.n - b.rd);
		memcpy(out + n, b.v.get() + b.rd, take * sizeof(acb_msg_t));
		n += (int)take;
		b.rd += take;
		if (b.rd == b.n) c->outq.pop_front();
	}
	c->outq_count -= (size_t)n;
	return n;
}

extern "C" int acb_block_fec_batch(acb_ctx_t *c, acb_msg_t *msgs, int n, int *keep)
{
	if (!c || !msgs || !keep || n < 0) return fail(ACB_ERR_ARG, "bad argument");
	if (int r = ctx_use(c)) return r;
	if (n == 0) return 0;
	std::vector<RawFrame> raw(n);
	memset(raw.data(), 0, (size_t)n * sizeof(RawFrame));
	for (int i = 0; i < n; i++) {
		raw[i].len = msgs[i].len; raw[i].err = msgs[i].err; raw[i].chn = msgs[i].chn;
		memcpy(raw[i].txt, msgs[i].txt, ACB_TXTMAX);
		raw[i].crc[0] = msgs[i].crc[0]; raw[i].crc[1] = msgs[i].crc[1];
	}
	RawFrame *d = nullptr;
	RingCtl *dc = nullptr, hc;
	memset(&hc, 0, sizeof(hc));
	hc.count = (unsigned)n;
	cudaError_t e = cudaMalloc(&d, (size_t)n * sizeof(RawFrame));
	if (e == cudaSuccess) e = cudaMalloc(&dc, sizeof(RingCtl));
	if (e == cudaSuccess) e = cudaMemcpyAsync(d, raw.data(), (size_t)n * sizeof(RawFrame), cudaMemcpyHostToDevice, c->s_d2h);   /* same stream as the kernel */
	if (e == cudaSuccess) e = cudaMemcpyAsync(dc, &hc, sizeof(hc), cudaMemcpyHostToDevice, c->s_d2h);
	if (e == cudaSuccess) e = (cudaError_t)launch_block_fec(d, dc, (unsigned)n, c->s_d2h);
	if (e == cudaSuccess) e = cudaMemcpyAsync(raw.data(), d, (size_t)n * sizeof(RawFrame), cudaMemcpyDeviceToHost, c->s_d2h);
	if (e == cudaSuccess) e = cudaStreamSynchronize(c->s_d2h);
	cudaFree(d);
	cudaFree(dc);
	if (e != cudaSuccess) return fail(ACB_ERR_CUDA, "block FEC batch: %s", cudaGetErrorString(e));
	int kept = 0;
	for (int i = 0; i < n; i++) {
		keep[i] = raw[i].pad0 == 1;
		kept += keep[i];
		if (keep[i]) {
			msgs[i].err = raw[i].err;
			memcpy(msgs[i].txt, raw[i].txt, ACB_TXTMAX);
		}
	}
	return kept;
}

extern "C" int acb_pending(acb_ctx_t *c)
{
	if (!c) return fail(ACB_ERR_ARG, "null context");
	std::lock_guard<std::mutex> lk(c->mtx);
	return (int)c->outq_count;
}

extern "C" int acb_read_dm(acb_ctx_t *c, float *out, size_t nfloats)
{
	if (!c || !out) return fail(ACB_ERR_ARG, "null argument");
	if (int r = ctx_use(c)) return r;
	const size_t have = (size_t)c->cfg.nstreams * c->last_nsamp * c->cfg.nch;
	if (nfloats > have) return fail(ACB_ERR_ARG, "asked for %zu floats, last submit produced %zu", nfloats, have);
	CU(cudaStreamSynchronize(c->s_comp));
	CU(cudaStreamSynchronize(c->s_dem));
	CU(cudaMemcpyAsync(out, c->d_dm[c->last_dm], nfloats * sizeof(float), cudaMemcpyDeviceToHost, c->s_copy));
	CU(cudaStreamSynchronize(c->s_copy));
	return ACB_OK;
}

static void to_api(const ChainState &s, acb_chan_state_t *o)
{
	memset(o, 0, sizeof(*o));
	o->MskPhi = s.phi; o->MskDf = s.df; o->MskLvlSum = s.lvlsum; o->MskClk = s.clk;
	o->MskBitCount = s.bitcount; o->MskS = s.S; o->idx = s.idx; o->nbits = s.nbits;
	o->Acarsstate = s.state; o->outbits = s.outbits; o->blk_len = s.blk_len; o->blk_err = s.blk_err;
	o->pos = s.pos; o->soh_pos = s.soh_pos;
	memcpy(o->inb_re, s.inb_re, sizeof(o->inb_re));
	memcpy(o->inb_im, s.inb_im, sizeof(o->inb_im));
	o->blk_crc[0] = s.crc[0]; o->blk_crc[1] = s.crc[1];
	memcpy(o->blk_txt, s.txt, ACB_TXTMAX);
}

static void from_api(const acb_chan_state_t *i, ChainState &s)
{
	memset(&s, 0, sizeof(s));
	s.phi = i->MskPhi; s.df = i->MskDf; s.lvlsum = i->MskLvlSum; s.clk = i->MskClk;
	s.bitcount = i->MskBitCount; s.S = i->MskS; s.idx = i->idx % FLEN; s.nbits = i->nbits;
	s.state = i->Acarsstate; s.outbits = i->outbits & 0xffu; s.blk_len = i->blk_len; s.blk_err = i->blk_err;
	s.pos = i->pos; s.soh_pos = i->soh_pos;
	memcpy(s.inb_re, i->inb_re, sizeof(s.inb_re));
	memcpy(s.inb_im, i->inb_im, sizeof(s.inb_im));
	s.crc[0] = i->blk_crc[0]; s.crc[1] = i->blk_crc[1];
	memcpy(s.txt, i->blk_txt, ACB_TXTMAX);
}

extern "C" int acb_get_state(acb_ctx_t *c, int stream, int chn, acb_chan_state_t *out)
{
	if (!c || !out) return fail(ACB_ERR_ARG, "null argument");
	if (stream < 0 || stream >= c->cfg.nstreams || chn < 0 || chn >= c->cfg.nch) return fail(ACB_ERR_ARG, "stream/chn out of range");
	if (int r = ctx_use(c)) return r;
	ChainState s;
	if (int r = sync_streams(c)) return r;
	CU(cudaMemcpyAsync(&s, c->d_state + (size_t)stream * c->cfg.nch + chn, sizeof(s), cudaMemcpyDeviceToHost, c->s_copy));
	CU(cudaStreamSynchronize(c->s_copy));
	to_api(s, out);
	return ACB_OK;
}

extern "C" int acb_set_state(acb_ctx_t *c, int stream, int chn, const acb_chan_state_t *in)
{
	if (!c || !in) return fail(ACB_ERR_ARG, "null argument");
	if (stream < 0 || stream >= c->cfg.nstreams || chn < 0 || chn >= c->cfg.nch) return fail(ACB_ERR_ARG, "stream/chn out of range");
	if (in->blk_len < 0 || in->blk_len > 248) return fail(ACB_ERR_ARG, "blk_len out of range");
	if (int r = ctx_use(c)) return r;
	ChainState s;
	from_api(in, s);
	if (int r = sync_streams(c)) return r;
	if (int r = upload(c, c->d_state + (size_t)stream * c->cfg.nch + chn, &s, sizeof(s))) return r;
	return ACB_OK;
}

extern "C" int acb_get_stats(acb_ctx_t *c, acb_stats_t *out, int reset)
{
	if (!c || !out) return fail(ACB_ERR_ARG, "null argument");
	std::lock_guard<std::mutex> lk(c->mtx);
	*out = c->stats;
	if (reset) memset(&c->stats, 0, sizeof(c->stats));
	return ACB_OK;
}

extern "C" int acb_get_decode_stats(acb_ctx_t *c, acb_decode_stats_t *out, size_t n, int reset)
{
	if (!c || !out) return fail(ACB_ERR_ARG, "null argument");
	if (!c->decode_stats) return fail(ACB_ERR_ARG, "context was not created with ACB_FLAG_DECODE_STATS");
	if (n < c->dstats.size()) return fail(ACB_ERR_ARG, "n=%zu < nstreams*nch=%zu", n, c->dstats.size());
	std::lock_guard<std::mutex> lk(c->dstats_mtx);
	memcpy(out, c->dstats.data(), c->dstats.size() * sizeof(acb_decode_stats_t));
	if (reset) memset(c->dstats.data(), 0, c->dstats.size() * sizeof(acb_decode_stats_t));
	return ACB_OK;
}

extern "C" int acb_get_level_stats(acb_ctx_t *c, acb_input_level_t *in, size_t n_in, acb_chan_level_t *ch, size_t n_ch, int reset)
{
	if (!c) return fail(ACB_ERR_ARG, "null context");
	if (!c->level_stats) return fail(ACB_ERR_ARG, "context was not created with ACB_FLAG_LEVEL_STATS");
	if (in && n_in < c->lin.size()) return fail(ACB_ERR_ARG, "n_in=%zu < nstreams=%zu", n_in, c->lin.size());
	if (ch && n_ch < c->lch.size()) return fail(ACB_ERR_ARG, "n_ch=%zu < nstreams*nch=%zu", n_ch, c->lch.size());
	std::lock_guard<std::mutex> lk(c->lstats_mtx);
	if (in) memcpy(in, c->lin.data(), c->lin.size() * sizeof(acb_input_level_t));
	if (ch) memcpy(ch, c->lch.data(), c->lch.size() * sizeof(acb_chan_level_t));
	if (reset) {                 /* the open windows stay on the device: the alignment is kept */
		memset(c->lin.data(), 0, c->lin.size() * sizeof(acb_input_level_t));
		memset(c->lch.data(), 0, c->lch.size() * sizeof(acb_chan_level_t));
	}
	return ACB_OK;
}

extern "C" int acb_get_freq_stats(acb_ctx_t *c, acb_chan_freq_t *out, size_t n, int reset)
{
	if (!c || !out) return fail(ACB_ERR_ARG, "null argument");
	if (!c->freq_stats) return fail(ACB_ERR_ARG, "context was not created with ACB_FLAG_FREQ_STATS");
	if (n < c->fch.size()) return fail(ACB_ERR_ARG, "n=%zu < nstreams*nch=%zu", n, c->fch.size());
	std::lock_guard<std::mutex> lk(c->lstats_mtx);
	memcpy(out, c->fch.data(), c->fch.size() * sizeof(acb_chan_freq_t));
	if (reset) clear_freq_sums(c->fch.data(), c->fch.size());
	return ACB_OK;
}

extern "C" int acb_freq_error(const acb_chan_freq_t *ch, int nch, int K, double *offset_hz, double *coherence, double *ppm)
{
	if (!ch || nch < 1 || K < 2) return fail(ACB_ERR_ARG, "null table, nch < 1 or K < 2");
	const double scale = (double)ACB_INTRATE * K / (2.0 * M_PI * (K / 2));
	double wsum = 0.0, wppm = 0.0;
	for (int c = 0; c < nch; c++) {
		const double mag = hypot(ch[c].s_re, ch[c].s_im);
		const double off = ch[c].pairs ? scale * atan2(ch[c].s_im, ch[c].s_re) : 0.0;
		if (offset_hz) offset_hz[c] = off;
		if (coherence) coherence[c] = ch[c].pairs && ch[c].mag_sum > 0 ? mag / ch[c].mag_sum : 0.0;
		if (ch[c].pairs && ch[c].freq_hz > 0) {
			wsum += mag;
			wppm += mag * off / ch[c].freq_hz;
		}
	}
	if (ppm) *ppm = wsum > 0 ? 1e6 * wppm / wsum : 0.0;
	return ACB_OK;
}

/* ---- moving streams (acb_save_streams / acb_load_streams) ----
 *
 * Blob: a 64-byte header (MvHead), then `count` records of record_bytes each.  A record is a 32-byte host part (MvRecHead),
 * the device regions of mv_layout at 16-byte aligned offsets (copied verbatim by k_stream_pack / k_stream_unpack), then
 * the host statistics: nch acb_decode_stats_t (ACB_FLAG_DECODE_STATS), one acb_input_level_t and nch acb_chan_level_t
 * (ACB_FLAG_LEVEL_STATS), nch acb_chan_freq_t (ACB_FLAG_FREQ_STATS: the NCO tables are rebuilt from their steps).  The CRC-32 (IEEE, as zlib's crc32) covers every byte from offset 16 to the end. */
namespace {
constexpr char MV_MAGIC[8] = { 'A', 'C', 'B', 'S', 'T', 'R', 'M', 0 };
/* The records copy these layouts verbatim, so a blob of one version means them: change any of them (a field moved, a
 * size, a table's order) and MV_VERSION must change with it, or old blobs would load without error and decode wrong.
 * The asserts pin what the version stands for today. */
constexpr uint32_t MV_VERSION = 1;
static_assert(sizeof(ChainState) == 432 && offsetof(ChainState, state) == 44 && offsetof(ChainState, pos) == 64 &&
              offsetof(ChainState, inb_re) == 80 && offsetof(ChainState, crc) == 168 && offsetof(ChainState, txt) == 176,
              "ChainState changed: bump MV_VERSION");
static_assert(sizeof(LevelCarry) == 16 && offsetof(LevelCarry, rows) == 8, "LevelCarry changed: bump MV_VERSION");
static_assert(CH_GROUP == 8 && WB_CTILE == 256 && WB_CB == 4 && WB_META == 546, "table layouts changed: bump MV_VERSION");
static_assert(sizeof(acb_decode_stats_t) == 120 && sizeof(acb_input_level_t) == 32 && sizeof(acb_chan_level_t) == 40 &&
              sizeof(acb_chan_freq_t) == 56, "statistics changed: bump MV_VERSION");
}

static size_t round16(size_t x) { return (x + 15) & ~(size_t)15; }

/* The record of a configuration; the same for every context of it, whatever its nstreams, max_blocks or device */
MvLayout acb::mv_layout(int in_kind, int K, int taps, int nch, int form, int flags)
{
	MvLayout L{};
	int hpad = 0, taps_pad = 0;
	taps_geometry(in_kind, K, taps, (ChanForm)form, hpad, taps_pad);
	const size_t ngrp = (size_t)(nch + CH_GROUP - 1) / CH_GROUP, nct = (size_t)(nch + WB_CTILE - 1) / WB_CTILE;
	size_t off = sizeof(MvRecHead);
	auto add = [&](int tag, size_t bytes) {
		L.tag[L.nreg] = tag;
		L.off[L.nreg] = off;
		L.bytes[L.nreg] = bytes;
		L.nreg++;
		off += round16(bytes);
	};
	add(R_STATE, (size_t)nch * sizeof(ChainState));
	if (in_kind != IN_KIND_U8IQ) add(R_IN, round16(((size_t)hpad + K) * 4));     /* history + carry (< K samples) */
	else if (hpad) add(R_IN, (size_t)hpad * 2);
	add(R_WF, ngrp * taps_pad * CH_GROUP * 2 * sizeof(float));
	if (form == CHAN_DFT || form == CHAN_RDFT || form == CHAN_OVL_FAST || form == CHAN_OVL_RDFT) {
		add(R_TW, ngrp * CH_GROUP * (K / 4) * 2 * sizeof(float));
		add(R_TWMETA, ngrp * sizeof(unsigned));
	}
	if (form == CHAN_WB || form == CHAN_WB_REAL) add(R_WBMETA, nct * WB_META * sizeof(int));
	if (flags & ACB_FLAG_LEVEL_STATS) add(R_LCARRY, (size_t)nch * sizeof(LevelCarry));
	L.off_dstats = off;
	if (flags & ACB_FLAG_DECODE_STATS) off += (size_t)nch * sizeof(acb_decode_stats_t);
	L.off_lin = off;
	L.off_lch = off + sizeof(acb_input_level_t);
	if (flags & ACB_FLAG_LEVEL_STATS) off += sizeof(acb_input_level_t) + (size_t)nch * sizeof(acb_chan_level_t);
	L.off_fch = off;
	if (flags & ACB_FLAG_FREQ_STATS) off += (size_t)nch * sizeof(acb_chan_freq_t);
	L.rec_bytes = round16(off);
	return L;
}

static MvLayout ctx_layout(const acb_ctx *c)
{
	return mv_layout(c->in_kind, c->cfg.K, c->taps, c->cfg.nch, c->form, c->cfg.flags & MV_FLAGS);
}

/* CRC-32 (IEEE, as zlib's crc32), eight bytes per step (slicing-by-8): moving a whole context is host-bound, and this
 * runs over every byte of a blob on save and on load */
static uint32_t crc32_update(uint32_t crc, const uint8_t *p, size_t n)
{
	struct Tables {
		uint32_t t[8][256];
		Tables()
		{
			for (uint32_t i = 0; i < 256; i++) {
				uint32_t v = i;
				for (int k = 0; k < 8; k++) v = v & 1 ? 0xEDB88320u ^ (v >> 1) : v >> 1;
				t[0][i] = v;
			}
			for (int k = 1; k < 8; k++)
				for (int i = 0; i < 256; i++) t[k][i] = (t[k - 1][i] >> 8) ^ t[0][t[k - 1][i] & 0xff];
		}
	};
	static const Tables T;                       /* initialised once, thread-safely */
	crc = ~crc;
	for (; n >= 8; n -= 8, p += 8) {
		uint32_t a, b;
		memcpy(&a, p, 4);                        /* the blob is little-endian, as the host is */
		memcpy(&b, p + 4, 4);
		a ^= crc;
		crc = T.t[7][a & 0xff] ^ T.t[6][(a >> 8) & 0xff] ^ T.t[5][(a >> 16) & 0xff] ^ T.t[4][a >> 24] ^ T.t[3][b & 0xff] ^
		      T.t[2][(b >> 8) & 0xff] ^ T.t[1][(b >> 16) & 0xff] ^ T.t[0][b >> 24];
	}
	for (; n; n--, p++) crc = T.t[0][(crc ^ *p) & 0xff] ^ (crc >> 8);
	return ~crc;
}

void acb::mv_seal(void *blob, size_t size, int count)
{
	MvHead h;
	memcpy(&h, blob, sizeof(h));
	h.count = count;
	memcpy(blob, &h, sizeof(h));
	const uint32_t crc = crc32_update(0, (const uint8_t *)blob + 16, size - 16);
	memcpy((uint8_t *)blob + offsetof(MvHead, crc), &crc, 4);
}

extern "C" int acb_streams_blob_check(const void *blob, size_t size, acb_streams_blob_info_t *out)
{
	if (!blob) return fail(ACB_ERR_ARG, "null blob");
	if (size < sizeof(MvHead)) return fail(ACB_ERR_ARG, "blob of %zu bytes is shorter than its header", size);
	MvHead h;
	memcpy(&h, blob, sizeof(h));
	if (memcmp(h.magic, MV_MAGIC, sizeof(MV_MAGIC))) return fail(ACB_ERR_ARG, "not a stream blob (magic)");
	if (h.version != MV_VERSION) return fail(ACB_ERR_ARG, "blob format version %u, this library reads %u", h.version, MV_VERSION);
	if (h.in_kind < IN_KIND_U8IQ || h.in_kind > IN_KIND_CS16IQ || h.K < 1 || h.K > ACB_MAXK || h.taps < 1 ||
	    h.taps > ACB_MAXTAPS_PER_K * h.K || h.nch < 1 || h.form < CHAN_EXACT || h.form > CHAN_WB_REAL || (h.flags & ~MV_FLAGS) ||
	    h.count < 1)
		return fail(ACB_ERR_ARG, "blob header out of range");
	const MvLayout L = mv_layout(h.in_kind, h.K, h.taps, h.nch, h.form, h.flags);
	if (h.record_bytes != L.rec_bytes) return fail(ACB_ERR_ARG, "blob records of %llu bytes, the configuration's are %zu",
	                                               (unsigned long long)h.record_bytes, L.rec_bytes);
	if ((size - sizeof(MvHead)) / L.rec_bytes != (size_t)h.count || (size - sizeof(MvHead)) % L.rec_bytes)
		return fail(ACB_ERR_ARG, "blob of %zu bytes does not hold %d records of %zu bytes", size, h.count, L.rec_bytes);
	if (crc32_update(0, (const uint8_t *)blob + 16, size - 16) != h.crc) return fail(ACB_ERR_ARG, "blob CRC mismatch");
	if (out) {
		out->in_kind = h.in_kind; out->K = h.K; out->taps = h.taps; out->nch = h.nch; out->form = h.form; out->flags = h.flags;
		out->group_unit = h.group_unit; out->group_period = h.group_period; out->count = h.count; out->record_bytes = h.record_bytes;
	}
	return ACB_OK;
}

extern "C" size_t acb_streams_blob_bytes(acb_ctx_t *c, int n)
{
	if (!c || n < 1) return 0;
	return sizeof(MvHead) + (size_t)n * ctx_layout(c).rec_bytes;
}

/* n distinct streams in range */
static int mv_check_list(const acb_ctx *c, const int *streams, int n)
{
	if (n < 1 || n > c->cfg.nstreams) return fail(ACB_ERR_ARG, "n=%d outside 1..nstreams=%d", n, c->cfg.nstreams);
	std::vector<unsigned char> seen(c->cfg.nstreams, 0);
	for (int i = 0; i < n; i++) {
		if (streams[i] < 0 || streams[i] >= c->cfg.nstreams) return fail(ACB_ERR_ARG, "stream %d out of range", streams[i]);
		if (seen[streams[i]]++) return fail(ACB_ERR_ARG, "stream %d listed twice", streams[i]);
	}
	return ACB_OK;
}

/* room for the list and n records in both stagings, once the last load's unpack has read the device one */
static int mv_stage(acb_ctx *c, size_t bytes)
{
	if (c->mv_pending) {
		CU(cudaEventSynchronize(c->ev_mv));
		c->mv_pending = false;
	}
	if (bytes <= c->mv_cap) return ACB_OK;
	cudaFree(c->d_mv);
	cudaFreeHost(c->h_mv);
	c->d_mv = c->h_mv = nullptr;
	c->mv_cap = 0;
	CU(cudaMalloc(&c->d_mv, bytes));
	CU(cudaHostAlloc(&c->h_mv, bytes, cudaHostAllocDefault));
	c->mv_cap = bytes;
	return ACB_OK;
}

/* where each region of L lives in this context */
static StreamRegions mv_regions(const acb_ctx *c, const MvLayout &L)
{
	StreamRegions R{};
	R.nreg = L.nreg;
	for (int k = 0; k < L.nreg; k++) {
		StreamRegion &g = R.r[k];
		g.bytes = L.bytes[k];
		g.off = L.off[k];
		g.stride = L.bytes[k];
		switch (L.tag[k]) {
		case R_STATE: g.base = (uint8_t *)c->d_state; break;
		case R_IN:
			if (c->real_input) {
				g.base = (uint8_t *)c->d_real[c->real_buf];     /* [history | carry] in front of the next submit's samples */
				g.stride = c->real_cap * sizeof(float);
			} else {
				g.base = c->d_hist;
			}
			break;
		case R_WF: g.base = (uint8_t *)c->d_wf; break;
		case R_TW: g.base = (uint8_t *)c->d_tw; break;
		case R_TWMETA: g.base = (uint8_t *)c->d_twmeta; break;
		case R_WBMETA: g.base = (uint8_t *)c->d_wbmeta; break;
		case R_LCARRY: g.base = (uint8_t *)c->d_lcarry; break;
		}
	}
	return R;
}

void acb::mv_fingerprint(acb_ctx_t *c, MvHead &h)
{
	h = MvHead{};
	memcpy(h.magic, MV_MAGIC, sizeof(MV_MAGIC));
	h.version = MV_VERSION;
	h.in_kind = c->in_kind; h.K = c->cfg.K; h.taps = c->taps; h.nch = c->cfg.nch; h.form = c->form; h.flags = c->cfg.flags & MV_FLAGS;
	h.group_unit = c->real_input ? c->group_unit : 0;
	h.group_period = c->real_input ? c->group_period : 0;
	h.record_bytes = ctx_layout(c).rec_bytes;
}

extern "C" int acb_save_streams(acb_ctx_t *c, const int *streams, int n, void *blob, size_t cap)
{
	if (!c || !streams || !blob) return fail(ACB_ERR_ARG, "null argument");
	if (int r = mv_check_list(c, streams, n)) return r;
	const MvLayout L = ctx_layout(c);
	const size_t rec = L.rec_bytes, need = sizeof(MvHead) + (size_t)n * rec, lb = round16((size_t)n * sizeof(int));
	if (cap < need) return fail(ACB_ERR_ARG, "cap=%zu < %zu bytes", cap, need);
	if (int r = ctx_use(c)) return r;
	/* every submit made so far, as acb_sync collects them (an overflow stays for acb_collect / acb_sync to report) */
	while (!c->inflight.empty())
		if (int r = collect_oldest(c)) return r;
	if (int r = sync_streams(c)) return r;
	wait_consumer(c, c->jobs_queued);
	if (c->consumer_err[0]) return fail(ACB_ERR_CUDA, "%s", c->consumer_err);
	if (int r = mv_stage(c, lb + (size_t)n * rec)) return r;
	memcpy(c->h_mv, streams, (size_t)n * sizeof(int));
	CU(cudaMemcpyAsync(c->d_mv, c->h_mv, (size_t)n * sizeof(int), cudaMemcpyHostToDevice, c->s_comp));
	/* the pack writes each region's bytes only: the padding up to the next 16-byte offset would otherwise carry whatever
	 * the staging buffer held before, and equal states would not give equal blobs */
	CU(cudaMemsetAsync(c->d_mv + lb, 0, (size_t)n * rec, c->s_comp));
	int launched = 0;
	if (int r = launch_stream_move(mv_regions(c, L), (const int *)c->d_mv, n, c->d_mv + lb, rec, false, c->s_comp, launched))
		return fail(ACB_ERR_CUDA, "stream pack launch: %s", cudaGetErrorString((cudaError_t)r));
	c->stats.kernel_launches += launched;
	CU(cudaMemcpyAsync(c->h_mv + lb, c->d_mv + lb, (size_t)n * rec, cudaMemcpyDeviceToHost, c->s_comp));
	CU(cudaStreamSynchronize(c->s_comp));
	uint8_t *const out = (uint8_t *)blob;
	MvHead h;
	mv_fingerprint(c, h);
	memcpy(out, &h, sizeof(h));
	memcpy(out + sizeof(MvHead), c->h_mv + lb, (size_t)n * rec);
	const int nch = c->cfg.nch;
	for (int i = 0; i < n; i++) {
		const int s = streams[i];
		uint8_t *r = out + sizeof(MvHead) + (size_t)i * rec;
		const MvRecHead rh{ c->pos[s], c->real_input ? (uint64_t)c->carry[s] : 0, c->fast_ok[s], 0, 0 };
		memcpy(r, &rh, sizeof(rh));
		for (int k = 0; c->real_input && k < L.nreg; k++) {
			/* what lies past the history and carry is no state: zeros, so that equal states give equal blobs */
			const size_t used = ((size_t)c->hpad + c->carry[s]) * sizeof(float);
			if (L.tag[k] == R_IN) memset(r + L.off[k] + used, 0, L.bytes[k] - used);
		}
		if (c->decode_stats) {
			std::lock_guard<std::mutex> lk(c->dstats_mtx);
			memcpy(r + L.off_dstats, &c->dstats[(size_t)s * nch], (size_t)nch * sizeof(acb_decode_stats_t));
		}
		if (c->level_stats) {
			std::lock_guard<std::mutex> lk(c->lstats_mtx);
			memcpy(r + L.off_lin, &c->lin[s], sizeof(acb_input_level_t));
			memcpy(r + L.off_lch, &c->lch[(size_t)s * nch], (size_t)nch * sizeof(acb_chan_level_t));
		}
		if (c->freq_stats) {
			std::lock_guard<std::mutex> lk(c->lstats_mtx);
			memcpy(r + L.off_fch, &c->fch[(size_t)s * nch], (size_t)nch * sizeof(acb_chan_freq_t));
		}
	}
	mv_seal(out, need, n);
	return ACB_OK;
}

/* Everything acb_load_streams refuses, checked before anything changes: the blob itself, its fingerprint against the
 * context's, n, and the record fields the device indexes with (a corrupt blob with a valid CRC must not write out of
 * bounds) */
int acb::mv_validate(acb_ctx_t *c, const void *blob, size_t size, int n)
{
	acb_streams_blob_info_t info;
	if (int r = acb_streams_blob_check(blob, size, &info)) return r;
	const int flags = c->cfg.flags & MV_FLAGS;
	if (info.in_kind != c->in_kind || info.K != c->cfg.K || info.taps != c->taps || info.nch != c->cfg.nch || info.form != c->form)
		return fail(ACB_ERR_ARG, "blob of kind %d, K=%d, taps=%d, nch=%d, form %d; the context is %d, %d, %d, %d, %d", info.in_kind, info.K,
		            info.taps, info.nch, info.form, c->in_kind, c->cfg.K, c->taps, c->cfg.nch, (int)c->form);
	if (info.flags != flags) return fail(ACB_ERR_ARG, "blob statistics flags %d, the context's %d", info.flags, flags);
	if (c->real_input && (info.group_unit != c->group_unit || info.group_period != c->group_period))
		return fail(ACB_ERR_ARG, "blob emission groups (%d, %llu) differ from the context's (%d, %llu)", info.group_unit,
		            (unsigned long long)info.group_period, c->group_unit, (unsigned long long)c->group_period);
	if (n != info.count) return fail(ACB_ERR_ARG, "n=%d, the blob holds %d records", n, info.count);
	const MvLayout L = ctx_layout(c);
	const int nch = c->cfg.nch;
	for (int i = 0; i < n; i++) {
		const uint8_t *r = (const uint8_t *)blob + sizeof(MvHead) + (size_t)i * L.rec_bytes;
		MvRecHead rh;
		memcpy(&rh, r, sizeof(rh));
		if (rh.carry >= (uint64_t)(c->real_input ? c->cfg.K : 1) || rh.fast_ok > 1) return fail(ACB_ERR_ARG, "record %d: carry / plan out of range", i);
		for (int k = 0; k < L.nreg; k++) {
			if (L.tag[k] == R_STATE) {
				for (int ch = 0; ch < nch; ch++) {
					ChainState st;
					memcpy(&st, r + L.off[k] + (size_t)ch * sizeof(ChainState), sizeof(st));
					if (st.idx >= (unsigned)FLEN || st.blk_len < 0 || st.blk_len > 248 || st.outbits > 0xffu)
						return fail(ACB_ERR_ARG, "record %d: chain %d's state out of range", i, ch);
				}
			} else if (L.tag[k] == R_WBMETA) {
				const int ntab = c->in_kind == IN_KIND_CS16IQ ? 2 : 1;
				for (size_t z = 0; z < L.bytes[k] / (WB_META * sizeof(int)); z++) {
					int m[WB_META];
					memcpy(m, r + L.off[k] + z * WB_META * sizeof(int), sizeof(m));
					bool ok = m[0] >= 0 && m[0] <= WB_SLOTS / WB_CB && m[1] >= 0 && m[1] < ntab;
					for (int j = 0; ok && j < WB_SLOTS; j++)
						ok = m[3 + 2 * j] >= -1 && m[3 + 2 * j] < nch && m[2 + 2 * j] > -c->cfg.K && m[2 + 2 * j] < c->cfg.K;
					if (!ok) return fail(ACB_ERR_ARG, "record %d: wideband plan out of range", i);
				}
			}
		}
	}
	return ACB_OK;
}

extern "C" int acb_load_streams(acb_ctx_t *c, const int *streams, int n, const void *blob, size_t size)
{
	if (!c || !streams || !blob) return fail(ACB_ERR_ARG, "null argument");
	if (int r = mv_check_list(c, streams, n)) return r;
	if (int r = mv_validate(c, blob, size, n)) return r;
	if (int r = ctx_use(c)) return r;
	const MvLayout L = ctx_layout(c);
	const size_t rec = L.rec_bytes, lb = round16((size_t)n * sizeof(int));
	const uint8_t *const in = (const uint8_t *)blob + sizeof(MvHead);
	if (int r = mv_stage(c, lb + (size_t)n * rec)) return r;
	memcpy(c->h_mv, streams, (size_t)n * sizeof(int));
	memcpy(c->h_mv + lb, in, (size_t)n * rec);
	/* as acb_reset_stream: the chain states behind the demods already queued, the input side, tables and open windows
	 * behind the channelizer, level kernels and tail moves (all on the channelizer stream), and everything ahead of the
	 * next submit's append and kernels */
	CU(cudaEventRecord(c->ev_join, c->s_dem));
	CU(cudaStreamWaitEvent(c->s_comp, c->ev_join, 0));
	CU(cudaMemcpyAsync(c->d_mv, c->h_mv, lb + (size_t)n * rec, cudaMemcpyHostToDevice, c->s_comp));
	int launched = 0;
	if (int r = launch_stream_move(mv_regions(c, L), (const int *)c->d_mv, n, c->d_mv + lb, rec, true, c->s_comp, launched))
		return fail(ACB_ERR_CUDA, "stream unpack launch: %s", cudaGetErrorString((cudaError_t)r));
	c->stats.kernel_launches += launched;
	CU(cudaEventRecord(c->ev_mv, c->s_comp));
	c->mv_pending = true;
	CU(cudaEventRecord(c->ev_join, c->s_comp));
	CU(cudaStreamWaitEvent(c->s_dem, c->ev_join, 0));
	CU(cudaStreamWaitEvent(c->s_copy, c->ev_join, 0));
	const int nch = c->cfg.nch;
	for (int i = 0; i < n; i++) {
		const int s = streams[i];
		const uint8_t *r = in + (size_t)i * rec;
		MvRecHead rh;
		memcpy(&rh, r, sizeof(rh));
		c->pos[s] = rh.pos;
		if (c->real_input) c->carry[s] = (size_t)rh.carry;
		c->fast_ok[s] = (unsigned char)rh.fast_ok;
		/* the slot's counts become the blob's; submits made before the load are not counted (acb_reset_stream's rule) */
		if (c->decode_stats) {
			std::lock_guard<std::mutex> lk(c->dstats_mtx);
			memcpy(&c->dstats[(size_t)s * nch], r + L.off_dstats, (size_t)nch * sizeof(acb_decode_stats_t));
			c->dstats_from[s] = c->nsubmit;
		}
		if (c->freq_stats) {
			/* the submits before the load are not counted for this stream (below), so the table may change under them */
			std::vector<double> freq(nch), step(nch);
			for (int ch = 0; ch < nch; ch++) {
				acb_chan_freq_t f;
				memcpy(&f, r + L.off_fch + (size_t)ch * sizeof(f), sizeof(f));
				freq[ch] = f.freq_hz, step[ch] = f.step;
			}
			if (int e = set_freq_plan(c, s, freq.data(), step.data())) return e;
		}
		if (c->dev_stats) {
			std::lock_guard<std::mutex> lk(c->lstats_mtx);
			if (c->level_stats) {
				memcpy(&c->lin[s], r + L.off_lin, sizeof(acb_input_level_t));
				memcpy(&c->lch[(size_t)s * nch], r + L.off_lch, (size_t)nch * sizeof(acb_chan_level_t));
			}
			if (c->freq_stats) memcpy(&c->fch[(size_t)s * nch], r + L.off_fch, (size_t)nch * sizeof(acb_chan_freq_t));
			c->lstats_from[s] = c->nsubmit;
		}
	}
	return ACB_OK;
}
