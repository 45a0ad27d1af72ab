/*
 * acb_multi_*: one process, several GPUs (include/acars_b200.h).  Host-side only: it fronts one acb_ctx_t per
 * device and splits either the streams or the channels among them; the devices never talk to each other
 * (SURVEY.md §8e: channels share nothing but the read-only matched filter, streams share nothing).
 * The reference has no counterpart (one thread serves all channels, rtl.c:344-360); what it fixes for us is the
 * emission order the merged output must keep: u8 IQ per 1024-sample block, then channel, then time (rtl.c:357-360);
 * the streaming front-ends (real input, CS16) per emission group of acb_set_emission_groups.  Every context orders
 * each submit's frames by (group number counted from the stream's start, stream, channel, time); this layer keeps each
 * stream's position after every submit not yet collected, because a message does not say which submit it came from.
 */
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <deque>
#include <vector>

#include "../../include/acars_b200.h"
#include "acb_internal.h"

using acb::fail;

struct Part {
	acb_ctx_t *ctx;
	int s0, ns;       /* streams served */
	int c0, nc;       /* channels served */
};

struct acb_multi {
	acb_config_t cfg;
	int mode;
	bool streaming;                    /* ACB_FLAG_REAL_INPUT or ACB_FLAG_CS16_INPUT: arbitrary submit lengths, emission groups */
	std::vector<Part> parts;
	std::deque<acb_msg_t> outq;
	std::vector<acb_msg_t> scratch;
	int group_unit;
	unsigned long long group_period;
	std::vector<unsigned long long> spos;   /* per (global) stream: envelope rows since create / reset */
	/* the submits not yet collected, oldest first: each stream's position after it (a message belongs to the first
	 * submit whose end lies beyond its pos) and which parts ran it (acb_multi_collect collects those) */
	struct Sub { std::vector<unsigned long long> end; std::vector<unsigned char> part; };
	std::deque<Sub> subs;
};

static void split(int n, int parts, int i, int *lo, int *cnt)
{
	const int base = n / parts, extra = n % parts;
	*lo = i * base + std::min(i, extra);
	*cnt = base + (i < extra ? 1 : 0);
}

extern "C" int acb_multi_create(const acb_config_t *cfg, const int *devices, int ndev, int mode, acb_multi_t **out)
{
	if (!cfg || !devices || !out || ndev < 1) return ACB_ERR_ARG;
	if (mode != ACB_MULTI_SPLIT_STREAMS && mode != ACB_MULTI_SPLIT_CHANNELS) return ACB_ERR_ARG;
	acb_multi *m = new acb_multi();
	m->cfg = *cfg;
	m->mode = mode;
	m->streaming = (cfg->flags & (ACB_FLAG_REAL_INPUT | ACB_FLAG_CS16_INPUT)) != 0;
	m->group_unit = ACB_GROUP_SUBMIT;
	m->group_period = 0;
	m->spos.assign(cfg->nstreams > 0 ? cfg->nstreams : 0, 0);
	*out = m;
	const int total = mode == ACB_MULTI_SPLIT_STREAMS ? cfg->nstreams : cfg->nch;
	for (int i = 0; i < ndev; i++) {
		Part p;
		p.ctx = nullptr;
		p.s0 = 0; p.ns = cfg->nstreams; p.c0 = 0; p.nc = cfg->nch;
		if (mode == ACB_MULTI_SPLIT_STREAMS) split(total, ndev, i, &p.s0, &p.ns);
		else split(total, ndev, i, &p.c0, &p.nc);
		if (p.ns == 0 || p.nc == 0) continue;             /* more devices than work: this one stays idle */
		acb_config_t c = *cfg;
		c.device = devices[i];
		c.nstreams = p.ns;
		c.nch = p.nc;
		const int r = acb_create(&c, &p.ctx);
		if (p.ctx) m->parts.push_back(p);
		if (r != ACB_OK) return r;                       /* the caller destroys what exists */
	}
	return m->parts.empty() ? ACB_ERR_ARG : ACB_OK;
}

extern "C" void acb_multi_destroy(acb_multi_t *m)
{
	if (!m) return;
	for (auto &p : m->parts) acb_destroy(p.ctx);
	delete m;
}

extern "C" int acb_multi_parts(acb_multi_t *m) { return m ? (int)m->parts.size() : ACB_ERR_ARG; }
extern "C" acb_ctx_t *acb_multi_part(acb_multi_t *m, int i) { return m && i >= 0 && i < (int)m->parts.size() ? m->parts[i].ctx : nullptr; }

extern "C" int acb_multi_set_plan(acb_multi_t *m, int stream, const unsigned *freqs_hz, int nch, unsigned *fc_out)
{
	if (!m || !freqs_hz || nch != m->cfg.nch || stream < 0 || stream >= m->cfg.nstreams) return ACB_ERR_ARG;
	/* one centre for all channels of the stream (chooseFc, rtl.c:131-168), whoever serves them */
	const unsigned fc = acb_choose_fc(freqs_hz, nch, m->cfg.K);
	if (fc == 0) return ACB_ERR_PLAN;
	if (fc_out) *fc_out = fc;
	for (auto &p : m->parts) {
		if (stream < p.s0 || stream >= p.s0 + p.ns) continue;
		if (int r = acb_set_plan_at(p.ctx, stream - p.s0, freqs_hz + p.c0, p.nc, fc)) return r;
	}
	return ACB_OK;
}

/* Channel split: every part serves some of the stream's channels, so Fc is chosen once over all of them and every part
 * builds its tables around it (each part choosing over its own subset would get a different centre). */
extern "C" int acb_multi_set_plan_air(acb_multi_t *m, int stream, const unsigned *freqs_hz, int nch, unsigned *fc_out)
{
	if (!m || !freqs_hz || nch != m->cfg.nch || stream < 0 || stream >= m->cfg.nstreams) return fail(ACB_ERR_ARG, "bad argument");
	if (!(m->cfg.flags & ACB_FLAG_REAL_INPUT)) return fail(ACB_ERR_ARG, "not a real-input multi-context");
	unsigned lo = freqs_hz[0], hi = freqs_hz[0];
	for (int i = 1; i < nch; i++) { lo = std::min(lo, freqs_hz[i]); hi = std::max(hi, freqs_hz[i]); }
	const unsigned fc = acb_air_choose_fc(lo, hi);           /* air.c:42-64, as acb_set_plan_air */
	if (fc_out) *fc_out = fc;
	for (auto &p : m->parts) {
		if (stream < p.s0 || stream >= p.s0 + p.ns) continue;
		if (int r = acb_set_plan_air_at(p.ctx, stream - p.s0, freqs_hz + p.c0, p.nc, fc)) return r;
	}
	return ACB_OK;
}

extern "C" int acb_multi_set_plan_cs16(acb_multi_t *m, int stream, const unsigned *freqs_hz, int nch, int variant, unsigned fc_hz,
                                       unsigned *fc_out)
{
	if (!m || !freqs_hz || nch != m->cfg.nch || stream < 0 || stream >= m->cfg.nstreams) return fail(ACB_ERR_ARG, "bad argument");
	if (!(m->cfg.flags & ACB_FLAG_CS16_INPUT)) return fail(ACB_ERR_ARG, "not a CS16 multi-context");
	if (variant != ACB_CS16_SOAPY && variant != ACB_CS16_SDRPLAY) return fail(ACB_ERR_ARG, "unknown CS16 variant");
	const unsigned fc = fc_hz ? fc_hz : acb_choose_fc(freqs_hz, nch, m->cfg.K);      /* as acb_set_plan_cs16 */
	if (fc == 0) return fail(ACB_ERR_PLAN, "Frequencies too far apart");
	if (fc_out) *fc_out = fc;
	for (auto &p : m->parts) {
		if (stream < p.s0 || stream >= p.s0 + p.ns) continue;
		if (int r = acb_set_plan_cs16(p.ctx, stream - p.s0, freqs_hz + p.c0, p.nc, variant, fc, nullptr)) return r;
	}
	return ACB_OK;
}

extern "C" int acb_multi_set_wf(acb_multi_t *m, int stream, const float *wf, int nch)
{
	if (!m || !wf || nch != m->cfg.nch || stream < 0 || stream >= m->cfg.nstreams) return ACB_ERR_ARG;
	const int taps = m->cfg.taps ? m->cfg.taps : m->cfg.K;
	for (auto &p : m->parts) {
		if (stream < p.s0 || stream >= p.s0 + p.ns) continue;
		if (int r = acb_set_wf(p.ctx, stream - p.s0, wf + (size_t)p.c0 * taps * 2, p.nc)) return r;
	}
	return ACB_OK;
}

extern "C" int acb_multi_reset(acb_multi_t *m)
{
	if (!m) return ACB_ERR_ARG;
	for (auto &p : m->parts)
		if (int r = acb_reset(p.ctx)) return r;
	m->outq.clear();
	std::fill(m->spos.begin(), m->spos.end(), 0);
	m->subs.clear();
	return ACB_OK;
}

/* A submit went to the parts marked in `ran`: stream s advanced by rows[s] */
static void record_submit(acb_multi *m, const std::vector<size_t> &rows, std::vector<unsigned char> &&ran)
{
	for (size_t s = 0; s < rows.size(); s++) m->spos[s] += rows[s];
	m->subs.push_back(acb_multi::Sub{ m->spos, std::move(ran) });
}

extern "C" int acb_multi_set_emission_groups(acb_multi_t *m, int unit, uint64_t period)
{
	if (!m) return fail(ACB_ERR_ARG, "null argument");
	for (auto &p : m->parts)
		if (int r = acb_set_emission_groups(p.ctx, unit, period)) return r;     /* validates unit and period */
	m->group_unit = unit;
	m->group_period = period;
	return ACB_OK;
}

extern "C" int acb_multi_submit_host(acb_multi_t *m, const uint8_t *iq, size_t stream_stride, int nblk)
{
	if (!m || !iq) return ACB_ERR_ARG;
	if (m->streaming) return fail(ACB_ERR_ARG, "not a u8-IQ multi-context: use acb_multi_submit_real_host / acb_multi_submit_cs16_host");
	/* asynchronous per device (pinned source): every GPU pulls its part over its own PCIe link at once */
	for (auto &p : m->parts)
		if (int r = acb_submit_host(p.ctx, iq + (size_t)p.s0 * stream_stride, stream_stride, nblk)) return r;
	record_submit(m, std::vector<size_t>(m->cfg.nstreams, (size_t)nblk * ACB_OUTBLK), std::vector<unsigned char>(m->parts.size(), 1));
	return ACB_OK;
}

/* Ragged u8: a stream split hands each part its streams' counts (a part whose counts are all 0 sits the submit out), a
 * channel split hands every part all of them.  The counts are checked here, before any part reads anything. */
extern "C" int acb_multi_submit_host_ragged(acb_multi_t *m, const uint8_t *iq, size_t stream_stride, const int *nblk)
{
	if (!m || !iq || !nblk) return fail(ACB_ERR_ARG, "null argument");
	if (m->streaming) return fail(ACB_ERR_ARG, "not a u8-IQ multi-context: use acb_multi_submit_real_host_ragged / acb_multi_submit_cs16_host_ragged");
	const int n = m->cfg.nstreams;
	int maxb = 0;
	for (int s = 0; s < n; s++) {
		if (nblk[s] < 0 || nblk[s] > m->cfg.max_blocks) return fail(ACB_ERR_ARG, "nblk[%d]=%d outside 0..%d", s, nblk[s], m->cfg.max_blocks);
		maxb = std::max(maxb, nblk[s]);
	}
	if (maxb == 0) return fail(ACB_ERR_ARG, "every stream's nblk is 0");
	if (n > 1 && stream_stride < (size_t)maxb * ACB_OUTBLK * m->cfg.K * 2) return fail(ACB_ERR_ARG, "stream_stride smaller than the largest input");
	if (stream_stride % 16) return fail(ACB_ERR_ARG, "stream_stride must be a multiple of 16 bytes");
	std::vector<unsigned char> ran(m->parts.size(), 0);
	for (size_t i = 0; i < m->parts.size(); i++) {
		const Part &p = m->parts[i];
		if (std::all_of(nblk + p.s0, nblk + p.s0 + p.ns, [](int b) { return b == 0; })) continue;
		if (int r = acb_submit_host_ragged(p.ctx, iq + (size_t)p.s0 * stream_stride, stream_stride, nblk + p.s0)) return r;
		ran[i] = 1;
	}
	std::vector<size_t> rows(n);
	for (int s = 0; s < n; s++) rows[s] = (size_t)nblk[s] * ACB_OUTBLK;
	record_submit(m, rows, std::move(ran));
	return ACB_OK;
}

/* The streaming submits: every part gets its streams' rows (stream split) or the whole input (channel split), each
 * pulling it over its own link.  In a channel split every part carries the same remainders, so all must produce the same
 * rows.  `ns` != NULL: the ragged calls, stream s bringing ns[s] samples; a stream-split part whose counts are all 0 sits
 * the submit out.  The lockstep calls return the rows every stream produced, the ragged ones the largest and nout[s]. */
static int submit_streaming(acb_multi *m, int flag, const void *x, const void *x2, size_t sample_bytes, size_t stride, size_t nsamples,
                            const size_t *ns = nullptr, size_t *nout_s = nullptr)
{
	if (!(m->cfg.flags & flag))
		return fail(ACB_ERR_ARG, flag == ACB_FLAG_REAL_INPUT ? "multi-context was not created with ACB_FLAG_REAL_INPUT"
		                                                     : "multi-context was not created with ACB_FLAG_CS16_INPUT");
	const int n = m->cfg.nstreams;
	size_t nmax = ns ? 0 : nsamples;
	for (int s = 0; ns && s < n; s++) nmax = std::max(nmax, ns[s]);
	if (ns && nmax == 0) return fail(ACB_ERR_ARG, "every stream's nsamples is 0");
	/* a part with one stream does not check this itself */
	if (n > 1 && stride < nmax) return fail(ACB_ERR_ARG, "stream stride smaller than one stream's input");
	std::vector<size_t> rows(n, 0), got(n, 0);
	std::vector<unsigned char> ran(m->parts.size(), 0);
	bool first = true;
	int nout = -1;
	for (size_t i = 0; i < m->parts.size(); i++) {
		const Part &p = m->parts[i];
		if (ns && std::all_of(ns + p.s0, ns + p.s0 + p.ns, [](size_t c) { return c == 0; })) continue;
		const size_t off = (size_t)p.s0 * stride * sample_bytes;
		const void *a = (const char *)x + off, *b = x2 ? (const char *)x2 + off : nullptr;
		int r;
		if (ns) {
			size_t *o = &got[p.s0];
			const size_t *c = ns + p.s0;
			r = flag == ACB_FLAG_REAL_INPUT ? acb_submit_real_host_ragged(p.ctx, (const float *)a, stride, c, o)
			    : b ? acb_submit_cs16_planar_host_ragged(p.ctx, (const int16_t *)a, (const int16_t *)b, stride, c, o)
			        : acb_submit_cs16_host_ragged(p.ctx, (const int16_t *)a, stride, c, o);
		} else {
			r = flag == ACB_FLAG_REAL_INPUT ? acb_submit_real_host(p.ctx, (const float *)a, stride, nsamples)
			    : b ? acb_submit_cs16_planar_host(p.ctx, (const int16_t *)a, (const int16_t *)b, stride, nsamples)
			        : acb_submit_cs16_host(p.ctx, (const int16_t *)a, stride, nsamples);
			std::fill(got.begin() + p.s0, got.begin() + p.s0 + p.ns, r < 0 ? 0 : (size_t)r);
		}
		if (r < 0) return r;
		if (!first && (ns ? !std::equal(got.begin() + p.s0, got.begin() + p.s0 + p.ns, rows.begin() + p.s0) && m->mode == ACB_MULTI_SPLIT_CHANNELS
		                  : r != nout))
			return fail(ACB_ERR_CUDA, "parts of a multi-context produced different envelope samples");
		std::copy(got.begin() + p.s0, got.begin() + p.s0 + p.ns, rows.begin() + p.s0);
		nout = std::max(nout, r);
		ran[i] = r > 0;
		first = false;
	}
	if (nout > 0) record_submit(m, rows, std::move(ran));
	if (nout_s) std::copy(rows.begin(), rows.end(), nout_s);
	return nout;
}

extern "C" int acb_multi_submit_real_host(acb_multi_t *m, const float *x, size_t stream_stride_samples, size_t nsamples)
{
	if (!m || !x) return fail(ACB_ERR_ARG, "null argument");
	return submit_streaming(m, ACB_FLAG_REAL_INPUT, x, nullptr, sizeof(float), stream_stride_samples, nsamples);
}

extern "C" int acb_multi_submit_cs16_host(acb_multi_t *m, const int16_t *iq, size_t stream_stride_samples, size_t nsamples)
{
	if (!m || !iq) return fail(ACB_ERR_ARG, "null argument");
	return submit_streaming(m, ACB_FLAG_CS16_INPUT, iq, nullptr, 2 * sizeof(int16_t), stream_stride_samples, nsamples);
}

extern "C" int acb_multi_submit_cs16_planar_host(acb_multi_t *m, const int16_t *xi, const int16_t *xq, size_t stream_stride_samples,
                                                 size_t nsamples)
{
	if (!m || !xi || !xq) return fail(ACB_ERR_ARG, "null argument");
	return submit_streaming(m, ACB_FLAG_CS16_INPUT, xi, xq, sizeof(int16_t), stream_stride_samples, nsamples);
}

extern "C" int acb_multi_submit_real_host_ragged(acb_multi_t *m, const float *x, size_t stream_stride_samples, const size_t *nsamples,
                                                 size_t *nout)
{
	if (!m || !x || !nsamples) return fail(ACB_ERR_ARG, "null argument");
	return submit_streaming(m, ACB_FLAG_REAL_INPUT, x, nullptr, sizeof(float), stream_stride_samples, 0, nsamples, nout);
}

extern "C" int acb_multi_submit_cs16_host_ragged(acb_multi_t *m, const int16_t *iq, size_t stream_stride_samples, const size_t *nsamples,
                                                 size_t *nout)
{
	if (!m || !iq || !nsamples) return fail(ACB_ERR_ARG, "null argument");
	return submit_streaming(m, ACB_FLAG_CS16_INPUT, iq, nullptr, 2 * sizeof(int16_t), stream_stride_samples, 0, nsamples, nout);
}

extern "C" int acb_multi_submit_cs16_planar_host_ragged(acb_multi_t *m, const int16_t *xi, const int16_t *xq, size_t stream_stride_samples,
                                                        const size_t *nsamples, size_t *nout)
{
	if (!m || !xi || !xq || !nsamples) return fail(ACB_ERR_ARG, "null argument");
	return submit_streaming(m, ACB_FLAG_CS16_INPUT, xi, xq, sizeof(int16_t), stream_stride_samples, 0, nsamples, nout);
}

/* pull what every part has queued, translate to global indices, merge in emission order */
static int gather(acb_multi *m)
{
	acb_msg_t buf[64];
	m->scratch.clear();
	for (auto &p : m->parts)
		for (int n; (n = acb_drain(p.ctx, buf, 64)) > 0;)
			for (int i = 0; i < n; i++) {
				buf[i].stream += p.s0;
				buf[i].chn += p.c0;
				m->scratch.push_back(buf[i]);
			}
	/* (submit, group number counted from the stream's start, stream, channel, time), as one context's consumer orders
	 * its submits (context.cu) */
	struct Key { size_t sub; unsigned long long grp; };
	std::vector<Key> key(m->scratch.size());
	for (size_t i = 0; i < key.size(); i++) {
		const acb_msg_t &x = m->scratch[i];
		size_t sub = 0;
		while (sub < m->subs.size() && m->subs[sub].end[x.stream] <= x.pos) sub++;
		key[i] = Key{ sub, acb::group_number(!m->streaming, m->group_unit, m->group_period, m->cfg.K, x.pos) };
	}
	std::vector<size_t> order(key.size());
	for (size_t i = 0; i < order.size(); i++) order[i] = i;
	std::stable_sort(order.begin(), order.end(), [m, &key](size_t ia, size_t ib) {
		const acb_msg_t &a = m->scratch[ia], &b = m->scratch[ib];
		if (key[ia].sub != key[ib].sub) return key[ia].sub < key[ib].sub;
		if (key[ia].grp != key[ib].grp) return key[ia].grp < key[ib].grp;
		if (a.stream != b.stream) return a.stream < b.stream;
		if (a.chn != b.chn) return a.chn < b.chn;
		return a.pos < b.pos;
	});
	for (size_t i : order) m->outq.push_back(m->scratch[i]);
	return (int)m->outq.size();
}

extern "C" int acb_multi_collect(acb_multi_t *m)
{
	if (!m) return ACB_ERR_ARG;
	int err = 0;
	for (size_t i = 0; i < m->parts.size(); i++) {      /* the parts that ran the oldest submit */
		if (!m->subs.empty() && !m->subs.front().part[i]) continue;
		const int r = acb_collect(m->parts[i].ctx);
		if (r < 0 && !err) err = r;
	}
	const int n = gather(m);
	if (!m->subs.empty()) m->subs.pop_front();          /* the oldest submit is merged */
	return err ? err : n;
}

extern "C" int acb_multi_sync(acb_multi_t *m)
{
	if (!m) return ACB_ERR_ARG;
	int err = 0;
	for (auto &p : m->parts) { const int r = acb_sync(p.ctx); if (r < 0 && !err) err = r; }
	const int n = gather(m);
	m->subs.clear();
	return err ? err : n;
}

/* The submits in flight are collected first (as acb_multi_sync does): a message's submit is known from its stream's
 * positions, which restart here. */
extern "C" int acb_multi_reset_stream(acb_multi_t *m, int stream)
{
	if (!m) return fail(ACB_ERR_ARG, "null argument");
	if (stream < 0 || stream >= m->cfg.nstreams) return fail(ACB_ERR_ARG, "stream %d out of range", stream);
	const int r = acb_multi_sync(m);
	if (r < 0) return r;
	for (auto &p : m->parts) {
		if (stream < p.s0 || stream >= p.s0 + p.ns) continue;
		if (int e = acb_reset_stream(p.ctx, stream - p.s0)) return e;
	}
	m->spos[stream] = 0;
	return ACB_OK;
}

extern "C" int acb_multi_drain(acb_multi_t *m, acb_msg_t *out, int max)
{
	if (!m || (!out && max > 0)) return ACB_ERR_ARG;
	int n = 0;
	while (n < max && !m->outq.empty()) { out[n++] = m->outq.front(); m->outq.pop_front(); }
	return n;
}

static Part *find(acb_multi *m, int stream, int chn)
{
	for (auto &p : m->parts)
		if (stream >= p.s0 && stream < p.s0 + p.ns && chn >= p.c0 && chn < p.c0 + p.nc) return &p;
	return nullptr;
}

extern "C" int acb_multi_get_state(acb_multi_t *m, int stream, int chn, acb_chan_state_t *out)
{
	Part *p = m ? find(m, stream, chn) : nullptr;
	return p ? acb_get_state(p->ctx, stream - p->s0, chn - p->c0, out) : ACB_ERR_ARG;
}

extern "C" int acb_multi_set_state(acb_multi_t *m, int stream, int chn, const acb_chan_state_t *in)
{
	Part *p = m ? find(m, stream, chn) : nullptr;
	return p ? acb_set_state(p->ctx, stream - p->s0, chn - p->c0, in) : ACB_ERR_ARG;
}

/* each part's table, placed at the global indices of its chains */
extern "C" int acb_multi_get_decode_stats(acb_multi_t *m, acb_decode_stats_t *out, size_t n, int reset)
{
	if (!m || !out) return fail(ACB_ERR_ARG, "null argument");
	const int nch = m->cfg.nch;
	if (n < (size_t)m->cfg.nstreams * nch) return fail(ACB_ERR_ARG, "n=%zu < nstreams*nch", n);
	std::vector<acb_decode_stats_t> part;
	for (auto &p : m->parts) {
		part.resize((size_t)p.ns * p.nc);
		if (int r = acb_get_decode_stats(p.ctx, part.data(), part.size(), reset)) return r;
		for (int s = 0; s < p.ns; s++)
			for (int c = 0; c < p.nc; c++) out[(size_t)(p.s0 + s) * nch + p.c0 + c] = part[(size_t)s * p.nc + c];
	}
	return ACB_OK;
}

/* each part's tables at the global indices of its streams and chains; in a channel split every part reads every sample,
 * and the input table is part 0's */
extern "C" int acb_multi_get_level_stats(acb_multi_t *m, acb_input_level_t *in, size_t n_in, acb_chan_level_t *ch, size_t n_ch, int reset)
{
	if (!m) return fail(ACB_ERR_ARG, "null argument");
	const int nch = m->cfg.nch;
	if (in && n_in < (size_t)m->cfg.nstreams) return fail(ACB_ERR_ARG, "n_in=%zu < nstreams", n_in);
	if (ch && n_ch < (size_t)m->cfg.nstreams * nch) return fail(ACB_ERR_ARG, "n_ch=%zu < nstreams*nch", n_ch);
	std::vector<acb_input_level_t> pin;
	std::vector<acb_chan_level_t> pch;
	for (size_t i = 0; i < m->parts.size(); i++) {
		const Part &p = m->parts[i];
		pin.resize(p.ns);
		pch.resize((size_t)p.ns * p.nc);
		if (int r = acb_get_level_stats(p.ctx, pin.data(), pin.size(), pch.data(), pch.size(), reset)) return r;
		if (in && (m->mode == ACB_MULTI_SPLIT_STREAMS || i == 0))
			for (int s = 0; s < p.ns; s++) in[p.s0 + s] = pin[s];
		if (ch)
			for (int s = 0; s < p.ns; s++)
				for (int c = 0; c < p.nc; c++) ch[(size_t)(p.s0 + s) * nch + p.c0 + c] = pch[(size_t)s * p.nc + c];
	}
	return ACB_OK;
}

/* each part's table, placed at the global indices of its chains */
extern "C" int acb_multi_get_freq_stats(acb_multi_t *m, acb_chan_freq_t *out, size_t n, int reset)
{
	if (!m || !out) return fail(ACB_ERR_ARG, "null argument");
	const int nch = m->cfg.nch;
	if (n < (size_t)m->cfg.nstreams * nch) return fail(ACB_ERR_ARG, "n=%zu < nstreams*nch", n);
	std::vector<acb_chan_freq_t> part;
	for (auto &p : m->parts) {
		part.resize((size_t)p.ns * p.nc);
		if (int r = acb_get_freq_stats(p.ctx, part.data(), part.size(), reset)) return r;
		for (int s = 0; s < p.ns; s++)
			for (int c = 0; c < p.nc; c++) out[(size_t)(p.s0 + s) * nch + p.c0 + c] = part[(size_t)s * p.nc + c];
	}
	return ACB_OK;
}

/* ---- moving streams: a blob is the one a single context of cfg gives, whatever the split ----
 * A stream split saves each stream on the part that owns it (every part has cfg's fingerprint but nstreams).  In a
 * channel split every part holds every stream but only channels [c0, c0 + nc) of it, in tables laid out for nc channels;
 * a record is converted between a part's layout and the full one on the host (chan_record), the input side and the input
 * levels taken from part 0, which reads the same samples as every part. */
using acb::MvHead;
using acb::MvLayout;
using acb::MvRecHead;

static int multi_list(acb_multi *m, const int *streams, int n)
{
	if (!streams || n < 1 || n > m->cfg.nstreams) return fail(ACB_ERR_ARG, "n=%d outside 1..nstreams", n);
	std::vector<unsigned char> seen(m->cfg.nstreams, 0);
	for (int i = 0; i < n; i++) {
		if (streams[i] < 0 || streams[i] >= m->cfg.nstreams) return fail(ACB_ERR_ARG, "stream %d out of range", streams[i]);
		if (seen[streams[i]]++) return fail(ACB_ERR_ARG, "stream %d listed twice", streams[i]);
	}
	return ACB_OK;
}

static size_t part_of(const acb_multi *m, int stream)
{
	size_t i = 0;
	while (stream >= m->parts[i].s0 + m->parts[i].ns) i++;
	return i;
}

static MvLayout layout_of(const MvHead &h, int nch)
{
	return acb::mv_layout(h.in_kind, h.K, h.taps, nch, h.form, h.flags);
}

/* Channel split: record `part` (layout P, channels [c0, c0 + nc)) to or from record `full` (layout F, nch channels).
 * to_full: the part's channels go to their places, part 0 also gives the host part, the input side and the input levels,
 * and fast_ok is the AND over the parts (the caller starts it at 1), as one context planning all channels would find;
 * the wideband plan's bins are gathered into kbin and its etab noted, the plan itself is rebuilt by the caller.
 * to part: the part's channels are taken out, and its wideband plan is rebuilt from the full plan's bins. */
static void chan_record(const MvHead &h, const MvLayout &F, const MvLayout &P, int c0, int nc, int nch, bool first, uint8_t *part,
                        uint8_t *full, bool to_full, std::vector<int> &kbin, int &etab)
{
	auto mv = [to_full](uint8_t *p, uint8_t *f, size_t n) { to_full ? memcpy(f, p, n) : memcpy(p, f, n); };
	MvRecHead ph, fh;
	memcpy(&ph, part, sizeof(ph));
	memcpy(&fh, full, sizeof(fh));
	if (to_full) {
		if (first) fh = MvRecHead{ ph.pos, ph.carry, fh.fast_ok, 0, 0 };
		fh.fast_ok &= ph.fast_ok;
		memcpy(full, &fh, sizeof(fh));
	} else {
		memcpy(part, &fh, sizeof(fh));
	}
	const int N2 = h.K / 4;
	for (int k = 0; k < F.nreg; k++) {
		uint8_t *fr = full + F.off[k], *pr = part + P.off[k];
		switch (F.tag[k]) {
		case acb::R_STATE: mv(pr, fr + (size_t)c0 * sizeof(acb::ChainState), (size_t)nc * sizeof(acb::ChainState)); break;
		case acb::R_LCARRY: mv(pr, fr + (size_t)c0 * sizeof(acb::LevelCarry), (size_t)nc * sizeof(acb::LevelCarry)); break;
		case acb::R_IN:
			if (!to_full || first) mv(pr, fr, F.bytes[k]);
			break;
		case acb::R_WF: {                            /* [group][tap][8 channels] (c, d) */
			const size_t fg = (size_t)(nch + 7) / 8, tp = F.bytes[k] / (fg * acb::CH_GROUP * 2 * sizeof(float));
			for (int c = 0; c < nc; c++) {
				const int g = c0 + c;
				for (size_t t = 0; t < tp; t++)
					mv(pr + (((size_t)(c / 8) * tp + t) * 8 + c % 8) * 8, fr + (((size_t)(g / 8) * tp + t) * 8 + g % 8) * 8, 8);
			}
			break;
		}
		case acb::R_TW:                              /* [group][8 channels][K/4] (Tr, Ti): channel-major */
			mv(pr, fr + (size_t)c0 * N2 * 2 * sizeof(float), (size_t)nc * N2 * 2 * sizeof(float));
			break;
		case acb::R_TWMETA: {                        /* per group: 2-bit k mod 4 at 2*slot, 2-bit (k/2) mod 4 at 16 + 2*slot */
			uint32_t *pw = (uint32_t *)pr, *fw = (uint32_t *)fr;
			if (!to_full) memset(pr, 0, P.bytes[k]);
			for (int c = 0; c < nc; c++) {
				const int g = c0 + c;
				const uint32_t *sw = to_full ? &pw[c / 8] : &fw[g / 8];
				uint32_t *dw = to_full ? &fw[g / 8] : &pw[c / 8];
				const int ss = to_full ? c % 8 : g % 8, ds = to_full ? g % 8 : c % 8;
				for (int b : { 0, 16 }) {
					const uint32_t v = (*sw >> (b + 2 * ss)) & 3u;
					*dw = (*dw & ~(3u << (b + 2 * ds))) | (v << (b + 2 * ds));
				}
			}
			break;
		}
		case acb::R_WBMETA: {
			if (to_full) {
				for (size_t z = 0; z < P.bytes[k] / (acb::WB_META * sizeof(int)); z++) {
					const int *pm = (const int *)pr + z * acb::WB_META;
					etab = pm[1];
					for (int j = 0; j < std::min(pm[0] * acb::WB_CB, acb::WB_SLOTS); j++)     /* the slots in use only */
						if (pm[3 + 2 * j] >= 0 && pm[3 + 2 * j] < nc) kbin[c0 + pm[3 + 2 * j]] = pm[2 + 2 * j];
				}
			} else {
				acb::wb_meta(h.in_kind, nc, kbin.data() + c0, etab, (int *)pr);
			}
			break;
		}
		}
	}
	if (h.flags & ACB_FLAG_DECODE_STATS)
		mv(part + P.off_dstats, full + F.off_dstats + (size_t)c0 * sizeof(acb_decode_stats_t), (size_t)nc * sizeof(acb_decode_stats_t));
	if (h.flags & ACB_FLAG_LEVEL_STATS) {
		if (!to_full || first) mv(part + P.off_lin, full + F.off_lin, sizeof(acb_input_level_t));
		mv(part + P.off_lch, full + F.off_lch + (size_t)c0 * sizeof(acb_chan_level_t), (size_t)nc * sizeof(acb_chan_level_t));
	}
	if (h.flags & ACB_FLAG_FREQ_STATS)
		mv(part + P.off_fch, full + F.off_fch + (size_t)c0 * sizeof(acb_chan_freq_t), (size_t)nc * sizeof(acb_chan_freq_t));
}

/* the bins of a full record's wideband plan (0 for a stream not on the raster, whose plan is unused) */
static void wb_bins(const MvLayout &F, const uint8_t *full, int nch, std::vector<int> &kbin, int &etab)
{
	MvRecHead fh;
	memcpy(&fh, full, sizeof(fh));
	std::fill(kbin.begin(), kbin.end(), 0);
	for (int k = 0; k < F.nreg; k++) {
		if (F.tag[k] != acb::R_WBMETA) continue;
		for (size_t z = 0; z < F.bytes[k] / (acb::WB_META * sizeof(int)); z++) {
			const int *fm = (const int *)(full + F.off[k]) + z * acb::WB_META;
			etab = fm[1];
			for (int j = 0; fh.fast_ok && j < std::min(fm[0] * acb::WB_CB, acb::WB_SLOTS); j++)     /* the slots in use only */
				if (fm[3 + 2 * j] >= 0 && fm[3 + 2 * j] < nch) kbin[fm[3 + 2 * j]] = fm[2 + 2 * j];
		}
	}
}

/* the full layout: part 0's fingerprint (every part's but nch) with all of cfg's channels */
static MvHead full_head(acb_multi *m)
{
	MvHead h;
	acb::mv_fingerprint(m->parts[0].ctx, h);
	h.nch = m->cfg.nch;
	h.record_bytes = layout_of(h, h.nch).rec_bytes;
	return h;
}

extern "C" size_t acb_multi_streams_blob_bytes(acb_multi_t *m, int n)
{
	if (!m || n < 1) return 0;
	return acb::MV_HEAD_BYTES + (size_t)n * full_head(m).record_bytes;
}

/* Each part saves its streams (collecting its own submits in flight; their messages wait in the part's queue until the
 * next acb_multi_collect / acb_multi_sync merges them), and the records go to their places in the caller's order */
extern "C" int acb_multi_save_streams(acb_multi_t *m, const int *streams, int n, void *blob, size_t cap)
{
	if (!m || !blob) return fail(ACB_ERR_ARG, "null argument");
	if (int r = multi_list(m, streams, n)) return r;
	const MvHead h = full_head(m);
	const MvLayout F = layout_of(h, h.nch);
	const size_t rec = F.rec_bytes, need = acb::MV_HEAD_BYTES + (size_t)n * rec;
	if (cap < need) return fail(ACB_ERR_ARG, "cap=%zu < %zu bytes", cap, need);
	uint8_t *const out = (uint8_t *)blob, *const recs = out + acb::MV_HEAD_BYTES;
	memcpy(out, &h, sizeof(h));
	std::vector<uint8_t> tmp;
	if (m->mode == ACB_MULTI_SPLIT_STREAMS) {
		for (size_t p = 0; p < m->parts.size(); p++) {
			std::vector<int> local, where;
			for (int i = 0; i < n; i++)
				if (part_of(m, streams[i]) == p) local.push_back(streams[i] - m->parts[p].s0), where.push_back(i);
			if (local.empty()) continue;
			tmp.resize(acb::MV_HEAD_BYTES + local.size() * rec);
			if (int r = acb_save_streams(m->parts[p].ctx, local.data(), (int)local.size(), tmp.data(), tmp.size())) return r;
			for (size_t j = 0; j < local.size(); j++)
				memcpy(recs + (size_t)where[j] * rec, tmp.data() + acb::MV_HEAD_BYTES + j * rec, rec);
		}
	} else {
		memset(recs, 0, (size_t)n * rec);
		for (int i = 0; i < n; i++) {
			MvRecHead fh{ 0, 0, 1, 0, 0 };
			memcpy(recs + (size_t)i * rec, &fh, sizeof(fh));
		}
		std::vector<std::vector<int>> kbin(n, std::vector<int>(m->cfg.nch, 0));
		std::vector<int> etab(n, 0);
		for (size_t p = 0; p < m->parts.size(); p++) {
			const Part &q = m->parts[p];
			const MvLayout P = layout_of(h, q.nc);
			tmp.resize(acb::MV_HEAD_BYTES + (size_t)n * P.rec_bytes);
			if (int r = acb_save_streams(q.ctx, streams, n, tmp.data(), tmp.size())) return r;
			for (int i = 0; i < n; i++)
				chan_record(h, F, P, q.c0, q.nc, m->cfg.nch, p == 0, tmp.data() + acb::MV_HEAD_BYTES + (size_t)i * P.rec_bytes,
				            recs + (size_t)i * rec, true, kbin[i], etab[i]);
		}
		for (int k = 0; k < F.nreg; k++) {
			if (F.tag[k] != acb::R_WBMETA) continue;
			for (int i = 0; i < n; i++) {
				MvRecHead fh;
				memcpy(&fh, recs + (size_t)i * rec, sizeof(fh));
				if (!fh.fast_ok) std::fill(kbin[i].begin(), kbin[i].end(), 0);     /* not on the raster: the plan is unused */
				acb::wb_meta(h.in_kind, m->cfg.nch, kbin[i].data(), etab[i], (int *)(recs + (size_t)i * rec + F.off[k]));
			}
		}
	}
	acb::mv_seal(out, need, n);
	return ACB_OK;
}

/* Every part's records are made into a blob of its own and checked against that part before anything changes; then the
 * submits in flight are collected (as acb_multi_reset_stream: the merge tells a message's submit by its stream's
 * position), each part loads, and each stream's position becomes the record's */
extern "C" int acb_multi_load_streams(acb_multi_t *m, const int *streams, int n, const void *blob, size_t size)
{
	if (!m || !blob) return fail(ACB_ERR_ARG, "null argument");
	if (int r = multi_list(m, streams, n)) return r;
	acb_streams_blob_info_t info;
	if (int r = acb_streams_blob_check(blob, size, &info)) return r;
	if (info.nch != m->cfg.nch || info.count != n) return fail(ACB_ERR_ARG, "blob of %d channels and %d records, the call %d and %d", info.nch,
	                                                          info.count, m->cfg.nch, n);
	MvHead h;
	memcpy(&h, blob, sizeof(h));
	const MvLayout F = layout_of(h, h.nch);
	const uint8_t *const in = (const uint8_t *)blob + acb::MV_HEAD_BYTES;
	std::vector<std::vector<uint8_t>> pb(m->parts.size());
	std::vector<std::vector<int>> local(m->parts.size());
	std::vector<int> kbin(m->cfg.nch);
	for (size_t p = 0; p < m->parts.size(); p++) {
		const Part &q = m->parts[p];
		const MvLayout P = layout_of(h, q.nc);
		MvHead ph = h;
		ph.nch = q.nc;
		ph.record_bytes = P.rec_bytes;
		pb[p].assign((const uint8_t *)&ph, (const uint8_t *)&ph + sizeof(ph));
		for (int i = 0; i < n; i++) {
			if (m->mode == ACB_MULTI_SPLIT_STREAMS) {
				if (part_of(m, streams[i]) != p) continue;
				pb[p].insert(pb[p].end(), in + (size_t)i * F.rec_bytes, in + (size_t)(i + 1) * F.rec_bytes);
			} else {
				int etab = 0;
				wb_bins(F, in + (size_t)i * F.rec_bytes, m->cfg.nch, kbin, etab);
				const size_t at = pb[p].size();
				pb[p].resize(at + P.rec_bytes, 0);
				chan_record(h, F, P, q.c0, q.nc, m->cfg.nch, p == 0, pb[p].data() + at, const_cast<uint8_t *>(in + (size_t)i * F.rec_bytes),
				            false, kbin, etab);
			}
			local[p].push_back(streams[i] - q.s0);
		}
		if (local[p].empty()) continue;
		acb::mv_seal(pb[p].data(), pb[p].size(), (int)local[p].size());
		if (int r = acb::mv_validate(q.ctx, pb[p].data(), pb[p].size(), (int)local[p].size())) return r;
	}
	const int r0 = acb_multi_sync(m);
	if (r0 < 0) return r0;
	for (size_t p = 0; p < m->parts.size(); p++)
		if (!local[p].empty())
			if (int r = acb_load_streams(m->parts[p].ctx, local[p].data(), (int)local[p].size(), pb[p].data(), pb[p].size())) return r;
	for (int i = 0; i < n; i++) {
		MvRecHead rh;
		memcpy(&rh, in + (size_t)i * F.rec_bytes, sizeof(rh));
		m->spos[streams[i]] = rh.pos;
	}
	return ACB_OK;
}
