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
