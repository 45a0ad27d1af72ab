/*
 * TEST INFRASTRUCTURE — NOT PRODUCT CODE.
 *
 * The host emulation of the demodulator loop (demod_emul.cpp, included whole: the same accessor, environment and
 * tables) with the counting kernels' accessor: the frame synchroniser's events of frame_sm.h reach event(), as they
 * reach DevFrameAccStats in k_demod2_stats, so tests/test_decode_stats_oracle.py can hold the device loop's own
 * definition of the decode statistics to the restatement's on the CPU.  Built by tests/decode_stats_refs.py with g++
 * -O2 -ffp-contract=off.
 */
#include "demod_emul.cpp"

/* counts[EV_*] of frame_sm.h; EV_SHORT for an emitted block under 13 bytes (no ring here: no EV_LOST) */
struct HostFrameAccCounted : HostFrameAcc {
	unsigned long long *counts;
	void event(int e) { counts[e]++; }
	void frame_emit()
	{
		if (r.blk_len < 13) counts[EV_SHORT]++;
		HostFrameAcc::frame_emit();
	}
};

/* demod_emul's call with the counts added to counts[EV_COUNT] */
extern "C" int demod_emul_counted(acb_chan_state_t *st, const float *dm, int nsamp, int stride, int f2f, EmulFrame *frames,
                                  int maxframes, unsigned long long *counts)
{
	static DemodShared<1> sm;
	static bool init = false;
	if (!init) {
		float h[FLENO];
		acb_build_h(h);
		for (int o = 0; o <= MFLTOVER; o++) {
			float t[12];
			for (int j = 0; j < 12; j++) t[j] = j < FLEN ? h[o + MFLTOVER * j] : 0.f;
			for (int q = 0; q < 3; q++) { sm.h2[o][q].x = t[4 * q]; sm.h2[o][q].y = t[4 * q + 1]; sm.h2[o][q].z = t[4 * q + 2]; sm.h2[o][q].w = t[4 * q + 3]; }
		}
		double tc[128], ts[128];
		acb_build_sincos_table(tc, ts);
		for (int k = 0; k < 64; k++) { sm.tcos[k].x = tc[2 * k]; sm.tcos[k].y = tc[2 * k + 1]; sm.tsin[k].x = ts[2 * k]; sm.tsin[k].y = ts[2 * k + 1]; }
		init = true;
	}
	DemodRegs r;
	r.phi = st->MskPhi; r.df = st->MskDf; r.lvlsum = st->MskLvlSum; r.clk = st->MskClk; r.bitcount = st->MskBitCount;
	r.S = st->MskS; r.idx = st->idx % FLEN; r.nbits = st->nbits; r.state = st->Acarsstate; r.outbits = st->outbits;
	r.blk_len = st->blk_len; r.blk_err = st->blk_err; r.pos = st->pos; r.soh_pos = st->soh_pos;
	for (int k = 0; k < FLEN; k++) {
		DcF2 v;
		v.x = st->inb_re[k]; v.y = st->inb_im[k];
		sm.ring[k][0] = v;
		sm.ring[k + FLEN][0] = v;
	}
	HostFrameAccCounted acc{ { r, st, frames, maxframes, 0 }, counts };
	if (f2f) demod_run<1, true, true, HostEnv>(r, sm, dm, stride, nsamp, 0, 0, acc);
	else demod_run<1, false, true, HostEnv>(r, sm, dm, stride, nsamp, 0, 0, acc);
	st->MskPhi = r.phi; st->MskDf = r.df; st->MskLvlSum = r.lvlsum; st->MskClk = r.clk; st->MskBitCount = r.bitcount;
	st->MskS = r.S; st->idx = r.idx; st->nbits = r.nbits; st->Acarsstate = r.state; st->outbits = r.outbits;
	st->blk_len = r.blk_len; st->blk_err = r.blk_err; st->pos = r.pos; st->soh_pos = r.soh_pos;
	for (int k = 0; k < FLEN; k++) { st->inb_re[k] = sm.ring[k][0].x; st->inb_im[k] = sm.ring[k][0].y; }
	return acc.n;
}
