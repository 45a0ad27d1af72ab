/*
 * Front-end test host for the shim libraries (libacarsdec_compat*.so, one per WITH_* macro): the globals
 * (acarsdec.c:34-57), an outputmsg() sink and acarsdec.c's init/run/close order for ONE front-end, chosen by the macro
 * this file is compiled with.  Unlike the reference program built under oracle/_ref, it needs nothing but the product's
 * headers and libraries, so it always runs the shim as built from this tree.
 *
 *   -DWITH_RTL      fehost <K> <u8 IQ file> <MHz>...        initRtl / runRtlSample / runRtlClose
 *   -DWITH_AIR      fehost <float32 file> <MHz>...          initAirspy / runAirspySample (rate: ACARSDEC_B200_AIRRATE)
 *   -DWITH_SOAPY    fehost <K> <CS16 file> <MHz>...         initSoapy / runSoapySample / runSoapyClose
 *   -DWITH_SDRPLAY  fehost <MHz>...                         initSdrplay / runSdrplaySample (file: ACARSDEC_B200_CAPTURE)
 *
 * Every delivered block is printed as: chn len err crc txt(hex).  Exit status 1 when the front-end's init fails.
 */
#define _GNU_SOURCE
#include <stdio.h>
#include <stdlib.h>
#include "acarsdec_compat.h"

channel_t channel[MAXNBCHANNELS];
unsigned int nbch;
int verbose = 0;
int signalExit = 0;
#ifdef WITH_RTL
int gain = -100, ppm = 0, rtlMult = 160;
#endif
#ifdef WITH_AIR
int gain = 18;
#endif
#ifdef WITH_SOAPY
int rateMult = 160, freq = 0, ppm = 0;
double gain = -10.0;
#endif
#ifdef WITH_SDRPLAY
int gain = -100, ppm = 0;
#endif

void outputmsg(const msgblk_t *blk)
{
	printf("%d %d %d %02x%02x ", blk->chn, blk->len, blk->err, blk->crc[0], blk->crc[1]);
	for (int i = 0; i < blk->len; i++) printf("%02x", (unsigned char)blk->txt[i]);
	printf("\n");
	fflush(stdout);
}

static int init_decoders(void)
{
	for (unsigned n = 0; n < nbch; n++) {          /* acarsdec.c:445-454 */
		channel[n].chn = n;
		if (initMsk(&channel[n])) return 1;
		if (initAcars(&channel[n])) return 1;
	}
	return 0;
}

int main(int argc, char **argv)
{
	int res;
#if defined(WITH_RTL) || defined(WITH_SOAPY)
	if (argc < 4) return 2;
#ifdef WITH_RTL
	rtlMult = atoi(argv[1]);
	if (initRtl(argv, 2)) { fprintf(stderr, "Unable to init input\n"); return 1; }
#else
	rateMult = atoi(argv[1]);
	if (initSoapy(argv, 2)) { fprintf(stderr, "Unable to init input\n"); return 1; }
#endif
#else
	if (argc < 2) return 2;
#ifdef WITH_AIR
	if (initAirspy(argv, 1)) { fprintf(stderr, "Unable to init input\n"); return 1; }
#else
	if (initSdrplay(argv, 1)) { fprintf(stderr, "Unable to init input\n"); return 1; }
#endif
#endif
	if (init_decoders()) { fprintf(stderr, "Unable to init internal decoders\n"); return 1; }
#if defined(WITH_RTL)
	res = runRtlSample();
	if (!res) res = runRtlClose();
#elif defined(WITH_AIR)
	res = runAirspySample();
#elif defined(WITH_SOAPY)
	res = runSoapySample();
	if (!res) res = runSoapyClose();
#else
	res = runSdrplaySample();
#endif
	deinitAcars();
	return res ? 1 : 0;
}
