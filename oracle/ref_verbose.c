/*
 * TEST INFRASTRUCTURE — NOT PRODUCT CODE.
 *
 * The reference's -v switch (acarsdec.c's `verbose`) for oracle/_ref/libacarsref_verbose.so (recipe: oracle/verbose.mk),
 * which is libacarsref_O2.so's sources (ref_harness.c, the unmodified acars.c in place through ref_acars_tap.c, msk.c)
 * plus this file.  Once set, decodeAcars and blk_thread print their per-event lines on stderr (acars.c:101-206,
 * 311-354); tests/test_decode_stats_oracle.py counts them by kind and channel against the restatement's counts
 * (tests/host/decode_stats_oracle.c).
 */
extern int verbose;

void ref_set_verbose(int v) { verbose = v; }
