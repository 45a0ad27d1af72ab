# TEST INFRASTRUCTURE.  Builds
#   _ref/libacarsref_verbose.so   libacarsref_O2.so's sources (ref_harness.c, the UNMODIFIED acars.c in place through
#                                 ref_acars_tap.c, msk.c) plus ref_verbose.c, which makes the reference's -v switch
#                                 reachable: its per-event stderr lines, counted by tests/test_decode_stats_oracle.py
#                                 against the restatement's decode statistics
# Run by __graft_entry__.build() beside the Makefile.  Needs the reference source tree (REF); where it is absent nothing
# is built and whatever _ref/ already holds is kept.
REF ?= /root/reference
CC ?= gcc
STRICT = -O2 -ffp-contract=off
COMMON = -fPIC -shared -std=gnu11 -w
REFSRC = ref_harness.c ref_acars_tap.c $(REF)/msk.c ref_verbose.c
REFINC = -DWITH_RTL -Istub -I$(REF)

all:
	@if [ -d $(REF) ]; then $(MAKE) -f verbose.mk _ref/libacarsref_verbose.so; \
	else echo "oracle: $(REF) absent, keeping prebuilt _ref/"; fi

_ref/libacarsref_verbose.so: ref_harness.c ref_acars_tap.c ref_verbose.c stub/rtl-sdr.h
	mkdir -p _ref && $(CC) $(STRICT) $(COMMON) $(REFINC) -o $@ $(REFSRC) -lm -lpthread
