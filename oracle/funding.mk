# oracle/funding.mk — TEST INFRASTRUCTURE: the reference's funding-output script, as gossipd computes it.
#
#   make -C oracle -f funding.mk   -> oracle/_ref/libcln_funding.so
#
# Compiles the reference's unmodified bitcoin/script.c (bitcoin_redeem_2of2, scriptpubkey_p2wsh) with what it links
# against, and links it with funding_harness.c and the objects of the `cln` target of oracle/Makefile (bitcoin/pubkey.c,
# the libwally amalgamation, tal, and cln_harness.c's stand-ins).  Run that target first.  Without those objects (no Core
# Lightning source tree), whatever _ref already holds is kept.
REF ?= $(or $(CLN_SRC),/root/reference)
W = $(REF)/external/libwally-core
CC ?= gcc
CLN_INC = -I _ref/clncfg -I $(REF) -I $(REF)/ccan -I $(W)/include -I $(W)/src/secp256k1/include
FUNDING_SRCS = bitcoin/script.c common/pseudorand.c ccan/ccan/isaac/isaac64.c \
  ccan/ccan/crypto/siphash24/siphash24.c

all:
	@if [ -f $(REF)/bitcoin/script.c ] && [ -f _ref/libcln_ref.so ]; then $(MAKE) -f funding.mk _ref/libcln_funding.so; \
	else echo "reference tree or _ref/libcln_ref.so absent: keeping prebuilt oracle/_ref"; fi

_ref/libcln_funding.so: funding_harness.c funding.mk _ref/libcln_ref.so
	mkdir -p _ref/fundobj
	for f in $(FUNDING_SRCS); do $(CC) -O2 -fPIC -w $(CLN_INC) -c $(REF)/$$f -o _ref/fundobj/`echo $$f | tr / _`.o || exit 1; done
	$(CC) -O2 -fPIC -Wall $(CLN_INC) -c funding_harness.c -o _ref/fundobj/funding_harness.o
	$(CC) -shared -Wl,--no-undefined -o $@ _ref/clnobj/*.o _ref/fundobj/*.o -lpthread

.PHONY: all
