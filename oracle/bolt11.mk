# oracle/bolt11.mk — TEST INFRASTRUCTURE: the reference's BOLT11 decoder, unmodified.
#
#   make -C oracle -f bolt11.mk   -> oracle/_ref/libcln_bolt11.so
#
# Compiles common/bolt11.c with the files it needs (bech32, bech32_util, hash_u5, features, amount, chainparams, script and
# their own needs) where they lie under $(REF) (a Core Lightning source tree: $CLN_SRC if set, else /root/reference)
# together with bolt11_harness.c, linked against _ref/libcln_ref.so (oracle/Makefile target `cln`: node_id, pubkey, the
# wire layer, tal and libsecp256k1 with the recovery module).  bolt11.c includes lightningd/lightningd.h for nothing the
# decoder uses; bolt11_stub/lightningd/lightningd.h stands in for it and is searched first, and bolt11_stub/stubs.c
# defines the few symbols the linked files name but the decoder never reaches.
# Without a source tree, or before the `cln` target has run, whatever _ref already holds is kept.
REF ?= $(or $(CLN_SRC),/root/reference)
W = $(REF)/external/libwally-core
CC ?= gcc
B11_SRCS = common/bolt11.c common/bech32.c common/bech32_util.c common/hash_u5.c common/features.c common/amount.c \
  bitcoin/script.c bitcoin/short_channel_id.c bitcoin/chainparams.c common/pseudorand.c \
  ccan/ccan/isaac/isaac64.c ccan/ccan/crypto/siphash24/siphash24.c
B11_INC = -I bolt11_stub -I gossmap_inc -I _ref/clncfg -I $(REF) -I $(REF)/ccan -I $(W)/include -I $(W)/src/secp256k1/include

all:
	@if [ -f $(REF)/common/bolt11.c ] && [ -f _ref/libcln_ref.so ]; then $(MAKE) -f bolt11.mk _ref/libcln_bolt11.so; \
	else echo "reference tree or _ref/libcln_ref.so absent: keeping prebuilt oracle/_ref"; fi

_ref/libcln_bolt11.so: bolt11_harness.c bolt11_stub/stubs.c bolt11_stub/lightningd/lightningd.h bolt11.mk _ref/libcln_ref.so
	mkdir -p _ref/b11obj
	for f in $(B11_SRCS); do $(CC) -O2 -fPIC -w $(B11_INC) -c $(REF)/$$f -o _ref/b11obj/`echo $$f | tr / _`.o || exit 1; done
	$(CC) -O2 -fPIC -Wall $(B11_INC) -c bolt11_harness.c -o _ref/b11obj/bolt11_harness.o
	$(CC) -O2 -fPIC -Wall $(B11_INC) -c bolt11_stub/stubs.c -o _ref/b11obj/stubs.o
	$(CC) -shared -Wl,--no-undefined -o $@ _ref/b11obj/*.o -L _ref -lcln_ref -Wl,-rpath,'$$ORIGIN'

.PHONY: all
