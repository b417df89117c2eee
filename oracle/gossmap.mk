# oracle/gossmap.mk — TEST INFRASTRUCTURE: the reference's gossip_store loader, unmodified.
#
#   make -C oracle -f gossmap.mk   -> oracle/_ref/libcln_gossmap.so
#
# Compiles common/gossmap.c with what it needs (common/amount.c, common/fp16.c, common/node_id.c and the ccan modules
# below) where they lie under $(REF) (a Core Lightning source tree: $CLN_SRC if set, else /root/reference), together with
# gossmap_harness.c.  CCAN's config.h is the one the `cln` target of oracle/Makefile produced with the reference's own
# configurator.  gossmap.c includes two headers the CLN build generates from wire CSVs, which the source tree does not
# hold; gossmap_inc/ holds stand-ins (message type numbers and two prototypes) and is searched first.  Without a source
# tree, or before the `cln` target has run, whatever _ref already holds is kept.
REF ?= $(or $(CLN_SRC),/root/reference)
W = $(REF)/external/libwally-core
CC ?= gcc
GM_SRCS = common/gossmap.c common/amount.c common/fp16.c common/node_id.c ccan/ccan/crc32c/crc32c.c \
  ccan/ccan/htable/htable.c ccan/ccan/tal/tal.c ccan/ccan/tal/str/str.c ccan/ccan/take/take.c ccan/ccan/list/list.c \
  ccan/ccan/str/str.c ccan/ccan/str/hex/hex.c ccan/ccan/err/err.c ccan/ccan/mem/mem.c
GM_INC = -I gossmap_inc -I _ref/clncfg -I $(REF) -I $(REF)/ccan -I $(W)/include -I $(W)/src/secp256k1/include

all:
	@if [ -f $(REF)/common/gossmap.c ] && [ -f _ref/clncfg/config.h ]; then $(MAKE) -f gossmap.mk _ref/libcln_gossmap.so; \
	else echo "reference tree or _ref/clncfg/config.h absent: keeping prebuilt oracle/_ref"; fi

_ref/libcln_gossmap.so: gossmap_harness.c gossmap.mk gossmap_inc/wire/peer_wiregen.h gossmap_inc/common/gossip_store_wiregen.h
	mkdir -p _ref/gmobj
	for f in $(GM_SRCS); do $(CC) -O2 -fPIC -w $(GM_INC) -c $(REF)/$$f -o _ref/gmobj/`echo $$f | tr / _`.o || exit 1; done
	$(CC) -O2 -fPIC -Wall -Wno-unused-parameter $(GM_INC) -c gossmap_harness.c -o _ref/gmobj/gossmap_harness.o
	$(CC) -shared -Wl,--no-undefined -o $@ _ref/gmobj/*.o

.PHONY: all
