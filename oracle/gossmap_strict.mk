# oracle/gossmap_strict.mk — TEST INFRASTRUCTURE: the reference's gossip_store loader, loading as gossipd does at start-up.
#
#   make -C oracle -f gossmap_strict.mk   -> oracle/_ref/libcln_gossmap_strict.so
#
# Links gossmap_strict_harness.c with the objects oracle/gossmap.mk compiled (common/gossmap.c unmodified, what it needs,
# and gossmap_harness.c for the stand-ins gossmap.c links against).  Run gossmap.mk first.  Without those objects (no
# Core Lightning source tree), whatever _ref already holds is kept.
REF ?= $(or $(CLN_SRC),/root/reference)
W = $(REF)/external/libwally-core
CC ?= gcc
GM_INC = -I gossmap_inc -I _ref/clncfg -I $(REF) -I $(REF)/ccan -I $(W)/include -I $(W)/src/secp256k1/include

all:
	@if [ -f $(REF)/common/gossmap.c ] && [ -f _ref/libcln_gossmap.so ]; then $(MAKE) -f gossmap_strict.mk _ref/libcln_gossmap_strict.so; \
	else echo "reference tree or _ref/libcln_gossmap.so absent: keeping prebuilt oracle/_ref"; fi

_ref/libcln_gossmap_strict.so: gossmap_strict_harness.c gossmap_strict.mk _ref/libcln_gossmap.so
	mkdir -p _ref/gmstrict
	$(CC) -O2 -fPIC -Wall -Wno-unused-parameter $(GM_INC) -c gossmap_strict_harness.c -o _ref/gmstrict/gossmap_strict_harness.o
	$(CC) -shared -Wl,--no-undefined -o $@ _ref/gmobj/*.o _ref/gmstrict/gossmap_strict_harness.o

.PHONY: all
