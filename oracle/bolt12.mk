# oracle/bolt12.mk — TEST INFRASTRUCTURE: the reference's BOLT12 signature hashing, unmodified.
#
#   make -C oracle -f bolt12.mk   -> oracle/_ref/libcln_bolt12.so
#
# Compiles common/bolt12_merkle.c, common/bigsize.c, wire/tlvstream.c, ccan/ccan/ilog/ilog.c and ccan/ccan/asort/asort.c
# where they lie under $(REF) (a Core Lightning source tree: $CLN_SRC if set, else /root/reference) together with
# bolt12_harness.c, linked against _ref/libcln_ref.so (oracle/Makefile target `cln`: bitcoin/signature.c, the wire layer,
# tal and libsecp256k1).  bolt12_merkle.h includes the generated wire/bolt12_wiregen.h, which the source tree does not
# hold; a stand-in that includes only what bolt12_merkle.c uses is written to _ref/b12inc and searched first.
# Without a source tree, or before the `cln` target has run, whatever _ref already holds is kept.
REF ?= $(or $(CLN_SRC),/root/reference)
W = $(REF)/external/libwally-core
CC ?= gcc
B12_SRCS = common/bolt12_merkle.c common/bigsize.c wire/tlvstream.c ccan/ccan/ilog/ilog.c ccan/ccan/asort/asort.c
B12_INC = -I _ref/b12inc -I _ref/clncfg -I $(REF) -I $(REF)/ccan -I $(W)/include -I $(W)/src/secp256k1/include

all:
	@if [ -f $(REF)/common/bolt12_merkle.c ] && [ -f _ref/libcln_ref.so ]; then $(MAKE) -f bolt12.mk _ref/libcln_bolt12.so; \
	else echo "reference tree or _ref/libcln_ref.so absent: keeping prebuilt oracle/_ref"; fi

_ref/libcln_bolt12.so: bolt12_harness.c bolt12.mk _ref/libcln_ref.so
	mkdir -p _ref/b12inc/wire _ref/b12obj
	printf '#include <common/bigsize.h>\n#include <wire/tlvstream.h>\n#include <bitcoin/signature.h>\n' > _ref/b12inc/wire/bolt12_wiregen.h
	for f in $(B12_SRCS); do $(CC) -O2 -fPIC -w $(B12_INC) -c $(REF)/$$f -o _ref/b12obj/`echo $$f | tr / _`.o || exit 1; done
	$(CC) -O2 -fPIC -Wall $(B12_INC) -c bolt12_harness.c -o _ref/b12obj/bolt12_harness.o
	$(CC) -shared -Wl,--no-undefined -o $@ _ref/b12obj/*.o -L _ref -lcln_ref -Wl,-rpath,'$$ORIGIN'

.PHONY: all
