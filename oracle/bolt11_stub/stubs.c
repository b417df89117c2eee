/*
 * oracle/bolt11_stub/stubs.c — TEST INFRASTRUCTURE: the common/utils.c functions common/bolt11.c names, written for the
 * oracle build (oracle/bolt11.mk) instead of linking common/utils.c, whose globals libcln_ref.so already defines.
 *
 * utf8_str checks with the utf8_check libcln_ref.so carries (oracle/cln_harness.c: it accepts every buffer), so the
 * oracle never refuses a `d` field for its UTF-8; the device does not check it either (cln_sigverify.h).
 * str_lowering is only reached through to_canonical_invstr, which the oracle never calls.
 */
#include "config.h"
#include <ccan/take/take.h>
#include <ccan/tal/tal.h>
#include <common/randbytes.h>
#include <common/utils.h>
#include <stdlib.h>
#include <string.h>

char *utf8_str(const tal_t *ctx, const u8 *buf TAKES, size_t buflen) {
    char *ret = NULL;
    if (utf8_check(buf, buflen)) {
        ret = tal_arr(ctx, char, buflen + 1);
        memcpy(ret, buf, buflen);
        ret[buflen] = '\0';
    }
    if (taken(buf)) tal_free(buf);
    return ret;
}

char *str_lowering(const void *ctx, const char *string TAKES) {
    (void)ctx; (void)string;
    abort();
}

/* common/randbytes.c needs libsodium; bitcoin/script.c and common/pseudorand.c name these, the decoder never reaches them */
void randbytes_(void *bytes, size_t num_bytes, u64 *offset) {
    (void)bytes; (void)num_bytes; (void)offset;
    abort();
}
bool randbytes_overridden(void) {
    abort();
}
