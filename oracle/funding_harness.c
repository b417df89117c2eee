/*
 * oracle/funding_harness.c — TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * The script gossipd expects a channel's funding output to have (gossipd/gossmap_manage.c:696-699):
 * scriptpubkey_p2wsh(bitcoin_redeem_2of2(bitcoin_key_1, bitcoin_key_2)), computed by the reference's own unmodified
 * bitcoin/script.c and bitcoin/pubkey.c.  Linked by oracle/funding.mk with the objects of the `cln` target of
 * oracle/Makefile.  Flat C entry points for ctypes.  Output: oracle/_ref/libcln_funding.so.
 */
#include "config.h"
#include <bitcoin/pubkey.h>
#include <bitcoin/script.h>
#include <ccan/tal/tal.h>
#include <common/randbytes.h>
#include <common/utils.h>
#include <secp256k1.h>
#include <stdlib.h>
#include <string.h>

/* stand-ins for common/randbytes.c (libsodium): script.c links pseudorand.c for its hash-table seeds, which the functions
 * below never use */
void randbytes_(void *bytes, size_t num_bytes, u64 *offset) { (void)offset; memset(bytes, 0, num_bytes); }
bool randbytes_overridden(void) { return true; }

static void setup(void) {
    if (!secp256k1_ctx) secp256k1_ctx = secp256k1_context_create(SECP256K1_CONTEXT_VERIFY | SECP256K1_CONTEXT_SIGN);
}

/* out34 = scriptpubkey_p2wsh(bitcoin_redeem_2of2(key1, key2)); 0 if a key does not parse or the script is not 34 bytes */
int cln_funding_script(const u8 *key1_33, const u8 *key2_33, u8 *out34) {
    struct pubkey k1, k2;
    setup();
    if (!pubkey_from_der(key1_33, 33, &k1) || !pubkey_from_der(key2_33, 33, &k2)) return 0;
    u8 *redeem = bitcoin_redeem_2of2(NULL, &k1, &k2);
    u8 *spk = scriptpubkey_p2wsh(NULL, redeem);
    int ok = tal_bytelen(spk) == 34;
    if (ok) memcpy(out34, spk, 34);
    tal_free(redeem);
    tal_free(spk);
    return ok;
}

static int by_scid(const void *a, const void *b) {
    const u64 x = *(const u64 *)a, y = *(const u64 *)b;
    return x < y ? -1 : x > y;
}

/* What lightningd and gossipd do per announcement on one core, for timing: the script from the keys (parsed from their
 * 33 bytes, as fromwire does), then the output looked up by scid (bsearch over scid_sorted, n_out entries; the script
 * of entry i at script34 + 34 * i) and the scripts compared.  match[i] = 1 found with the same script, 0 otherwise. */
void cln_funding_check_batch(const u8 *keys66, const u64 *scid, size_t n, const u64 *scid_sorted, const u8 *script34,
                             size_t n_out, u8 *match) {
    setup();
    for (size_t i = 0; i < n; i++) {
        u8 want[34];
        const u64 *hit = bsearch(&scid[i], scid_sorted, n_out, sizeof(u64), by_scid);
        match[i] = cln_funding_script(keys66 + 66 * i, keys66 + 66 * i + 33, want) && hit &&
                   !memcmp(script34 + 34 * (size_t)(hit - scid_sorted), want, 34);
    }
}
