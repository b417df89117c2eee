/*
 * oracle/bolt11_harness.c — TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * The reference's own bolt11_decode (common/bolt11.c:980-1062) and bolt11_decode_nosig (:748-975) on an invoice string,
 * compiled unmodified by oracle/bolt11.mk, and libsecp256k1's secp256k1_ecdsa_recover on its own.  Flat C entry points for
 * ctypes.  Output: oracle/_ref/libcln_bolt11.so.
 */
#include "config.h"
#include <bitcoin/pubkey.h>
#include <common/bolt11.h>
#include <common/node_id.h>
#include <common/utils.h>
#include <secp256k1.h>
#include <secp256k1_recovery.h>
#include <stdlib.h>
#include <string.h>
#include <sys/mman.h>
#include <sys/wait.h>
#include <unistd.h>

/* the globals live in libcln_ref.so (oracle/cln_harness.c); set them up if nothing has yet */
static void setup(void) {
    if (!secp256k1_ctx)
        secp256k1_ctx = secp256k1_context_create(SECP256K1_CONTEXT_VERIFY | SECP256K1_CONTEXT_SIGN);
    if (!tmpctx) tmpctx = tal(NULL, char);
}

static void copy_msg(char *out, size_t cap, const char *msg) {
    memset(out, 0, cap);
    if (msg) strncpy(out, msg, cap - 1);
}

/* buf[0 .. len) with a NUL appended is the string bolt11_decode receives (so it ends at the first NUL in buf).
 * bolt11_decode with no features, no description and no chain.
 * Returns bit 0: bolt11_decode returned an invoice; bit 1: bolt11_decode_nosig did.  node33: its receiver_id (zeros when it
 * failed); hash32: bolt11_decode_nosig's signing hash (zeros when it failed); fail / nosig_fail: the failure messages. */
int cln_bolt11_check(const char *buf, size_t len, uint8_t *node33, uint8_t *hash32, char *fail_out, char *nosig_fail_out) {
    setup();
    const tal_t *ctx = tal(NULL, char);
    char *fail = NULL, *nosig_fail = NULL;
    struct sha256 hash;
    const u5 *sig;
    bool have_n;
    int r = 0;
    char *str = tal_arr(ctx, char, len + 1);
    memcpy(str, buf, len);
    str[len] = '\0';
    memset(node33, 0, 33);
    memset(hash32, 0, 32);
    struct bolt11 *b = bolt11_decode_nosig(ctx, str, NULL, NULL, NULL, &hash, &sig, &have_n, &nosig_fail);
    if (b) {
        r |= 2;
        memcpy(hash32, hash.u.u8, 32);
    }
    b = bolt11_decode(ctx, str, NULL, NULL, NULL, &fail);
    if (b) {
        r |= 1;
        memcpy(node33, b->receiver_id.k, 33);
    }
    copy_msg(fail_out, 256, fail);
    copy_msg(nosig_fail_out, 256, nosig_fail);
    tal_free(ctx);
    tal_free(tmpctx);
    tmpctx = tal(NULL, char);
    return r;
}

/* secp256k1_ecdsa_recoverable_signature_parse_compact + secp256k1_ecdsa_recover; returns 1 with the compressed key, 0 when
 * either refuses (out33 zeros) */
int cln_ecdsa_recover(const uint8_t *sig64, int recid, const uint8_t *msg32, uint8_t *out33) {
    setup();
    secp256k1_ecdsa_recoverable_signature s;
    secp256k1_pubkey pk;
    size_t len = 33;
    memset(out33, 0, 33);
    if (!secp256k1_ecdsa_recoverable_signature_parse_compact(secp256k1_ctx, &s, sig64, recid)) return 0;
    if (!secp256k1_ecdsa_recover(secp256k1_ctx, &pk, &s, msg32)) return 0;
    secp256k1_ec_pubkey_serialize(secp256k1_ctx, out33, &len, &pk, SECP256K1_EC_COMPRESSED);
    return 1;
}

/* bolt11_decode alone (no features, description or chain) over n invoices, the way a caller decodes them: ok[i] = 1 where
 * it returns an invoice.  The invoices are split over procs forked processes; returns 0, or -1 if a process failed. */
int cln_bolt11_decode_batch(const uint8_t *blob, const uint64_t *off, const uint32_t *len, size_t n, int *ok, int procs) {
    setup();
    if (procs < 1) procs = 1;
    if ((size_t)procs > n) procs = n ? (int)n : 1;
    int *shared = mmap(NULL, (n ? n : 1) * sizeof(int), PROT_READ | PROT_WRITE, MAP_SHARED | MAP_ANONYMOUS, -1, 0);
    if (shared == MAP_FAILED) return -1;
    pid_t *pids = calloc(procs, sizeof(pid_t));
    int rc = 0;
    for (int w = 0; w < procs; w++) {
        size_t lo = n * w / procs, hi = n * (w + 1) / procs;
        pid_t pid = fork();
        if (pid == 0) {
            for (size_t i = lo; i < hi; i++) {
                const tal_t *ctx = tal(NULL, char);
                char *fail = NULL, *str = tal_arr(ctx, char, len[i] + 1);
                memcpy(str, blob + off[i], len[i]);
                str[len[i]] = '\0';
                shared[i] = bolt11_decode(ctx, str, NULL, NULL, NULL, &fail) != NULL;
                tal_free(ctx);
                tal_free(tmpctx);
                tmpctx = tal(NULL, char);
            }
            _exit(0);
        }
        if (pid < 0) rc = -1;
        pids[w] = pid;
    }
    for (int w = 0; w < procs; w++) {
        int st = 0;
        if (pids[w] > 0 && (waitpid(pids[w], &st, 0) < 0 || !WIFEXITED(st) || WEXITSTATUS(st) != 0)) rc = -1;
    }
    if (rc == 0) memcpy(ok, shared, n * sizeof(int));
    munmap(shared, (n ? n : 1) * sizeof(int));
    free(pids);
    return rc;
}
