/*
 * oracle/bolt12_harness.c — TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * The reference's own bolt12_check_signature path (common/bolt12.c:80-92) on a raw TLV stream: fromwire_tlv with any
 * type allowed (wire/tlvstream.c:144-300), merkle_tlv and sighash_from_merkle (common/bolt12_merkle.c:160-220) and
 * check_schnorr_sig (bitcoin/signature.c:408-430), all compiled unmodified by oracle/bolt12.mk.  Flat C entry points for
 * ctypes.  Output: oracle/_ref/libcln_bolt12.so.
 */
#include "config.h"
#include <bitcoin/pubkey.h>
#include <bitcoin/signature.h>
#include <common/bolt12_merkle.h>
#include <common/utils.h>
#include <secp256k1.h>
#include <stdlib.h>
#include <string.h>
#include <sys/mman.h>
#include <sys/wait.h>
#include <unistd.h>
#include <wire/tlvstream.h>

/* wire/tlvstream.c's tlvstream_set_short_channel_id needs it (bitcoin/short_channel_id.c is not in libcln_ref.so); the
 * BOLT12 path never calls it */
void towire_short_channel_id(u8 **pptr, struct short_channel_id short_channel_id) {
    (void)pptr; (void)short_channel_id;
    abort();
}

/* the globals live in libcln_ref.so (oracle/cln_harness.c); set them up if nothing has yet */
static void setup(void) {
    if (!secp256k1_ctx) secp256k1_ctx = secp256k1_context_create(SECP256K1_CONTEXT_VERIFY | SECP256K1_CONTEXT_SIGN);
    if (!tmpctx) tmpctx = tal(NULL, char);
}

/* 1 / 0 = bolt12_check_signature's answer for these fields, key 02||x and signature; -1 = fromwire_tlv refuses the stream
 * or it holds no field (merkle_tlv asserts on that).  merkle32_out / sighash32_out: zeros for -1. */
int cln_bolt12_check(const u8 *stream, size_t len, const char *messagename, const char *fieldname, const u8 *xonly32,
                     const u8 *sig64, u8 *merkle32_out, u8 *sighash32_out) {
    setup();
    memset(merkle32_out, 0, 32);
    memset(sighash32_out, 0, 32);
    tal_t *ctx = tal(NULL, char);
    struct tlv_field *fields = tal_arr(ctx, struct tlv_field, 0);
    const u8 *cursor = stream;
    size_t max = len;
    if (!fromwire_tlv(&cursor, &max, NULL, 0, ctx, &fields, FROMWIRE_TLV_ANY_TYPE, NULL, NULL) || tal_count(fields) == 0) {
        tal_free(ctx);
        return -1;
    }
    struct sha256 m, sh;
    merkle_tlv(fields, &m);
    sighash_from_merkle(messagename, fieldname, &m, &sh);
    memcpy(merkle32_out, m.u.u8, 32);
    memcpy(sighash32_out, sh.u.u8, 32);
    u8 der[33];
    struct pubkey key;
    struct bip340sig sig;
    int r = 0;
    der[0] = 2;
    memcpy(der + 1, xonly32, 32);
    memcpy(sig.u8, sig64, 64);
    if (pubkey_from_der(der, 33, &key)) r = check_schnorr_sig(&sh, &key.pubkey, &sig) ? 1 : 0;
    tal_free(ctx);
    return r;
}

/* The same for n streams (stream i = blob[off[i] .. off[i]+len[i])), spread over `procs` worker processes: the CPU
 * baseline.  tal is not thread-safe (merkle_tlv allocates from the NULL parent), so the workers are forked processes
 * writing into shared memory; all of them have exited when this returns.  Returns 0, or -1 if a worker failed. */
int cln_bolt12_check_batch(const u8 *blob, const uint64_t *off, const uint32_t *len, size_t n, const char *messagename,
                           const char *fieldname, const u8 *xonly32, const u8 *sig64, int *status, int procs) {
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
            u8 m[32], h[32];
            for (size_t i = lo; i < hi; i++)
                shared[i] = cln_bolt12_check(blob + off[i], len[i], messagename, fieldname, xonly32 + 32 * i, sig64 + 64 * i, m, h);
            _exit(0);
        }
        if (pid < 0) rc = -1;
        pids[w] = pid;
    }
    for (int w = 0; w < procs; w++) {
        int st = 0;
        if (pids[w] > 0 && (waitpid(pids[w], &st, 0) < 0 || !WIFEXITED(st) || WEXITSTATUS(st) != 0)) rc = -1;
    }
    if (rc == 0) memcpy(status, shared, n * sizeof(int));
    munmap(shared, (n ? n : 1) * sizeof(int));
    free(pids);
    return rc;
}
