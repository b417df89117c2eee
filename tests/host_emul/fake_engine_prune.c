/*
 * fake_engine_prune.c — a stand-in for the engine's gossip_store prune (sv_gossip_prune_count, sv_prune_gossip_store_host
 * of cln_sigverify.h), linked beside fake_engine.c or fake_engine_timed.c so that sv_prune_gossip_store_fd
 * (lightning_b200/csrc/gossip_store_fd.c), the verifier subdaemon's prune requests and the drop-in's gossip_store_prune
 * can be tested without a GPU (tests/test_sigverifyd_prune_fake.py).  It deletes a fixed set of records for fixed reasons,
 * which the test recomputes:
 *   walk    from offset 1 while a whole 12-byte header fits; a record whose message runs past the end stops it
 *           (stop SV_GS_PARTIAL, end_offset its offset), else the walk ends at the end (SV_GS_EOF)
 *   delete  record r (0-based, in walk order) when r % 3 == 1 and its flags do not have bit 0x8000 yet, for reason
 *           1 + (r / 3) % 8 (SV_GP_BAD_CRC .. SV_GP_UNKNOWN); reverified counts the SV_GP_SIGNATURE deletions
 * A major version other than 0, len 0 or rec_capacity below the record count: SV_ERR_ARG, nothing written.  Each call
 * appends "sv_prune_gossip_store_host 0 <records> <len>" to $FAKE_ENGINE_LOG.  Like fake_engine_timed.c, a
 * "sv_prune_gossip_store_host=<ms>" entry in $FAKE_ENGINE_DELAY holds each call that long, between a
 * "begin sv_prune_gossip_store_host 0" and an "end sv_prune_gossip_store_host 0" line in $FAKE_ENGINE_TRACE.
 */
#define _POSIX_C_SOURCE 200809L /* nanosleep */
#include "../../include/cln_sigverify.h"

#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>

#define FN "sv_prune_gossip_store_host"

static void append(const char *var, const char *line) {
    const char *path = getenv(var);
    FILE *f = path ? fopen(path, "a") : NULL;
    if (!f) return;
    fputs(line, f);
    fclose(f);
}
static long prune_delay_ms(void) {
    const char *d = getenv("FAKE_ENGINE_DELAY");
    size_t fl = strlen(FN);
    while (d && *d) {
        if (!strncmp(d, FN, fl) && d[fl] == '=') return strtol(d + fl + 1, NULL, 10);
        d = strchr(d, ',');
        if (d) d++;
    }
    return 0;
}

/* the walk: each record's offset into offs (if given); returns the record count, *end and *stop where it ended */
static size_t walk(const uint8_t *s, size_t len, uint64_t *end, int32_t *stop, uint64_t *offs) {
    size_t off = 1, r = 0;
    *stop = SV_GS_EOF;
    while (off + 12 <= len) {
        size_t mlen = ((size_t)s[off + 2] << 8) | s[off + 3];
        if (off + 12 + mlen > len) { *stop = SV_GS_PARTIAL; break; }
        if (offs) offs[r] = off;
        r++;
        off += 12 + mlen;
    }
    *end = off < len ? off : len;
    return r;
}

size_t sv_gossip_prune_count(const uint8_t *store, size_t len) {
    uint64_t end;
    int32_t stop;
    return store && len ? walk(store, len, &end, &stop, NULL) : 0;
}

int sv_prune_gossip_store_host(sv_ctx *ctx, const uint8_t *store, size_t len, const uint8_t *chain_hash32, uint8_t *out,
                               uint64_t *rec_off, uint16_t *rec_type, int *rec_status, uint8_t *rec_pruned,
                               size_t rec_capacity, sv_gossip_prune_summary *sum) {
    (void)chain_hash32;
    char line[128];
    long ms = prune_delay_ms();
    append("FAKE_ENGINE_TRACE", "begin " FN " 0\n");
    if (ms > 0) {
        struct timespec t = {ms / 1000, (ms % 1000) * 1000000L};
        while (nanosleep(&t, &t) != 0) {}
    }
    append("FAKE_ENGINE_TRACE", "end " FN " 0\n");
    if (!ctx || !store || !out || !len || !sum || (store[0] >> 5)) return SV_ERR_ARG;
    uint64_t end;
    int32_t stop;
    size_t n = walk(store, len, &end, &stop, NULL);
    snprintf(line, sizeof line, FN " 0 %zu %zu\n", n, len);
    append("FAKE_ENGINE_LOG", line);
    if (n > rec_capacity || (n && (!rec_off || !rec_type || !rec_status || !rec_pruned))) return SV_ERR_ARG;
    if (out != store) memcpy(out, store, len);
    walk(store, len, &end, &stop, rec_off);
    sv_gossip_prune_summary S;
    memset(&S, 0, sizeof S);
    S.version = store[0];
    S.stop = stop;
    S.end_offset = end;
    S.records = n;
    for (size_t r = 0; r < n; r++) {
        const uint64_t o = rec_off[r];
        rec_type[r] = (uint16_t)(o + 14 <= len ? (store[o + 12] << 8) | store[o + 13] : 0);
        rec_status[r] = 0;
        rec_pruned[r] = 0;
        if (r % 3 != 1 || (out[o] & 0x80)) continue;
        const uint8_t why = (uint8_t)(1 + (r / 3) % 8);
        out[o] |= 0x80;
        rec_pruned[r] = why;
        S.pruned++;
        uint64_t *by[9] = {NULL, &S.bad_crc, &S.truncated, &S.message, &S.redundant, &S.no_channel, &S.signature, &S.amount,
                           &S.unknown};
        (*by[why])++;
        S.reverified += why == SV_GP_SIGNATURE;
    }
    *sum = S;
    return SV_OK;
}
