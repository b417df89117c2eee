/*
 * fake_engine_repair.c — a stand-in for the engine's gossip_store prune (sv_gossip_prune_count, sv_prune_gossip_store_host
 * of cln_sigverify.h) whose walk stops where gossmap's does on a torn store, linked beside fake_engine.c or
 * fake_engine_timed.c so that sv_repair_gossip_store_fd (lightning_b200/csrc/gossip_store_fd.c), the verifier subdaemon's
 * repair requests and the drop-in's gossip_store_repair can be tested without a GPU
 * (tests/test_sigverifyd_repair_fake.py).  It deletes a fixed set of records for fixed reasons, which the test recomputes:
 *   walk    from offset 1 while 13 bytes are left (a shorter tail is a torn header: stop SV_GS_EOF, end_offset < len).
 *           A record without bit 0x2000 stops it (SV_GS_INCOMPLETE); one with bit 0x8000 is stepped over (so a deleted
 *           record running past the end leaves end_offset > len); one running past the end stops it (SV_GS_PARTIAL), as
 *           does a type 4105 (SV_GS_ENDED) and a type 256 with fewer than 22 bytes after it (SV_GS_NO_AMOUNT).  The
 *           record it stops at is not an entry, so summary.records counts one record fewer than the engine's walk
 *           gives for a stopped store (gs_walk emits the record it stops at too); the cut does not read it.
 *           end_offset is the stop's offset, or where the walk ran out.
 *   delete  entry r (0-based, in walk order) when r % 3 == 1 and it is not deleted yet, for reason 1 + (r / 3) % 8
 *           (SV_GP_BAD_CRC .. SV_GP_UNKNOWN); reverified counts the SV_GP_SIGNATURE deletions
 * A major version other than 0, len 0 or rec_capacity below the entry count: SV_ERR_ARG, nothing written.  Each call
 * appends "sv_prune_gossip_store_host 0 <entries> <len>" to $FAKE_ENGINE_LOG, and writes a "begin" and an "end" line to
 * $FAKE_ENGINE_TRACE as fake_engine_prune.c does ($FAKE_ENGINE_DELAY "sv_prune_gossip_store_host=<ms>" holds it between).
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

/* the walk: each entry's offset into offs (if given); returns the entry count, *end and *stop where it ended */
static size_t walk(const uint8_t *s, size_t len, uint64_t *end, int32_t *stop, uint64_t *offs) {
    uint64_t off = 1;
    size_t r = 0;
    *stop = SV_GS_EOF;
    while (off + 12 < len) {
        const unsigned flags = ((unsigned)s[off] << 8) | s[off + 1];
        const uint64_t mlen = ((uint64_t)s[off + 2] << 8) | s[off + 3];
        const unsigned type = off + 14 <= len ? ((unsigned)s[off + 12] << 8) | s[off + 13] : 0;
        if (!(flags & 0x2000)) { *stop = SV_GS_INCOMPLETE; break; }
        if (!(flags & 0x8000)) {
            if (off + 12 + mlen > len) { *stop = SV_GS_PARTIAL; break; }
            if (type == 4105) { *stop = SV_GS_ENDED; break; }
            if (type == 256 && off + 12 + mlen + 22 > len) { *stop = SV_GS_NO_AMOUNT; break; }
        }
        if (offs) offs[r] = off;
        r++;
        off += 12 + mlen;
    }
    *end = off;
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
