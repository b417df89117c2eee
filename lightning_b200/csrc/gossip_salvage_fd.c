/*
 * gossip_salvage_fd.c — sv_salvage_gossip_store_fd (cln_sigverify.h): salvage a gossip_store FILE in place, then repair
 * it.  Plain C, linked into libcln_sigverify.so.  It reads the file, calls sv_salvage_gossip_store_host and writes back
 * only the 4 bytes of flags and length of each header the salvage changed, then runs sv_repair_gossip_store_fd.
 */
#define _GNU_SOURCE
#include "../../include/cln_sigverify.h"
#include "gossip_store_fd.h"

#include <errno.h>
#include <stdlib.h>

/* the 4 bytes of flags and length of the header at off, as the salvage wrote them into out */
static int write_header(int fd, const uint8_t *out, uint64_t off) { return gsfd_write_at(fd, out + off, 4, off); }

/* the header after the one at p in out, by its length */
static uint64_t next_filler(const uint8_t *out, uint64_t p) { return p + 12 + (((uint64_t)out[p + 2] << 8) | out[p + 3]); }

/* the salvage's header writes, one action at a time in store order.  The headers of an action chain from its offset to
 * where the records resume: one for a restored header, the fillers for a bridge.  A bridge's fillers are written from the
 * last to the first, and synced before the first one overwrites the damaged header: until that 4-byte write reaches the
 * disk, the walk still reads the damaged header and never reaches the others, so a crash or a power loss at any point
 * leaves the store as it was or with the whole bridge.  (A bridge has a filler per 64 KiB of its span, so finding each
 * one from the first is cheap.) */
static int write_salvage(int fd, const uint8_t *out, const uint64_t *off, const uint64_t *resume, size_t n) {
    for (size_t a = 0; a < n; a++) {
        size_t k = 0;
        for (uint64_t p = off[a]; p < resume[a]; p = next_filler(out, p)) k++;
        while (k--) {
            uint64_t p = off[a];
            for (size_t i = 0; i < k; i++) p = next_filler(out, p);
            if (k == 0 && next_filler(out, p) < resume[a] && gsfd_sync(fd) < 0) return -1;
            if (write_header(fd, out, p) < 0) return -1;
        }
    }
    return 0;
}

int sv_salvage_gossip_store_fd(sv_ctx *ctx, int fd, uint64_t len, const uint8_t *chain_hash32, sv_gossip_prune_summary *summary,
                               sv_gossip_salvage_summary *salvage, uint64_t *new_len) {
    if (!ctx || !summary || !salvage) { errno = EINVAL; return SV_ERR_ARG; }
    int chk = gsfd_check(fd, len);
    if (chk != SV_OK) return chk;
    uint8_t *store = (uint8_t *)malloc((size_t)len), *out = (uint8_t *)malloc((size_t)len);
    size_t cap = 1024;
    uint64_t *act_off = NULL, *act_resume = NULL;
    uint8_t *act_kind = NULL;
    sv_gossip_salvage_summary sv;
    int rc = SV_ERR_NOMEM, e = 0;
    if (!store || !out) goto out;
    if (gsfd_read_all(fd, store, (size_t)len) < 0) { rc = SV_ERR_IO; e = errno; goto out; }
    for (;;) { /* again with room for every action, in the rare store with more breaks than the first guess */
        free(act_off); free(act_resume); free(act_kind);
        act_off = (uint64_t *)malloc(8 * cap);
        act_resume = (uint64_t *)malloc(8 * cap);
        act_kind = (uint8_t *)malloc(cap);
        if (!act_off || !act_resume || !act_kind) { rc = SV_ERR_NOMEM; goto out; }
        rc = sv_salvage_gossip_store_host(ctx, store, (size_t)len, out, act_off, act_resume, act_kind, cap, &sv);
        if (rc != SV_OK) { e = rc == SV_ERR_ARG ? EINVAL : 0; goto out; }
        if (sv.breaks <= cap) break;
        cap = (size_t)sv.breaks;
    }
    if (sv.breaks) {
        if (write_salvage(fd, out, act_off, act_resume, (size_t)sv.breaks) < 0 || gsfd_sync(fd) < 0) {
            rc = SV_ERR_IO;
            e = errno;
            goto out;
        }
    }
    free(store); free(out); free(act_off); free(act_resume); free(act_kind);
    rc = sv_repair_gossip_store_fd(ctx, fd, len, chain_hash32, summary, new_len);
    if (rc == SV_OK) *salvage = sv;
    return rc;
out:
    free(store); free(out); free(act_off); free(act_resume); free(act_kind);
    if (e) errno = e;
    return rc;
}
