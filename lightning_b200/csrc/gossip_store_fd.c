/*
 * gossip_store_fd.c — sv_prune_gossip_store_fd and sv_repair_gossip_store_fd (cln_sigverify.h): prune a gossip_store
 * FILE in place, and cut a torn tail off it.  Plain C, linked into libcln_sigverify.so.  It reads the file, calls the
 * engine's public prune entry points (sv_gossip_prune_count, sv_prune_gossip_store_host) and writes back only the flags of
 * the records they deleted, the way gossipd deletes a record (gossip_store_del, gossipd/gossip_store.c:572-638: the be16
 * flags at the record's header, bit 0x8000 set).  The repair then truncates the file where the prune's walk stopped at a
 * torn append (sv_gossip_prune_cut), as gossipd does to a store it upgrades (gossipd/gossip_store.c:319).
 */
#define _GNU_SOURCE
#include "../../include/cln_sigverify.h"
#include "gossip_store_fd.h"

#include <errno.h>
#include <fcntl.h>
#include <stdlib.h>
#include <string.h>
#include <sys/stat.h>
#include <unistd.h>

#define IO_CHUNK ((size_t)1 << 30) /* bytes per pread / pwrite call */

int gsfd_read_all(int fd, uint8_t *p, size_t len) {
    size_t got = 0;
    while (got < len) {
        size_t want = len - got < IO_CHUNK ? len - got : IO_CHUNK;
        ssize_t r = pread(fd, p + got, want, (off_t)got);
        if (r < 0 && errno == EINTR) continue;
        if (r < 0) return -1;
        if (r == 0) { errno = EIO; return -1; }
        got += (size_t)r;
    }
    return 0;
}

int gsfd_write_at(int fd, const uint8_t *p, size_t len, uint64_t off) {
    while (len) {
        ssize_t w = pwrite(fd, p, len, (off_t)off);
        if (w < 0 && errno == EINTR) continue;
        if (w <= 0) { if (w == 0) errno = EIO; return -1; }
        p += w;
        len -= (size_t)w;
        off += (uint64_t)w;
    }
    return 0;
}

int gsfd_sync(int fd) {
    while (fsync(fd) < 0)
        if (errno != EINTR) return -1;
    return 0;
}

/* the tail rule on the walk summary alone: where the torn append begins */
static uint64_t tail_cut(const sv_gossip_prune_summary *s, uint64_t len) {
    switch (s->stop) {
    case SV_GS_INCOMPLETE: /* a torn append: the record the walk stopped at and everything after it go */
    case SV_GS_PARTIAL:
    case SV_GS_NO_AMOUNT:
    case SV_GS_EOF:        /* only a torn header (1 to 12 bytes the walk never reads) lies between end_offset and len */
        return s->end_offset < len ? s->end_offset : len;
    default:               /* SV_GS_ENDED: the store was replaced, not torn */
        return len;
    }
}

/* The first live channel_announcement of store[0, cut) without the 22 bytes of its channel_amount record before cut
 * (gossmap.c:488-492 checks the room by length alone), or cut if there is none.  gossipd writes a record with flags 0 and
 * sets COMPLETED in a second write, so a crash between the two during the amount's append leaves a whole amount record
 * the walk stops at (SV_GS_INCOMPLETE): cut there, the announcement would end the store with no room for it. */
static uint64_t announcement_without_room(const uint8_t *store, uint64_t cut) {
    uint64_t off = 1;
    while (off + 12 + 2 <= cut) {
        const unsigned flags = ((unsigned)store[off] << 8) | store[off + 1];
        const uint64_t mlen = ((uint64_t)store[off + 2] << 8) | store[off + 3];
        const unsigned type = ((unsigned)store[off + 12] << 8) | store[off + 13];
        if (off + 12 + mlen > cut) break;
        if (!(flags & 0x8000) && type == 256 && off + 12 + mlen + 12 + 2 + 8 > cut) return off;
        off += 12 + mlen;
    }
    return cut;
}

uint64_t sv_gossip_prune_cut(const sv_gossip_prune_summary *s, const uint8_t *pruned, uint64_t len) {
    if (!s || !pruned) return len;
    uint64_t cut = tail_cut(s, len);
    if (cut == len) return len;
    /* an announcement left without room for its amount ends the store at it; again for one before it (never for a
     * store gossipd wrote, where every announcement is followed by its 22-byte amount record) */
    for (uint64_t at; (at = announcement_without_room(pruned, cut)) < cut;) cut = at;
    return cut;
}

int gsfd_check(int fd, uint64_t len) {
    struct stat st;
    int fl = fcntl(fd, F_GETFL);
    if (fl < 0) return SV_ERR_IO; /* errno EBADF: not an open descriptor */
    if (fstat(fd, &st) < 0) return SV_ERR_IO;
    if (!S_ISREG(st.st_mode) || len < 1 || len > (uint64_t)st.st_size || len > SIZE_MAX) { errno = EINVAL; return SV_ERR_ARG; }
    if ((fl & O_ACCMODE) != O_RDWR) { errno = EBADF; return SV_ERR_IO; } /* the deletions could not be written */
    return SV_OK;
}

/* sv_prune_gossip_store_fd; with cut, also where the repair ends the file (sv_gossip_prune_cut of the pruned store) */
static int prune_file(sv_ctx *ctx, int fd, uint64_t len, const uint8_t *chain_hash32, sv_gossip_prune_summary *summary,
                      uint64_t *cut) {
    if (!ctx || !summary) { errno = EINVAL; return SV_ERR_ARG; }
    int chk = gsfd_check(fd, len);
    if (chk != SV_OK) return chk;
    uint8_t *store = (uint8_t *)malloc((size_t)len);
    if (!store) return SV_ERR_NOMEM;
    int rc = SV_ERR_IO, e = 0;
    uint64_t *rec_off = NULL;
    uint16_t *rec_type = NULL;
    int *rec_status = NULL;
    uint8_t *rec_pruned = NULL;
    if (gsfd_read_all(fd, store, (size_t)len) < 0) { e = errno; goto out; }
    size_t cap = sv_gossip_prune_count(store, (size_t)len);
    rec_off = (uint64_t *)malloc(8 * (cap + 1));
    rec_type = (uint16_t *)malloc(2 * (cap + 1));
    rec_status = (int *)malloc(sizeof(int) * (cap + 1));
    rec_pruned = (uint8_t *)malloc(cap + 1);
    if (!rec_off || !rec_type || !rec_status || !rec_pruned) { rc = SV_ERR_NOMEM; goto out; }
    rc = sv_prune_gossip_store_host(ctx, store, (size_t)len, chain_hash32, store, rec_off, rec_type, rec_status, rec_pruned,
                                    cap, summary);
    if (rc != SV_OK) { e = rc == SV_ERR_ARG ? EINVAL : 0; goto out; }
    for (uint64_t r = 0; r < summary->records; r++)
        if (rec_pruned[r] && gsfd_write_at(fd, store + rec_off[r], 2, rec_off[r]) < 0) { rc = SV_ERR_IO; e = errno; goto out; }
    if (gsfd_sync(fd) < 0) { rc = SV_ERR_IO; e = errno; goto out; }
    if (cut) *cut = sv_gossip_prune_cut(summary, store, len);
out:
    free(store); free(rec_off); free(rec_type); free(rec_status); free(rec_pruned);
    if (e) errno = e;
    return rc;
}

int sv_prune_gossip_store_fd(sv_ctx *ctx, int fd, uint64_t len, const uint8_t *chain_hash32, sv_gossip_prune_summary *summary) {
    return prune_file(ctx, fd, len, chain_hash32, summary, NULL);
}

int sv_repair_gossip_store_fd(sv_ctx *ctx, int fd, uint64_t len, const uint8_t *chain_hash32, sv_gossip_prune_summary *summary,
                              uint64_t *new_len) {
    uint64_t cut;
    int rc = prune_file(ctx, fd, len, chain_hash32, summary, &cut);
    if (rc != SV_OK) return rc;
    /* the deletions are on disk before the file shrinks: a crash in between leaves a pruned store with its torn tail */
    if (cut < len) {
        int r;
        while ((r = ftruncate(fd, (off_t)cut)) < 0 && errno == EINTR) {}
        if (r < 0 || gsfd_sync(fd) < 0) return SV_ERR_IO;
    }
    if (new_len) *new_len = cut;
    return SV_OK;
}

