/*
 * gossip_store_fd.c — sv_prune_gossip_store_fd (cln_sigverify.h): prune a gossip_store FILE in place.  Plain C, linked
 * into libcln_sigverify.so.  It reads the file, calls the engine's public prune entry points (sv_gossip_prune_count,
 * sv_prune_gossip_store_host) and writes back only the flags of the records they deleted, the way gossipd deletes a
 * record (gossip_store_del, gossipd/gossip_store.c:572-638: the be16 flags at the record's header, bit 0x8000 set).
 */
#define _GNU_SOURCE
#include "../../include/cln_sigverify.h"

#include <errno.h>
#include <fcntl.h>
#include <stdlib.h>
#include <string.h>
#include <sys/stat.h>
#include <unistd.h>

#define IO_CHUNK ((size_t)1 << 30) /* bytes per pread / pwrite call */

/* len bytes from offset 0; -1 with errno on failure (EIO: the file ended early) */
static int read_all(int fd, uint8_t *p, size_t len) {
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

static int write_at(int fd, const uint8_t *p, size_t len, uint64_t off) {
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

int sv_prune_gossip_store_fd(sv_ctx *ctx, int fd, uint64_t len, const uint8_t *chain_hash32, sv_gossip_prune_summary *summary) {
    struct stat st;
    if (!ctx || !summary) { errno = EINVAL; return SV_ERR_ARG; }
    int fl = fcntl(fd, F_GETFL);
    if (fl < 0) return SV_ERR_IO; /* errno EBADF: not an open descriptor */
    if (fstat(fd, &st) < 0) return SV_ERR_IO;
    if (!S_ISREG(st.st_mode) || len < 1 || len > (uint64_t)st.st_size || len > SIZE_MAX) { errno = EINVAL; return SV_ERR_ARG; }
    if ((fl & O_ACCMODE) != O_RDWR) { errno = EBADF; return SV_ERR_IO; } /* the deletions could not be written */
    uint8_t *store = (uint8_t *)malloc((size_t)len);
    if (!store) return SV_ERR_NOMEM;
    int rc = SV_ERR_IO, e = 0;
    uint64_t *rec_off = NULL;
    uint16_t *rec_type = NULL;
    int *rec_status = NULL;
    uint8_t *rec_pruned = NULL;
    if (read_all(fd, store, (size_t)len) < 0) { e = errno; goto out; }
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
        if (rec_pruned[r] && write_at(fd, store + rec_off[r], 2, rec_off[r]) < 0) { rc = SV_ERR_IO; e = errno; goto out; }
    while (fsync(fd) < 0) {
        if (errno == EINTR) continue;
        rc = SV_ERR_IO;
        e = errno;
        break;
    }
out:
    free(store); free(rec_off); free(rec_type); free(rec_status); free(rec_pruned);
    if (e) errno = e;
    return rc;
}
