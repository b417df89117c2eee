/*
 * oracle/gossmap_strict_harness.c — TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * Loads a gossip_store with the reference's own common/gossmap.c as gossipd does at start-up (gossmap_load_initial,
 * gossipd/gossmap_manage.c:525): expected_len = the store's length, so the load refuses a bad checksum, a truncated
 * record, a redundant announcement, an unknown record type and a walk that stops short of the end (common/gossmap.c:862,
 * :885, :895, :922, :1428-1438).  Reports the channel table as gossmap_harness.c does, and each node's current
 * node_announcement.  Linked by oracle/gossmap_strict.mk with the objects of oracle/gossmap.mk (gossmap.c unmodified, and
 * gossmap_harness.c for the stand-ins gossmap.c links against).  Flat C entry point for ctypes.
 * Output: oracle/_ref/libcln_gossmap_strict.so.
 *
 * As in gossmap_harness.c, each load runs in a forked child that sends its answer back through a pipe: gossmap asserts
 * or exits on some stores, and the caller survives whatever it does.
 */
#include "config.h"
#include <bitcoin/short_channel_id.h>
#include <ccan/tal/tal.h>
#include <common/gossmap.h>
#include <common/utils.h>
#include <fcntl.h>
#include <signal.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/resource.h>
#include <sys/wait.h>
#include <unistd.h>

static void quiet(void *cbarg, enum log_level level, const char *fmt, ...) {}

static int write_all(int fd, const void *p, size_t n) {
    const char *c = p;
    while (n) {
        ssize_t w = write(fd, c, n);
        if (w <= 0) return -1;
        c += w;
        n -= (size_t)w;
    }
    return 0;
}

static int by_cann_off(const void *a, const void *b) {
    const u64 *x = a, *y = b;
    return x[1] < y[1] ? -1 : x[1] > y[1];
}

static int by_u64(const void *a, const void *b) {
    const u64 *x = a, *y = b;
    return *x < *y ? -1 : *x > *y;
}

/* the child: load strictly, then send [channel count or -1][map_end][count x (scid, cann_off, cupdate_off[0],
 * cupdate_off[1])][node count][node count x nann_off] */
static void child(const char *path, int fd, u64 len) {
    tmpctx = tal(NULL, char);
    struct gossmap *map = gossmap_load_(NULL, path, len, quiet, NULL, NULL);
    s64 n = -1, nn = 0;
    u64 end = 0, total;
    u64 *rows = NULL, *nodes = NULL;
    if (map) {
        n = 0;
        for (struct gossmap_chan *c = gossmap_first_chan(map); c; c = gossmap_next_chan(map, c)) n++;
        rows = calloc(n ? n : 1, 4 * sizeof(u64));
        s64 i = 0;
        for (struct gossmap_chan *c = gossmap_first_chan(map); c; c = gossmap_next_chan(map, c), i++) {
            rows[4 * i] = gossmap_chan_scid(map, c).u64;
            rows[4 * i + 1] = c->cann_off;
            rows[4 * i + 2] = c->cupdate_off[0];
            rows[4 * i + 3] = c->cupdate_off[1];
        }
        qsort(rows, n, 4 * sizeof(u64), by_cann_off);
        end = gossmap_lengths(map, &total);
        for (struct gossmap_node *d = gossmap_first_node(map); d; d = gossmap_next_node(map, d)) nn++;
        nodes = calloc(nn ? nn : 1, sizeof(u64));
        i = 0;
        for (struct gossmap_node *d = gossmap_first_node(map); d; d = gossmap_next_node(map, d)) nodes[i++] = d->nann_off;
        qsort(nodes, nn, sizeof(u64), by_u64);
    }
    if (write_all(fd, &n, 8) || write_all(fd, &end, 8)) _exit(3);
    if (n >= 0 && ((n > 0 && write_all(fd, rows, (size_t)n * 32)) || write_all(fd, &nn, 8) ||
                   (nn > 0 && write_all(fd, nodes, (size_t)nn * 8))))
        _exit(3);
    _exit(0);
}

/* Returns the channel count (rows up to cap written to chans: scid, cann_off, cupdate_off[0], cupdate_off[1], sorted by
 * cann_off; offsets are of messages, 12 past their record header) with *map_end = gossmap_lengths() and *n_nodes, the
 * nann_off of every node up to ncap in nodes (the message offset of its current node_announcement, 0 if none), sorted
 * ascending; -1 if gossmap refuses the store; -2 if the load did not return; -3 if no temporary file could be written. */
long long cln_gossmap_load_strict(const u8 *store, size_t len, u64 *map_end, u64 *chans, size_t cap, u64 *nodes,
                                  size_t ncap, u64 *n_nodes) {
    const char *dir = getenv("TMPDIR");
    char *path = malloc(strlen(dir ? dir : "/tmp") + 32);
    sprintf(path, "%s/gossmap_strict.XXXXXX", dir ? dir : "/tmp");
    int tfd = mkstemp(path);
    *map_end = 0;
    *n_nodes = 0;
    if (tfd < 0 || write_all(tfd, store, len)) {
        if (tfd >= 0) { close(tfd); unlink(path); }
        free(path);
        return -3;
    }
    close(tfd);
    int p[2];
    if (pipe(p)) { unlink(path); free(path); return -3; }
    fflush(NULL);
    pid_t pid = fork();
    if (pid == 0) {
        close(p[0]);
        /* no gossmap log lines or assertion messages in the test output, no crash handler of the caller, no core files */
        int null = open("/dev/null", O_WRONLY);
        if (null >= 0) dup2(null, 2);
        signal(SIGABRT, SIG_DFL);
        signal(SIGSEGV, SIG_DFL);
        struct rlimit no_core = {0, 0};
        setrlimit(RLIMIT_CORE, &no_core);
        child(path, p[1], len);
    }
    close(p[1]);
    /* read everything before waiting: a large table does not fit the pipe */
    size_t have = 0, size = 4096;
    u8 *buf = malloc(size);
    for (;;) {
        if (have == size) buf = realloc(buf, size *= 2);
        ssize_t r = read(p[0], buf + have, size - have);
        if (r <= 0) break;
        have += (size_t)r;
    }
    close(p[0]);
    int st = 0;
    long long ret = -2;
    if (pid > 0 && waitpid(pid, &st, 0) == pid && WIFEXITED(st) && WEXITSTATUS(st) == 0 && have >= 16) {
        s64 n, nn;
        memcpy(&n, buf, 8);
        memcpy(map_end, buf + 8, 8);
        if (n == -1) {
            ret = -1;
        } else if (n >= 0 && have >= 24 + (size_t)n * 32) {
            memcpy(&nn, buf + 16 + (size_t)n * 32, 8);
            if (nn >= 0 && have == 24 + (size_t)n * 32 + (size_t)nn * 8) {
                memcpy(chans, buf + 16, (size_t)(n < (s64)cap ? n : (s64)cap) * 32);
                memcpy(nodes, buf + 24 + (size_t)n * 32, (size_t)(nn < (s64)ncap ? nn : (s64)ncap) * 8);
                *n_nodes = (u64)nn;
                ret = n;
            }
        }
    }
    free(buf);
    unlink(path);
    free(path);
    return ret;
}
