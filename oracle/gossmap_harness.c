/*
 * oracle/gossmap_harness.c — TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * Loads a gossip_store with the reference's own common/gossmap.c (compiled unmodified by oracle/gossmap.mk) and reports
 * the channel table it ends with.  Flat C entry point for ctypes.  Output: oracle/_ref/libcln_gossmap.so.
 *
 * gossmap reads a store through a file, and some stores end it: map_copy asserts when a read runs past the end of the
 * store, and an ENDED record makes reopen_store look for the next file and errx when it is not one.  So each load runs in
 * a forked child that sends its answer back through a pipe; the caller survives whatever gossmap does.
 */
#include "config.h"
#include <bitcoin/short_channel_id.h>
#include <bitcoin/signature.h>
#include <ccan/tal/str/str.h>
#include <ccan/tal/tal.h>
#include <common/gossip_store_wiregen.h>
#include <common/gossmap.h>
#include <common/pseudorand.h>
#include <common/sciddir_or_pubkey.h>
#include <common/utils.h>
#include <wire/wire.h>
#include <fcntl.h>
#include <signal.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/resource.h>
#include <sys/wait.h>
#include <unistd.h>
#include <wire/peer_wiregen.h>

/* ---- what gossmap.c, amount.c and node_id.c link against but a plain load never needs from the rest of CLN ---- */
/* local modifications only (gossmap_apply_localmods), never called here */
u8 *towire_channel_update(const tal_t *ctx, const secp256k1_ecdsa_signature *signature,
                          const struct bitcoin_blkid *chain_hash, struct short_channel_id short_channel_id, u32 timestamp,
                          u8 message_flags, u8 channel_flags, u16 cltv_expiry_delta, struct amount_msat htlc_minimum_msat,
                          u32 fee_base_msat, u32 fee_proportional_millionths, struct amount_msat htlc_maximum_msat) {
    abort();
}
/* only with a dying callback, and the load passes none */
bool fromwire_gossip_store_chan_dying(const void *p, struct short_channel_id *scid, u32 *blockheight) { abort(); }
/* the node table's hash: any fixed seed gives the same table */
const struct siphash_seed *siphash_seed(void) {
    static struct siphash_seed seed;
    return &seed;
}
uint64_t pseudorand_u64_(uint64_t *offset) { return 0; }
/* log text only: the harness's log callback drops it */
char *fmt_short_channel_id(const tal_t *ctx, struct short_channel_id scid) { return tal_strdup(ctx, ""); }
char *tal_hexstr(const tal_t *ctx, const void *data, size_t len) { return tal_strdup(ctx, ""); }
char *tal_hex(const tal_t *ctx, const tal_t *data) { return tal_strdup(ctx, ""); }
/* key parsing, signatures, wire encoding and chain parameters: amount.c and node_id.c helpers a load never calls */
const tal_t *tmpctx;
secp256k1_context *secp256k1_ctx;
const struct chainparams *chainparams;
bool check_signed_hash(const struct sha256_double *hash, const secp256k1_ecdsa_signature *signature,
                       const struct pubkey *key) { abort(); }
bool sciddir_or_pubkey_from_node_id(struct sciddir_or_pubkey *sciddpk, const struct node_id *node_id) { abort(); }
void towire(u8 **pptr, const void *data, size_t len) { abort(); }
void towire_u64(u8 **pptr, u64 v) { abort(); }
const u8 *fromwire(const u8 **cursor, size_t *max, void *copy, size_t n) { abort(); }
u64 fromwire_u64(const u8 **cursor, size_t *max) { abort(); }
int secp256k1_ec_pubkey_parse(const secp256k1_context *ctx, secp256k1_pubkey *pubkey, const unsigned char *input,
                              size_t inputlen) { abort(); }
int secp256k1_ec_pubkey_serialize(const secp256k1_context *ctx, unsigned char *output, size_t *outputlen,
                                  const secp256k1_pubkey *pubkey, unsigned int flags) { abort(); }

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

/* the child: load, then send [count or -1][map_end][count x (scid, cann_off, cupdate_off[0], cupdate_off[1])] */
static void child(const char *path, int fd) {
    tmpctx = tal(NULL, char);
    struct gossmap *map = gossmap_load_(NULL, path, 0, quiet, NULL, NULL);
    s64 n = -1;
    u64 end = 0, total;
    u64 *rows = NULL;
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
    }
    if (write_all(fd, &n, 8) || write_all(fd, &end, 8) || (n > 0 && write_all(fd, rows, (size_t)n * 32))) _exit(3);
    _exit(0);
}

/* Loads the store (version byte first) as gossmap_load does with no expected length, mmap on (so every checksum is
 * tested).  Returns the channel count (rows up to cap written to chans: scid, cann_off, cupdate_off[0], cupdate_off[1],
 * sorted by cann_off; offsets are of messages, 12 past their record header) with *map_end = gossmap_lengths(); -1 if
 * gossmap refuses the store (major version); -2 if the load did not return (an assert, errx or signal in gossmap). */
long long cln_gossmap_load(const u8 *store, size_t len, u64 *map_end, u64 *chans, size_t cap) {
    const char *dir = getenv("TMPDIR");
    char *path = malloc(strlen(dir ? dir : "/tmp") + 32);
    sprintf(path, "%s/gossmap_oracle.XXXXXX", dir ? dir : "/tmp");
    int tfd = mkstemp(path);
    *map_end = 0;
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
        /* gossmap's own log lines and assertion messages would only clutter the test output, and so would a crash
         * handler the caller installed (an assert ends the child with SIGABRT); no core files either */
        int null = open("/dev/null", O_WRONLY);
        if (null >= 0) dup2(null, 2);
        signal(SIGABRT, SIG_DFL);
        signal(SIGSEGV, SIG_DFL);
        struct rlimit no_core = {0, 0};
        setrlimit(RLIMIT_CORE, &no_core);
        child(path, p[1]);
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
        s64 n;
        memcpy(&n, buf, 8);
        memcpy(map_end, buf + 8, 8);
        if (n >= 0 && have == 16 + (size_t)n * 32) {
            memcpy(chans, buf + 16, (size_t)(n < (s64)cap ? n : (s64)cap) * 32);
            ret = n;
        } else if (n == -1) {
            ret = -1;
        }
    }
    free(buf);
    unlink(path);
    free(path);
    return ret;
}
