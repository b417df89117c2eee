/*
 * fake_engine_timed.c — the fake engine (fake_engine.c, included below with its entry points renamed) for callers with
 * several contexts on several threads, such as the verifier subdaemon's two engine workers
 * (tests/test_sigverifyd_workers.py).  Every answer and every $FAKE_ENGINE_LOG line is fake_engine.c's; two variables,
 * both unset by default, add time and a trace:
 *   FAKE_ENGINE_DELAY  "<function>=<ms>,..."  each call of a listed entry point waits that long before it answers
 *   FAKE_ENGINE_TRACE  a file that gets "begin <function> <context>" when a call starts and "end <function> <context>"
 *                      when it has waited its delay; contexts are numbered from 1 in the order sv_create made them
 * Trace lines and the fake's log lines are written under one lock, so they are whole and in the order they happened.
 */
#define _POSIX_C_SOURCE 200809L /* nanosleep */
#include <pthread.h>
#include <time.h>

#define sv_create fake_sv_create
#define sv_verify_host fake_sv_verify_host
#define sv_verify_tx_host fake_sv_verify_tx_host
#define sv_verify_bolt12_tagged_host fake_sv_verify_bolt12_tagged_host
#define sv_sha256d_host fake_sv_sha256d_host
#define sv_pubkey_parse_host fake_sv_pubkey_parse_host
#define sv_verify_gossip_host fake_sv_verify_gossip_host
#define sv_verify_gossip_burst_host fake_sv_verify_gossip_burst_host
#include "fake_engine.c"
#undef sv_create
#undef sv_verify_host
#undef sv_verify_tx_host
#undef sv_verify_bolt12_tagged_host
#undef sv_sha256d_host
#undef sv_pubkey_parse_host
#undef sv_verify_gossip_host
#undef sv_verify_gossip_burst_host

#define MAX_CONTEXTS 64
static pthread_mutex_t timed_mu = PTHREAD_MUTEX_INITIALIZER;
static const sv_ctx *contexts[MAX_CONTEXTS]; /* context k + 1 */
static int ncontexts;

/* the context's number, 0 if it is not one sv_create made (call with timed_mu held) */
static int context_id(const sv_ctx *ctx) {
    for (int k = 0; k < ncontexts; k++)
        if (contexts[k] == ctx) return k + 1;
    return 0;
}
static void trace(const char *ev, const char *fn, const sv_ctx *ctx) {
    const char *path = getenv("FAKE_ENGINE_TRACE");
    FILE *f = path ? fopen(path, "a") : NULL;
    if (!f) return;
    fprintf(f, "%s %s %d\n", ev, fn, context_id(ctx));
    fclose(f);
}
/* $FAKE_ENGINE_DELAY's milliseconds for fn, 0 if it lists none */
static long delay_ms(const char *fn) {
    const char *d = getenv("FAKE_ENGINE_DELAY");
    size_t fl = strlen(fn);
    while (d && *d) {
        if (!strncmp(d, fn, fl) && d[fl] == '=') return strtol(d + fl + 1, NULL, 10);
        d = strchr(d, ',');
        if (d) d++;
    }
    return 0;
}
/* a call's start: its begin line, its delay, its end line; returns with timed_mu held for the fake's own call */
static void enter(const char *fn, const sv_ctx *ctx) {
    long ms = delay_ms(fn);
    pthread_mutex_lock(&timed_mu);
    trace("begin", fn, ctx);
    pthread_mutex_unlock(&timed_mu);
    if (ms > 0) {
        struct timespec t = {ms / 1000, (ms % 1000) * 1000000L};
        while (nanosleep(&t, &t) != 0) {}
    }
    pthread_mutex_lock(&timed_mu);
    trace("end", fn, ctx);
}
#define TIMED(fn, ...)                        \
    do {                                      \
        enter(#fn, ctx);                      \
        int rc_ = fake_##fn(__VA_ARGS__);     \
        pthread_mutex_unlock(&timed_mu);      \
        return rc_;                           \
    } while (0)

int sv_create(sv_ctx **out, int device) {
    int rc = fake_sv_create(out, device);
    pthread_mutex_lock(&timed_mu);
    if (rc == SV_OK && ncontexts < MAX_CONTEXTS) contexts[ncontexts++] = *out;
    pthread_mutex_unlock(&timed_mu);
    return rc;
}

int sv_verify_host(sv_ctx *ctx, int kind, const uint8_t *msg32, const uint8_t *key, const uint8_t *sig64, size_t n,
                   uint8_t *verdicts) {
    TIMED(sv_verify_host, ctx, kind, msg32, key, sig64, n, verdicts);
}

int sv_verify_tx_host(sv_ctx *ctx, int kind, const sv_tx *txs, const uint8_t *scripts, size_t scripts_len,
                      const uint8_t *key, const uint8_t *sig64, size_t n, uint8_t *verdicts, uint8_t *sighash32_out) {
    TIMED(sv_verify_tx_host, ctx, kind, txs, scripts, scripts_len, key, sig64, n, verdicts, sighash32_out);
}

int sv_verify_bolt12_tagged_host(sv_ctx *ctx, size_t ntags, const char *const *messagenames, const char *const *fieldnames,
                                 const uint32_t *tag_of, const uint8_t *blob, size_t blob_len, const uint64_t *off,
                                 const uint32_t *len, const uint8_t *xonly32, const uint8_t *sig64, size_t n, int *status,
                                 uint8_t *sighash32_out) {
    TIMED(sv_verify_bolt12_tagged_host, ctx, ntags, messagenames, fieldnames, tag_of, blob, blob_len, off, len, xonly32,
          sig64, n, status, sighash32_out);
}

int sv_sha256d_host(sv_ctx *ctx, const uint8_t *data, size_t data_len, const uint64_t *off, const uint32_t *len, size_t n,
                    uint8_t *out32) {
    TIMED(sv_sha256d_host, ctx, data, data_len, off, len, n, out32);
}

int sv_pubkey_parse_host(sv_ctx *ctx, const uint8_t *key33, size_t n, uint8_t *xy64, uint8_t *ok) {
    TIMED(sv_pubkey_parse_host, ctx, key33, n, xy64, ok);
}

int sv_verify_gossip_host(sv_ctx *ctx, const uint8_t *blob, size_t blob_len, const uint64_t *msg_off, const uint32_t *msg_len,
                          size_t n_msgs, const uint8_t *cu_signers33, int *status) {
    TIMED(sv_verify_gossip_host, ctx, blob, blob_len, msg_off, msg_len, n_msgs, cu_signers33, status);
}

int sv_verify_gossip_burst_host(sv_ctx *ctx, const uint8_t chain_hash32[32], const uint8_t *blob, size_t blob_len,
                                const uint64_t *msg_off, const uint32_t *msg_len, size_t n_msgs, const uint8_t *signer_kind,
                                const uint8_t *signers33, int *status) {
    TIMED(sv_verify_gossip_burst_host, ctx, chain_hash32, blob, blob_len, msg_off, msg_len, n_msgs, signer_kind, signers33,
          status);
}
