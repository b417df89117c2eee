/*
 * fake_engine.c — a stand-in for libcln_sigverify.so with the entry points the verifier subdaemon (sigverifyd.c) calls,
 * so the daemon and the drop-in's client mode (cln_dropin.c) can be tested without a GPU
 * (tests/test_sigverifyd_fake_engine.py).  Every result is FNV-1a (64-bit) over the bytes of its item, a function the
 * test recomputes:
 *   sv_verify_host         verdict  h(kind, msg32, key, sig64) % 3
 *   sv_verify_tx_host      verdict  h(kind, key, sig64, the sv_tx fields, each span's u32le length and bytes) % 3;
 *                          sighash  fill(h, 32)
 *   sv_verify_bolt12_tagged_host  status h(messagename, 0, fieldname, 0, stream, xonly32, sig64) % 3 - 1; sighash fill(h, 32)
 *   sv_sha256d_host        fill(h(buffer), 32)
 *   sv_pubkey_parse_host   ok h(key33) % 3, xy fill(h, 64)
 *   sv_verify_gossip_host  status h(message, signer33) % 6 - 1
 *   sv_verify_gossip_burst_host  status h(chain32, message, signer_kind, signer33) % 10 - 4
 * where fill(h, n)[k] = the low byte of FNV-1a continued from h over the one byte k.  Integers enter as little-endian
 * bytes.  Each call appends "<function> <kind> <n> <blob bytes>" to the file named by $FAKE_ENGINE_LOG.  A span out of
 * range or a tag index past the table is SV_ERR_ARG, as the engine's own checks make it.
 *
 * Built with -DFAKE_ENGINE_NO_CONTEXT (into the drop-in library), sv_create aborts: client mode must never reach an
 * in-process path.  The other in-process entry points the drop-in references always abort.
 */
#include "../../include/cln_sigverify.h"

#include <stdio.h>
#include <stdlib.h>
#include <string.h>

struct sv_ctx { int unused; };

static uint64_t fnv(uint64_t h, const void *p, size_t n) {
    const uint8_t *b = (const uint8_t *)p;
    for (size_t i = 0; i < n; i++) h = (h ^ b[i]) * 0x100000001b3ull;
    return h;
}
#define FNV0 0xcbf29ce484222325ull
static uint64_t fnv_u32(uint64_t h, uint32_t v) {
    uint8_t b[4] = {(uint8_t)v, (uint8_t)(v >> 8), (uint8_t)(v >> 16), (uint8_t)(v >> 24)};
    return fnv(h, b, 4);
}
static uint64_t fnv_u64(uint64_t h, uint64_t v) { return fnv_u32(fnv_u32(h, (uint32_t)v), (uint32_t)(v >> 32)); }
static void fill(uint64_t h, uint8_t *out, size_t n) {
    for (size_t k = 0; k < n; k++) {
        uint8_t b = (uint8_t)k;
        out[k] = (uint8_t)fnv(h, &b, 1);
    }
}
static void log_call(const char *fn, int kind, size_t n, size_t bytes) {
    const char *path = getenv("FAKE_ENGINE_LOG");
    FILE *f = path ? fopen(path, "a") : NULL;
    if (!f) return;
    fprintf(f, "%s %d %zu %zu\n", fn, kind, n, bytes);
    fclose(f);
}
static int span_ok(size_t blob_len, uint64_t off, uint64_t len) { return off <= blob_len && len <= blob_len - off; }

int sv_create(sv_ctx **out, int device) {
    (void)device;
#ifdef FAKE_ENGINE_NO_CONTEXT
    fprintf(stderr, "fake engine: sv_create called\n");
    abort();
#endif
    *out = (sv_ctx *)calloc(1, sizeof(sv_ctx));
    return *out ? SV_OK : SV_ERR_NOMEM;
}
void sv_destroy(sv_ctx *ctx) { free(ctx); }
const char *sv_last_error(const sv_ctx *ctx) { (void)ctx; return "fake engine: bad argument"; }
size_t sv_key_size(int kind) { return kind == SV_KIND_ECDSA33 ? 33 : kind == SV_KIND_ECDSA_XY ? 64 : kind == SV_KIND_SCHNORR ? 32 : 0; }

int sv_verify_host(sv_ctx *ctx, int kind, const uint8_t *msg32, const uint8_t *key, const uint8_t *sig64, size_t n,
                   uint8_t *verdicts) {
    (void)ctx;
    size_t ks = sv_key_size(kind);
    log_call("sv_verify_host", kind, n, 0);
    if (!ks) return SV_ERR_ARG;
    for (size_t i = 0; i < n; i++) {
        uint8_t k = (uint8_t)kind;
        uint64_t h = fnv(fnv(fnv(fnv(FNV0, &k, 1), msg32 + 32 * i, 32), key + ks * i, ks), sig64 + 64 * i, 64);
        verdicts[i] = (uint8_t)(h % 3);
    }
    return SV_OK;
}

int sv_verify_tx_host(sv_ctx *ctx, int kind, const sv_tx *txs, const uint8_t *scripts, size_t scripts_len,
                      const uint8_t *key, const uint8_t *sig64, size_t n, uint8_t *verdicts, uint8_t *sighash32_out) {
    (void)ctx;
    size_t ks = sv_key_size(kind);
    log_call("sv_verify_tx_host", kind, n, scripts_len);
    if (kind != SV_KIND_ECDSA33 && kind != SV_KIND_ECDSA_XY) return SV_ERR_ARG;
    for (size_t i = 0; i < n; i++) {
        const sv_tx *t = &txs[i];
        const uint32_t offs[4] = {t->script_off, t->out_script_off, t->prevouts_off, t->sequences_off};
        const uint32_t lens[4] = {t->script_len, t->out_script_len, t->prevouts_len, t->sequences_len};
        uint8_t k = (uint8_t)kind;
        uint64_t h = fnv(fnv(fnv(FNV0, &k, 1), key + ks * i, ks), sig64 + 64 * i, 64);
        h = fnv_u32(fnv_u32(fnv_u32(fnv_u32(h, t->version), t->locktime), t->sequence), t->sighash_type);
        h = fnv_u32(fnv(h, t->prev_txid, 32), t->prev_index);
        h = fnv_u64(fnv_u64(fnv_u32(h, t->flags), t->input_amount), t->output_amount);
        for (int s = 0; s < 4; s++) {
            if (!span_ok(scripts_len, offs[s], lens[s])) return SV_ERR_ARG;
            h = fnv(fnv_u32(h, lens[s]), scripts + offs[s], lens[s]);
        }
        verdicts[i] = (uint8_t)(h % 3);
        if (sighash32_out) fill(h, sighash32_out + 32 * i, 32);
    }
    return SV_OK;
}

int sv_verify_bolt12_tagged_host(sv_ctx *ctx, size_t ntags, const char *const *messagenames, const char *const *fieldnames,
                                 const uint32_t *tag_of, const uint8_t *blob, size_t blob_len, const uint64_t *off,
                                 const uint32_t *len, const uint8_t *xonly32, const uint8_t *sig64, size_t n, int *status,
                                 uint8_t *sighash32_out) {
    (void)ctx;
    log_call("sv_verify_bolt12_tagged_host", 0, n, blob_len);
    for (size_t i = 0; i < n; i++) {
        if (tag_of[i] >= ntags || !span_ok(blob_len, off[i], len[i])) return SV_ERR_ARG;
        const char *mn = messagenames[tag_of[i]], *fn = fieldnames[tag_of[i]];
        uint64_t h = fnv(fnv(FNV0, mn, strlen(mn) + 1), fn, strlen(fn) + 1);
        h = fnv(fnv(fnv(h, blob + off[i], len[i]), xonly32 + 32 * i, 32), sig64 + 64 * i, 64);
        status[i] = (int)(h % 3) - 1;
        if (sighash32_out) fill(h, sighash32_out + 32 * i, 32);
    }
    return SV_OK;
}

int sv_sha256d_host(sv_ctx *ctx, const uint8_t *data, size_t data_len, const uint64_t *off, const uint32_t *len, size_t n,
                    uint8_t *out32) {
    (void)ctx;
    log_call("sv_sha256d_host", 0, n, data_len);
    for (size_t i = 0; i < n; i++) {
        if (!span_ok(data_len, off[i], len[i])) return SV_ERR_ARG;
        fill(fnv(FNV0, data + off[i], len[i]), out32 + 32 * i, 32);
    }
    return SV_OK;
}

int sv_pubkey_parse_host(sv_ctx *ctx, const uint8_t *key33, size_t n, uint8_t *xy64, uint8_t *ok) {
    (void)ctx;
    log_call("sv_pubkey_parse_host", 0, n, 0);
    for (size_t i = 0; i < n; i++) {
        uint64_t h = fnv(FNV0, key33 + 33 * i, 33);
        ok[i] = (uint8_t)(h % 3);
        fill(h, xy64 + 64 * i, 64);
    }
    return SV_OK;
}

int sv_verify_gossip_host(sv_ctx *ctx, const uint8_t *blob, size_t blob_len, const uint64_t *msg_off, const uint32_t *msg_len,
                          size_t n_msgs, const uint8_t *cu_signers33, int *status) {
    (void)ctx;
    static const uint8_t none[33];
    log_call("sv_verify_gossip_host", 0, n_msgs, blob_len);
    for (size_t i = 0; i < n_msgs; i++) {
        if (!span_ok(blob_len, msg_off[i], msg_len[i])) return SV_ERR_ARG;
        uint64_t h = fnv(fnv(FNV0, blob + msg_off[i], msg_len[i]), cu_signers33 ? cu_signers33 + 33 * i : none, 33);
        status[i] = (int)(h % 6) - 1;
    }
    return SV_OK;
}

int sv_verify_gossip_burst_host(sv_ctx *ctx, const uint8_t chain_hash32[32], const uint8_t *blob, size_t blob_len,
                                const uint64_t *msg_off, const uint32_t *msg_len, size_t n_msgs, const uint8_t *signer_kind,
                                const uint8_t *signers33, int *status) {
    (void)ctx;
    static const uint8_t none[33];
    log_call("sv_verify_gossip_burst_host", 0, n_msgs, blob_len);
    for (size_t i = 0; i < n_msgs; i++) {
        uint8_t kind = signer_kind ? signer_kind[i] : 0;
        if (kind > 2 || !span_ok(blob_len, msg_off[i], msg_len[i])) return SV_ERR_ARG;
        uint64_t h = fnv(fnv(fnv(FNV0, chain_hash32, 32), blob + msg_off[i], msg_len[i]), &kind, 1);
        h = fnv(h, signers33 ? signers33 + 33 * i : none, 33);
        status[i] = (int)(h % 10) - 4;
    }
    return SV_OK;
}

/* in-process only: client mode never calls them */
int sv_verify_samekey_host(sv_ctx *ctx, int kind, const uint8_t *key, const uint8_t *msg32, const uint8_t *sig64, size_t n,
                           uint8_t *verdicts) {
    (void)ctx; (void)kind; (void)key; (void)msg32; (void)sig64; (void)n; (void)verdicts;
    fprintf(stderr, "fake engine: sv_verify_samekey_host called\n");
    abort();
}
int sv_verify_bolt12_host(sv_ctx *ctx, const char *messagename, const char *fieldname, const uint8_t *blob, size_t blob_len,
                          const uint64_t *off, const uint32_t *len, const uint8_t *xonly32, const uint8_t *sig64, size_t n,
                          int *status, uint8_t *sighash32_out) {
    (void)ctx; (void)messagename; (void)fieldname; (void)blob; (void)blob_len; (void)off; (void)len; (void)xonly32;
    (void)sig64; (void)n; (void)status; (void)sighash32_out;
    fprintf(stderr, "fake engine: sv_verify_bolt12_host called\n");
    abort();
}
