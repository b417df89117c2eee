/*
 * fake_engine_bolt11.c — sv_verify_bolt11_host for the fake engine (tests/host_emul/fake_engine.c), linked beside it by
 * tests/test_sigverifyd_bolt11_fake.py so that the verifier subdaemon's sigverifyd_bolt11 path and the drop-in's
 * bolt11_check_signature in client mode can be tested without a GPU.  The answer is FNV-1a (64-bit) over the invoice's
 * span (every byte of it, a NUL included: the daemon must route the bytes, not read them), as in fake_engine.c:
 *   status h % 3 - 1;  node_id33 fill(h, 33) where the status is 1, zeros elsewhere
 * Each call appends "sv_verify_bolt11_host 0 <n> <blob bytes>" to $FAKE_ENGINE_LOG.  A span out of range is SV_ERR_ARG,
 * as the engine's own checks make it; hash32_out, when given, is zeroed.
 */
#include "../../include/cln_sigverify.h"

#include <stdio.h>
#include <stdlib.h>
#include <string.h>

static uint64_t b11_fnv(uint64_t h, const void *p, size_t n) {
    const uint8_t *b = (const uint8_t *)p;
    for (size_t i = 0; i < n; i++) h = (h ^ b[i]) * 0x100000001b3ull;
    return h;
}

int sv_verify_bolt11_host(sv_ctx *ctx, const uint8_t *blob, size_t blob_len, const uint64_t *off, const uint32_t *len,
                          size_t n, int *status, uint8_t *node_id33_out, uint8_t *hash32_out) {
    (void)ctx;
    const char *path = getenv("FAKE_ENGINE_LOG");
    FILE *f = path ? fopen(path, "a") : NULL;
    if (f) {
        fprintf(f, "sv_verify_bolt11_host 0 %zu %zu\n", n, blob_len);
        fclose(f);
    }
    for (size_t i = 0; i < n; i++) {
        if (off[i] > blob_len || len[i] > blob_len - off[i]) return SV_ERR_ARG;
        uint64_t h = b11_fnv(0xcbf29ce484222325ull, blob + off[i], len[i]);
        status[i] = (int)(h % 3) - 1;
        for (size_t k = 0; k < 33; k++) {
            uint8_t b = (uint8_t)k;
            node_id33_out[33 * i + k] = status[i] == 1 ? (uint8_t)b11_fnv(h, &b, 1) : 0;
        }
        if (hash32_out) memset(hash32_out + 32 * i, 0, 32);
    }
    return SV_OK;
}
