/*
 * fake_engine_bolt11.c — sv_verify_bolt11_host for the fake engine (tests/host_emul/fake_engine.c), linked beside it by
 * tests/test_sigverifyd_bolt11_fake.py so that the verifier subdaemon's sigverifyd_bolt11 path and the drop-in's
 * bolt11_check_signature in client mode can be tested without a GPU.  The answer is FNV-1a (64-bit) over the invoice's
 * span (every byte of it, a NUL included: the daemon must route the bytes, not read them), as in fake_engine.c:
 *   status h % 3 - 1;  node_id33 fill(h, 33) where the status is 1, zeros elsewhere
 * Each call logs "sv_verify_bolt11_host 0 <n> <blob bytes>" and can be delayed and traced (fake_engine.h).  A span out
 * of range is SV_ERR_ARG, as the engine's own checks make it; hash32_out, when given, is zeroed.
 */
#include "fake_engine.h"

#include <string.h>

int sv_verify_bolt11_host(sv_ctx *ctx, const uint8_t *blob, size_t blob_len, const uint64_t *off, const uint32_t *len,
                          size_t n, int *status, uint8_t *node_id33_out, uint8_t *hash32_out) {
    fake_call("sv_verify_bolt11_host", ctx, 0, n, blob_len);
    for (size_t i = 0; i < n; i++) {
        if (!span_ok(blob_len, off[i], len[i])) return SV_ERR_ARG;
        uint64_t h = fnv(FNV0, blob + off[i], len[i]);
        status[i] = (int)(h % 3) - 1;
        if (status[i] == 1)
            fill(h, node_id33_out + 33 * i, 33);
        else
            memset(node_id33_out + 33 * i, 0, 33);
        if (hash32_out) memset(hash32_out + 32 * i, 0, 32);
    }
    return SV_OK;
}
