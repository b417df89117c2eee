/*
 * fake_engine_grind.c — sv_grind_tx_fee_host for the fake engine (tests/host_emul/fake_engine.c), linked beside it by
 * tests/test_sigverifyd_fee_grind.py so that the verifier subdaemon's sigverifyd_fee_grind path and the drop-in's
 * check_tx_sig_grind_fee in client mode can be tested without a GPU.  The answer is FNV-1a (64-bit), as in fake_engine.c:
 *   h = h(kind, key, sig64, version, locktime, sequence, sighash_type, prev_txid, prev_index, input_amount, each span's u32le
 *         length and bytes (witness script, output script), weight (u64le), min_feerate, max_feerate)
 *   none if min_feerate > max_feerate or h % 3 == 0, else feerate min + (h >> 8) % (max - min + 1), fee feerate * weight / 1000
 * Each call logs "sv_grind_tx_fee_host <kind> 1 <scripts_len>" and can be delayed and traced (fake_engine.h).  Flags
 * other than 0, a weight of 2^32 or more and spans out of range are SV_ERR_ARG, as the engine's own checks make them.
 */
#include "fake_engine.h"

int sv_grind_tx_fee_host(sv_ctx *ctx, int kind, const sv_tx *tx, const uint8_t *scripts, size_t scripts_len,
                         const uint8_t *key, const uint8_t *sig64, uint64_t weight, uint32_t min_feerate,
                         uint32_t max_feerate, int64_t *feerate_out, uint64_t *fee_out) {
    fake_call("sv_grind_tx_fee_host", ctx, kind, 1, scripts_len);
    size_t ks = sv_key_size(kind);
    if ((kind != SV_KIND_ECDSA33 && kind != SV_KIND_ECDSA_XY) || tx->flags || (weight >> 32) ||
        !span_ok(scripts_len, tx->script_off, tx->script_len) ||
        !span_ok(scripts_len, tx->out_script_off, tx->out_script_len))
        return SV_ERR_ARG;
    uint8_t k = (uint8_t)kind;
    uint64_t h = fnv(fnv(fnv(FNV0, &k, 1), key, ks), sig64, 64);
    h = fnv_le(fnv_le(fnv_le(fnv_le(h, tx->version, 4), tx->locktime, 4), tx->sequence, 4), tx->sighash_type, 4);
    h = fnv_le(fnv_le(fnv(h, tx->prev_txid, 32), tx->prev_index, 4), tx->input_amount, 8);
    h = fnv(fnv_le(h, tx->script_len, 4), scripts + tx->script_off, tx->script_len);
    h = fnv(fnv_le(h, tx->out_script_len, 4), scripts + tx->out_script_off, tx->out_script_len);
    h = fnv_le(fnv_le(fnv_le(h, weight, 8), min_feerate, 4), max_feerate, 4);
    *feerate_out = -1;
    *fee_out = 0;
    if (min_feerate <= max_feerate && h % 3) {
        uint64_t r = min_feerate + (h >> 8) % ((uint64_t)max_feerate - min_feerate + 1);
        *feerate_out = (int64_t)r;
        *fee_out = r * weight / 1000;
    }
    return SV_OK;
}
