/* TEST-ONLY: exposes the generated C codec of sigverifyd_tx / sigverifyd_tx_reply to ctypes
 * (tests/test_sigverifyd_tx_codec.py) */
#include "../../lightning_b200/csrc/sigverifyd_wiregen.h"

/* arrays[] = the 14 per-transaction arrays in wire order: version, locktime, sequence, sighash_type, prev_index, flags,
 * prev_txid, input_amount, output_amount, script_len, outputs_len, prevouts_len, sequences_len, sigs (big-endian bytes) */
size_t shim_towire_tx(uint8_t *out, size_t cap, uint64_t req_id, uint8_t kind, uint32_t keylen, const uint8_t *key,
                      uint32_t n, const uint8_t *const *arrays, uint32_t bloblen, const uint8_t *blob, uint8_t want_sighash) {
    const uint8_t *const *a = arrays;
    return towire_sigverifyd_tx(out, cap, req_id, kind, keylen, key, n, a[0], a[1], a[2], a[3], a[4], a[5], a[6], a[7], a[8],
                                a[9], a[10], a[11], a[12], bloblen, blob, a[13], want_sighash);
}
/* returns 1 and fills the scalar fields [kind, keylen, n, bloblen, want_sighash] and the offsets of the views [key, the 13
 * per-transaction arrays before the blob in wire order, blob, sigs], 0 if the message does not parse */
int shim_fromwire_tx(const uint8_t *p, size_t len, uint64_t *req_id, uint32_t *scalars, size_t *offs) {
    struct sigverifyd_tx t;
    if (!fromwire_sigverifyd_tx(p, len, &t)) return 0;
    *req_id = t.req_id;
    scalars[0] = t.kind; scalars[1] = t.keylen; scalars[2] = t.n; scalars[3] = t.bloblen; scalars[4] = t.want_sighash;
    const uint8_t *v[16] = {t.key, t.version, t.locktime, t.sequence, t.sighash_type, t.prev_index, t.flags, t.prev_txid,
                            t.input_amount, t.output_amount, t.script_len, t.outputs_len, t.prevouts_len, t.sequences_len,
                            t.blob, t.sigs};
    for (int i = 0; i < 16; i++) offs[i] = (size_t)(v[i] - p);
    return 1;
}
size_t shim_towire_tx_reply(uint8_t *out, size_t cap, uint64_t req_id, uint32_t n, const uint8_t *verdicts,
                            uint32_t nsighash, const uint8_t *sighashes) {
    return towire_sigverifyd_tx_reply(out, cap, req_id, n, verdicts, nsighash, sighashes);
}
/* scalars: [n, nsighash]; offs: [verdicts, sighashes] */
int shim_fromwire_tx_reply(const uint8_t *p, size_t len, uint64_t *req_id, uint32_t *scalars, size_t *offs) {
    struct sigverifyd_tx_reply r;
    if (!fromwire_sigverifyd_tx_reply(p, len, &r)) return 0;
    *req_id = r.req_id;
    scalars[0] = r.n; scalars[1] = r.nsighash;
    offs[0] = (size_t)(r.verdicts - p); offs[1] = (size_t)(r.sighashes - p);
    return 1;
}
