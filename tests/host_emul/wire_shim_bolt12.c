/* TEST-ONLY: exposes the generated C codec of sigverifyd_bolt12 / sigverifyd_bolt12_reply to ctypes
 * (tests/test_sigverifyd_bolt12_codec.py) */
#include "../../lightning_b200/csrc/sigverifyd_wiregen.h"

size_t shim_towire_bolt12(uint8_t *out, size_t cap, uint64_t req_id, uint16_t mnlen, const uint8_t *messagename,
                          uint16_t fnlen, const uint8_t *fieldname, uint32_t n, const uint8_t *lens, uint32_t bloblen,
                          const uint8_t *blob, const uint8_t *xonly, const uint8_t *sigs, uint8_t want_sighash) {
    return towire_sigverifyd_bolt12(out, cap, req_id, mnlen, messagename, fnlen, fieldname, n, lens, bloblen, blob, xonly,
                                    sigs, want_sighash);
}
/* returns 1 and fills the scalar fields [mnlen, fnlen, n, bloblen, want_sighash] and the offsets of the views
 * [messagename, fieldname, lens, blob, xonly, sigs], 0 if the message does not parse */
int shim_fromwire_bolt12(const uint8_t *p, size_t len, uint64_t *req_id, uint32_t *scalars, size_t *offs) {
    struct sigverifyd_bolt12 b;
    if (!fromwire_sigverifyd_bolt12(p, len, &b)) return 0;
    *req_id = b.req_id;
    scalars[0] = b.mnlen; scalars[1] = b.fnlen; scalars[2] = b.n; scalars[3] = b.bloblen; scalars[4] = b.want_sighash;
    offs[0] = (size_t)(b.messagename - p); offs[1] = (size_t)(b.fieldname - p); offs[2] = (size_t)(b.lens - p);
    offs[3] = (size_t)(b.blob - p); offs[4] = (size_t)(b.xonly - p); offs[5] = (size_t)(b.sigs - p);
    return 1;
}
size_t shim_towire_bolt12_reply(uint8_t *out, size_t cap, uint64_t req_id, uint32_t n, const uint8_t *status,
                                uint32_t nsighash, const uint8_t *sighashes) {
    return towire_sigverifyd_bolt12_reply(out, cap, req_id, n, status, nsighash, sighashes);
}
/* scalars: [n, nsighash]; offs: [status, sighashes] */
int shim_fromwire_bolt12_reply(const uint8_t *p, size_t len, uint64_t *req_id, uint32_t *scalars, size_t *offs) {
    struct sigverifyd_bolt12_reply r;
    if (!fromwire_sigverifyd_bolt12_reply(p, len, &r)) return 0;
    *req_id = r.req_id;
    scalars[0] = r.n; scalars[1] = r.nsighash;
    offs[0] = (size_t)(r.status - p); offs[1] = (size_t)(r.sighashes - p);
    return 1;
}
