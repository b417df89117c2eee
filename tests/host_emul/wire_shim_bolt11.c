/* TEST-ONLY: exposes the generated C codec of sigverifyd_bolt11 / sigverifyd_bolt11_reply to ctypes
 * (tests/test_sigverifyd_bolt11_codec.py) */
#include "../../lightning_b200/csrc/sigverifyd_wiregen.h"

size_t shim_towire_bolt11(uint8_t *out, size_t cap, uint64_t req_id, uint32_t n, const uint8_t *lens, uint32_t bloblen,
                          const uint8_t *blob) {
    return towire_sigverifyd_bolt11(out, cap, req_id, n, lens, bloblen, blob);
}
/* returns 1 and fills the scalar fields [n, bloblen] and the offsets of the views [lens, blob], 0 if the message does not
 * parse */
int shim_fromwire_bolt11(const uint8_t *p, size_t len, uint64_t *req_id, uint32_t *scalars, size_t *offs) {
    struct sigverifyd_bolt11 b;
    if (!fromwire_sigverifyd_bolt11(p, len, &b)) return 0;
    *req_id = b.req_id;
    scalars[0] = b.n; scalars[1] = b.bloblen;
    offs[0] = (size_t)(b.lens - p); offs[1] = (size_t)(b.blob - p);
    return 1;
}
size_t shim_towire_bolt11_reply(uint8_t *out, size_t cap, uint64_t req_id, uint32_t n, const uint8_t *status,
                                const uint8_t *node_ids) {
    return towire_sigverifyd_bolt11_reply(out, cap, req_id, n, status, node_ids);
}
/* scalars: [n]; offs: [status, node_ids] */
int shim_fromwire_bolt11_reply(const uint8_t *p, size_t len, uint64_t *req_id, uint32_t *scalars, size_t *offs) {
    struct sigverifyd_bolt11_reply r;
    if (!fromwire_sigverifyd_bolt11_reply(p, len, &r)) return 0;
    *req_id = r.req_id;
    scalars[0] = r.n;
    offs[0] = (size_t)(r.status - p); offs[1] = (size_t)(r.node_ids - p);
    return 1;
}
