/* TEST-ONLY: exposes the generated C codec of sigverifyd_sha256d / sigverifyd_pubkey and their replies to ctypes
 * (tests/test_sigverifyd_misc_codec.py) */
#include "../../lightning_b200/csrc/sigverifyd_wiregen.h"

size_t shim_towire_sha256d(uint8_t *out, size_t cap, uint64_t req_id, uint32_t n, const uint8_t *lens, uint32_t bloblen,
                           const uint8_t *blob) {
    return towire_sigverifyd_sha256d(out, cap, req_id, n, lens, bloblen, blob);
}
/* scalars: [n, bloblen]; offs: [lens, blob] */
int shim_fromwire_sha256d(const uint8_t *p, size_t len, uint64_t *req_id, uint32_t *scalars, size_t *offs) {
    struct sigverifyd_sha256d s;
    if (!fromwire_sigverifyd_sha256d(p, len, &s)) return 0;
    *req_id = s.req_id;
    scalars[0] = s.n; scalars[1] = s.bloblen;
    offs[0] = (size_t)(s.lens - p); offs[1] = (size_t)(s.blob - p);
    return 1;
}
size_t shim_towire_sha256d_reply(uint8_t *out, size_t cap, uint64_t req_id, uint32_t n, const uint8_t *hashes) {
    return towire_sigverifyd_sha256d_reply(out, cap, req_id, n, hashes);
}
/* scalars: [n]; offs: [hashes] */
int shim_fromwire_sha256d_reply(const uint8_t *p, size_t len, uint64_t *req_id, uint32_t *scalars, size_t *offs) {
    struct sigverifyd_sha256d_reply r;
    if (!fromwire_sigverifyd_sha256d_reply(p, len, &r)) return 0;
    *req_id = r.req_id;
    scalars[0] = r.n;
    offs[0] = (size_t)(r.hashes - p);
    return 1;
}
size_t shim_towire_pubkey(uint8_t *out, size_t cap, uint64_t req_id, uint32_t n, const uint8_t *keys) {
    return towire_sigverifyd_pubkey(out, cap, req_id, n, keys);
}
/* scalars: [n]; offs: [keys] */
int shim_fromwire_pubkey(const uint8_t *p, size_t len, uint64_t *req_id, uint32_t *scalars, size_t *offs) {
    struct sigverifyd_pubkey k;
    if (!fromwire_sigverifyd_pubkey(p, len, &k)) return 0;
    *req_id = k.req_id;
    scalars[0] = k.n;
    offs[0] = (size_t)(k.keys - p);
    return 1;
}
size_t shim_towire_pubkey_reply(uint8_t *out, size_t cap, uint64_t req_id, uint32_t n, const uint8_t *ok, const uint8_t *xy) {
    return towire_sigverifyd_pubkey_reply(out, cap, req_id, n, ok, xy);
}
/* scalars: [n]; offs: [ok, xy] */
int shim_fromwire_pubkey_reply(const uint8_t *p, size_t len, uint64_t *req_id, uint32_t *scalars, size_t *offs) {
    struct sigverifyd_pubkey_reply r;
    if (!fromwire_sigverifyd_pubkey_reply(p, len, &r)) return 0;
    *req_id = r.req_id;
    scalars[0] = r.n;
    offs[0] = (size_t)(r.ok - p); offs[1] = (size_t)(r.xy - p);
    return 1;
}
