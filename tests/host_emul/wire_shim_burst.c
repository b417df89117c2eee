/* TEST-ONLY: exposes the generated C codec of sigverifyd_gossip_burst and its reply to ctypes
 * (tests/test_sigverifyd_gossip_burst_codec.py) */
#include "../../lightning_b200/csrc/sigverifyd_wiregen.h"

size_t shim_towire_gossip_burst(uint8_t *out, size_t cap, uint64_t req_id, const uint8_t *chain_hash, uint32_t n,
                                const uint8_t *lens, const uint8_t *signer_kind, const uint8_t *signers, uint32_t bloblen,
                                const uint8_t *blob) {
    return towire_sigverifyd_gossip_burst(out, cap, req_id, chain_hash, n, lens, signer_kind, signers, bloblen, blob);
}
/* scalars: [n, bloblen]; offs: [chain_hash, lens, signer_kind, signers, blob] */
int shim_fromwire_gossip_burst(const uint8_t *p, size_t len, uint64_t *req_id, uint32_t *scalars, size_t *offs) {
    struct sigverifyd_gossip_burst g;
    if (!fromwire_sigverifyd_gossip_burst(p, len, &g)) return 0;
    *req_id = g.req_id;
    scalars[0] = g.n; scalars[1] = g.bloblen;
    offs[0] = (size_t)(g.chain_hash - p); offs[1] = (size_t)(g.lens - p); offs[2] = (size_t)(g.signer_kind - p);
    offs[3] = (size_t)(g.signers - p); offs[4] = (size_t)(g.blob - p);
    return 1;
}
size_t shim_towire_gossip_burst_reply(uint8_t *out, size_t cap, uint64_t req_id, uint32_t n, const uint8_t *status) {
    return towire_sigverifyd_gossip_burst_reply(out, cap, req_id, n, status);
}
/* scalars: [n]; offs: [status] */
int shim_fromwire_gossip_burst_reply(const uint8_t *p, size_t len, uint64_t *req_id, uint32_t *scalars, size_t *offs) {
    struct sigverifyd_gossip_burst_reply r;
    if (!fromwire_sigverifyd_gossip_burst_reply(p, len, &r)) return 0;
    *req_id = r.req_id;
    scalars[0] = r.n;
    offs[0] = (size_t)(r.status - p);
    return 1;
}
