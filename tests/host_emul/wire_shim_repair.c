/* TEST-ONLY: exposes the generated C codec of sigverifyd_gossip_store_repair and its reply to ctypes
 * (tests/test_sigverifyd_repair_fake.py) */
#include "../../lightning_b200/csrc/sigverifyd_wiregen.h"

size_t shim_towire_repair(uint8_t *out, size_t cap, uint64_t req_id, uint8_t has_chain, const uint8_t *chain_hash, uint64_t len) {
    return towire_sigverifyd_gossip_store_repair(out, cap, req_id, has_chain, chain_hash, len);
}
/* u64s: [req_id, has_chain, len]; *chain_off: where chain_hash is in p */
int shim_fromwire_repair(const uint8_t *p, size_t len, uint64_t *u64s, size_t *chain_off) {
    struct sigverifyd_gossip_store_repair m;
    if (!fromwire_sigverifyd_gossip_store_repair(p, len, &m)) return 0;
    u64s[0] = m.req_id; u64s[1] = m.has_chain; u64s[2] = m.len;
    *chain_off = (size_t)(m.chain_hash - p);
    return 1;
}
/* v: [req_id, err, version, stop, end_offset, records, pruned, bad_crc, truncated, message, redundant, no_channel,
 * signature, amount, unknown, reverified, new_len] */
size_t shim_towire_repair_reply(uint8_t *out, size_t cap, const uint64_t *v) {
    return towire_sigverifyd_gossip_store_repair_reply(out, cap, v[0], (uint32_t)v[1], (uint32_t)v[2], (uint32_t)v[3], v[4],
                                                       v[5], v[6], v[7], v[8], v[9], v[10], v[11], v[12], v[13], v[14], v[15],
                                                       v[16]);
}
int shim_fromwire_repair_reply(const uint8_t *p, size_t len, uint64_t *v) {
    struct sigverifyd_gossip_store_repair_reply r;
    if (!fromwire_sigverifyd_gossip_store_repair_reply(p, len, &r)) return 0;
    const uint64_t w[17] = {r.req_id, r.err, r.version, r.stop, r.end_offset, r.records, r.pruned, r.bad_crc, r.truncated,
                            r.message, r.redundant, r.no_channel, r.signature, r.amount, r.unknown, r.reverified, r.new_len};
    memcpy(v, w, sizeof w);
    return 1;
}
