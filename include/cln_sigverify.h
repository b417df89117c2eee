/*
 * cln_sigverify.h — C ABI of the H100 batched secp256k1 verification engine (libcln_sigverify.so).
 *
 * This is the drop-in boundary behind Core Lightning's bitcoin/signature.h surface.  Plain C,
 * plain pointers and sizes; no CUDA, torch or libsecp256k1 types appear in any signature.
 *
 * Reference interfaces each entry point replaces (paths relative to the CLN tree):
 *
 *   sv_verify_host(SV_KIND_ECDSA_XY, ...)   check_signed_hash()          bitcoin/signature.c:174-192
 *                                           (hash32, secp256k1_ecdsa_signature, struct pubkey)
 *   sv_verify_host(SV_KIND_ECDSA33, ...)    check_signed_hash_nodeid()   common/node_id.c:72-80
 *                                           (33-byte node_id decompressed per call, then as above)
 *   sv_verify_host(SV_KIND_SCHNORR, ...)    check_schnorr_sig()          bitcoin/signature.c:408-430
 *   sv_verify_host_raw(...)                 sha256_double() + the above  bitcoin/shadouble.c:7-11,
 *                                           as used by gossipd/sigcheck.c:9-43, 45-115, 118-164 and,
 *                                           with a BIP143 preimage as the span, check_tx_sig()
 *                                           bitcoin/signature.c:194-221 (the per-HTLC loop of
 *                                           channeld/channeld.c:2215-2232)
 *   sv_verify_bolt12_host(...)              bolt12_check_signature()     common/bolt12.c:80-92: merkle_tlv()
 *                                           common/bolt12_merkle.c:160-194 over the fields fromwire_tlv()
 *                                           wire/tlvstream.c:144-300 parses, sighash_from_merkle() :210-220,
 *                                           check_schnorr_sig(); callers plugins/offers_invreq_hook.c:634-637,
 *                                           plugins/offers_inv_hook.c:177-179, plugins/fetchinvoice.c:256-260,
 *                                           :1501-1507, lightningd/offer.c:88-89, devtools/bolt12-cli.c:319-321
 *   sv_verify_bolt12_tagged_host(...)       the same checks, many callers' tags in one batch (the verifier
 *                                           subdaemon serves the plugins' bolt12_check_signature calls with it)
 *   sv_verify_bolt11_host(...)              bolt11_decode()'s signature step common/bolt11.c:980-1062 (bech32,
 *                                           the field walk of bolt11_decode_nosig :887-936, hash_u5's signing hash,
 *                                           then secp256k1_ecdsa_verify against `n` or secp256k1_ecdsa_recover);
 *                                           run by every invoice string given to pay, xpay, renepay, decode,
 *                                           listsendpays and listinvoices
 *   sv_verify_gossip_burst_host(...)        gossipd's signature gate over a burst: parse, node-id order and chain
 *                                           gates gossipd/gossmap_manage.c:659-670, :1048-1051, sigcheck_*, and the
 *                                           pending map that gives a channel_update its signer (:695-703,
 *                                           :1060-1097), or the source peer's private-update check (:1099-1110)
 *   sv_verify_gossip_store_host(...)        gossmap's map_catchup over a whole gossip_store (common/gossmap.c:815-937:
 *                                           record walk, crc32c) plus every signature it never checks, with the
 *                                           signer its channel table gives
 *   sv_grind_tx_fee_host(...)               onchaind's grind_htlc_tx_fee loop over check_tx_sig
 *                                           onchaind/onchaind.c:389-437, every candidate feerate in one call
 *   sv_sha256d_host(...)                    sha256_double()              bitcoin/shadouble.c:7-11
 *   sv_pubkey_parse_host(...)               pubkey_from_der()            bitcoin/pubkey.c:14-24
 *   sv_enqueue_* / sv_flush                 the deferral queue a batching caller (gossipd ingest,
 *                                           SURVEY.md §8f N1) sits on; synchronous check_* = enqueue 1 + flush
 *   sv_verify_device(...)                   same kernels on device-resident arrays (bench / multi-GPU)
 *
 * Verdict semantics are those of the reference, bit for bit, INCLUDING the parse-time rejects CLN
 * performs before check_signed_hash (r >= n, s >= n: wire/fromwire.c:188-199; bad pubkey:
 * bitcoin/pubkey.c:102-113): a verdict byte is 1 iff libsecp256k1 would parse the key, parse the
 * signature and return 1 from secp256k1_ecdsa_verify / secp256k1_schnorrsig_verify.
 *
 * Error convention (SURVEY.md §8b): a verification failure is verdict 0, never an error code.
 * Engine failures (no device, CUDA error, out of memory) return a negative sv_status and leave the
 * verdict buffer untouched; there is NO CPU fallback.  The check_* drop-in wrappers in
 * cln_dropin.h abort() on engine failure, matching CLN's "internal error is fatal" style.
 *
 * Threading: one sv_ctx per thread/process (CLN daemons are single-threaded event loops).  Calls on one context
 * share its device scratch (work records, per-thread tables): issue them one at a time, on one stream at a time.
 */
#ifndef CLN_SIGVERIFY_H
#define CLN_SIGVERIFY_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct sv_ctx sv_ctx;

/* item kinds (layout of the key array; msg is always 32 bytes, sig always 64 bytes) */
#define SV_KIND_ECDSA33 0  /* key = 33-byte SEC1 compressed (02/03 || x)           sig = r_be32 || s_be32 */
#define SV_KIND_ECDSA_XY 1 /* key = 64 bytes x_be32 || y_be32 (pre-decompressed)   sig = r_be32 || s_be32 */
#define SV_KIND_SCHNORR 2  /* key = 32-byte x-only (BIP-340)                        sig = R.x_be32 || s_be32 */

typedef enum {
    SV_OK = 0,
    SV_ERR_NO_DEVICE = -1,
    SV_ERR_CUDA = -2,
    SV_ERR_NOMEM = -3,
    SV_ERR_ARG = -4,
    SV_ERR_IO = -5 /* sv_prune_gossip_store_fd: the file could not be read, written or synced; errno is kept */
} sv_status;

/* Create an engine on CUDA device `device` (ordinal).  Allocates the stream, builds the 34 MiB
 * fixed-base table on the device (kernel K4) and the per-thread scratch.  */
int sv_create(sv_ctx **out, int device);
void sv_destroy(sv_ctx *ctx);
/* last error text for this context (or for a failed sv_create when ctx == NULL) */
const char *sv_last_error(const sv_ctx *ctx);
/* size of the key element for a kind (33 / 64 / 32), or 0 */
size_t sv_key_size(int kind);

/* ---- synchronous batch verification, HOST buffers (SoA): msg32[n][32], key[n][keysize], sig64[n][64];
 *      verdicts[n] receives 0/1.  Copies in, runs the kernels, copies out, returns when done. ---- */
int sv_verify_host(sv_ctx *ctx, int kind, const uint8_t *msg32, const uint8_t *key, const uint8_t *sig64,
                   size_t n, uint8_t *verdicts);

/* Batches of at most `small_max` signatures (default = capacity = 8192; 0 disables) take the LATENCY path: one launch
 * of a kernel that spreads each verification over three warps (key side / scalar side in parallel, then the two GLV
 * half-ladders and the fixed-base comb in parallel, joined by full Jacobian additions), inputs and verdicts passing
 * through a pinned, device-mapped staging block (no copy commands, no allocation).  Larger batches take the throughput
 * kernels.  Verdicts are identical on both paths (tests/test_gpu_small.py). */
int sv_set_small_max(sv_ctx *ctx, size_t small_max);
size_t sv_get_small_max(const sv_ctx *ctx);

/* ---- MIXED batch (BASELINE config C3: interleaved ECDSA + BIP-340): kinds[i] is the SV_KIND_* tag of item i, keys sit
 *      in 64-byte slots (the first 33 / 64 / 32 bytes are the key).  The batch is split per kind on the device (index
 *      lists by warp-aggregated atomics, gather, per-kind kernels, scatter); verdicts come back in item order; an
 *      unknown tag yields verdict 0. ---- */
int sv_verify_mixed_host(sv_ctx *ctx, const uint8_t *kinds, const uint8_t *msg32, const uint8_t *key64,
                         const uint8_t *sig64, size_t n, uint8_t *verdicts);
int sv_verify_mixed_device(sv_ctx *ctx, const void *d_kinds, const void *d_msg32, const void *d_key64,
                           const void *d_sig64, size_t n, void *d_verdicts, void *stream);

/* ---- same, but the message hash is computed on the device: item i signs
 *      SHA256d(data[off[i] .. off[i]+len[i])).  Several items may share one span (the four
 *      signatures of a channel_announcement do). ---- */
int sv_verify_host_raw(sv_ctx *ctx, int kind, const uint8_t *data, size_t data_len, const uint64_t *off,
                       const uint32_t *len, const uint8_t *key, const uint8_t *sig64, size_t n,
                       uint8_t *verdicts);

/* ---- gossip ingest with DEVICE-side slicing (SURVEY.md §8f N1; replaces the per-message work of
 *      gossipd/sigcheck.c:9-164 and the field extraction of wire/peer_wiregen.c for the three gossip messages):
 *      blob = concatenated raw wire messages (2-byte type included), msg_off/msg_len locate them.  The device finds
 *      the signatures, keys and signed regions itself, hashes (SHA-256d) and verifies.  status[m] = 0 all signatures
 *      good; 1..4 = first bad signature in the reference's order (node_signature_1, node_signature_2,
 *      bitcoin_signature_1, bitcoin_signature_2; node_announcement / channel_update: 1); -1 = not a gossip message,
 *      shorter than the message's fixed layout (every field of wire/peer_wire.csv:340-377 up to and including the
 *      variable-length features / addresses arrays must be present, as the generated fromwire_* require), a signature
 *      with r or s >= n, or an undecodable bitcoin_key.  NOT checked: the TLV stream that may follow a
 *      node_announcement (node_ann_tlvs) — a caller that consumes those still parses them itself.  channel_update is signed by a node the caller looks up in its gossmap: cu_signers33[m] (33 bytes per
 *      MESSAGE, ignored for other types; NULL if the batch has no channel_update). ---- */
int sv_verify_gossip_host(sv_ctx *ctx, const uint8_t *blob, size_t blob_len, const uint64_t *msg_off,
                          const uint32_t *msg_len, size_t n_msgs, const uint8_t *cu_signers33, int *status);

/* ---- gossip BURST: a batch of raw gossip messages of any mix of types (a peer's channel_announcement followed by its
 *      channel_updates, as initial sync and query_short_channel_ids deliver them), where an update's signer may be found
 *      among the batch's own announcements.  status[m] is what gossipd's signature gate decides:
 *        channel_announcement / node_announcement: as sv_verify_gossip_host (0, 1..4, -1), and for a channel_announcement
 *          -4 if node_id_1 is not below node_id_2 (gossipd/gossmap_manage.c:659-663), else -3 if its chain_hash is not
 *          chain_hash32 (:669-670).  A message the wire parser refuses is -1 before either gate, as in gossipd.  A gated
 *          announcement reports no signature verdict.
 *        channel_update: -1 as sv_verify_gossip_host, else -3 if its chain_hash is not chain_hash32 (:1048-1051), else by
 *          signer_kind[m]:
 *          1  signers33[m] is the node the caller's gossmap gives for the update's direction (sv_verify_gossip_host's
 *             meaning; the batch is not consulted): 0 or 1.
 *          0  the channel is the FIRST channel_announcement at an index j < m with the same short_channel_id whose final
 *             status is 0 (gossipd's pending map, :695-703, :1060-1097: an announcement that fails sigcheck is never
 *             added, a later one of the same scid can be, an update that arrives first finds no channel).  The signer is
 *             its node_id_1 if channel_flags & 1 == 0, else its node_id_2: 0 or 1.  No such announcement: -2.
 *          2  as 0; if no announcement resolves, signers33[m] is the source peer and the update is checked as gossipd's
 *             private-update path does (:1099-1110): 5 if it verifies under the peer, -2 otherwise.
 *      Every channel_announcement reports its own signatures, duplicates included.  Not decided here (policy, not
 *      signatures): timestamp_reasonable, txout confirmation, node_announcements of nodes without channels.  For a
 *      gossip_store, sv_verify_gossip_store_funding_host decides the txout from lightningd's own tables.
 *      signer_kind == NULL means all 0; signers33 (33 bytes per MESSAGE) may be NULL only when no channel_update has kind 1
 *      or 2; a signer_kind above 2 (any message) is SV_ERR_ARG.  Resolution never reaches outside the call.  On the device:
 *      an scid table of the gated announcements, one resolve thread per update and ONE verification launch for all
 *      items; only when an update's candidate announcement itself fails does a second, small round run
 *      (sv_last_gossip_repairs reports how many updates it took). ---- */
int sv_verify_gossip_burst_host(sv_ctx *ctx, const uint8_t chain_hash32[32], const uint8_t *blob, size_t blob_len,
                                const uint64_t *msg_off, const uint32_t *msg_len, size_t n_msgs, const uint8_t *signer_kind,
                                const uint8_t *signers33, int *status);
unsigned sv_last_gossip_repairs(const sv_ctx *ctx);

/* ---- a whole GOSSIP_STORE (common/gossip_store.h layout: version byte, then records of a 12-byte header and a message),
 *      audited before gossmap loads it.  gossmap's map_catchup (common/gossmap.c:815-937) trusts the store: it checks each
 *      record's CRC-32C and no signature.  This call walks the store exactly as map_catchup does, checks every checksum it
 *      would check, and verifies every channel_announcement, node_announcement and channel_update it would load.
 *
 *      Walk (host, headers only): from offset 1 while off + 12 < len.  A record without the COMPLETED flag stops it
 *      (SV_GS_INCOMPLETE); a DELETED record is skipped unchecked (SV_GS_DELETED); a record running past the end stops it
 *      (SV_GS_PARTIAL), as does a message under 2 bytes (SV_GS_TRUNCATED), a checksum mismatch (SV_GS_BAD_CRC: crc32c with
 *      the header timestamp as start value), a gossip_store_ended record (SV_GS_ENDED) and a channel_announcement that
 *      holds its channel but has no room for the amount record after it (SV_GS_NO_AMOUNT, gossmap.c:488-492).  Records of
 *      types 4101, 4103, 4106, 4107 are SV_GS_STORE_RECORD, any other type SV_GS_UNKNOWN.  Records after a BAD_CRC or
 *      NO_AMOUNT stop are SV_GS_NOT_REACHED and are not verified.
 *
 *      Messages: rec_status is what sv_verify_gossip_host reports (0, 1..4, -1).  With chain_hash32, the gates of
 *      sv_verify_gossip_burst_host apply too (-4 node ids out of order, -3 another chain); NULL means no gates.  A
 *      channel_update is signed by the channel gossmap holds for its scid at the update's position: the first
 *      non-deleted channel_announcement of the scid holds it (whatever its own status), a later one is redundant and
 *      never signs, a non-deleted gossip_store_delete_chan frees the scid for the next announcement.  The signer is
 *      node_id_1 or node_id_2 by channel_flags & 1.  An update whose scid has no channel at its position is -2 (after -1
 *      and -3).  As gossmap does, these fields are read at their fixed offsets from the message start even where the
 *      message is shorter (an announcement through node_id_2, an update through htlc_maximum_msat, a delete_chan's
 *      scid): the bytes come from the records after it.  Only a record whose reads would pass the end of the store, where
 *      gossmap's load asserts, takes no part in the channel table.
 *
 *      rec_off / rec_type / rec_status (and rec_holder, optional): one entry per record the walk reads, in store order;
 *      rec_holder is the header offset of the announcement holding the channel, for a channel_update and for a redundant
 *      channel_announcement, else UINT64_MAX.  rec_capacity below sv_gossip_store_count(store, len), or a major version
 *      other than 0 (gossmap.c:958-963): SV_ERR_ARG, nothing written.  The store is staged on the device for the call only.
 *      On the device: the checksums (the first bad one cuts the walk), the slicing, gates, hashing and verification of
 *      sv_verify_gossip_host, and the channel table (events sorted by scid, one thread walks each scid). ---- */
#define SV_GS_EOF 0 /* summary.stop only: the walk reached the end of the store */
#define SV_GS_DELETED 16
#define SV_GS_STORE_RECORD 17
#define SV_GS_UNKNOWN 18
#define SV_GS_NOT_REACHED 19
#define SV_GS_INCOMPLETE 32
#define SV_GS_PARTIAL 33
#define SV_GS_TRUNCATED 34
#define SV_GS_BAD_CRC 35
#define SV_GS_ENDED 36
#define SV_GS_NO_AMOUNT 37
typedef struct {
    uint32_t version;                 /* the store's version byte */
    int32_t stop;                     /* SV_GS_EOF or the status of the record the walk stopped at */
    uint64_t end_offset;              /* gossmap's map_end: the offset of that record, or where the walk ran out */
    uint64_t ended_equivalent_offset; /* stop == SV_GS_ENDED: the record's equivalent_offset */
    uint64_t records;                 /* entries written */
    uint64_t good, bad_signature, malformed, no_channel, wrong_chain, bad_order; /* messages: 0, 1..4, -1, -2, -3, -4 */
    uint64_t deleted, store_records, unknown, not_reached;
    uint64_t redundant_announcements; /* reached channel_announcements of an scid whose channel was already held */
    uint64_t updates_without_channel; /* reached channel_updates (read inside the store) whose scid held no channel */
} sv_gossip_store_summary;
size_t sv_gossip_store_count(const uint8_t *store, size_t len);
int sv_verify_gossip_store_host(sv_ctx *ctx, const uint8_t *store, size_t len, const uint8_t *chain_hash32,
                                uint64_t *rec_off, uint16_t *rec_type, int *rec_status, uint64_t *rec_holder,
                                size_t rec_capacity, sv_gossip_store_summary *summary);
/* profiling mode (sv_set_profiling): ms4 = host header walk, H2D copy of the store, checksum kernel, the rest of the call */
int sv_get_last_gossip_store_timing(sv_ctx *ctx, float *ms4);

/* ---- PRUNE a gossip_store: mark every record gossmap should not trust as deleted, so that gossipd's strict load
 *      (gossmap_load_initial, gossipd/gossmap_manage.c:525: must_be_clean, common/gossmap.c:862, :885, :895, :922,
 *      :1428-1438) accepts the store and keeps every record that verifies.  gossipd drops a record the same way
 *      (gossip_store_del, gossipd/gossip_store.c:572-638): bit 0x8000 of the record's flags, set in place.  The checksum
 *      covers the timestamp and the message only (csum_matches, common/gossmap.c:800-812), and map_catchup skips a deleted
 *      record before it looks at its length or checksum (:844-847), so every other record reads as before.  gossmap takes
 *      the last live channel_update per direction and the last live node_announcement per node (update_channel :585-610,
 *      node_announcement :650-668): deleting a bad newest record makes the previous verified one current again.
 *
 *      out (len bytes; may equal store) differs from store only in bit 0x8000 of the flags of the deleted records.
 *      rec_pruned[r] = 0 (kept, or deleted already) or the SV_GP_* reason record r is deleted for:
 *        1. Walk: sv_verify_gossip_store_host's, except that a record with a bad checksum (SV_GP_BAD_CRC) or a message
 *           under 2 bytes (SV_GP_TRUNCATED) is deleted and the walk goes on past it.  INCOMPLETE, PARTIAL and ENDED still
 *           stop it; nothing at or after the stop is touched.
 *        2. First round: the statuses of sv_verify_gossip_store_host (with the chain gates when chain_hash32 is given) over
 *           the records the walk left live.  A channel_announcement or node_announcement whose status is not 0, and a
 *           channel_update whose status is -1 or -3, is deleted (SV_GP_MESSAGE).
 *        3. Second round: the channel table again, with the announcements of rule 2 deleted (the first live announcement
 *           of an scid holds it, a delete_chan frees it).  An announcement redundant in it is deleted (SV_GP_REDUNDANT:
 *           the strict load refuses one, gossmap.c:895-896).  An update whose scid holds no channel at its position is
 *           deleted (SV_GP_NO_CHANNEL).  An update whose signer changed is verified again under the new node (same
 *           SHA-256d digest) and deleted if it fails (SV_GP_SIGNATURE), as is one that failed under an unchanged signer.
 *           One round is enough: updates never hold channels, and deleting a redundant announcement changes no holder.
 *        4. The channel_amount record directly after a deleted channel_announcement is deleted with it (SV_GP_AMOUNT), as
 *           gossip_store_del does.
 *        5. A record of an unknown type is deleted (SV_GP_UNKNOWN: the strict load refuses one, gossmap.c:918-923).
 *        6. Nothing else: node_announcements of nodes left without channels stay (gossmap ignores them).
 *      An announcement kept that has no room for its amount record stops the walk as in the audit (SV_GS_NO_AMOUNT): it
 *      and every record after it are left as they are.
 *      rec_status[r] is the record's first-round status: sv_verify_gossip_store_host's, except SV_GS_BAD_CRC and
 *      SV_GS_TRUNCATED for records the walk went past.  rec_capacity below sv_gossip_prune_count(store, len) (which is
 *      sv_gossip_store_count plus the truncated records walked past), or a major version other than 0: SV_ERR_ARG,
 *      nothing written.
 *      On the device, besides the audit's kernels: a checksum flag per record, a mark kernel (deletions and the event
 *      mask), k_store_resolve again over the already sorted events, the updates whose signer changed gathered into a
 *      compact list and verified with their kept digests, and one thread per deleted record setting its flag bit. ---- */
#define SV_GP_KEPT 0
#define SV_GP_BAD_CRC 1
#define SV_GP_TRUNCATED 2
#define SV_GP_MESSAGE 3
#define SV_GP_REDUNDANT 4
#define SV_GP_NO_CHANNEL 5
#define SV_GP_SIGNATURE 6
#define SV_GP_AMOUNT 7
#define SV_GP_UNKNOWN 8
typedef struct {
    uint32_t version;    /* the store's version byte */
    int32_t stop;        /* SV_GS_EOF or the status of the record the walk stopped at */
    uint64_t end_offset; /* where the walk stopped (the offset of that record) or ran out */
    uint64_t records;    /* entries written */
    uint64_t pruned;     /* records this call deleted: the sum of the reasons below */
    uint64_t bad_crc, truncated, message, redundant, no_channel, signature, amount, unknown; /* SV_GP_1..8 */
    uint64_t reverified; /* updates verified again under a new signer */
} sv_gossip_prune_summary;
size_t sv_gossip_prune_count(const uint8_t *store, size_t len);
int sv_prune_gossip_store_host(sv_ctx *ctx, const uint8_t *store, size_t len, const uint8_t *chain_hash32, uint8_t *out,
                               uint64_t *rec_off, uint16_t *rec_type, int *rec_status, uint8_t *rec_pruned,
                               size_t rec_capacity, sv_gossip_prune_summary *summary);
/* profiling mode: ms4 = host header walk, first round (H2D of the store, checksums, the audit's kernels), second round
 * (mark, resolution, compaction, re-verification), flag write and copy back */
int sv_get_last_gossip_prune_timing(sv_ctx *ctx, float *ms4);

/* ---- FUNDING of a gossip_store's channels: the audit and the prune above, plus the check gossipd makes before it lets a
 *      channel_announcement in from a peer and which a store not written by this node's gossipd never had.  gossipd asks
 *      lightningd for the announcement's txout (gossipd/gossmap_manage.c:748-751) and drops the announcement unless an
 *      unspent output exists and its script is the P2WSH of the 2-of-2 of the announcement's bitcoin keys; it then writes
 *      the announcement and a channel_amount record with the output's amount (:850-852), which gossmap takes as the
 *      channel's capacity (common/gossmap.c:1473-1499).  lightningd answers from two tables (get_txout,
 *      lightningd/gossip_control.c:78-115): the unspent P2WSH outputs of the blocks it processed (utxoset, spendheight
 *      NULL, wallet_outpoint_for_scid) and the heights of those blocks (blocks, wallet_have_block).  The caller passes
 *      them as sv_funding_table; lightning_b200/funding.py reads them from lightningd.sqlite3.
 *
 *      One verdict per record (rec_funding).  Every live channel_announcement the walk reaches whose message status is 0
 *      gets one of SV_GF_FUNDED..SV_GF_AMOUNT, redundant ones included; every other record SV_GF_NONE.  With
 *      scid = block << 40 | txindex << 16 | outnum, read from the announcement:
 *        SV_GF_DYING      the record's header has GOSSIP_STORE_DYING_BIT (0x0800): gossipd has seen the spend and deletes
 *                         the channel at its deadline (gossipd/gossmap_manage.c:1420-1433).  Whatever the table says.
 *        SV_GF_FUNDED     the table has an output at scid whose 34-byte script is 0x00 0x20 || SHA-256(script) of the
 *                         2-of-2 (bitcoin_redeem_2of2, bitcoin/script.c:151-167: OP_2 <ka> <kb> OP_2 OP_CHECKMULTISIG with
 *                         the 33-byte keys in memcmp order, pubkey_cmp bitcoin/pubkey.c:84-90), and the record directly
 *                         after the announcement (by the header's length, whatever its flags, as gossmap_chan_get_capacity
 *                         reads it, common/gossmap.c:1488-1495) is a channel_amount (4101) holding the output's amount.
 *        SV_GF_UNCHECKED  no output at scid and block is not a processed height: lightningd would ask bitcoind
 *                         (getfilteredblock, lightningd/gossip_control.c:104-112), which this call cannot.
 *        SV_GF_NO_TXOUT   no output at scid and block is a processed height (the wallet_have_block branch, :97-103):
 *                         gossipd ignores the announcement (gossipd/gossmap_manage.c:791-810).
 *        SV_GF_SCRIPT     the output's script is not that P2WSH (:696-699, :812-819).
 *        SV_GF_AMOUNT     the script matches, but the next record is not a channel_amount or holds another amount: gossipd
 *                         would have written the txout's amount (:850-852).
 *      The audit (sv_verify_gossip_store_funding_host) writes exactly what sv_verify_gossip_store_host writes, plus
 *      rec_funding and *fsummary (fsummary->deleted = 0).  Records at or after a BAD_CRC or NO_AMOUNT stop get SV_GF_NONE.
 *
 *      The prune (sv_prune_gossip_store_funding_host) extends rule 2 of sv_prune_gossip_store_host: a channel_announcement
 *      whose first-round status is 0 and whose verdict is SV_GF_NO_TXOUT, SV_GF_SCRIPT or SV_GF_AMOUNT is deleted
 *      (SV_GP_FUNDING).  SV_GF_UNCHECKED and SV_GF_DYING are kept.  Rules 3 to 6 then run unchanged: the second channel
 *      table gives the scid to a later live announcement or to none, the updates are verified again under the new holder
 *      or deleted, and the channel_amount record goes with its announcement.  No other round is needed: a funding
 *      deletion is one more announcement masked out of the second round, exactly as a failing one.  So when no
 *      announcement is deleted for funding, every output equals sv_prune_gossip_store_host's; summary->pruned counts the
 *      funding deletions as well, and fsummary->deleted says how many there were.  rec_funding is NONE at and after a
 *      NO_AMOUNT stop.
 *
 *      The table: scid[n_outputs] unique (a duplicate is SV_ERR_ARG, nothing written), any order; satoshis and script34
 *      (34 bytes) per output; blocks[n_blocks] any order.  It is staged on the device for the call and sorted there (CUB
 *      radix sort); k_store_funding runs one thread per candidate announcement: the 2-of-2 script in registers, its
 *      SHA-256, the scid and the block by binary search, and the amount record and the header flags read from the staged
 *      store.  Otherwise the arguments and errors are those of the calls without the table. ---- */
#define SV_GF_NONE 0
#define SV_GF_FUNDED 1
#define SV_GF_UNCHECKED 2
#define SV_GF_DYING 3
#define SV_GF_NO_TXOUT 4
#define SV_GF_SCRIPT 5
#define SV_GF_AMOUNT 6
#define SV_GP_FUNDING 9
typedef struct {
    const uint64_t *scid;     /* n_outputs, unique, any order: block << 40 | txindex << 16 | outnum */
    const uint64_t *satoshis; /* n_outputs */
    const uint8_t *script34;  /* 34 bytes per output (lightningd keeps P2WSH outputs only) */
    size_t n_outputs;
    const uint32_t *blocks;   /* processed block heights, any order */
    size_t n_blocks;
} sv_funding_table;
typedef struct {
    uint64_t checked;  /* announcements given a verdict: the sum of the six below */
    uint64_t funded, unchecked, no_txout, script, amount, dying;
    uint64_t deleted;  /* the prune: announcements deleted for funding (SV_GP_FUNDING); the audit: 0 */
} sv_gossip_funding_summary;
int sv_verify_gossip_store_funding_host(sv_ctx *ctx, const uint8_t *store, size_t len, const uint8_t *chain_hash32,
                                        const sv_funding_table *table, uint64_t *rec_off, uint16_t *rec_type,
                                        int *rec_status, uint64_t *rec_holder, uint8_t *rec_funding, size_t rec_capacity,
                                        sv_gossip_store_summary *summary, sv_gossip_funding_summary *fsummary);
int sv_prune_gossip_store_funding_host(sv_ctx *ctx, const uint8_t *store, size_t len, const uint8_t *chain_hash32,
                                       const sv_funding_table *table, uint8_t *out, uint64_t *rec_off, uint16_t *rec_type,
                                       int *rec_status, uint8_t *rec_pruned, uint8_t *rec_funding, size_t rec_capacity,
                                       sv_gossip_prune_summary *summary, sv_gossip_funding_summary *fsummary);
/* profiling mode: ms2 = the last funding call's table staging and sort, and its k_store_funding (device events) */
int sv_get_last_gossip_funding_timing(sv_ctx *ctx, float *ms2);

/* ---- PRUNE a gossip_store FILE in place: the store is bytes [0, len) of fd, which must be a regular file opened for
 *      reading and writing.  The store is read (pread) into host memory and pruned by sv_prune_gossip_store_host with out
 *      == store; then, for each record it deleted, the two-byte big-endian flags field (the first two bytes of the
 *      record's 12-byte header) is written back (pwrite) with bit 0x8000 set, as gossip_store_del does, and the file is
 *      synced (fsync).  No other byte of the file changes, so every checksum stays valid.  *summary is the host call's.
 *      fd not a regular file, len 0 or larger than the file: SV_ERR_ARG, nothing read, errno EINVAL.  A store the host
 *      call refuses (a major version other than 0): SV_ERR_ARG, errno EINVAL, nothing written.  fd not open for reading
 *      and writing: SV_ERR_IO, errno EBADF, nothing read.  A failed or short read, a failed write or fsync: SV_ERR_IO with
 *      that errno (EIO for a short read); the flags written before a failed write stay (each is a deletion of its own).
 *      The other engine errors (SV_ERR_NOMEM, SV_ERR_CUDA, ...) are returned as the host call returns them.  The verifier
 *      subdaemon serves this call for its clients (sigverifyd_gossip_store_prune: the fd travels over its socket). ---- */
int sv_prune_gossip_store_fd(sv_ctx *ctx, int fd, uint64_t len, const uint8_t *chain_hash32, sv_gossip_prune_summary *summary);

/* ---- REPAIR a gossip_store FILE in place: prune it (sv_prune_gossip_store_fd, everything it does and refuses), then cut
 *      a torn tail off it.  gossipd only appends, so a crash during gossip_store_add leaves a last record without
 *      GOSSIP_STORE_COMPLETED_BIT, a record running past the end of the file, fewer than 13 trailing bytes, or a
 *      channel_announcement without its channel_amount record; gossmap's strict start-up load refuses each (its walk stops
 *      short of expected_len, common/gossmap.c:1428-1438).  The cut, where the file ends afterwards, is
 *      sv_gossip_prune_cut(summary, pruned store, len):
 *        stop SV_GS_INCOMPLETE, SV_GS_PARTIAL or SV_GS_NO_AMOUNT:  summary.end_offset (the record the walk stopped at);
 *        stop SV_GS_EOF with end_offset < len (a torn header):      end_offset;
 *        anything else, SV_GS_ENDED included (a replaced store):    len, and the call is exactly the prune.
 *      When the cut is below len and would leave a live channel_announcement without the 22 bytes of its channel_amount
 *      record before it (gossmap.c:488-492), the store ends at that announcement instead (repeated while that leaves
 *      another one so).  gossipd writes a record with flags 0 and sets COMPLETED in a second one-byte write
 *      (gossipd/gossip_store.c:64-77), so a crash between the two during the amount's append leaves a whole amount record
 *      without COMPLETED after a complete announcement: the walk stops INCOMPLETE at the amount, and the announcement must
 *      go with it.  A strict load with expected_len = the cut accepts the repaired store, and it holds what a load of the
 *      pruned store holds up to its walk's stop, minus such an announcement: a lenient load of the torn store reads the
 *      incomplete amount record's bytes and keeps that channel, the repaired store does not (gossipd learns it again
 *      from its peers).  Order of writes: the deleted flags, fsync, then (cut < len) ftruncate(fd, cut) and fsync again,
 *      so a crash in between leaves a store whose pruned prefix is still valid; the bytes after len go too.  *new_len (may
 *      be NULL) = the cut, written on SV_OK only.  A failed ftruncate or fsync: SV_ERR_IO with its errno, the flags
 *      already written stay.  The verifier subdaemon serves this call for its clients (sigverifyd_gossip_store_repair).
 *      sv_gossip_prune_cut is that rule alone, for a store pruned in host memory (pruned: the len bytes the prune wrote,
 *      whose deleted flags it reads; NULL summary or pruned: len). ---- */
int sv_repair_gossip_store_fd(sv_ctx *ctx, int fd, uint64_t len, const uint8_t *chain_hash32, sv_gossip_prune_summary *summary,
                              uint64_t *new_len);
uint64_t sv_gossip_prune_cut(const sv_gossip_prune_summary *summary, const uint8_t *pruned, uint64_t len);

/* ---- SALVAGE a gossip_store past damaged record headers.  Every walk above follows the length in each record's header,
 *      as map_catchup does, so one flipped bit in a record's flags or length sends it into the middle of a message, where
 *      it soon stops (SV_GS_INCOMPLETE) and the repair cuts the file there: every record after the damage is lost though
 *      it is intact.  The salvage finds where the records resume and mends the chain of lengths with a few header
 *      writes, so the prune and the repair keep them.
 *
 *      A SOUND record at offset o: its 12-byte header and its message lie inside the store, COMPLETED is set, len >= 2,
 *      the type is 256, 257, 258, 4101, 4103, 4105, 4106 or 4107, and crc32c(timestamp, msg[0, len)) is the header's
 *      crc.  The deleted bit does not matter (gossipd's deletions keep a valid checksum).  The walk starts at offset 1 and
 *      goes on while 12 bytes of header fit before the end.  A sound record is stepped over by its length; a sound,
 *      non-deleted gossip_store_ended record stops the walk.  At a record t that is not sound:
 *        1. If COMPLETED is set and t + 12 + len is sound, the length is right: t is left to the prune, which deletes it
 *           (SV_GP_BAD_CRC, SV_GP_TRUNCATED or SV_GP_UNKNOWN), and the walk goes on at t + 12 + len.
 *        2. Else let q be the smallest sound offset with q >= t + 14.  If there is none, t is the tail: the walk stops and
 *           leaves it to sv_gossip_prune_cut.  The end of the store is never a q, so a torn tail is repaired exactly as
 *           sv_repair_gossip_store_fd repairs it without the salvage.
 *        3. RESTORE when q - t - 12 <= 65535 and crc32c(timestamp(t), store[t + 12, q)) == crc(t): len = q - t - 12 is
 *           written and COMPLETED set, the other flag bits kept.  The record is whole again and the prune judges it.
 *        4. Else BRIDGE [t, q) with filler records: flags DELETED | COMPLETED, a length in [2, 65535], as few as cover the
 *           span, their sizes as even as possible (the first span % k one byte longer).  Only each filler's 4 bytes of
 *           flags and length are written.  gossmap skips a deleted record by its length before it looks at anything else
 *           (common/gossmap.c:842-847), and gossipd's compaction (gossipd/compactd.c copy_records) reads len - 2 bytes of
 *           every record, deleted or not, hence the 14-byte minimum.
 *        The walk goes on at q.  A span [t, q) that already holds exactly the fillers rule 4 would write is not a break
 *      (fillers are never sound, so a salvaged store leads the walk there again).  For a message of 2 bytes or more, rule 1 is "COMPLETED and t + 12 + len == q"; for a
 *      shorter one (SV_GS_TRUNCATED, which ends before any q can lie) it keeps the sound record right after it.
 *      A store without a break (a torn tail included) is not changed; a salvaged store has no break left, so a second
 *      salvage writes nothing.  Known limit: a sound record that an attacker embeds in the damaged record's own payload is
 *      taken as q.  It still goes through the prune, where every signed message is verified; the store's own record
 *      types carry no signature.
 *
 *      sv_salvage_gossip_store_host: out (len bytes; may equal store) is store with the header writes.  One action per
 *      break, in store order: act_off = t, act_resume = q, act_kind = SV_SALVAGE_RESTORED or SV_SALVAGE_BRIDGED; at most
 *      act_capacity are listed (the arrays may be NULL when it is 0), summary->breaks counts them all.  A major version
 *      other than 0: SV_ERR_ARG, nothing written.  On the device: k_salvage_filter (one thread per byte offset: the
 *      header tests, and an order-preserving compaction of the candidates through a per-block count and cub's scan of
 *      the counts), then k_salvage_crc (the slice-by-8 checksum, one thread per candidate, a warp per candidate over
 *      1,024 bytes).  The host walks the store with the sorted sound offsets (a galloping binary search, header bytes
 *      only), and k_salvage_restore checks each break's restore CRC on the device, one warp per break.
 *
 *      sv_salvage_gossip_store_fd: the salvage on bytes [0, len) of fd, then fsync, then exactly sv_repair_gossip_store_fd
 *      (*summary and *new_len are its).  Each action is written back (pwrite) as 4 bytes of flags and length per header;
 *      a bridge's fillers are written from the last to the first and synced (fsync) before the first one overwrites the
 *      damaged header at t.  Until that 4-byte write reaches the disk the walk still stops at the damaged header and never
 *      reads the other fillers, so a crash or a power loss at any point leaves each break as it was or whole.  Arguments,
 *      errors and errno are those of sv_repair_gossip_store_fd; *salvage is written on SV_OK.  The verifier subdaemon
 *      serves this call for its clients (sigverifyd_gossip_store_salvage: the fd travels over its socket). ---- */
#define SV_SALVAGE_RESTORED 1
#define SV_SALVAGE_BRIDGED 2
typedef struct {
    uint64_t breaks;        /* records restored or bridged */
    uint64_t restored, bridged;
    uint64_t bridged_bytes; /* bytes the bridges cover */
    uint64_t fillers;       /* filler records written */
    uint64_t sound;         /* sound offsets found in the store */
} sv_gossip_salvage_summary;
int sv_salvage_gossip_store_host(sv_ctx *ctx, const uint8_t *store, size_t len, uint8_t *out, uint64_t *act_off,
                                 uint64_t *act_resume, uint8_t *act_kind, size_t act_capacity,
                                 sv_gossip_salvage_summary *summary);
int sv_salvage_gossip_store_fd(sv_ctx *ctx, int fd, uint64_t len, const uint8_t *chain_hash32,
                               sv_gossip_prune_summary *summary, sv_gossip_salvage_summary *salvage, uint64_t *new_len);
/* profiling mode: ms3 = the two filter passes with the scan, the checksum kernel (device events around the kernels
 * only), the host walk */
int sv_get_last_gossip_salvage_timing(sv_ctx *ctx, float *ms3);

/* L2 residency hint for the throughput kernels (default on): the G comb table and the per-thread multiples tables are
 * marked persisting through a stream access-policy window, the rest of the stream's traffic streaming.  0 switches it off
 * for streams not yet seen (measurement aid). */
int sv_set_l2_policy(sv_ctx *ctx, int on);

/* ---- BIP-340 BATCH verification by random linear combination (SURVEY.md 8f N3; BIP-340 "Batch Verification").  The batch
 *      is cut into groups of 1024 signatures; each group's equation  sum a_i R_i + sum a_i e_i P_i - (sum a_i s_i) G = 0
 *      is evaluated with a per-warp bucket method (about half the field work of one-by-one verification); the members of
 *      a group whose equation fails are re-verified one by one, so every verdict is the one sv_verify_host(SV_KIND_SCHNORR)
 *      gives, up to the 2^-127 chance that random a_i hide a bad signature.  Meant for batches that are almost all valid
 *      (a bad signature costs its whole group the fast path).  seed32: 32 bytes the signers could not predict (NULL: taken
 *      from getrandom()); a seed the signers can learn lets them make invalid signatures pass, as
 *      tests/test_gpu_batch_rlc.py shows.  groups_total / groups_failed (optional) report how the batch went. ---- */
int sv_verify_schnorr_batch_host(sv_ctx *ctx, const uint8_t *msg32, const uint8_t *xonly32, const uint8_t *sig64, size_t n,
                                 const uint8_t *seed32, uint8_t *verdicts, uint32_t *groups_total, uint32_t *groups_failed);

/* Key de-duplication (SURVEY.md 8f N3): sv_verify_gossip_host looks for repeated keys in batches above the small-batch limit (and >= 4096 signatures)
 * (exact hash table over the 33 key bytes, on the device); when at least 40 % of the items repeat a key, every DISTINCT
 * key is decoded and its multiples table built once and the curve kernel indexes those tables.  Verdicts are unchanged.
 * sv_set_dedup(ctx, 0) switches the search off; sv_last_distinct_keys reports what the last gossip batch contained. */
int sv_set_dedup(sv_ctx *ctx, int on);
unsigned sv_last_distinct_keys(const sv_ctx *ctx);

/* Compressed-key ECDSA (SV_KIND_ECDSA33) batches above the small-batch limit never take the square root of
 * secp256k1_eckey_pubkey_parse (eckey_impl.h:17-20 -> group_impl.h:334-346): the unknown y only scales Z, the final
 * comparison becomes linear in y and is settled by one batched division (lightning_b200/csrc/verify.cuh, "without the
 * square root").  Verdicts are identical; sv_set_nosqrt(ctx, 0) selects the plain flow (A/B measurements, tests). */
int sv_set_nosqrt(sv_ctx *ctx, int on);

/* ---- n ECDSA signatures by ONE key (SURVEY.md §8a a16 / §8f N3: every HTLC signature of a commitment_signed is made
 *      with remote_htlckey, channeld/channeld.c:2154,2215-2232).  The key is decoded and its multiples table built once;
 *      each verification skips the per-signature square root and table build.  kind: SV_KIND_ECDSA33 or _XY; key is
 *      ONE key of that kind. ---- */
int sv_verify_samekey_host(sv_ctx *ctx, int kind, const uint8_t *key, const uint8_t *msg32, const uint8_t *sig64,
                           size_t n, uint8_t *verdicts);

/* ---- check_tx_sig with the BIP143 sighash computed ON THE DEVICE (SURVEY.md §8f N2).  Replaces, for the one-input
 *      one-output commitment-HTLC transactions of channeld/channeld.c:2215-2232 (shape: common/htlc_tx.c:10-69),
 *      bitcoin_tx_hash_for_sig (bitcoin/signature.c:120-151) -> wally_tx_get_btc_signature_hash ->
 *      bip143_signature_hash (libwally tx_io.c:660-765) + check_signed_hash.  The host passes only the fields of the
 *      preimage; scripts live in one blob.  Multi-output / multi-input transactions (the commitment transaction itself,
 *      check_tx_sig in general) pass their serialised outputs / outpoints through the SV_TX_* flags.  sighash32_out (optional, n x 32) returns the computed sighashes.
 *      A sighash_type libwally does not hash for a segwit-v0 Bitcoin input (tx_io.c:972-1009: anything but 0, 1, 2, 3,
 *      0x81, 0x82, 0x83) gives verdict 0 and a zero sighash, whatever the signature. ---- */
#define SV_TX_OUTPUTS_SERIALIZED 1u /* the out_script span holds the already-serialised outputs to commit to (amount ||
                                       CompactSize || script, concatenated: all outputs for SIGHASH_ALL, the one at the
                                       input's index for SIGHASH_SINGLE); output_amount is ignored */
#define SV_TX_INPUTS_SERIALIZED 2u  /* multi-input transaction: the prevouts span holds every outpoint (36 bytes each), the
                                       sequences span every nSequence (4 bytes each) — hashPrevouts / hashSequence are
                                       taken over them; prev_txid/prev_index/sequence still describe THE input being signed */
#define SV_TX_OUTPUTS_ZERO 4u       /* hashOutputs is 32 zero bytes (SIGHASH_SINGLE with no output at the input's index,
                                       libwally tx_io.c:725) */
typedef struct {
    uint32_t version, locktime, sequence, sighash_type; /* sighash_type: SIGHASH_ALL 1 / NONE 2 / SINGLE 3, | 0x80 ANYONECANPAY,
                                                           or 0 (hashed as ALL); any other value is refused */
    uint8_t prev_txid[32];                              /* as serialised in the transaction (internal byte order) */
    uint32_t prev_index;
    uint32_t script_off, script_len;                    /* witness script (scriptCode) inside `scripts`, any length */
    uint32_t out_script_off, out_script_len;            /* scriptPubKey of the single output inside `scripts` (or the
                                                           serialised outputs, see SV_TX_OUTPUTS_SERIALIZED) */
    uint32_t flags;                                     /* 0 for the one-input one-output HTLC shape, or SV_TX_* above */
    uint64_t input_amount, output_amount;               /* satoshi */
    uint32_t prevouts_off, prevouts_len;                /* SV_TX_INPUTS_SERIALIZED only */
    uint32_t sequences_off, sequences_len;
} sv_tx;
int sv_verify_tx_host(sv_ctx *ctx, int kind, const sv_tx *txs, const uint8_t *scripts, size_t scripts_len,
                      const uint8_t *key, const uint8_t *sig64, size_t n, uint8_t *verdicts, uint8_t *sighash32_out);

/* onchaind's HTLC fee grind (onchaind/onchaind.c:389-437) as one call: the first feerate f in [min_feerate, max_feerate],
 * ascending, whose fee = f*weight/1000 (common/amount.c:698-707 amount_tx_fee) makes sig64 verify under key for the
 * transaction *tx with its single output set to input_amount - fee.  A feerate whose fee equals the previous feerate's
 * is skipped; the walk ends at the first fee above input_amount, as the reference loop does.  *feerate_out = -1 when
 * none verifies (including a signature, key or sighash type the reference would refuse: the types sv_verify_tx_host
 * refuses give -1 without a candidate checked).  tx->output_amount is ignored; tx->flags
 * must be 0 (one input, one output); weight < 2^32.  Verdict per candidate = sv_verify_tx_host's.
 *      kind: SV_KIND_ECDSA33 or _XY.  min_feerate > max_feerate: none found, no launch.  weight 0: one candidate, fee 0.
 *      Spans out of range, a non-zero flags, weight >= 2^32 and NULL required pointers: SV_ERR_ARG.  On the device: one
 *      warp computes s^-1, u2*Q and the preimage through nSequence once (k_grind_setup), then one thread per feerate
 *      (k_grind) hashes its output and adds u1*G; the range runs in ascending chunks of 2^20 feerates from min_feerate and
 *      the call returns after the first chunk with a match.  *fee_out: the matching fee (0 when none). */
int sv_grind_tx_fee_host(sv_ctx *ctx, int kind, const sv_tx *tx, const uint8_t *scripts, size_t scripts_len,
                         const uint8_t *key, const uint8_t *sig64, uint64_t weight, uint32_t min_feerate,
                         uint32_t max_feerate, int64_t *feerate_out, uint64_t *fee_out);

/* ---- BOLT12 signatures with the message hash computed ON THE DEVICE: bolt12_check_signature (common/bolt12.c:80-92)
 *      for n TLV streams.  Stream i is blob[off[i] .. off[i]+len[i]), the raw TLV bytes of an offer, invoice_request or
 *      invoice (signature fields included: they are outside the Merkle tree).  The device parses each stream as
 *      fromwire_tlv with any type allowed does (wire/tlvstream.c:144-300: minimal BigSize type and length, strictly
 *      increasing types, no length past the end), builds merkle_tlv's root (common/bolt12_merkle.c:160-194), hashes it
 *      with the tag "lightning" || messagename || fieldname (sighash_from_merkle, :210-220) and verifies BIP-340 exactly as
 *      sv_verify_host(SV_KIND_SCHNORR) does: xonly32[i] is the key's x coordinate (check_schnorr_sig drops the parity,
 *      bitcoin/signature.c:412-423), sig64[i] the signature.
 *      status[i] = 1  bolt12_check_signature would return true;
 *                  0  it would return false (including an x that is not on the curve, r >= p, s >= n);
 *                 -1  the stream is not one CLN's TLV parser produces fields from, or it is empty.
 *      sighash32_out (optional, n x 32) returns the sighashes, zeros where status is -1.  No bound on fields per stream or
 *      value length beyond the 32-bit span length.  Spans out of range or NULL required pointers: SV_ERR_ARG. ---- */
int sv_verify_bolt12_host(sv_ctx *ctx, const char *messagename, const char *fieldname, const uint8_t *blob,
                          size_t blob_len, const uint64_t *off, const uint32_t *len, const uint8_t *xonly32,
                          const uint8_t *sig64, size_t n, int *status, uint8_t *sighash32_out);
/* ---- the same for streams signed under DIFFERENT tags, in one pass (one launch sequence): stream i is hashed with the
 *      tag "lightning" || messagenames[tag_of[i]] || fieldnames[tag_of[i]].  Callers that collect checks of several kinds
 *      (the verifier subdaemon: invoice and invoice_request signatures of many clients) verify them together.  status and
 *      sighash32_out as for sv_verify_bolt12_host.  No bound on ntags or on the length of a name.  SV_ERR_ARG also when
 *      ntags == 0 with n > 0, a tag_of[i] >= ntags, or a NULL name. ---- */
int sv_verify_bolt12_tagged_host(sv_ctx *ctx, size_t ntags, const char *const *messagenames, const char *const *fieldnames,
                                 const uint32_t *tag_of, const uint8_t *blob, size_t blob_len, const uint64_t *off,
                                 const uint32_t *len, const uint8_t *xonly32, const uint8_t *sig64, size_t n,
                                 int *status, uint8_t *sighash32_out);

/* ---- BOLT11 invoice signatures, everything on the device: bolt11_decode's signature step (common/bolt11.c:980-1062)
 *      for n invoice strings.  Invoice i is blob[off[i] .. off[i]+len[i]), read up to its first NUL byte as strlen would
 *      read it, exactly as bolt11_decode receives it (no "lightning:" prefix is stripped; callers lower-case and strip it
 *      with to_canonical_invstr).  No bound on invoice length beyond the 32-bit span.
 *      status[i] = -1  the structure that locates the signed bytes and the key is unsound: bech32_decode refuses the
 *                      string (fewer than 8 characters, a character outside 33..126, mixed case, no '1', fewer than 6
 *                      checksum characters, a bad checksum) or gives BECH32M; the 35-bit timestamp cannot be read; the
 *                      tagged-field walk fails (a tag or length it cannot read, a field longer than what is left); the walk
 *                      does not end with exactly 104 words for the signature; the first 53-word `n` field (a later one
 *                      is an unknown field) has a non-zero trailing bit or is not a valid compressed key;
 *                   0  the signature step refuses: recovery id above 3, r >= n or s >= n; with `n`,
 *                      secp256k1_ecdsa_verify is false (high-S included); without `n`, secp256k1_ecdsa_recover fails
 *                      (r = 0, s = 0, recid & 2 with r + n >= p, R.x off the curve, Q = infinity; high-S is accepted);
 *                   1  the signature step accepts.
 *      node_id33_out (n x 33): the receiver_id bolt11_decode would set (the `n` key, or the recovered key compressed)
 *      where status is 1, zeros elsewhere.  hash32_out (optional, n x 32): hash_u5's signing hash, SHA-256 of the
 *      lowercased hrp and every word before the signature packed to bytes and zero-padded; zeros where status is -1.
 *      NOT checked on the device (field values the caller's own decode handles, so an invoice bolt11_decode refuses for
 *      one of them can still get status 1): the hrp's "ln" prefix, chain and amount; whether p, s and one of d / h are
 *      present; trailing bits of p / h / s; UTF-8 in d; x, c, f, r, m; 9 against our_features; h against a description.
 *      Spans out of range or NULL required pointers: SV_ERR_ARG.  n == 0 is valid. ---- */
int sv_verify_bolt11_host(sv_ctx *ctx, const uint8_t *blob, size_t blob_len, const uint64_t *off, const uint32_t *len,
                          size_t n, int *status, uint8_t *node_id33_out, uint8_t *hash32_out);

/* ---- DEVICE buffers (same SoA layout, device pointers); asynchronous on `stream`
 *      (a cudaStream_t passed as void*; NULL = the context's own stream).  d_verdicts[n] bytes;
 *      d_bitmap, if non-NULL, receives ceil(n/32) little-endian 32-bit words, bit i%32 of word i/32. ---- */
int sv_verify_device(sv_ctx *ctx, int kind, const void *d_msg32, const void *d_key, const void *d_sig64, size_t n,
                     void *d_verdicts, void *d_bitmap, void *stream);
int sv_sync(sv_ctx *ctx, void *stream);
/* the context's own cudaStream_t (as void*), e.g. to record timing events on it */
void *sv_get_stream(const sv_ctx *ctx);

/* ---- deferral queue: enqueue returns the item's index in the pending batch; sv_flush verifies all
 *      pending items of every kind and writes one verdict byte per item in enqueue order. ---- */
long sv_enqueue(sv_ctx *ctx, int kind, const uint8_t msg32[32], const uint8_t *key, const uint8_t sig64[64]);
size_t sv_pending(const sv_ctx *ctx);
int sv_flush(sv_ctx *ctx, uint8_t *verdicts, size_t capacity);

/* ---- helpers of the bitcoin/ surface that are pure functions of bytes ---- */
/* out32[i] = SHA256d(data[off[i]..off[i]+len[i]))   (bitcoin/shadouble.c:7) */
int sv_sha256d_host(sv_ctx *ctx, const uint8_t *data, size_t data_len, const uint64_t *off, const uint32_t *len,
                    size_t n, uint8_t *out32);
/* pubkey_from_der semantics for a batch: key33[n][33] -> xy64[n][64] (x||y big-endian), ok[n] = 0/1 */
int sv_pubkey_parse_host(sv_ctx *ctx, const uint8_t *key33, size_t n, uint8_t *xy64, uint8_t *ok);

/* ---- device-side self test of the arithmetic (TEST SUPPORT; model: libsecp256k1 tests.c:3023-3176 field self-tests,
 *      :2354 scalar tests).  Runs ONE primitive of the engine's inline-PTX arithmetic on caller operands, one GPU thread
 *      per item: a[n][8], b[n][8] little-endian 32-bit limbs in; out[n][16] limbs out (result in out[0..7]; flags or the
 *      high half in out[8..15], see the list).  Field results are in the engine's WEAK form (any value < 2^256
 *      congruent to the residue) unless stated. ---- */
enum {
    SV_ST_FE_MUL = 0,        /* a*b mod p */
    SV_ST_FE_SQR = 1,        /* a^2 */
    SV_ST_FE_ADD = 2,        /* a+b */
    SV_ST_FE_SUB = 3,        /* a-b */
    SV_ST_FE_NEG = 4,        /* -a */
    SV_ST_FE_NORMALIZE = 5,  /* canonical a; out[8] = (a == 0 mod p), out[9] = (a >= p), out[10] = (a == b mod p) */
    SV_ST_FE_INV = 6,        /* a^(p-2) */
    SV_ST_FE_SQRT = 7,       /* a^((p+1)/4); out[8] = 1 iff it squares back to a */
    SV_ST_FE_MUL3 = 8,
    SV_ST_FE_MUL8 = 9,
    SV_ST_FE_MUL_SMALL = 10, /* a * (b[0] & 0xFFFF) */
    SV_ST_FE_DBL = 11,
    SV_ST_FE_B32 = 12,       /* a = 32 big-endian bytes (memory order): set_b32 -> get_b32 round trip; out[8] = (value < p) */
    SV_ST_U256_MUL_WIDE = 13, /* full 512-bit product in out[0..15] */
    SV_ST_U256_SQR_WIDE = 14,
    SV_ST_FE_REDUCE512 = 15,  /* (a + b*2^256) mod p */
    SV_ST_U256_ADD = 16,      /* out[8] = carry */
    SV_ST_U256_SUB = 17,      /* out[8] = borrow */
    SV_ST_SC_MUL = 20,        /* a*b mod n (a, b < n), canonical */
    SV_ST_SC_SQR = 21,
    SV_ST_SC_ADD = 22,
    SV_ST_SC_NEGATE = 23,     /* out[8] = is_high(a), out[9] = is_zero(a), out[10] = (a >= n) */
    SV_ST_SC_INVERSE = 24,
    SV_ST_SC_REDUCE512 = 25,  /* (a + b*2^256) mod n */
    SV_ST_SC_SPLIT_LAMBDA = 26, /* r1 -> out[0..7], r2 -> out[8..15] */
    SV_ST_SC_SET_B32 = 27,    /* a = 32 big-endian bytes: reduced scalar, out[8] = overflow */
    SV_ST_ECMULT_GEN = 28,    /* a*G through the fixed-base comb table: affine x -> out[0..7], y -> out[8..15]; 0 -> zeros */
    SV_ST_PREPARE_U2 = 29,    /* b = u2: |k1| -> out[0..4], |k2| -> out[5..9] (sign in bit 159), both odd */
    SV_ST_PREPARE_U1 = 30,    /* a = u1: 16 signed comb digits -> out[0..15] */
    SV_ST_SC_INVERSE_VAR = 31, /* binary extended Euclid: same value as SV_ST_SC_INVERSE */
    SV_ST_FE_INV_VAR = 32     /* canonical 1/a mod p */
};
int sv_selftest_host(sv_ctx *ctx, int op, const uint32_t *a, const uint32_t *b, size_t n, uint32_t *out);

/* ---- device-side self test of the group law and the scalar-multiplication schedules (TEST SUPPORT).  One op per item:
 *      in[n][SV_STG_IN_WORDS] -> out[n][SV_STG_OUT_WORDS], 32-bit little-endian limbs.  A field element takes 8 words, a
 *      Jacobian point 25 (x, y, z, then the infinity flag); field outputs are in the engine's weak form.  In the list,
 *      "a" is the point at in[0..24], "b" the point at in[32..56] (affine: x, y only), "w" the work record built from
 *      in[32..36] = k1 and in[40..44] = k2 (magnitude, sign in bit 31 of the last word, as SV_ST_PREPARE_U2 returns them)
 *      and the comb digits of u1 = in[48..55]; "Q" is the affine point at in[0..15]. ---- */
#define SV_STG_IN_WORDS 64
#define SV_STG_OUT_WORDS 200
enum {
    SV_STG_GEJ_DOUBLE = 0,        /* 2a -> out[0..24] */
    SV_STG_GEJ_ADD_GE = 1,        /* a + b (b affine) -> out[0..24], rzr -> out[32..39]; in[60] bit 0: r aliases a */
    SV_STG_GEJ_ADD_GEJ = 2,       /* a + b -> out[0..24]; in[60] = 0: r separate, 1: r aliases a, 2: r aliases b */
    SV_STG_GE_SET_XO = 3,         /* x = in[0..7], odd = in[8]: x -> out[0..7], y -> out[8..15], out[16] = x^3+7 is a residue */
    SV_STG_QTABLE_BUILD = 4,      /* table of Q: entry e at out[24e..24e+23] (x, y, beta*x), zc -> out[192..199] */
    SV_STG_ECMULT_LADDER_Q = 5,   /* table of Q, then ecmult_ladder_q with w -> out[0..24] (true coordinates) */
    SV_STG_ECMULT_HALF_LADDER = 6, /* table of Q, then ecmult_half_ladder over the magnitude at in[32..36], lambda half iff
                                      in[60] != 0 -> out[0..24] on the scaled curve (true Z = Z * zc), zc -> out[32..39] */
    SV_STG_ECMULT_COMB_ADD = 7,   /* a + u1*G through ecmult_comb_add -> out[0..24] */
    SV_STG_SMALL_COMB = 8,        /* u1*G through small_comb (from infinity) -> out[0..24] */
    SV_STG_ECMULT_LADDER = 9,     /* table of Q, then ecmult_ladder with w (u1*G + u2*Q) -> out[0..24] */
    SV_STG_NS_LINEAR_FORM = 10    /* X1, Y1, Zs = in[0..7], [8..15], [16..23], c = in[24..31], T = in[32..55], r = in[56..63]:
                                     D, B, N, CG -> out[0..7], [8..15], [16..23], [24..31]; out[32] = exceptional */
};
int sv_selftest_group_host(sv_ctx *ctx, int op, const uint32_t *in, size_t n, uint32_t *out);

/* ---- synthetic workload generator (benchmark / test support; NOT constant time, no secrets):
 *      item i gets secret key and nonce derived from (seed, i); writes msg32, key (per kind) and a
 *      VALID low-S ECDSA / BIP-340 signature to device arrays. ---- */
int sv_synth_device(sv_ctx *ctx, int kind, uint64_t seed, size_t n, void *d_msg32, void *d_key, void *d_sig64,
                    void *stream);

/* ---- introspection for the benchmark ---- */
typedef struct {
    int device;
    int sm_count;
    int main_block;       /* threads per CTA of the curve-side kernel */
    int main_grid;        /* CTAs */
    int main_regs;        /* registers per thread (cudaFuncGetAttributes) */
    size_t gtable_bytes;
    size_t scratch_bytes;
    unsigned long long launches; /* kernels launched by this context so far, not counting cub's sorts and scans */
    size_t l2_persist_bytes;     /* persisting L2 carve-out behind the table-slab access-policy window (0: hint off) */
    size_t l2_max_persist_bytes; /* what the device would allow */
} sv_info;
int sv_get_info(const sv_ctx *ctx, sv_info *info);

/* per-kernel device timing: when enabled, every sv_verify_* call records CUDA events on its launch stream
 * around the scalar-side and curve-side kernels; read them back after synchronising. */
int sv_set_profiling(sv_ctx *ctx, int on);
int sv_get_last_timing(sv_ctx *ctx, float *prep_ms, float *main_ms);
/* the same for the last sv_verify_bolt12_host call: parse + Merkle + sighash kernels, then the verification kernels.
 * It and sv_get_last_bolt11_timing report what the last profiled call of their own entry point measured before it
 * returned, as the gossip_store getters do: a later call of any other entry point leaves them as they are, and before
 * the first such call they are 0. */
int sv_get_last_bolt12_timing(sv_ctx *ctx, float *merkle_ms, float *verify_ms);
/* the same for the last sv_verify_bolt11_host call: parse + hash kernels, then the verification and recovery kernels */
int sv_get_last_bolt11_timing(sv_ctx *ctx, float *parse_ms, float *curve_ms);

/* integer-pipe roofline probe: runs a dependent-chain IMAD.WIDE.U32 microbenchmark and returns the
 * achieved 32x32->64 multiply-accumulates per second on this device (the roofline denominator
 * SURVEY.md §8d asks to be measured, not assumed). */
int sv_probe_imad_peak(sv_ctx *ctx, double *imad_per_sec);
/* individual probes (see engine.cu k_probe_*): 0 IMAD.WIDE peak, 1 4-deep carry chains, 2 fe_mul/s, 3 fe_sqr/s,
 * 4 8-deep carry chains, 5 carry-save, 6 32-bit IMAD lo/hi, 7 IADD3 carry chains, 8 FP64 FMA,
 * 9 / 10: dependent fe_mul / fe_sqr per second of ONE thread on an otherwise idle device (small-batch latency model) */
int sv_probe(sv_ctx *ctx, int mode, double *ops_per_sec);

/* pinned host memory (cudaHostAlloc) for callers that want full-speed copies */
void *sv_host_alloc(size_t bytes);
void sv_host_free(void *p);

#ifdef __cplusplus
}
#endif
#endif
