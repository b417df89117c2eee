/*
 * cln_dropin.h — the reference's own entry points for the verification path, re-implemented on top
 * of the batch engine (cln_sigverify.h).  Same names, argument meaning and error behaviour as CLN:
 *
 *   check_signed_hash          bitcoin/signature.h:85    (bitcoin/signature.c:174-192)
 *   check_signed_hash_nodeid   common/node_id.h:80       (common/node_id.c:72-80)
 *   check_schnorr_sig          bitcoin/signature.h:129   (bitcoin/signature.c:408-430)
 *   sha256_double              bitcoin/shadouble.h       (bitcoin/shadouble.c:7-11)
 *   pubkey_from_der            bitcoin/pubkey.h          (bitcoin/pubkey.c:14-24)
 *   sigcheck_channel_announcement / _node_announcement / _channel_update
 *                              gossipd/sigcheck.h        (gossipd/sigcheck.c:45-115, 118-164, 9-43)
 *                              — here in BATCH form: n raw wire messages in, one status per message out
 *   check_tx_sigs_batch        the per-HTLC loop of channeld/channeld.c:2215-2232 (one shared key,
 *                              n sighashes, n signatures) as one launch
 *
 *   bolt12_check_signature     common/bolt12.h           (common/bolt12.c:80-92) — same signature; the TLV Merkle root
 *                              and sighash are computed on the device
 *   check_tx_sig               bitcoin/signature.h:120   (bitcoin/signature.c:194-221) — same signature; the BIP143
 *                              sighash (bitcoin_tx_hash_for_sig :120-151 -> libwally tx_io.c:660-765) is computed
 *                              on the device from the wally_tx fields
 *
 * A false return always means "signature invalid" (peer's fault).  Engine failures (no GPU, CUDA
 * error) abort() with a message on stderr, CLN's convention for internal errors
 * (bitcoin/signature.c:117,212,420; SURVEY.md §8b) — they are never reported as false.
 *
 * Types: inside CLN the real headers provide these (define CLN_TYPES_PROVIDED before including);
 * stand-alone, layout-compatible minimal definitions are supplied below.
 */
#ifndef CLN_DROPIN_H
#define CLN_DROPIN_H

#include <stdbool.h>
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#ifndef CLN_TYPES_PROVIDED
typedef unsigned char u8;
struct sha256 { union { uint32_t u32[8]; unsigned char u8[32]; } u; };  /* ccan/crypto/sha256/sha256.h */
struct sha256_double { struct sha256 sha; };                           /* bitcoin/shadouble.h:9-11 */
typedef struct { unsigned char data[64]; } secp256k1_ecdsa_signature;   /* secp256k1.h (opaque) */
typedef struct { unsigned char data[64]; } secp256k1_pubkey;            /* secp256k1.h (opaque) */
struct pubkey { secp256k1_pubkey pubkey; };                            /* bitcoin/pubkey.h:15-18 */
struct node_id { u8 k[33]; };                                          /* common/node_id.h:11-13 */
struct bip340sig { u8 u8[64]; };                                       /* bitcoin/signature.h:145-147 */
enum sighash_type { SIGHASH_ALL = 1, SIGHASH_NONE = 2, SIGHASH_SINGLE = 3, SIGHASH_ANYONECANPAY = 0x80 };
struct bitcoin_signature { secp256k1_ecdsa_signature s; enum sighash_type sighash_type; }; /* signature.h:47-50 */
/* libwally's public transaction structs (external/libwally-core/include/wally_transaction.h:89-155), Elements fields
 * included as CLN builds libwally (no WALLY_ABI_NO_ELEMENTS); only the fields BIP143 commits to are read. */
struct wally_tx_witness_stack;
struct wally_tx_input {
    unsigned char txhash[32];
    uint32_t index;
    uint32_t sequence;
    unsigned char *script;
    size_t script_len;
    struct wally_tx_witness_stack *witness;
    uint8_t features;
    unsigned char blinding_nonce[32];
    unsigned char entropy[32];
    unsigned char *issuance_amount;
    size_t issuance_amount_len;
    unsigned char *inflation_keys;
    size_t inflation_keys_len;
    unsigned char *issuance_amount_rangeproof;
    size_t issuance_amount_rangeproof_len;
    unsigned char *inflation_keys_rangeproof;
    size_t inflation_keys_rangeproof_len;
    struct wally_tx_witness_stack *pegin_witness;
};
struct wally_tx_output {
    uint64_t satoshi;
    unsigned char *script;
    size_t script_len;
    uint8_t features;
    unsigned char *asset;
    size_t asset_len;
    unsigned char *value;
    size_t value_len;
    unsigned char *nonce;
    size_t nonce_len;
    unsigned char *surjectionproof;
    size_t surjectionproof_len;
    unsigned char *rangeproof;
    size_t rangeproof_len;
};
struct wally_tx {
    uint32_t version;
    uint32_t locktime;
    struct wally_tx_input *inputs;
    size_t num_inputs;
    size_t inputs_allocation_len;
    struct wally_tx_output *outputs;
    size_t num_outputs;
    size_t outputs_allocation_len;
};
struct chainparams;
struct wally_psbt;
struct bitcoin_tx { struct wally_tx *wtx; const struct chainparams *chainparams; struct wally_psbt *psbt; }; /* bitcoin/tx.h:32-40 */
struct tlv_record_type;
struct tlv_field {                         /* wire/tlvstream.h:16-27 */
    const struct tlv_record_type *meta;
    uint64_t numtype;
    size_t length;
    u8 *value;
};
#endif

/* Optional: choose the CUDA device (default: $CLN_SIGVERIFY_DEVICE or 0).  The context is created
 * lazily on first use; one per process, as CLN's global secp256k1_ctx (common/utils.c:16). */
void cln_sigverify_init(int device);
void cln_sigverify_shutdown(void);

/* CLIENT MODE: share one GPU process (the verifier subdaemon cln_sigverifyd) instead of opening an engine context here.
 * It is on when $CLN_SIGVERIFYD_SOCKET names the daemon's unix socket (connected on the first check; a failed connect
 * aborts), or after one of these calls succeeds (0; -1 and errno when the socket cannot be reached):
 *   cln_sigverify_connect(path)   connect to the daemon's socket
 *   cln_sigverify_connect_fd(fd)  use an already-connected socket, e.g. a socketpair end inherited from the parent, the way
 *                                 lightningd hands fds to its subdaemons (the daemon side: cln_sigverifyd --fd N)
 * In client mode these functions send one request over the process's one connection and wait for the reply;
 * they never create a context:
 *   check_signed_hash, check_signed_hash_nodeid, check_schnorr_sig, check_tx_sigs_batch   (sigverifyd_verify)
 *   bolt12_check_signature                                                              (sigverifyd_bolt12)
 *   check_tx_sig, check_tx_sigs_bip143_batch                                            (sigverifyd_tx)
 *   check_tx_sig_grind_fee                                                              (sigverifyd_fee_grind)
 *   sigcheck_channel_announcement_batch / _node_announcement_batch / _channel_update_batch (sigverifyd_gossip)
 *   sigcheck_gossip_batch                                                               (sigverifyd_gossip_burst)
 *   sha256_double                                                                       (sigverifyd_sha256d)
 *   pubkey_from_der                                                                     (sigverifyd_pubkey)
 * check_tx_sig gates the sighash type before it sends anything; the BIP143 sighash is built on the daemon's device.
 * check_tx_sigs_bip143_batch sends requests of at most 65536 transactions and 64 MiB of scripts each.  pubkey_from_der
 * returns false for a length other than 33 without sending anything.  The daemon serves the requests of all its clients
 * together.  A lost daemon, a short read, an error reply, a reply to another request or a transaction or buffer too large
 * for one request abort() (an internal error, never a bad signature).  No function of this header opens a context in
 * client mode; cln_sigverify_init(), which creates one on purpose, is for the in-process variant.  Without the variable
 * and the calls, nothing changes. */
int cln_sigverify_connect(const char *socket_path);
int cln_sigverify_connect_fd(int fd);

/* NON-BLOCKING CLIENT MODE: many checks in flight from one process.  A blocking call holds at most one request at the
 * daemon; an event loop (ccan/io, libplugin) with many independent checks starts them as tickets instead, and the daemon
 * serves everything the process has sent in the same launches, as it serves many processes.  Each _start below takes the
 * arguments of the blocking function of the same name, plus where the answer goes and a continuation:
 *
 *   0    the answer is already in *ok / status and no callback follows: always in in-process mode (the _start calls the
 *        blocking function), and for the local gates, which send nothing: check_tx_sig's sighash-type gate,
 *        bolt12_check_signature's empty or not strictly ascending field array (false, as the device answers the blocking
 *        call), sigcheck_gossip_batch with n == 0.
 *   > 0  a ticket.  The answer is written to *ok / status[0..n), then done(arg) runs (done may be NULL).  The caller keeps
 *        that output memory alive until the callback; every input is copied before the _start returns.
 *
 * Verdicts, statuses and aborts are exactly the blocking function's: the request is built by the same code and the reply
 * passes the same checks.
 * Ordering: callbacks run in ticket order, each exactly once, and only from cln_sigverify_process() or
 * cln_sigverify_drain(), never from inside a _start or a blocking call.  A callback may call any function of this header,
 * _start and blocking ones included.
 * Blocking calls with tickets outstanding: the blocking call's request goes behind the unsent ones and it reads replies
 * until its own arrives, writing the earlier tickets' answers on the way; their callbacks wait for the next
 * cln_sigverify_process() (call it after such a blocking call: the socket may have nothing more to read).
 * Back-pressure: writes never block; what the socket does not take stays in a buffer of this library.  While 1,024
 * tickets await replies, or 64 MiB of requests are unsent, a _start first waits (as a blocking call would) until the
 * oldest are answered or written; their callbacks still wait for cln_sigverify_process().  One request's own limits are the
 * blocking function's (MAX_FRAME; a gossip burst is never split).
 * Errors: a lost daemon, a short read, an error reply, a malformed reply or a reply out of request order abort(), as in
 * blocking mode; nothing is ever reported as a bad signature.  cln_sigverify_shutdown() and a new connection discard the
 * outstanding tickets without running their callbacks. */
/* the continuation of a ticket */ typedef void (*cln_sigverify_done)(void *arg);

uint64_t check_signed_hash_start(const struct sha256_double *hash, const secp256k1_ecdsa_signature *signature,
                                 const struct pubkey *key, bool *ok, cln_sigverify_done done, void *arg);
uint64_t check_signed_hash_nodeid_start(const struct sha256_double *hash, const secp256k1_ecdsa_signature *signature,
                                        const struct node_id *id, bool *ok, cln_sigverify_done done, void *arg);
uint64_t check_schnorr_sig_start(const struct sha256 *hash, const secp256k1_pubkey *pubkey, const struct bip340sig *sig,
                                 bool *ok, cln_sigverify_done done, void *arg);
uint64_t check_tx_sig_start(const struct bitcoin_tx *tx, size_t input_num, const u8 *redeemscript, const u8 *witness_script,
                            const struct pubkey *key, const struct bitcoin_signature *sig, bool *ok, cln_sigverify_done done,
                            void *arg);
uint64_t bolt12_check_signature_start(const struct tlv_field *fields, const char *messagename, const char *fieldname,
                                      const struct pubkey *key, const struct bip340sig *sig, bool *ok,
                                      cln_sigverify_done done, void *arg);
uint64_t sigcheck_gossip_batch_start(const u8 *chain_hash32, const u8 *const *msgs, const size_t *lens, size_t n,
                                     const u8 *signer_kind, const struct node_id *signers, int *status,
                                     cln_sigverify_done done, void *arg);

/* The event loop's side.  cln_sigverify_fd(): the daemon socket to watch, -1 in in-process mode.
 * cln_sigverify_events(): POLLIN while tickets are outstanding, | POLLOUT while request bytes are unsent (0: nothing to
 * watch).  cln_sigverify_process(): never blocks; writes what the socket takes, reads what has arrived and runs the
 * callbacks of the answered tickets in ticket order; returns the number of tickets still outstanding.
 * cln_sigverify_drain(): blocks until no ticket is outstanding, running their callbacks. */
int cln_sigverify_fd(void);
short cln_sigverify_events(void);
size_t cln_sigverify_process(void);
void cln_sigverify_drain(void);

bool check_signed_hash(const struct sha256_double *hash, const secp256k1_ecdsa_signature *signature,
                       const struct pubkey *key);
bool check_signed_hash_nodeid(const struct sha256_double *hash, const secp256k1_ecdsa_signature *signature,
                              const struct node_id *id);
bool check_schnorr_sig(const struct sha256 *hash, const secp256k1_pubkey *pubkey, const struct bip340sig *sig);
void sha256_double(struct sha256_double *shadouble, const void *p, size_t len);
bool pubkey_from_der(const u8 *der, size_t len, struct pubkey *key);

/* bitcoin/signature.h:120.  Exactly one of redeemscript / witness_script is used (witness_script when non-NULL), both
 * are tal arrays in CLN: their length comes from tal_bytelen(), the input amount from psbt_input_get_amount(tx->psbt, in)
 * (bitcoin/signature.c:130).  Those two are CLN-internal functions: when this object is linked into a CLN daemon they are
 * picked up directly (weak references); a stand-alone user supplies them with cln_sigverify_set_tx_hooks(). */
bool check_tx_sig(const struct bitcoin_tx *tx, size_t input_num, const u8 *redeemscript, const u8 *witness_script,
                  const struct pubkey *key, const struct bitcoin_signature *sig);
void cln_sigverify_set_tx_hooks(size_t (*script_bytelen)(const void *tal_script),
                                uint64_t (*input_amount_sat)(const struct bitcoin_tx *tx, size_t input_num));

/* grind_htlc_tx_fee (onchaind/onchaind.c:389-437) in one call.  tx is NOT modified: on true the caller sets output 0 to
 * input - *fee_sat and finalizes, as the loop leaves it.  remotesig's sighash type is gated as check_tx_sig does.
 *      The record is built as check_tx_sig builds it (input amount from the same hook); a transaction that is not one
 *      input and one output aborts.  Semantics of the walk: sv_grind_tx_fee_host (cln_sigverify.h). */
bool check_tx_sig_grind_fee(const struct bitcoin_tx *tx, const u8 *witness_script, const struct pubkey *key,
                            const struct bitcoin_signature *remotesig, uint64_t weight, uint32_t min_feerate,
                            uint32_t max_feerate, uint64_t *fee_sat, uint32_t *feerate);

/* common/bolt12.h: bolt12_check_signature (common/bolt12.c:80-92).  fields is a tal array (its length comes from
 * tal_bytelen(fields) / sizeof(struct tlv_field), through the same weak tal_bytelen reference or hook as check_tx_sig);
 * the fields are serialised in array order into one TLV stream and sent to sv_verify_bolt12_host, which builds the
 * Merkle root and sighash on the device.  CLN only passes strictly ascending arrays (fromwire_tlv and tlv_update_fields
 * produce them), and for those the result is CLN's.  An array that is not strictly ascending by type, or is empty (merkle_tlv
 * asserts on that), is not a stream CLN's parser produces: the function returns false for it. */
bool bolt12_check_signature(const struct tlv_field *fields, const char *messagename, const char *fieldname,
                            const struct pubkey *key, const struct bip340sig *sig);

/* channeld HTLC loop: ok[i] = check_signed_hash(&hashes[i], &sigs[i].s, key) for one shared key. */
void check_tx_sigs_batch(const struct sha256_double *hashes, const struct bitcoin_signature *sigs,
                         const struct pubkey *key, size_t n, bool *ok);

/* The same loop with the BIP143 sighash ALSO computed on the device (row N2): check_tx_sig (bitcoin/signature.c:194-221)
 * for n one-input one-output transactions described by sv_tx records (cln_sigverify.h); the sighash type of each
 * signature is taken from sigs[i].sighash_type and gated exactly as check_tx_sig does (:206-211: only SIGHASH_ALL or
 * SIGHASH_SINGLE|SIGHASH_ANYONECANPAY, else false). */
struct sv_tx_fields; /* = sv_tx of cln_sigverify.h */
void check_tx_sigs_bip143_batch(const void *sv_tx_array, const u8 *scripts, size_t scripts_len,
                                const struct pubkey *key, const struct bitcoin_signature *sigs, size_t n, bool *ok);

/* gossipd: status[i] = 0 if every signature of message i verifies, else 1 + the index of the FIRST bad
 * signature in the reference's checking order (channel_announcement: node_signature_1, node_signature_2,
 * bitcoin_signature_1, bitcoin_signature_2 -> 1..4; node_announcement / channel_update: 1); -1 if the
 * message is too short / malformed to locate its fields.  msgs[i] is the complete wire message
 * (2-byte type included), lens[i] its length. */
void sigcheck_channel_announcement_batch(const u8 *const *msgs, const size_t *lens, size_t n, int *status);
void sigcheck_node_announcement_batch(const u8 *const *msgs, const size_t *lens, size_t n, int *status);
/* channel_update is signed by the node found in the gossmap: the caller supplies it. */
void sigcheck_channel_update_batch(const u8 *const *msgs, const size_t *lens, const struct node_id *signers,
                                   size_t n, int *status);

/* gossipd's signature gate over a burst of raw gossip messages of any types (sv_verify_gossip_burst_host in
 * cln_sigverify.h): a channel_update's signer comes from the batch's own channel_announcements (signer_kind[i] 0), from
 * signers[i] (1: the node the caller's gossmap gives), or from the batch with signers[i] as the source peer's fallback
 * (2).  status[i]: 0 ok, 1..4 first bad signature, 5 verified under the source peer, -1 malformed, -2 no channel, -3
 * another chain than chain_hash32, -4 node ids out of order.  signer_kind == NULL means all 0; signers may be NULL only
 * when no channel_update has kind 1 or 2.  The batch is never split (an update may resolve against any announcement
 * before it): in client mode it travels as ONE sigverifyd_gossip_burst request, and a batch too large for one frame
 * aborts. */
void sigcheck_gossip_batch(const u8 *chain_hash32, const u8 *const *msgs, const size_t *lens, size_t n, const u8 *signer_kind,
                           const struct node_id *signers, int *status);

#ifdef __cplusplus
}
#endif
#endif
