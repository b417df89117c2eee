/* oracle/gossmap_inc/wire/peer_wiregen.h — TEST INFRASTRUCTURE: stand-in for the header Core Lightning generates from
 * wire/peer_wire.csv, for compiling common/gossmap.c outside its build (oracle/gossmap.mk).  It holds the message type
 * numbers of peer_wire.csv (BOLT #1, #2, #7) and the one prototype gossmap.c calls; oracle/gossmap_harness.c stubs it. */
#ifndef LIGHTNING_WIRE_PEER_WIREGEN_H
#define LIGHTNING_WIRE_PEER_WIREGEN_H
#include "config.h"
#include <bitcoin/block.h>
#include <bitcoin/short_channel_id.h>
#include <ccan/short_types/short_types.h>
#include <ccan/tal/tal.h>
#include <common/amount.h>
#include <common/node_id.h>
#include <secp256k1.h>

enum peer_wire {
	WIRE_PROTOCOL_BATCH_ELEMENT = 0,
	WIRE_WARNING = 1,
	WIRE_STFU = 2,
	WIRE_PEER_STORAGE = 7,
	WIRE_PEER_STORAGE_RETRIEVAL = 9,
	WIRE_INIT = 16,
	WIRE_ERROR = 17,
	WIRE_PING = 18,
	WIRE_PONG = 19,
	WIRE_OPEN_CHANNEL = 32,
	WIRE_ACCEPT_CHANNEL = 33,
	WIRE_FUNDING_CREATED = 34,
	WIRE_FUNDING_SIGNED = 35,
	WIRE_CHANNEL_READY = 36,
	WIRE_SHUTDOWN = 38,
	WIRE_CLOSING_SIGNED = 39,
	WIRE_CLOSING_COMPLETE = 40,
	WIRE_CLOSING_SIG = 41,
	WIRE_OPEN_CHANNEL2 = 64,
	WIRE_ACCEPT_CHANNEL2 = 65,
	WIRE_TX_ADD_INPUT = 66,
	WIRE_TX_ADD_OUTPUT = 67,
	WIRE_TX_REMOVE_INPUT = 68,
	WIRE_TX_REMOVE_OUTPUT = 69,
	WIRE_TX_COMPLETE = 70,
	WIRE_TX_SIGNATURES = 71,
	WIRE_TX_INIT_RBF = 72,
	WIRE_TX_ACK_RBF = 73,
	WIRE_TX_ABORT = 74,
	WIRE_SPLICE_LOCKED = 77,
	WIRE_SPLICE = 80,
	WIRE_SPLICE_ACK = 81,
	WIRE_START_BATCH = 127,
	WIRE_UPDATE_ADD_HTLC = 128,
	WIRE_UPDATE_FULFILL_HTLC = 130,
	WIRE_UPDATE_FAIL_HTLC = 131,
	WIRE_COMMITMENT_SIGNED = 132,
	WIRE_REVOKE_AND_ACK = 133,
	WIRE_UPDATE_FEE = 134,
	WIRE_UPDATE_FAIL_MALFORMED_HTLC = 135,
	WIRE_CHANNEL_REESTABLISH = 136,
	WIRE_UPDATE_BLOCKHEIGHT = 137,
	WIRE_CHANNEL_ANNOUNCEMENT = 256,
	WIRE_NODE_ANNOUNCEMENT = 257,
	WIRE_CHANNEL_UPDATE = 258,
	WIRE_ANNOUNCEMENT_SIGNATURES = 259,
	WIRE_QUERY_SHORT_CHANNEL_IDS = 261,
	WIRE_REPLY_SHORT_CHANNEL_IDS_END = 262,
	WIRE_QUERY_CHANNEL_RANGE = 263,
	WIRE_REPLY_CHANNEL_RANGE = 264,
	WIRE_GOSSIP_TIMESTAMP_FILTER = 265,
	WIRE_ONION_MESSAGE = 513,
};

u8 *towire_channel_update(const tal_t *ctx, const secp256k1_ecdsa_signature *signature,
			  const struct bitcoin_blkid *chain_hash, struct short_channel_id short_channel_id, u32 timestamp,
			  u8 message_flags, u8 channel_flags, u16 cltv_expiry_delta, struct amount_msat htlc_minimum_msat,
			  u32 fee_base_msat, u32 fee_proportional_millionths, struct amount_msat htlc_maximum_msat);

#endif /* LIGHTNING_WIRE_PEER_WIREGEN_H */
