/* oracle/gossmap_inc/common/gossip_store_wiregen.h — TEST INFRASTRUCTURE: stand-in for the header Core Lightning
 * generates from common/gossip_store_wire.csv, for compiling common/gossmap.c outside its build (oracle/gossmap.mk).  It
 * holds the store-only message type numbers and the one prototype gossmap.c calls; oracle/gossmap_harness.c stubs it. */
#ifndef LIGHTNING_COMMON_GOSSIP_STORE_WIREGEN_H
#define LIGHTNING_COMMON_GOSSIP_STORE_WIREGEN_H
#include "config.h"
#include <bitcoin/short_channel_id.h>
#include <ccan/short_types/short_types.h>
#include <common/amount.h>
#include <common/node_id.h>
#include <common/pseudorand.h>

enum gossip_store_wire {
	WIRE_GOSSIP_STORE_CHANNEL_AMOUNT = 4101,
	WIRE_GOSSIP_STORE_PRIVATE_UPDATE_OBS = 4102,
	WIRE_GOSSIP_STORE_DELETE_CHAN = 4103,
	WIRE_GOSSIP_STORE_PRIVATE_CHANNEL_OBS = 4104,
	WIRE_GOSSIP_STORE_ENDED = 4105,
	WIRE_GOSSIP_STORE_CHAN_DYING = 4106,
	WIRE_GOSSIP_STORE_UUID = 4107,
};

bool fromwire_gossip_store_chan_dying(const void *p, struct short_channel_id *scid, u32 *blockheight);

#endif /* LIGHTNING_COMMON_GOSSIP_STORE_WIREGEN_H */
