/*
 * sigverifyd_proto.h — what the verifier subdaemon (sigverifyd.c) and its client (cln_dropin.c) must agree on beyond
 * the generated codec (sigverifyd_wiregen.h): the frame limit, the largest store a prune request may name, and how a
 * negative status travels in a u8 status array.
 */
#pragma once
#include <stdint.h>

#define MAX_ITEMS (1u << 20)               /* signatures, buffers or keys in one request */
#define MAX_FRAME (32u + MAX_ITEMS * 161u) /* the longest message the daemon reads; a longer length prefix closes the connection */
/* the longest gossip_store a sigverifyd_gossip_store_prune request may name: a longer one is answered EFBIG and never
 * reaches the engine (the store is staged whole in host and device memory, and the daemon is shared) */
#define MAX_PRUNE_STORE ((uint64_t)4 << 30)

/* statuses -4..-1 travel as 252..255, 0..5 as themselves */
static inline uint8_t status_to_wire(int s) { return (uint8_t)(s < 0 ? 256 + s : s); }
static inline int status_from_wire(uint8_t b) { return b >= 252 ? (int)b - 256 : b; }
