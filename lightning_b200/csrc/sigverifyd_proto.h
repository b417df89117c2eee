/*
 * sigverifyd_proto.h — what the verifier subdaemon (sigverifyd.c) and its client (cln_dropin.c) must agree on beyond
 * the generated codec (sigverifyd_wiregen.h): the frame limit, and how a negative status travels in a u8 status array.
 */
#pragma once
#include <stdint.h>

#define MAX_ITEMS (1u << 20)               /* signatures, buffers or keys in one request */
#define MAX_FRAME (32u + MAX_ITEMS * 161u) /* the longest message the daemon reads; a longer length prefix closes the connection */

/* statuses -4..-1 travel as 252..255, 0..5 as themselves */
static inline uint8_t status_to_wire(int s) { return (uint8_t)(s < 0 ? 256 + s : s); }
static inline int status_from_wire(uint8_t b) { return b >= 252 ? (int)b - 256 : b; }
