/* Stand-in for lightningd/lightningd.h, which common/bolt11.c includes although the decoder uses nothing of the daemon.
 * The real header pulls in the whole daemon; the oracle build (oracle/bolt11.mk) searches this directory first.  What
 * bolt11.c does take from it by way of its includes: tmpctx and secp256k1_ctx, and struct secret. */
#ifndef LIGHTNING_ORACLE_BOLT11_STUB_LIGHTNINGD_H
#define LIGHTNING_ORACLE_BOLT11_STUB_LIGHTNINGD_H
#include "config.h"
#include <bitcoin/privkey.h>
#include <common/utils.h>
#endif
