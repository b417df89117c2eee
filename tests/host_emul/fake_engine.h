/*
 * fake_engine.h — what every part of the fake engine shares (fake_engine.c and the optional fake_engine_grind.c,
 * fake_engine_bolt11.c and fake_engine_prune.c linked beside it): the hash its answers are made of and its
 * instrumentation.
 *
 * Answers are FNV-1a (64-bit) over an item's bytes, integers entering as little-endian bytes; fill(h, n)[k] is the low
 * byte of FNV-1a continued from h over the one byte k.  The tests recompute both.
 *
 * Instrumentation, driven by three variables, each unset by default (then it does nothing):
 *   FAKE_ENGINE_LOG    a file that gets "<function> <kind> <n> <blob bytes>" for each call (fake_log)
 *   FAKE_ENGINE_DELAY  "<function>=<ms>,...": each call of a listed entry point waits that long (fake_enter)
 *   FAKE_ENGINE_TRACE  a file that gets "begin <function> <context>" when a call starts and "end <function> <context>"
 *                      when it has waited its delay; contexts are numbered from 1 in the order sv_create made them, 0
 *                      for a pointer sv_create did not return
 * Log and trace lines are written under one lock, so they are whole and in the order they happened.
 */
#pragma once
#include "../../include/cln_sigverify.h"

#include <stddef.h>
#include <stdint.h>

#define FNV0 0xcbf29ce484222325ull

static inline uint64_t fnv(uint64_t h, const void *p, size_t n) {
    const uint8_t *b = (const uint8_t *)p;
    for (size_t i = 0; i < n; i++) h = (h ^ b[i]) * 0x100000001b3ull;
    return h;
}
/* the n low bytes of v, little-endian */
static inline uint64_t fnv_le(uint64_t h, uint64_t v, int n) {
    uint8_t b[8];
    for (int i = 0; i < n; i++) b[i] = (uint8_t)(v >> (8 * i));
    return fnv(h, b, (size_t)n);
}
static inline void fill(uint64_t h, uint8_t *out, size_t n) {
    for (size_t k = 0; k < n; k++) {
        uint8_t b = (uint8_t)k;
        out[k] = (uint8_t)fnv(h, &b, 1);
    }
}
static inline int span_ok(size_t blob_len, uint64_t off, uint64_t len) { return off <= blob_len && len <= blob_len - off; }

/* a call's begin line, its delay and its end line */
void fake_enter(const char *fn, const sv_ctx *ctx);
/* a call's log line */
void fake_log(const char *fn, int kind, size_t n, size_t bytes);
/* both, as every entry point but the prune starts */
static inline void fake_call(const char *fn, const sv_ctx *ctx, int kind, size_t n, size_t bytes) {
    fake_enter(fn, ctx);
    fake_log(fn, kind, n, bytes);
}
