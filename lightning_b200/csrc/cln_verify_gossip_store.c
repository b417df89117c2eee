/* cln_verify_gossip_store — audit a Core Lightning gossip_store before lightningd loads it.
 *
 *   cln_verify_gossip_store [--chain HEX] [--device N] [--funding TABLE] [--prune OUT [--cut-tail]] FILE
 *
 * Walks the store as gossmap does, checks every record checksum and verifies every signature on the GPU
 * (sv_verify_gossip_store_host).  Prints a summary and one line per failing record (offset, type, status).
 * --chain HEX (32-byte chain hash as it appears on the wire) adds gossipd's chain and node-order gates.
 *
 * Exit code: 0  every reached record is good and the walk ended at the end of the store, an incomplete or partial
 *               last record (a live store's tail can look like either) or a gossip_store_ended record;
 *            1  some signature, gate or channel resolution failed;
 *            2  the walk stopped at a bad checksum, a truncated record or an announcement without its amount;
 *            3  usage, I/O or engine error.
 *
 * --prune OUT: writes OUT, a copy of FILE with every record gossmap should not trust marked deleted
 * (sv_prune_gossip_store_host), and never writes FILE.  Prints the deletions per reason, then audits OUT as above.
 * Exit code: 0  OUT is clean: its audit finds no bad signature, malformed message, update without a channel, other
 *               chain, node ids out of order, redundant announcement or unknown record, and its walk reaches the end of
 *               the store, so gossipd's strict load accepts it;
 *            1  OUT is written but not clean (its walk stops before the end: an incomplete, partial or ended record,
 *               or an announcement without its amount record);
 *            3  usage, I/O or engine error (OUT may be missing).
 *
 * --cut-tail (with --prune): OUT also ends where the prune's walk stopped at a torn append (sv_gossip_prune_cut: an
 * incomplete or partial record, an announcement without its amount record, or a torn header; an announcement the cut
 * would leave without its amount record goes too), as
 * sv_repair_gossip_store_fd cuts a file in place.  Prints where it cut, then audits OUT as --prune does.
 *
 * --funding TABLE: also checks every announcement against lightningd's funding outputs (TABLE as written by
 * `python -m lightning_b200.funding export`; sv_verify_gossip_store_funding_host).  Prints the funding counts and one
 * line per announcement gossipd would have refused (no unspent output, wrong script, wrong amount record).  Without
 * --prune it exits 1 if there is one (unless a worse code applies).  With --prune it deletes them too
 * (sv_prune_gossip_store_funding_host), and OUT's audit runs with the table: OUT is clean only if no announcement in it
 * is refused.  Announcements in blocks lightningd never processed (unchecked) and dying channels are printed and never
 * change the exit code. */
#include <errno.h>
#include <inttypes.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "../../include/cln_sigverify.h"

static const char *status_name(int s) {
    switch (s) {
    case 0: return "ok";
    case 1: case 2: case 3: case 4: return "bad signature";
    case -1: return "malformed";
    case -2: return "no channel";
    case -3: return "other chain";
    case -4: return "node ids out of order";
    case SV_GS_DELETED: return "deleted";
    case SV_GS_STORE_RECORD: return "store record";
    case SV_GS_UNKNOWN: return "unknown type";
    case SV_GS_NOT_REACHED: return "not reached";
    case SV_GS_INCOMPLETE: return "incomplete";
    case SV_GS_PARTIAL: return "partial";
    case SV_GS_TRUNCATED: return "truncated";
    case SV_GS_BAD_CRC: return "bad checksum";
    case SV_GS_ENDED: return "ended";
    case SV_GS_NO_AMOUNT: return "no amount record";
    default: return "?";
    }
}

static int usage(void) {
    fprintf(stderr, "usage: cln_verify_gossip_store [--chain HEX] [--device N] [--funding TABLE] [--prune OUT [--cut-tail]] "
                    "FILE\n");
    return 3;
}

static const char *const reason_name[] = {"kept", "bad checksum", "truncated", "failing message", "redundant announcement",
                                          "update without a channel", "bad signature under the new signer",
                                          "amount record of a deleted announcement", "unknown record type",
                                          "announcement gossipd would refuse for its funding output"};
static const char *const funding_name[] = {"-", "funded", "unchecked (block not processed)", "dying",
                                           "no unspent output", "script is not the 2-of-2", "amount record differs"};

/* the funding table file (lightning_b200/funding.py): "CLNFUND1", u64 n_outputs, u64 n_blocks (little-endian), then
 * n_outputs x [scid u64, satoshis u64, script 34 bytes], then n_blocks x [height u32] */
typedef struct {
    sv_funding_table t;
    uint64_t *scid, *sats;
    uint8_t *script;
    uint32_t *blocks;
} funding_file;

static uint64_t le64(const uint8_t *p) {
    uint64_t v = 0;
    for (int i = 7; i >= 0; i--) v = (v << 8) | p[i];
    return v;
}

static int load_funding(const char *path, funding_file *F) {
    FILE *f = fopen(path, "rb");
    if (!f) { fprintf(stderr, "%s: %s\n", path, strerror(errno)); return -1; }
    uint8_t h[24], e[50], b[4];
    if (fread(h, 1, 24, f) != 24 || memcmp(h, "CLNFUND1", 8)) {
        fprintf(stderr, "%s: not a funding table\n", path);
        fclose(f);
        return -1;
    }
    const uint64_t n = le64(h + 8), nb = le64(h + 16);
    if (n > ((uint64_t)1 << 32) || nb > ((uint64_t)1 << 32)) { fprintf(stderr, "%s: not a funding table\n", path); fclose(f); return -1; }
    F->scid = malloc((n ? n : 1) * 8);
    F->sats = malloc((n ? n : 1) * 8);
    F->script = malloc((n ? n : 1) * 34);
    F->blocks = malloc((nb ? nb : 1) * 4);
    if (!F->scid || !F->sats || !F->script || !F->blocks) { fprintf(stderr, "out of memory\n"); fclose(f); return -1; }
    for (uint64_t i = 0; i < n; i++) {
        if (fread(e, 1, 50, f) != 50) { fprintf(stderr, "%s: truncated\n", path); fclose(f); return -1; }
        F->scid[i] = le64(e);
        F->sats[i] = le64(e + 8);
        memcpy(F->script + 34 * i, e + 16, 34);
    }
    for (uint64_t i = 0; i < nb; i++) {
        if (fread(b, 1, 4, f) != 4) { fprintf(stderr, "%s: truncated\n", path); fclose(f); return -1; }
        F->blocks[i] = (uint32_t)b[0] | (uint32_t)b[1] << 8 | (uint32_t)b[2] << 16 | (uint32_t)b[3] << 24;
    }
    if (fread(b, 1, 1, f) != 0) { fprintf(stderr, "%s: trailing bytes\n", path); fclose(f); return -1; }
    fclose(f);
    F->t = (sv_funding_table){F->scid, F->sats, F->script, (size_t)n, F->blocks, (size_t)nb};
    return 0;
}

/* prints the funding counts; returns the number of refused announcements */
static uint64_t print_funding(const char *what, const sv_gossip_funding_summary *g) {
    printf("  funding (%s): %" PRIu64 " announcements checked: %" PRIu64 " funded, %" PRIu64 " unchecked, %" PRIu64
           " dying, %" PRIu64 " no unspent output, %" PRIu64 " wrong script, %" PRIu64 " wrong amount\n",
           what, g->checked, g->funded, g->unchecked, g->dying, g->no_txout, g->script, g->amount);
    return g->no_txout + g->script + g->amount;
}

/* one audit of a store: each record's offset, type, status and (with a table) funding verdict, and the summaries */
typedef struct {
    size_t n;
    uint64_t *off;
    uint16_t *type;
    int *status;
    uint8_t *fund;
    sv_gossip_store_summary s;
    sv_gossip_funding_summary g;
} audit_result;

/* sv_verify_gossip_store_host, or with a table sv_verify_gossip_store_funding_host; returns 0, or 3 (the exit code)
 * after saying why it failed */
static int audit(sv_ctx *ctx, const uint8_t *store, size_t len, const uint8_t *chain, const sv_funding_table *table,
                 audit_result *a) {
    const size_t n = a->n = sv_gossip_store_count(store, len);
    a->off = malloc((n ? n : 1) * sizeof *a->off);
    a->type = malloc((n ? n : 1) * sizeof *a->type);
    a->status = malloc((n ? n : 1) * sizeof *a->status);
    a->fund = malloc(n ? n : 1);
    if (!a->off || !a->type || !a->status || !a->fund) { fprintf(stderr, "out of memory\n"); return 3; }
    int rc = table ? sv_verify_gossip_store_funding_host(ctx, store, len, chain, table, a->off, a->type, a->status, NULL,
                                                         a->fund, n, &a->s, &a->g)
                   : sv_verify_gossip_store_host(ctx, store, len, chain, a->off, a->type, a->status, NULL, n, &a->s);
    if (rc != SV_OK) {
        fprintf(stderr, "%s: %d %s\n", table ? "sv_verify_gossip_store_funding_host" : "sv_verify_gossip_store_host", rc,
                sv_last_error(ctx));
        return 3;
    }
    return 0;
}

static void audit_free(audit_result *a) { free(a->off); free(a->type); free(a->status); free(a->fund); }

/* --prune: write the pruned copy (cut_tail: without its torn tail), report it, audit it; returns the exit code */
static int prune(sv_ctx *ctx, const char *path, const uint8_t *store, size_t len, const uint8_t *chain, const char *outp,
                 int cut_tail, const sv_funding_table *table) {
    size_t n = sv_gossip_prune_count(store, len);
    uint64_t *off = malloc((n ? n : 1) * sizeof *off);
    uint16_t *type = malloc((n ? n : 1) * sizeof *type);
    int *status = malloc((n ? n : 1) * sizeof *status);
    uint8_t *why = malloc(n ? n : 1), *fund = malloc(n ? n : 1), *out = malloc(len);
    if (!off || !type || !status || !why || !fund || !out) { fprintf(stderr, "out of memory\n"); return 3; }
    sv_gossip_prune_summary p;
    sv_gossip_funding_summary g;
    int rc = table ? sv_prune_gossip_store_funding_host(ctx, store, len, chain, table, out, off, type, status, why, fund, n,
                                                        &p, &g)
                   : sv_prune_gossip_store_host(ctx, store, len, chain, out, off, type, status, why, n, &p);
    if (rc != SV_OK) {
        fprintf(stderr, "%s: %d %s\n", table ? "sv_prune_gossip_store_funding_host" : "sv_prune_gossip_store_host", rc,
                sv_last_error(ctx));
        return 3;
    }
    for (size_t i = 0; i < n; i++)
        if (why[i]) printf("deleted @%" PRIu64 " type %u: %s (status %d)\n", off[i], type[i], reason_name[why[i]], status[i]);
    const size_t wlen = cut_tail ? (size_t)sv_gossip_prune_cut(&p, out, len) : len;
    FILE *f = fopen(outp, "wb");
    if (!f || fwrite(out, 1, wlen, f) != wlen || fclose(f)) { fprintf(stderr, "%s: %s\n", outp, strerror(errno)); return 3; }
    printf("gossip_store %s: %" PRIu64 " records, walk stopped: %s at %" PRIu64 "; %" PRIu64 " deleted into %s\n", path,
           p.records, p.stop ? status_name(p.stop) : "end of store", p.end_offset, p.pruned, outp);
    const uint64_t count[9] = {0, p.bad_crc, p.truncated, p.message, p.redundant, p.no_channel, p.signature, p.amount, p.unknown};
    for (int k = 1; k < 9; k++) printf("  %" PRIu64 " %s\n", count[k], reason_name[k]);
    if (table) printf("  %" PRIu64 " %s\n", g.deleted, reason_name[SV_GP_FUNDING]);
    printf("  %" PRIu64 " updates verified again under a new signer\n", p.reverified);
    if (table) print_funding(path, &g);
    if (cut_tail) printf("  torn tail: %zu bytes cut, %s ends at %zu\n", len - wlen, outp, wlen);
    len = wlen;
    audit_result a;
    if (audit(ctx, out, len, chain, table, &a)) return 3;
    const sv_gossip_store_summary s = a.s;
    const uint64_t refused = table ? print_funding(outp, &a.g) : 0;
    const int clean = s.stop == SV_GS_EOF && s.end_offset == len && !s.bad_signature && !s.malformed && !s.no_channel &&
                      !s.wrong_chain && !s.bad_order && !s.redundant_announcements && !s.unknown && !refused;
    printf("%s: %s (%" PRIu64 " good messages, %" PRIu64 " deleted records)\n", outp,
           clean ? "clean" : "NOT clean", s.good, s.deleted);
    free(off); free(type); free(status); free(why); free(fund); free(out);
    audit_free(&a);
    return clean ? 0 : 1;
}

int main(int argc, char **argv) {
    const char *path = NULL, *prune_out = NULL, *funding_path = NULL;
    uint8_t chain[32];
    int have_chain = 0, device = 0, cut_tail = 0;
    for (int i = 1; i < argc; i++) {
        if (!strcmp(argv[i], "--chain") && i + 1 < argc) {
            const char *h = argv[++i];
            if (strlen(h) != 64) return usage();
            for (int b = 0; b < 32; b++) {
                unsigned v;
                if (sscanf(h + 2 * b, "%2x", &v) != 1) return usage();
                chain[b] = (uint8_t)v;
            }
            have_chain = 1;
        } else if (!strcmp(argv[i], "--device") && i + 1 < argc) {
            device = atoi(argv[++i]);
        } else if (!strcmp(argv[i], "--prune") && i + 1 < argc) {
            prune_out = argv[++i];
        } else if (!strcmp(argv[i], "--funding") && i + 1 < argc) {
            funding_path = argv[++i];
        } else if (!strcmp(argv[i], "--cut-tail")) {
            cut_tail = 1;
        } else if (argv[i][0] == '-' || path) {
            return usage();
        } else {
            path = argv[i];
        }
    }
    if (!path || (cut_tail && !prune_out)) return usage();
    if (prune_out && !strcmp(prune_out, path)) {
        fprintf(stderr, "--prune: OUT must be another file than %s\n", path);
        return 3;
    }
    funding_file ff;
    const sv_funding_table *table = NULL;
    if (funding_path) {
        if (load_funding(funding_path, &ff)) return 3;
        table = &ff.t;
    }
    FILE *f = fopen(path, "rb");
    if (!f) { fprintf(stderr, "%s: %s\n", path, strerror(errno)); return 3; }
    size_t cap = 1 << 20, len = 0, got;
    uint8_t *store = malloc(cap);
    while (store && (got = fread(store + len, 1, cap - len, f)) > 0) {
        len += got;
        if (len == cap) store = realloc(store, cap *= 2);
    }
    fclose(f);
    if (!store || len == 0) { fprintf(stderr, "%s: empty or unreadable\n", path); return 3; }
    sv_ctx *ctx = NULL;
    if (sv_create(&ctx, device) != SV_OK) { fprintf(stderr, "engine: %s\n", sv_last_error(NULL)); return 3; }
    if (prune_out) {
        int code = prune(ctx, path, store, len, have_chain ? chain : NULL, prune_out, cut_tail, table);
        sv_destroy(ctx);
        free(store);
        return code;
    }
    audit_result a;
    int rc = audit(ctx, store, len, have_chain ? chain : NULL, table, &a);
    sv_destroy(ctx);
    if (rc) return rc;

    int failing = 0;
    for (size_t i = 0; i < a.n; i++) {
        int st = a.status[i];
        int bad = (st != 0 && st < SV_GS_DELETED) || st == SV_GS_BAD_CRC || st == SV_GS_TRUNCATED || st == SV_GS_NO_AMOUNT;
        if (bad) {
            printf("record @%" PRIu64 " type %u: %d (%s)\n", a.off[i], a.type[i], st, status_name(st));
            failing += st < SV_GS_DELETED;
        }
        if (table && a.fund[i] != SV_GF_NONE && a.fund[i] != SV_GF_FUNDED)
            printf("record @%" PRIu64 " type %u: funding %s\n", a.off[i], a.type[i], funding_name[a.fund[i]]);
    }
    const sv_gossip_store_summary s = a.s;
    printf("gossip_store %s: version %u, %" PRIu64 " bytes, %" PRIu64 " records, walk stopped: %s at %" PRIu64 "\n", path,
           s.version, (uint64_t)len, s.records, s.stop ? status_name(s.stop) : "end of store", s.end_offset);
    if (s.stop == SV_GS_ENDED) printf("  gossip_store_ended: equivalent_offset %" PRIu64 "\n", s.ended_equivalent_offset);
    printf("  messages: %" PRIu64 " good, %" PRIu64 " bad signature, %" PRIu64 " malformed, %" PRIu64 " no channel, %" PRIu64
           " other chain, %" PRIu64 " node ids out of order\n",
           s.good, s.bad_signature, s.malformed, s.no_channel, s.wrong_chain, s.bad_order);
    printf("  records: %" PRIu64 " deleted, %" PRIu64 " store records, %" PRIu64 " unknown, %" PRIu64 " not reached\n",
           s.deleted, s.store_records, s.unknown, s.not_reached);
    printf("  %" PRIu64 " redundant announcements, %" PRIu64 " updates without a channel\n", s.redundant_announcements,
           s.updates_without_channel);
    const uint64_t refused = table ? print_funding(path, &a.g) : 0;
    free(store);
    audit_free(&a);
    if (s.stop == SV_GS_BAD_CRC || s.stop == SV_GS_TRUNCATED || s.stop == SV_GS_NO_AMOUNT) return 2;
    return failing || refused ? 1 : 0;
}
