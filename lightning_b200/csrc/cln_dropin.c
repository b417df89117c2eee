/*
 * cln_dropin.c — host side of the drop-in (plain C, as the reference's bitcoin/signature.c is).
 * It only marshals bytes: opaque libsecp256k1 structs -> wire form, wire messages -> (span, key,
 * signature) items, and calls the batch C ABI.  No arithmetic happens on the host.
 *
 * Client mode: with $CLN_SIGVERIFYD_SOCKET set, or after cln_sigverify_connect() / cln_sigverify_connect_fd(), the
 * functions the verifier subdaemon has a message for send a request to it instead of creating an engine context of their
 * own: the blocking functions wait for the reply, the _start variants return a ticket whose answer a later
 * cln_sigverify_process() delivers (see cln_dropin.h).
 */
#define _GNU_SOURCE
#include "../../include/cln_dropin.h"
#include "../../include/cln_sigverify.h"
#include "sigverifyd_proto.h"
#include "sigverifyd_wiregen.h"

/* weak: the library's client mode is also linked against engine builds without the fee grind (the fake engine of the
 * client-mode CPU tests); check_tx_sig_grind_fee then works through the daemon only */
#pragma weak sv_grind_tx_fee_host

#include <errno.h>
#include <poll.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/socket.h>
#include <sys/un.h>
#include <unistd.h>

#if !defined(__BYTE_ORDER__) || __BYTE_ORDER__ != __ORDER_LITTLE_ENDIAN__
#error "opaque-struct conversion below assumes a little-endian 64-bit libsecp256k1 build"
#endif

static sv_ctx *g_ctx;
static int g_device = -1;

static void die(const char *what, int rc) {
    fprintf(stderr, "cln_sigverify: %s failed (%d): %s\n", what, rc, sv_last_error(g_ctx));
    abort(); /* internal error is fatal (CLN convention); never reported as "bad signature" */
}

/* ---- client mode: one connection to cln_sigverifyd per process ----
 * Every request, blocking or a ticket, joins one queue in request order.  Its frame is written as the socket takes it
 * (never blocking outside a wait), and the daemon answers one client in request order, so each reply belongs to the
 * oldest request still without one.  A ticket's reply is decoded into the caller's output at once and its callback waits
 * at the head of the queue for cln_sigverify_process(); a blocking call's reply is handed back to that call. */
#define MAX_TICKETS 1024                 /* tickets awaiting a reply before a _start waits */
#define MAX_UNSENT ((size_t)64 << 20)    /* request bytes not yet taken by the socket before a _start waits */

struct req {
    uint64_t id;              /* req_id; a ticket's number too */
    u8 *frame;                /* be32 length + message: owned by a ticket, borrowed from a blocking call */
    size_t len, sent;
    bool ticket, replied;
    uint16_t type;            /* a ticket's request type, its item count and where its answer goes */
    uint32_t n;
    bool *ok;
    int *status;
    cln_sigverify_done done;
    void *arg;
    u8 *reply;                /* a blocking call's reply message (malloc'ed) */
    size_t reply_len;
};
/* where a check's answer goes: NULL for a blocking call, else the ticket's callback */
struct later { cln_sigverify_done done; void *arg; };

static int g_sock = -1;
static int g_env_done;
static uint64_t g_req_id;
static struct req *g_q;           /* g_q[g_h .. g_t): the requests in order; g_s: the first not fully sent, g_r: the first */
static size_t g_h, g_t, g_s, g_r, g_qcap; /* without a reply */
static size_t g_unsent;           /* bytes of g_q[g_s ..) not yet sent */
static u8 *g_in;                  /* bytes received and not yet parsed */
static size_t g_in_len, g_in_cap;

static void die_daemon(const char *what) {
    fprintf(stderr, "cln_sigverify: verifier subdaemon: %s\n", what);
    abort(); /* a lost daemon is an internal error too: never reported as "bad signature" */
}

/* forget every queued request and partial reply (a new connection, or shutdown) */
static void drop_queue(void) {
    for (size_t i = g_h; i < g_t; i++) {
        if (g_q[i].ticket) free(g_q[i].frame);
        free(g_q[i].reply);
    }
    g_h = g_t = g_s = g_r = 0;
    g_unsent = g_in_len = 0;
}

int cln_sigverify_connect(const char *socket_path) {
    struct sockaddr_un addr;
    if (!socket_path || strlen(socket_path) >= sizeof addr.sun_path) return -1;
    int fd = socket(AF_UNIX, SOCK_STREAM | SOCK_CLOEXEC, 0);
    if (fd < 0) return -1;
    memset(&addr, 0, sizeof addr);
    addr.sun_family = AF_UNIX;
    memcpy(addr.sun_path, socket_path, strlen(socket_path));
    if (connect(fd, (struct sockaddr *)&addr, sizeof addr) < 0) {
        close(fd);
        return -1;
    }
    return cln_sigverify_connect_fd(fd);
}

int cln_sigverify_connect_fd(int fd) {
    if (fd < 0) return -1;
    if (g_sock >= 0) close(g_sock);
    drop_queue();
    g_sock = fd;
    g_env_done = 1;
    return 0;
}

/* true when the checks go to the subdaemon; the first call looks at $CLN_SIGVERIFYD_SOCKET */
static bool client(void) {
    if (!g_env_done) {
        g_env_done = 1;
        const char *path = getenv("CLN_SIGVERIFYD_SOCKET");
        if (path && *path && cln_sigverify_connect(path) < 0) {
            fprintf(stderr, "cln_sigverify: cannot connect to %s: %s\n", path, strerror(errno));
            abort();
        }
    }
    return g_sock >= 0;
}

static void ticket_reply(const struct req *q, const u8 *r, size_t rl);

/* one reply message: it answers the oldest request without a reply.  A sigverifyd_error reply, or a reply with another
 * req_id, is fatal. */
static void reply_arrived(const u8 *r, size_t rl) {
    struct sigverifyd_error e;
    if (fromwire_sigverifyd_error(r, rl, &e)) {
        fprintf(stderr, "cln_sigverify: verifier subdaemon refused request %llu (code %u)\n", (unsigned long long)e.req_id, e.code);
        abort();
    }
    if (g_r == g_t) die_daemon("reply to no request");
    struct req *q = &g_q[g_r];
    if (rl < 10 || wire_be(r + 2, 8) != q->id) die_daemon("reply out of order");
    if (q->ticket) {
        ticket_reply(q, r, rl);
    } else {
        if (!(q->reply = (u8 *)malloc(rl ? rl : 1))) die("malloc", -3);
        memcpy(q->reply, r, rl);
        q->reply_len = rl;
    }
    q->replied = true;
    g_r++;
}

/* writes what the socket takes now */
static void send_some(void) {
    while (g_s < g_t) {
        struct req *q = &g_q[g_s];
        ssize_t w = send(g_sock, q->frame + q->sent, q->len - q->sent, MSG_NOSIGNAL | MSG_DONTWAIT);
        if (w < 0 && errno == EINTR) continue;
        if (w < 0 && (errno == EAGAIN || errno == EWOULDBLOCK)) return;
        if (w <= 0) die_daemon("write failed");
        q->sent += (size_t)w;
        g_unsent -= (size_t)w;
        if (q->sent == q->len) {
            if (q->ticket) free(q->frame);
            q->frame = NULL;
            g_s++;
        }
    }
}

/* writes what the socket takes and, while a request awaits its reply, reads what has arrived and hands out every
 * complete reply; never blocks */
static void io_step(void) {
    send_some();
    if (g_r == g_t) return; /* nothing awaited: a closed connection is noticed by the next request */
    for (;;) {
        if (g_in_cap - g_in_len < 65536) {
            size_t cap = g_in_cap ? 2 * g_in_cap : 131072;
            u8 *p = (u8 *)realloc(g_in, cap);
            if (!p) die("malloc", -3);
            g_in = p;
            g_in_cap = cap;
        }
        ssize_t n = recv(g_sock, g_in + g_in_len, g_in_cap - g_in_len, MSG_DONTWAIT);
        if (n > 0) { g_in_len += (size_t)n; continue; }
        if (n < 0 && errno == EINTR) continue;
        if (n < 0 && (errno == EAGAIN || errno == EWOULDBLOCK)) break;
        die_daemon(n == 0 ? "connection closed" : "read failed");
    }
    size_t off = 0;
    while (g_in_len - off >= 4) {
        size_t rl = wire_be32(g_in + off);
        if (g_in_len - off - 4 < rl) break;
        reply_arrived(g_in + off + 4, rl);
        off += 4 + rl;
    }
    memmove(g_in, g_in + off, g_in_len - off);
    g_in_len -= off;
}

/* blocks until the socket can take bytes or has bytes (for an awaited reply), then does what it can */
static void io_wait(void) {
    struct pollfd p = {g_sock, (short)((g_r < g_t ? POLLIN : 0) | (g_unsent ? POLLOUT : 0)), 0};
    while (poll(&p, 1, -1) < 0)
        if (errno != EINTR) die_daemon("poll failed");
    io_step();
}

/* appends a request of len bytes (be32 length included) to the queue; returns its index */
static size_t push_req(uint64_t id, u8 *frame, size_t len, bool ticket) {
    if (g_h == g_t) g_h = g_t = g_s = g_r = 0;
    if (g_t == g_qcap) {
        if (g_h) { /* slide the live part down */
            memmove(g_q, g_q + g_h, (g_t - g_h) * sizeof *g_q);
            g_t -= g_h; g_s -= g_h; g_r -= g_h; g_h = 0;
        } else {
            size_t cap = g_qcap ? 2 * g_qcap : 64;
            struct req *p = (struct req *)realloc(g_q, cap * sizeof *g_q);
            if (!p) die("malloc", -3);
            g_q = p;
            g_qcap = cap;
        }
    }
    struct req *q = &g_q[g_t];
    memset(q, 0, sizeof *q);
    q->id = id;
    q->frame = frame;
    q->len = len;
    q->ticket = ticket;
    g_unsent += len;
    return g_t++;
}

/* frame[4..4+len) holds a request (CLN framing: the be32 length goes in frame[0..4)); returns the reply message, which
 * the caller frees.  The request goes behind every unsent one; the replies of earlier tickets are written to their
 * outputs on the way, their callbacks left for cln_sigverify_process(). */
static u8 *roundtrip(u8 *frame, size_t len, uint64_t req_id, size_t *reply_len) {
    wire_put(frame, len, 4);
    size_t at = push_req(req_id, frame, 4 + len, false);
    send_some();
    while (!g_q[at].replied) io_wait();
    u8 *r = g_q[at].reply;
    *reply_len = g_q[at].reply_len;
    g_t = g_s = g_r = at; /* the last request: nothing joins the queue while a blocking call waits */
    return r;
}

/* queues frame[4..4+len), a request whose reply ticket_reply() decodes into ok or status (n items), and returns its
 * ticket.  Above MAX_TICKETS tickets awaiting replies or MAX_UNSENT unsent bytes it first waits for the oldest. */
static uint64_t submit(u8 *frame, size_t len, uint64_t id, uint16_t type, uint32_t n, bool *ok, int *status,
                       const struct later *lt) {
    while (g_t - g_r >= MAX_TICKETS || g_unsent >= MAX_UNSENT) io_wait();
    wire_put(frame, len, 4);
    size_t at = push_req(id, frame, 4 + len, true); /* may move g_q */
    struct req *q = &g_q[at];
    q->type = type;
    q->n = n;
    q->ok = ok;
    q->status = status;
    q->done = lt->done;
    q->arg = lt->arg;
    send_some();
    return id;
}

int cln_sigverify_fd(void) { return client() ? g_sock : -1; }

short cln_sigverify_events(void) {
    if (g_sock < 0) return 0;
    return (short)((g_h < g_t ? POLLIN : 0) | (g_unsent ? POLLOUT : 0));
}

size_t cln_sigverify_process(void) {
    if (g_sock < 0) return 0;
    io_step();
    while (g_h < g_t && g_q[g_h].replied) { /* replies arrive in request order: the answered tickets are a prefix */
        struct req q = g_q[g_h++];
        if (q.done) q.done(q.arg); /* may queue or wait for requests of its own */
    }
    return g_t - g_h;
}

void cln_sigverify_drain(void) {
    while (cln_sigverify_process()) io_wait();
}

/* the sigverifyd_verify request for m checks of one kind (its frame: 4 bytes for the length, then the message) */
static u8 *verify_request(int kind, const u8 *msg32, const u8 *key, const u8 *sig64, uint32_t m, size_t *len, uint64_t *id) {
    const size_t ks = sv_key_size(kind);
    *len = 2 + 8 + 1 + 4 + 32 * (size_t)m + 4 + ks * m + 64 * (size_t)m;
    u8 *f = (u8 *)malloc(4 + *len);
    if (!f) die("malloc", -3);
    *id = ++g_req_id;
    towire_sigverifyd_verify(f + 4, *len, *id, (uint8_t)kind, m, msg32, (uint32_t)(ks * m), key, sig64);
    return f;
}
static void verify_reply(const u8 *r, size_t rl, uint32_t m, u8 *verdicts) {
    struct sigverifyd_verify_reply v;
    if (!fromwire_sigverifyd_verify_reply(r, rl, &v) || v.n != m) die_daemon("malformed verify reply");
    memcpy(verdicts, v.verdicts, m);
}

/* n verifications of one kind through sigverifyd_verify; verdicts[n] 0/1 */
static void remote_verify(int kind, const u8 *msg32, const u8 *key, const u8 *sig64, size_t n, u8 *verdicts) {
    const size_t ks = sv_key_size(kind), chunk = 1u << 16; /* well inside the daemon's frame limit */
    for (size_t s = 0; s < n; s += chunk) {
        uint32_t m = (uint32_t)(n - s < chunk ? n - s : chunk);
        size_t len, rl;
        uint64_t id;
        u8 *f = verify_request(kind, msg32 + 32 * s, key + ks * s, sig64 + 64 * s, m, &len, &id);
        u8 *r = roundtrip(f, len, id, &rl);
        verify_reply(r, rl, m, verdicts + s);
        free(r);
        free(f);
    }
}

static sv_ctx *ctx(void) {
    if (!g_ctx) {
        int dev = g_device;
        if (dev < 0) {
            const char *e = getenv("CLN_SIGVERIFY_DEVICE");
            dev = e ? atoi(e) : 0;
        }
        int rc = sv_create(&g_ctx, dev);
        if (rc != SV_OK) {
            fprintf(stderr, "cln_sigverify: sv_create(device %d) failed (%d): %s\n", dev, rc, sv_last_error(NULL));
            abort();
        }
    }
    return g_ctx;
}

void cln_sigverify_init(int device) {
    g_device = device;
    (void)ctx();
}
void cln_sigverify_shutdown(void) {
    if (g_ctx) sv_destroy(g_ctx);
    g_ctx = NULL;
    if (g_sock >= 0) close(g_sock);
    g_sock = -1;
    drop_queue();
}

/* libsecp256k1's opaque structs hold r,s / x,y as 4x64-bit little-endian limbs on 64-bit little-endian
 * builds (secp256k1.c:337-359, group_impl.h:968-986): 32 bytes little-endian each.  Inside CLN one would
 * call secp256k1_ecdsa_signature_serialize_compact / secp256k1_ec_pubkey_serialize instead
 * (INTEGRATION.md); the engine deliberately does not link libsecp256k1. */
static void rev32(u8 *out, const unsigned char *in) {
    for (int i = 0; i < 32; i++) out[i] = in[31 - i];
}
static void sig_to_wire(u8 out[64], const secp256k1_ecdsa_signature *s) {
    rev32(out, s->data);
    rev32(out + 32, s->data + 32);
}
static void pubkey_to_xy(u8 out[64], const secp256k1_pubkey *p) {
    rev32(out, p->data);
    rev32(out + 32, p->data + 32);
}

/* one verification of this kind: through the daemon in client mode, else in process.  With lt (client mode) it is a
 * ticket: the verdict goes to *ok when the reply arrives. */
static uint64_t verify_one(int kind, const u8 *msg32, const u8 *key, const u8 *sig64, bool *ok, const struct later *lt) {
    u8 v = 0;
    if (client()) {
        if (lt) {
            size_t len;
            uint64_t id;
            u8 *f = verify_request(kind, msg32, key, sig64, 1, &len, &id);
            return submit(f, len, id, WIRE_SIGVERIFYD_VERIFY, 1, ok, NULL, lt);
        }
        remote_verify(kind, msg32, key, sig64, 1, &v);
    } else {
        int rc = sv_verify_host(ctx(), kind, msg32, key, sig64, 1, &v);
        if (rc != SV_OK) die("sv_verify_host", rc);
    }
    *ok = v == 1;
    return 0;
}

static uint64_t signed_hash(const struct sha256_double *hash, const secp256k1_ecdsa_signature *signature,
                            const struct pubkey *key, bool *ok, const struct later *lt) {
    u8 sig[64], xy[64];
    sig_to_wire(sig, signature);
    pubkey_to_xy(xy, &key->pubkey);
    return verify_one(SV_KIND_ECDSA_XY, hash->sha.u.u8, xy, sig, ok, lt);
}
bool check_signed_hash(const struct sha256_double *hash, const secp256k1_ecdsa_signature *signature,
                       const struct pubkey *key) {
    bool ok;
    signed_hash(hash, signature, key, &ok, NULL);
    return ok;
}
uint64_t check_signed_hash_start(const struct sha256_double *hash, const secp256k1_ecdsa_signature *signature,
                                 const struct pubkey *key, bool *ok, cln_sigverify_done done, void *arg) {
    const struct later lt = {done, arg};
    return signed_hash(hash, signature, key, ok, &lt);
}

static uint64_t signed_hash_nodeid(const struct sha256_double *hash, const secp256k1_ecdsa_signature *signature,
                                   const struct node_id *id, bool *ok, const struct later *lt) {
    u8 sig[64];
    sig_to_wire(sig, signature);
    return verify_one(SV_KIND_ECDSA33, hash->sha.u.u8, id->k, sig, ok, lt);
}
bool check_signed_hash_nodeid(const struct sha256_double *hash, const secp256k1_ecdsa_signature *signature,
                              const struct node_id *id) {
    bool ok;
    signed_hash_nodeid(hash, signature, id, &ok, NULL);
    return ok;
}
uint64_t check_signed_hash_nodeid_start(const struct sha256_double *hash, const secp256k1_ecdsa_signature *signature,
                                        const struct node_id *id, bool *ok, cln_sigverify_done done, void *arg) {
    const struct later lt = {done, arg};
    return signed_hash_nodeid(hash, signature, id, ok, &lt);
}

static uint64_t schnorr_sig(const struct sha256 *hash, const secp256k1_pubkey *pubkey, const struct bip340sig *sig, bool *ok,
                            const struct later *lt) {
    /* signature.c:412-423: serialize compressed, drop the parity byte -> x-only key */
    u8 xy[64];
    pubkey_to_xy(xy, pubkey);
    return verify_one(SV_KIND_SCHNORR, hash->u.u8, xy, sig->u8, ok, lt);
}
bool check_schnorr_sig(const struct sha256 *hash, const secp256k1_pubkey *pubkey, const struct bip340sig *sig) {
    bool ok;
    schnorr_sig(hash, pubkey, sig, &ok, NULL);
    return ok;
}
uint64_t check_schnorr_sig_start(const struct sha256 *hash, const secp256k1_pubkey *pubkey, const struct bip340sig *sig,
                                 bool *ok, cln_sigverify_done done, void *arg) {
    const struct later lt = {done, arg};
    return schnorr_sig(hash, pubkey, sig, ok, &lt);
}

/* one buffer through sigverifyd_sha256d; a buffer too large for one frame aborts */
static void remote_sha256d(const u8 *p, size_t len, u8 out32[32]) {
    if (len > MAX_FRAME - (2 + 8 + 4 + 4 + 4)) die_daemon("buffer too large for one request");
    size_t mlen = 2 + 8 + 4 + 4 + 4 + len, rl;
    u8 *f = (u8 *)malloc(4 + mlen);
    if (!f) die("malloc", -3);
    u8 len_be[4];
    wire_put(len_be, len, 4);
    uint64_t id = ++g_req_id;
    towire_sigverifyd_sha256d(f + 4, mlen, id, 1, len_be, (uint32_t)len, p);
    u8 *r = roundtrip(f, mlen, id, &rl);
    struct sigverifyd_sha256d_reply h;
    if (!fromwire_sigverifyd_sha256d_reply(r, rl, &h) || h.n != 1) die_daemon("malformed sha256d reply");
    memcpy(out32, h.hashes, 32);
    free(r);
    free(f);
}

/* one 33-byte key through sigverifyd_pubkey: ok and x || y as sv_pubkey_parse_host gives them */
static void remote_pubkey(const u8 *der33, u8 xy[64], u8 *ok) {
    size_t mlen = 2 + 8 + 4 + 33, rl;
    u8 f[4 + 2 + 8 + 4 + 33];
    uint64_t id = ++g_req_id;
    towire_sigverifyd_pubkey(f + 4, mlen, id, 1, der33);
    u8 *r = roundtrip(f, mlen, id, &rl);
    struct sigverifyd_pubkey_reply k;
    if (!fromwire_sigverifyd_pubkey_reply(r, rl, &k) || k.n != 1) die_daemon("malformed pubkey reply");
    *ok = k.ok[0];
    memcpy(xy, k.xy, 64);
    free(r);
}

void sha256_double(struct sha256_double *shadouble, const void *p, size_t len) {
    uint64_t off = 0;
    uint32_t l = (uint32_t)len;
    u8 dummy = 0;
    if (client()) {
        remote_sha256d(len ? (const u8 *)p : &dummy, len, shadouble->sha.u.u8);
        return;
    }
    int rc = sv_sha256d_host(ctx(), len ? (const u8 *)p : &dummy, len, &off, &l, 1, shadouble->sha.u.u8);
    if (rc != SV_OK) die("sv_sha256d_host", rc);
}

bool pubkey_from_der(const u8 *der, size_t len, struct pubkey *key) {
    if (len != 33) return false; /* PUBKEY_CMPR_LEN, bitcoin/pubkey.c:16 */
    u8 xy[64], ok = 0;
    if (client()) {
        remote_pubkey(der, xy, &ok);
    } else {
        int rc = sv_pubkey_parse_host(ctx(), der, 1, xy, &ok);
        if (rc != SV_OK) die("sv_pubkey_parse_host", rc);
    }
    if (!ok) return false;
    rev32(key->pubkey.data, xy);
    rev32(key->pubkey.data + 32, xy + 32);
    return true;
}

/* ---- check_tx_sig (bitcoin/signature.c:194-221): gate on the sighash type, BIP143 sighash on the device from the
 * wally_tx fields (every output / outpoint is handed over serialised; the host hashes nothing), then the verification ---- */
struct amount_sat { uint64_t satoshis; };                                        /* common/amount.h */
extern size_t tal_bytelen(const void *ptr) __attribute__((weak));               /* ccan/tal/tal.h */
extern struct amount_sat psbt_input_get_amount(const struct wally_psbt *psbt, size_t in) __attribute__((weak)); /* bitcoin/psbt.h */
static size_t (*g_bytelen)(const void *);
static uint64_t (*g_input_sat)(const struct bitcoin_tx *, size_t);

void cln_sigverify_set_tx_hooks(size_t (*script_bytelen)(const void *), uint64_t (*input_amount_sat)(const struct bitcoin_tx *, size_t)) {
    g_bytelen = script_bytelen;
    g_input_sat = input_amount_sat;
}

/* the byte length of a tal array (NULL: 0), through the hook or CLN's own tal_bytelen; `who` names the caller in the
 * abort when neither is there */
static size_t tal_len(const void *p, const char *who) {
    if (g_bytelen) return p ? g_bytelen(p) : 0;
    if (tal_bytelen) return p ? tal_bytelen(p) : 0;
    die(who, -4);
    return 0;
}

static size_t put_varint(u8 *p, uint64_t v) { /* Bitcoin CompactSize */
    if (v < 0xfd) { p[0] = (u8)v; return 1; }
    if (v <= 0xffff) { p[0] = 0xfd; p[1] = (u8)v; p[2] = (u8)(v >> 8); return 3; }
    p[0] = 0xfe;
    for (int i = 0; i < 4; i++) p[1 + i] = (u8)(v >> (8 * i));
    return 5;
}
static size_t put_output(u8 *p, const struct wally_tx_output *o) {
    size_t n = 0;
    for (int i = 0; i < 8; i++) p[n++] = (u8)(o->satoshi >> (8 * i));
    n += put_varint(p + n, o->script_len);
    if (o->script_len) memcpy(p + n, o->script, o->script_len);
    return n + o->script_len;
}

/* the bytes of t's spans sv_verify_tx_host reads: witness script, outputs and, for a multi-input transaction, outpoints
 * and sequences; a span outside scripts[0 .. scripts_len) aborts, as the in-process call's SV_ERR_ARG does */
static uint64_t tx_span_bytes(const sv_tx *t, size_t scripts_len) {
    const bool in = (t->flags & SV_TX_INPUTS_SERIALIZED) != 0;
    if ((uint64_t)t->script_off + t->script_len > scripts_len || (uint64_t)t->out_script_off + t->out_script_len > scripts_len ||
        (in && ((uint64_t)t->prevouts_off + t->prevouts_len > scripts_len ||
                (uint64_t)t->sequences_off + t->sequences_len > scripts_len)))
        die("sv_tx: script span out of range", SV_ERR_ARG);
    return (uint64_t)t->script_len + t->out_script_len + (in ? (uint64_t)t->prevouts_len + t->sequences_len : 0);
}

/* the sigverifyd_tx request for the m transactions txs[0..m) by one key, whose spans hold `bytes` bytes of scripts (its
 * frame: 4 bytes for the length, then the message).  Each transaction's spans are copied out of scripts back to back: the
 * daemon derives the offsets.  A request too large for one frame aborts. */
static u8 *tx_request(int kind, const u8 *key, const sv_tx *txs, const u8 *scripts, const u8 *sig64, size_t m,
                      uint64_t bytes, size_t *len, uint64_t *id) {
    const size_t ks = sv_key_size(kind), per_tx = 6 * 4 + 32 + 2 * 8 + 4 * 4 + 64;
    uint64_t mlen64 = 2 + 8 + 1 + 4 + ks + 4 + per_tx * m + 4 + bytes + 1;
    if (mlen64 > MAX_FRAME) die_daemon("transaction too large for one request");
    size_t mlen = (size_t)mlen64;
    u8 *f = (u8 *)malloc(4 + mlen), *a = (u8 *)malloc((6 * 4 + 32 + 2 * 8 + 4 * 4) * m + bytes + 1);
    if (!f || !a) die("malloc", -3);
    u8 *ver = a, *lock = ver + 4 * m, *seq = lock + 4 * m, *sht = seq + 4 * m, *pidx = sht + 4 * m, *flg = pidx + 4 * m;
    u8 *txid = flg + 4 * m, *iamt = txid + 32 * m, *oamt = iamt + 8 * m, *sl = oamt + 8 * m, *ol = sl + 4 * m;
    u8 *pl = ol + 4 * m, *ql = pl + 4 * m, *blob = ql + 4 * m;
    size_t bo = 0;
    for (size_t i = 0; i < m; i++) {
        const sv_tx *t = &txs[i];
        const bool in = (t->flags & SV_TX_INPUTS_SERIALIZED) != 0;
        const uint32_t plen = in ? t->prevouts_len : 0, qlen = in ? t->sequences_len : 0;
        wire_put(ver + 4 * i, t->version, 4);
        wire_put(lock + 4 * i, t->locktime, 4);
        wire_put(seq + 4 * i, t->sequence, 4);
        wire_put(sht + 4 * i, t->sighash_type, 4);
        wire_put(pidx + 4 * i, t->prev_index, 4);
        wire_put(flg + 4 * i, t->flags, 4);
        memcpy(txid + 32 * i, t->prev_txid, 32);
        wire_put(iamt + 8 * i, t->input_amount, 8);
        wire_put(oamt + 8 * i, t->output_amount, 8);
        wire_put(sl + 4 * i, t->script_len, 4);
        wire_put(ol + 4 * i, t->out_script_len, 4);
        wire_put(pl + 4 * i, plen, 4);
        wire_put(ql + 4 * i, qlen, 4);
        if (t->script_len) memcpy(blob + bo, scripts + t->script_off, t->script_len);
        bo += t->script_len;
        if (t->out_script_len) memcpy(blob + bo, scripts + t->out_script_off, t->out_script_len);
        bo += t->out_script_len;
        if (plen) memcpy(blob + bo, scripts + t->prevouts_off, plen);
        bo += plen;
        if (qlen) memcpy(blob + bo, scripts + t->sequences_off, qlen);
        bo += qlen;
    }
    *id = ++g_req_id;
    towire_sigverifyd_tx(f + 4, mlen, *id, (uint8_t)kind, (uint32_t)ks, key, (uint32_t)m, ver, lock, seq, sht, pidx, flg,
                         txid, iamt, oamt, sl, ol, pl, ql, (uint32_t)bytes, blob, sig64, 0);
    free(a);
    *len = mlen;
    return f;
}
static void tx_reply(const u8 *r, size_t rl, size_t m, u8 *verdicts) {
    struct sigverifyd_tx_reply x;
    if (!fromwire_sigverifyd_tx_reply(r, rl, &x) || x.n != m) die_daemon("malformed tx reply");
    memcpy(verdicts, x.verdicts, m);
}

/* n transaction checks by one key through sigverifyd_tx, in requests of at most 65536 transactions and 64 MiB of spans
 * (a single larger transaction goes alone, and aborts if it does not fit in a frame); verdicts[n] as sv_verify_tx_host
 * gives them */
static void remote_tx(int kind, const u8 *key, const sv_tx *txs, const u8 *scripts, size_t scripts_len, const u8 *sig64,
                      size_t n, u8 *verdicts) {
    size_t s = 0;
    while (s < n) {
        size_t m = 0;
        uint64_t bytes = 0;
        while (s + m < n && m < 65536) {
            uint64_t b = tx_span_bytes(&txs[s + m], scripts_len);
            if (m && bytes + b > (64u << 20)) break;
            bytes += b;
            m++;
        }
        size_t mlen, rl;
        uint64_t id;
        u8 *f = tx_request(kind, key, txs + s, scripts, sig64 + 64 * s, m, bytes, &mlen, &id);
        u8 *r = roundtrip(f, mlen, id, &rl);
        tx_reply(r, rl, m, verdicts + s);
        free(r); free(f);
        s += m;
    }
}

/* "We only support a limited subset of sighash types." (signature.c:205-211) */
static bool sighash_type_supported(const struct bitcoin_signature *sig, bool have_witness_script) {
    if (sig->sighash_type == SIGHASH_ALL) return true;
    return have_witness_script && (int)sig->sighash_type == (SIGHASH_SINGLE | SIGHASH_ANYONECANPAY);
}

/* The record and span blob (returned, *blob_len bytes; the caller frees it) sv_verify_tx_host takes for input input_num of
 * tx signed under sig's sighash type, with script as the scriptCode and the input amount from the hook or
 * psbt_input_get_amount.  Every output / outpoint is handed over serialised, so the host hashes nothing.  With one_output
 * the transaction has exactly one input and one output (`who` aborts otherwise), and the record takes the single-output
 * form (flags 0): out_script is output 0's scriptPubKey alone, its amount goes in output_amount. */
static u8 *tx_record(const struct bitcoin_tx *tx, size_t input_num, const u8 *script, const struct bitcoin_signature *sig,
                     bool one_output, const char *who, sv_tx *t, size_t *blob_len) {
    const struct wally_tx *w = tx->wtx;
    if (input_num >= w->num_inputs) { /* assert(input_num < tx->wtx->num_inputs), signature.c:212 */
        fprintf(stderr, "cln_sigverify: %s: input %zu of %zu\n", who, input_num, w->num_inputs);
        abort();
    }
    if (one_output && (w->num_inputs != 1 || w->num_outputs != 1)) {
        fprintf(stderr, "cln_sigverify: %s: %zu inputs and %zu outputs, not one of each\n", who, w->num_inputs, w->num_outputs);
        abort();
    }
    size_t script_len = tal_len(script, "check_tx_sig: no tal_bytelen (cln_sigverify_set_tx_hooks)");
    uint64_t amount = 0;
    if (g_input_sat) amount = g_input_sat(tx, input_num);
    else if (psbt_input_get_amount) amount = psbt_input_get_amount(tx->psbt, input_num).satoshis;
    else die("check_tx_sig: no psbt_input_get_amount (cln_sigverify_set_tx_hooks)", -4);

    const bool single = ((int)sig->sighash_type & 0x1f) == SIGHASH_SINGLE;
    size_t out_bytes = 0;
    for (size_t i = 0; i < w->num_outputs; i++) out_bytes += 8 + 5 + w->outputs[i].script_len;
    size_t cap = script_len + out_bytes + 40 * w->num_inputs + 16;
    u8 *blob = (u8 *)malloc(cap);
    if (!blob) die("malloc", -3);
    memset(t, 0, sizeof *t);
    size_t n = 0;
    t->version = w->version;
    t->locktime = w->locktime;
    t->sequence = w->inputs[input_num].sequence;
    t->sighash_type = (uint32_t)sig->sighash_type;
    memcpy(t->prev_txid, w->inputs[input_num].txhash, 32);
    t->prev_index = w->inputs[input_num].index;
    t->input_amount = amount;
    t->script_off = (uint32_t)n;
    t->script_len = (uint32_t)script_len;
    if (script_len) memcpy(blob + n, script, script_len);
    n += script_len;
    t->out_script_off = (uint32_t)n;
    if (one_output) { /* ALL and SINGLE of input 0 both commit to output 0 alone (tx_io.c:714-731) */
        t->output_amount = w->outputs[0].satoshi;
        if (w->outputs[0].script_len) memcpy(blob + n, w->outputs[0].script, w->outputs[0].script_len);
        n += w->outputs[0].script_len;
    } else if (single) { /* the output at the input's index, or none (tx_io.c:725-731) */
        if (input_num < w->num_outputs) { n += put_output(blob + n, &w->outputs[input_num]); t->flags |= SV_TX_OUTPUTS_SERIALIZED; }
        else t->flags |= SV_TX_OUTPUTS_ZERO;
    } else {
        for (size_t i = 0; i < w->num_outputs; i++) n += put_output(blob + n, &w->outputs[i]);
        t->flags |= SV_TX_OUTPUTS_SERIALIZED;
    }
    t->out_script_len = (uint32_t)(n - t->out_script_off);
    if (w->num_inputs > 1) {
        t->flags |= SV_TX_INPUTS_SERIALIZED;
        t->prevouts_off = (uint32_t)n;
        for (size_t i = 0; i < w->num_inputs; i++) {
            memcpy(blob + n, w->inputs[i].txhash, 32);
            for (int b = 0; b < 4; b++) blob[n + 32 + b] = (u8)(w->inputs[i].index >> (8 * b));
            n += 36;
        }
        t->prevouts_len = (uint32_t)(n - t->prevouts_off);
        t->sequences_off = (uint32_t)n;
        for (size_t i = 0; i < w->num_inputs; i++) {
            for (int b = 0; b < 4; b++) blob[n + b] = (u8)(w->inputs[i].sequence >> (8 * b));
            n += 4;
        }
        t->sequences_len = (uint32_t)(n - t->sequences_off);
    }
    *blob_len = n;
    return blob;
}

static uint64_t tx_sig(const struct bitcoin_tx *tx, size_t input_num, const u8 *redeemscript, const u8 *witness_script,
                       const struct pubkey *key, const struct bitcoin_signature *sig, bool *ok, const struct later *lt) {
    *ok = false;
    if (!sighash_type_supported(sig, witness_script != NULL)) return 0;
    sv_tx t;
    size_t n;
    u8 *blob = tx_record(tx, input_num, witness_script ? witness_script : redeemscript, sig, false, "check_tx_sig", &t, &n);
    u8 xy[64], s64[64], v = 0;
    pubkey_to_xy(xy, &key->pubkey);
    sig_to_wire(s64, &sig->s);
    if (client()) {
        uint64_t ticket = 0;
        if (lt) {
            size_t len;
            u8 *f = tx_request(SV_KIND_ECDSA_XY, xy, &t, blob, s64, 1, tx_span_bytes(&t, n), &len, &ticket);
            ticket = submit(f, len, ticket, WIRE_SIGVERIFYD_TX, 1, ok, NULL, lt);
        } else {
            remote_tx(SV_KIND_ECDSA_XY, xy, &t, blob, n, s64, 1, &v);
            *ok = v == 1;
        }
        free(blob);
        return ticket;
    }
    int rc = sv_verify_tx_host(ctx(), SV_KIND_ECDSA_XY, &t, blob, n, xy, s64, 1, &v, NULL);
    free(blob);
    if (rc != SV_OK) die("sv_verify_tx_host", rc);
    *ok = v == 1;
    return 0;
}
bool check_tx_sig(const struct bitcoin_tx *tx, size_t input_num, const u8 *redeemscript, const u8 *witness_script,
                  const struct pubkey *key, const struct bitcoin_signature *sig) {
    bool ok;
    tx_sig(tx, input_num, redeemscript, witness_script, key, sig, &ok, NULL);
    return ok;
}
uint64_t check_tx_sig_start(const struct bitcoin_tx *tx, size_t input_num, const u8 *redeemscript, const u8 *witness_script,
                            const struct pubkey *key, const struct bitcoin_signature *sig, bool *ok, cln_sigverify_done done,
                            void *arg) {
    const struct later lt = {done, arg};
    return tx_sig(tx, input_num, redeemscript, witness_script, key, sig, ok, &lt);
}

/* one fee grind through sigverifyd_fee_grind: the record's two spans travel as they are */
static int64_t remote_grind(int kind, const u8 *key, const sv_tx *t, const u8 *blob, const u8 *sig64, uint64_t weight,
                            uint32_t min_feerate, uint32_t max_feerate, uint64_t *fee) {
    const size_t ks = sv_key_size(kind);
    uint64_t mlen64 = 2 + 8 + 1 + 4 + ks + 5 * 4 + 32 + 8 + 4 + (uint64_t)t->script_len + 4 + t->out_script_len + 64 + 8 + 4 + 4;
    if (mlen64 > MAX_FRAME) die_daemon("transaction too large for one request");
    size_t mlen = (size_t)mlen64, rl;
    u8 *f = (u8 *)malloc(4 + mlen);
    if (!f) die("malloc", -3);
    uint64_t id = ++g_req_id;
    towire_sigverifyd_fee_grind(f + 4, mlen, id, (uint8_t)kind, (uint32_t)ks, key, t->version, t->locktime, t->sequence,
                                t->sighash_type, t->prev_index, t->prev_txid, t->input_amount, t->script_len,
                                blob + t->script_off, t->out_script_len, blob + t->out_script_off, sig64, weight, min_feerate,
                                max_feerate);
    u8 *r = roundtrip(f, mlen, id, &rl);
    struct sigverifyd_fee_grind_reply g;
    if (!fromwire_sigverifyd_fee_grind_reply(r, rl, &g)) die_daemon("malformed fee grind reply");
    *fee = g.fee;
    int64_t feerate = g.found ? (int64_t)g.feerate : -1;
    free(r);
    free(f);
    return feerate;
}

bool check_tx_sig_grind_fee(const struct bitcoin_tx *tx, const u8 *witness_script, const struct pubkey *key,
                            const struct bitcoin_signature *remotesig, uint64_t weight, uint32_t min_feerate,
                            uint32_t max_feerate, uint64_t *fee_sat, uint32_t *feerate) {
    if (!sighash_type_supported(remotesig, witness_script != NULL)) return false;
    sv_tx t;
    size_t n;
    u8 *blob = tx_record(tx, 0, witness_script, remotesig, true, "check_tx_sig_grind_fee", &t, &n);
    u8 xy[64], s64[64];
    pubkey_to_xy(xy, &key->pubkey);
    sig_to_wire(s64, &remotesig->s);
    int64_t f = -1;
    uint64_t fee = 0;
    if (client()) {
        f = remote_grind(SV_KIND_ECDSA_XY, xy, &t, blob, s64, weight, min_feerate, max_feerate, &fee);
    } else {
        if (!sv_grind_tx_fee_host) die("check_tx_sig_grind_fee: this engine has no sv_grind_tx_fee_host", SV_ERR_ARG);
        int rc = sv_grind_tx_fee_host(ctx(), SV_KIND_ECDSA_XY, &t, blob, n, xy, s64, weight, min_feerate, max_feerate, &f, &fee);
        if (rc != SV_OK) die("sv_grind_tx_fee_host", rc);
    }
    free(blob);
    if (f < 0) return false;
    *fee_sat = fee;
    *feerate = (uint32_t)f;
    return true;
}

/* ---- bolt12_check_signature (common/bolt12.c:80-92): the fields go back to wire form (towire_tlvstream_raw's layout:
 * BigSize type, BigSize length, value), the device does merkle_tlv, sighash_from_merkle and check_schnorr_sig ---- */
static size_t put_bigsize(u8 *p, uint64_t v) { /* common/bigsize.c bigsize_put */
    size_t n = v < 0xfd ? 1 : v <= 0xffff ? 3 : v <= 0xffffffffu ? 5 : 9;
    if (n == 1) { p[0] = (u8)v; return 1; }
    p[0] = n == 3 ? 0xfd : n == 5 ? 0xfe : 0xff;
    for (size_t i = 1; i < n; i++) p[i] = (u8)(v >> (8 * (n - 1 - i)));
    return n;
}

/* the sigverifyd_bolt12 request for one stream (its frame: 4 bytes for the length, then the message) */
static u8 *bolt12_request(const char *messagename, const char *fieldname, const u8 *stream, size_t len, const u8 *xonly32,
                          const u8 *sig64, size_t *mlen, uint64_t *id) {
    size_t mnl = strlen(messagename), fnl = strlen(fieldname);
    if (mnl > 0xffff || fnl > 0xffff || len > 0xffffffffu) die("bolt12_check_signature: tag or stream too long", -4);
    *mlen = 2 + 8 + 2 + mnl + 2 + fnl + 4 + 4 + 4 + len + 32 + 64 + 1;
    u8 *f = (u8 *)malloc(4 + *mlen);
    if (!f) die("malloc", -3);
    u8 len_be[4];
    wire_put(len_be, len, 4);
    *id = ++g_req_id;
    towire_sigverifyd_bolt12(f + 4, *mlen, *id, (uint16_t)mnl, (const u8 *)messagename, (uint16_t)fnl, (const u8 *)fieldname, 1,
                             len_be, (uint32_t)len, stream, xonly32, sig64, 0);
    return f;
}
/* the stream's status (1, 0 or -1) */
static int bolt12_reply(const u8 *r, size_t rl) {
    struct sigverifyd_bolt12_reply b;
    if (!fromwire_sigverifyd_bolt12_reply(r, rl, &b) || b.n != 1) die_daemon("malformed bolt12 reply");
    return status_from_wire(b.status[0]);
}

/* one stream through sigverifyd_bolt12: its status (1, 0 or -1) */
static int remote_bolt12(const char *messagename, const char *fieldname, const u8 *stream, size_t len, const u8 *xonly32,
                         const u8 *sig64) {
    size_t mlen, rl;
    uint64_t id;
    u8 *f = bolt12_request(messagename, fieldname, stream, len, xonly32, sig64, &mlen, &id);
    u8 *r = roundtrip(f, mlen, id, &rl);
    int st = bolt12_reply(r, rl);
    free(r);
    free(f);
    return st;
}

/* an array CLN's TLV parser can produce: not empty, types strictly ascending */
static bool fields_ascending(const struct tlv_field *fields, size_t nf) {
    for (size_t i = 1; i < nf; i++)
        if (fields[i].numtype <= fields[i - 1].numtype) return false;
    return nf > 0;
}

static uint64_t bolt12_sig(const struct tlv_field *fields, const char *messagename, const char *fieldname,
                           const struct pubkey *key, const struct bip340sig *sig, bool *ok, const struct later *lt) {
    size_t nf = tal_len(fields, "bolt12_check_signature: no tal_bytelen (cln_sigverify_set_tx_hooks)") / sizeof(struct tlv_field);
    /* a ticket's local gate: the device refuses these streams too (status -1), so the blocking call's answer is false */
    if (lt && client() && !fields_ascending(fields, nf)) {
        *ok = false;
        return 0;
    }
    size_t total = 0;
    for (size_t i = 0; i < nf; i++) total += 18 + fields[i].length;
    if (total > 0xffffffffu) die("bolt12_check_signature: stream longer than 4 GiB", -4);
    u8 *blob = (u8 *)malloc(total ? total : 1);
    if (!blob) die("malloc", -3);
    size_t n = 0;
    for (size_t i = 0; i < nf; i++) {
        n += put_bigsize(blob + n, fields[i].numtype);
        n += put_bigsize(blob + n, fields[i].length);
        if (fields[i].length) memcpy(blob + n, fields[i].value, fields[i].length);
        n += fields[i].length;
    }
    uint64_t off = 0;
    uint32_t len = (uint32_t)n;
    u8 xy[64];
    int status = 0;
    pubkey_to_xy(xy, &key->pubkey); /* x-only: the first 32 bytes */
    if (client()) {
        uint64_t ticket = 0;
        if (lt) {
            size_t mlen;
            u8 *f = bolt12_request(messagename, fieldname, blob, n, xy, sig->u8, &mlen, &ticket);
            ticket = submit(f, mlen, ticket, WIRE_SIGVERIFYD_BOLT12, 1, ok, NULL, lt);
        } else {
            *ok = remote_bolt12(messagename, fieldname, blob, n, xy, sig->u8) == 1;
        }
        free(blob);
        return ticket;
    }
    int rc = sv_verify_bolt12_host(ctx(), messagename, fieldname, blob, n, &off, &len, xy, sig->u8, 1, &status, NULL);
    free(blob);
    if (rc != SV_OK) die("sv_verify_bolt12_host", rc);
    *ok = status == 1;
    return 0;
}
bool bolt12_check_signature(const struct tlv_field *fields, const char *messagename, const char *fieldname,
                            const struct pubkey *key, const struct bip340sig *sig) {
    bool ok;
    bolt12_sig(fields, messagename, fieldname, key, sig, &ok, NULL);
    return ok;
}
uint64_t bolt12_check_signature_start(const struct tlv_field *fields, const char *messagename, const char *fieldname,
                                      const struct pubkey *key, const struct bip340sig *sig, bool *ok,
                                      cln_sigverify_done done, void *arg) {
    const struct later lt = {done, arg};
    return bolt12_sig(fields, messagename, fieldname, key, sig, ok, &lt);
}

void check_tx_sigs_batch(const struct sha256_double *hashes, const struct bitcoin_signature *sigs,
                         const struct pubkey *key, size_t n, bool *ok) {
    if (n == 0) return;
    u8 *buf = (u8 *)malloc(n * (32 + 64 + 1));
    if (!buf) die("malloc", -3);
    u8 xy[64];
    u8 *msg = buf, *sig = buf + 32 * n, *v = sig + 64 * n;
    pubkey_to_xy(xy, &key->pubkey);
    for (size_t i = 0; i < n; i++) {
        memcpy(msg + 32 * i, hashes[i].sha.u.u8, 32);
        sig_to_wire(sig + 64 * i, &sigs[i].s);
    }
    if (client()) { /* per-item keys of one kind: the daemon coalesces them with every other client's */
        u8 *keys = (u8 *)malloc(64 * n);
        if (!keys) die("malloc", -3);
        for (size_t i = 0; i < n; i++) memcpy(keys + 64 * i, xy, 64);
        remote_verify(SV_KIND_ECDSA_XY, msg, keys, sig, n, v);
        free(keys);
    } else {
        /* one key for the whole loop: its multiples table is built once on the device */
        int rc = sv_verify_samekey_host(ctx(), SV_KIND_ECDSA_XY, xy, msg, sig, n, v);
        if (rc != SV_OK) die("sv_verify_samekey_host", rc);
    }
    for (size_t i = 0; i < n; i++) ok[i] = v[i] == 1;
    free(buf);
}

void check_tx_sigs_bip143_batch(const void *sv_tx_array, const u8 *scripts, size_t scripts_len,
                                const struct pubkey *key, const struct bitcoin_signature *sigs, size_t n, bool *ok) {
    if (n == 0) return;
    sv_tx *txs = (sv_tx *)malloc(n * sizeof(sv_tx));
    u8 *buf = (u8 *)malloc(n * (64 + 64 + 1));
    if (!txs || !buf) die("malloc", -3);
    memcpy(txs, sv_tx_array, n * sizeof(sv_tx));
    u8 *xy = buf, *sig = buf + 64 * n, *v = sig + 64 * n;
    for (size_t i = 0; i < n; i++) {
        txs[i].sighash_type = (uint32_t)sigs[i].sighash_type; /* the type committed to is the signature's */
        pubkey_to_xy(xy + 64 * i, &key->pubkey);
        sig_to_wire(sig + 64 * i, &sigs[i].s);
    }
    if (client()) { /* one key for the batch: the daemon coalesces it with every other client's transactions */
        remote_tx(SV_KIND_ECDSA_XY, xy, txs, scripts, scripts_len, sig, n, v);
    } else {
        int rc = sv_verify_tx_host(ctx(), SV_KIND_ECDSA_XY, txs, scripts, scripts_len, xy, sig, n, v, NULL);
        if (rc != SV_OK) die("sv_verify_tx_host", rc);
    }
    for (size_t i = 0; i < n; i++) {
        /* check_tx_sig's gate (signature.c:206-211); a witness script is always present on this path */
        bool type_ok = sigs[i].sighash_type == SIGHASH_ALL ||
                       (int)sigs[i].sighash_type == (SIGHASH_SINGLE | SIGHASH_ANYONECANPAY);
        ok[i] = type_ok && v[i] == 1;
    }
    free(txs);
    free(buf);
}

/* gossip messages through sigverifyd_gossip, in requests of at most 65536 messages and 64 MiB */
static void remote_gossip(const u8 *blob, const uint32_t *len, size_t n, const u8 *cu_signers33, int *status) {
    size_t s = 0, bo = 0;
    while (s < n) {
        size_t m = 0, bytes = 0;
        while (s + m < n && m < 65536 && (m == 0 || bytes + len[s + m] <= (64u << 20))) bytes += len[s + m++];
        size_t mlen = 2 + 8 + 4 + 4 * m + 33 * m + 4 + bytes, rl;
        u8 *f = (u8 *)malloc(4 + mlen), *lens = (u8 *)malloc(4 * m), *sg = (u8 *)calloc(m ? m : 1, 33);
        if (!f || !lens || !sg) die("malloc", -3);
        for (size_t i = 0; i < m; i++) wire_put(lens + 4 * i, len[s + i], 4);
        if (cu_signers33) memcpy(sg, cu_signers33 + 33 * s, 33 * m);
        uint64_t id = ++g_req_id;
        towire_sigverifyd_gossip(f + 4, mlen, id, (uint32_t)m, lens, sg, (uint32_t)bytes, blob + bo);
        u8 *r = roundtrip(f, mlen, id, &rl);
        struct sigverifyd_gossip_reply g;
        if (!fromwire_sigverifyd_gossip_reply(r, rl, &g) || g.n != m) die_daemon("malformed gossip reply");
        for (size_t i = 0; i < m; i++) status[s + i] = status_from_wire(g.status[i]);
        free(r); free(f); free(lens); free(sg);
        s += m;
        bo += bytes;
    }
}

/* the n messages back to back in one blob (returned, with its length in *total), their offsets and 32-bit lengths in *off
 * and *len; the caller frees all three */
static u8 *concat_msgs(const u8 *const *msgs, const size_t *lens, size_t n, size_t *total, uint64_t **off, uint32_t **len) {
    size_t t = 0;
    for (size_t i = 0; i < n; i++) t += lens[i];
    u8 *blob = (u8 *)malloc(t ? t : 1);
    *off = (uint64_t *)malloc(n * sizeof(uint64_t));
    *len = (uint32_t *)malloc(n * sizeof(uint32_t));
    if (!blob || !*off || !*len) die("malloc", -3);
    *total = t;
    t = 0;
    for (size_t i = 0; i < n; i++) {
        (*off)[i] = t;
        (*len)[i] = (uint32_t)lens[i];
        memcpy(blob + t, msgs[i], lens[i]);
        t += lens[i];
    }
    return blob;
}

/* ---- gossip: the raw wire messages go to the device as one blob; the DEVICE slices them the way
 * gossipd/sigcheck.c does (k_gossip_slice), hashes the signed regions and verifies (sv_verify_gossip_host) ---- */
static void gossip_batch(const u8 *const *msgs, const size_t *lens, size_t n, const struct node_id *signers,
                         uint16_t want_type, int *status) {
    if (n == 0) return;
    uint64_t *off;
    uint32_t *len;
    size_t total;
    u8 *blob = concat_msgs(msgs, lens, n, &total, &off, &len);
    if (client()) {
        remote_gossip(blob, len, n, signers ? signers[0].k : NULL, status);
    } else {
        int rc = sv_verify_gossip_host(ctx(), blob, total, off, len, n, signers ? signers[0].k : NULL, status);
        if (rc != SV_OK) die("sv_verify_gossip_host", rc);
    }
    for (size_t i = 0; i < n; i++) /* this entry point is typed: a message of another kind is malformed here */
        if (lens[i] < 2 || (uint16_t)((msgs[i][0] << 8) | msgs[i][1]) != want_type) status[i] = -1;
    free(blob); free(off); free(len);
}

void sigcheck_channel_announcement_batch(const u8 *const *msgs, const size_t *lens, size_t n, int *status) {
    gossip_batch(msgs, lens, n, NULL, 256, status);
}
void sigcheck_node_announcement_batch(const u8 *const *msgs, const size_t *lens, size_t n, int *status) {
    gossip_batch(msgs, lens, n, NULL, 257, status);
}
void sigcheck_channel_update_batch(const u8 *const *msgs, const size_t *lens, const struct node_id *signers,
                                   size_t n, int *status) {
    gossip_batch(msgs, lens, n, signers, 258, status); /* struct node_id is exactly 33 bytes: signers[] is the packed array */
}

/* the ONE sigverifyd_gossip_burst request of a burst: updates resolve against the whole batch, so it is never split (its
 * frame: 4 bytes for the length, then the message) */
static u8 *burst_request(const u8 *chain_hash32, const u8 *blob, size_t bytes, const size_t *len, size_t n,
                         const u8 *signer_kind, const u8 *signers33, size_t *mlen, uint64_t *id) {
    uint64_t mlen64 = 2 + 8 + 32 + 4 + (uint64_t)n * (4 + 1 + 33) + 4 + bytes;
    if (n > MAX_ITEMS || bytes > 0xffffffffu || mlen64 > MAX_FRAME) die_daemon("gossip burst too large for one request");
    *mlen = (size_t)mlen64;
    u8 *f = (u8 *)malloc(4 + *mlen), *lens = (u8 *)malloc(4 * n + 1), *kinds = (u8 *)calloc(n + 1, 1), *sg = (u8 *)calloc(n + 1, 33);
    if (!f || !lens || !kinds || !sg) die("malloc", -3);
    for (size_t i = 0; i < n; i++) wire_put(lens + 4 * i, len[i], 4);
    if (signer_kind) memcpy(kinds, signer_kind, n);
    if (signers33) memcpy(sg, signers33, 33 * n);
    *id = ++g_req_id;
    towire_sigverifyd_gossip_burst(f + 4, *mlen, *id, chain_hash32, (uint32_t)n, lens, kinds, sg, (uint32_t)bytes, blob);
    free(lens); free(kinds); free(sg);
    return f;
}
static void burst_reply(const u8 *r, size_t rl, size_t n, int *status) {
    struct sigverifyd_gossip_burst_reply g;
    if (!fromwire_sigverifyd_gossip_burst_reply(r, rl, &g) || g.n != n) die_daemon("malformed gossip burst reply");
    for (size_t i = 0; i < n; i++) status[i] = status_from_wire(g.status[i]);
}

static void remote_gossip_burst(const u8 *chain_hash32, const u8 *blob, size_t bytes, const size_t *len, size_t n,
                                const u8 *signer_kind, const u8 *signers33, int *status) {
    size_t mlen, rl;
    uint64_t id;
    u8 *f = burst_request(chain_hash32, blob, bytes, len, n, signer_kind, signers33, &mlen, &id);
    u8 *r = roundtrip(f, mlen, id, &rl);
    burst_reply(r, rl, n, status);
    free(r); free(f);
}

static uint64_t gossip_burst(const u8 *chain_hash32, const u8 *const *msgs, const size_t *lens, size_t n,
                             const u8 *signer_kind, const struct node_id *signers, int *status, const struct later *lt) {
    if (n == 0) return 0;
    uint64_t *off, ticket = 0;
    uint32_t *len;
    size_t total;
    u8 *blob = concat_msgs(msgs, lens, n, &total, &off, &len);
    if (client()) {
        if (lt) {
            size_t mlen;
            u8 *f = burst_request(chain_hash32, blob, total, lens, n, signer_kind, signers ? signers[0].k : NULL, &mlen, &ticket);
            ticket = submit(f, mlen, ticket, WIRE_SIGVERIFYD_GOSSIP_BURST, (uint32_t)n, NULL, status, lt);
        } else {
            remote_gossip_burst(chain_hash32, blob, total, lens, n, signer_kind, signers ? signers[0].k : NULL, status);
        }
    } else {
        int rc = sv_verify_gossip_burst_host(ctx(), chain_hash32, blob, total, off, len, n, signer_kind,
                                             signers ? signers[0].k : NULL, status);
        if (rc != SV_OK) die("sv_verify_gossip_burst_host", rc);
    }
    free(blob); free(off); free(len);
    return ticket;
}
void sigcheck_gossip_batch(const u8 *chain_hash32, const u8 *const *msgs, const size_t *lens, size_t n, const u8 *signer_kind,
                           const struct node_id *signers, int *status) {
    gossip_burst(chain_hash32, msgs, lens, n, signer_kind, signers, status, NULL);
}
uint64_t sigcheck_gossip_batch_start(const u8 *chain_hash32, const u8 *const *msgs, const size_t *lens, size_t n,
                                     const u8 *signer_kind, const struct node_id *signers, int *status,
                                     cln_sigverify_done done, void *arg) {
    const struct later lt = {done, arg};
    return gossip_burst(chain_hash32, msgs, lens, n, signer_kind, signers, status, &lt);
}

/* a ticket's reply through the blocking call's decoding, its answer written where the ticket said */
static void ticket_reply(const struct req *q, const u8 *r, size_t rl) {
    u8 v = 0;
    switch (q->type) {
    case WIRE_SIGVERIFYD_VERIFY: verify_reply(r, rl, 1, &v); *q->ok = v == 1; break;
    case WIRE_SIGVERIFYD_TX: tx_reply(r, rl, 1, &v); *q->ok = v == 1; break;
    case WIRE_SIGVERIFYD_BOLT12: *q->ok = bolt12_reply(r, rl) == 1; break;
    case WIRE_SIGVERIFYD_GOSSIP_BURST: burst_reply(r, rl, q->n, q->status); break;
    }
}
