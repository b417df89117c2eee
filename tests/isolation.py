"""Special items of every kind, and batch layouts that put each one at every offset of every batched stage.

Many stages of a verification share work between neighbouring items: one inversion mod n for 32 signatures (k_prep_inv),
one field inversion for 16 items (the final kernels), lane pairs and warps of the small-batch kernel, CTA barriers of the
throughput kernel, one group equation per 1024 BIP-340 signatures, one multiples table per distinct key.  An item that
takes a special path there (a parse failure, a key that does not decode, an exceptional addition handed to the plain
path) must not change the verdict of any other item of its unit.  The catalogue below lists such items per kind, each
with a verdict from a committed golden file or known by construction; the layouts place them among backgrounds of known
verdicts, so that a test can compare the whole verdict vector.

  block layout   `blocks` blocks of `size` items, block b holds the special at offset b: with 64 x 64 one batch puts it at
                 every offset of a 16- and a 32-item unit, of a small-batch CTA, both lanes of a pair and all 8 warps of a
                 256-thread CTA, in 4,096 items (at or below the default small_max)
  ragged tail    n = 4096 + r with the special as the last item, in a partial unit
  pairs          two specials of different classes in one 16-item unit, a seeded sample of offset pairs
  full units     a 32-item unit made entirely of one special

Backgrounds: all valid, or about 25 % rejected by a flipped message bit, so that valid and rejected items share every
batched product.  The GPU tests take theirs from the device generator, the host-build tests sign them with tests/ecc.py."""
import functools
import hashlib
import json
import os

import numpy as np

from tests import ecc
from tests import group_fixture as F
from tests import group_schedule as S

N, P = ecc.N, ecc.P
KEYLEN = {0: 33, 1: 64, 2: 32}
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

# how a special leaves the common path:
#   parse   rejected by the range checks of the signature or key bytes before any curve work (not pending in the final
#           kernels, "unusable" in k_final_schnorr)
#   key     a key in range that does not decode (off the curve)
#   exact   handed to the plain path by the flows without the square root (group_schedule.ns_trigger)
#   group   another exceptional addition of the constructed fixture
#   valid / invalid   everything else
CLASSES = ("parse", "key", "exact", "group", "valid", "invalid")


class Special:
    def __init__(self, label, kind, msg, key, sig, want, cls, d=None, sb_encoding=True):
        self.label, self.kind, self.cls, self.want = label, kind, cls, int(want)
        arr = lambda v, n: np.frombuffer(bytes(v), np.uint8).reshape(n).copy()
        self.msg, self.key, self.sig = arr(msg, 32), arr(key, KEYLEN[kind]), arr(sig, 64)
        self.d = d                    # secret key of the key, when known (ECDSA): the shared-key backgrounds are signed with it
        self.sb_encoding = sb_encoding  # BIP-340: the encoding check of batch verification passes

    def __repr__(self):
        return f"<{self.label} kind {self.kind} want {self.want} {self.cls}>"


def _h(*a):
    return int.from_bytes(hashlib.sha256(b"isolation/" + b"/".join(str(v).encode() for v in a)).digest(), "big")


def _b32(v):
    return np.frombuffer(int(v).to_bytes(32, "big"), np.uint8)


def _int(b):
    return int.from_bytes(bytes(b), "big")


def _is_x(x):
    """x < p is the x coordinate of a curve point"""
    return x < P and pow((x * x * x + 7) % P, (P - 1) // 2, P) in (0, 1)


def _off_curve_x(seed):
    x = _h("offx", seed) % P
    while _is_x(x):
        x += 1
    return x


BASE_D = _h("base-d") % N
BASE_MSG = hashlib.sha256(b"isolation/base-msg").digest()


def _ecdsa_base():
    pub33, xy = ecc.pubkey_create(BASE_D.to_bytes(32, "big"))
    return np.frombuffer(pub33, np.uint8), np.frombuffer(xy, np.uint8), np.frombuffer(ecc.ecdsa_sign(
        BASE_D.to_bytes(32, "big"), BASE_MSG), np.uint8)


def _with(sig, r=None, s=None):
    out = np.array(sig, np.uint8)
    if r is not None:
        out[:32] = _b32(r)
    if s is not None:
        out[32:] = _b32(s)
    return out


@functools.lru_cache(maxsize=None)
def ecdsa_catalogue(kind):
    """the ECDSA specials of `kind` (0: 33-byte keys, 1: 64-byte keys)"""
    assert kind in (0, 1)
    msg = np.frombuffer(BASE_MSG, np.uint8)
    pub33, xy, sig = _ecdsa_base()
    key = pub33 if kind == 0 else xy
    s0 = _int(sig[32:])
    out = []
    # signature encodings the parse refuses: the prep kernel multiplies 1 in their place
    for label, r, s in (("r=0", 0, None), ("s=0", None, 0), ("r=n", N, None), ("s=n", None, N),
                        ("r=s=2^256-1", 2**256 - 1, 2**256 - 1)):
        out.append(Special("sig." + label, kind, msg, key, _with(sig, r, s), 0, "parse", BASE_D))
    out.append(Special("sig.high_s", kind, msg, key, _with(sig, s=N - s0), 0, "parse", BASE_D))
    # keys that do not decode.  x = 0 is off the curve (7 is not a square mod p); the square root the decoder tries
    # instead lifts it to a point of order 3 on another curve of the form y^2 = x^3 + b, whose multiples reach a zero Z
    x0, y0 = _int(xy[:32]), _int(xy[32:])
    xo = _off_curve_x(kind)
    if kind == 0:
        pre = lambda b, rest: np.concatenate([[b], rest]).astype(np.uint8)
        for label, k, cls in (("key.prefix00", pre(0, pub33[1:]), "parse"), ("key.prefix04", pre(4, pub33[1:]), "parse"),
                              ("key.x>=p", pre(2, np.full(32, 0xFF)), "parse"), ("key.x_off_curve", pre(2, _b32(xo)), "key"),
                              ("key.x=0", pre(2, _b32(0)), "key")):
            out.append(Special(label, kind, msg, k, sig, 0, cls))
    else:
        for label, k, cls in (("key.x>=p", np.concatenate([np.full(32, 0xFF, np.uint8), _b32(y0)]), "parse"),
                              ("key.x_off_curve", np.concatenate([_b32(xo), _b32(y0)]), "key"),
                              ("key.y_off_curve", np.concatenate([_b32(x0), _b32((y0 + 1) % P)]), "key"),
                              ("key.x=0", np.concatenate([_b32(0), _b32(y0)]), "key")):
            out.append(Special(label, kind, msg, k, sig, 0, cls))
    # the constructed exceptional additions, with the reference's verdicts stored beside them
    fx = F.load()
    known = F.ecdsa_keys(fx)
    for i, label in enumerate(fx["ecdsa_label"]):
        m, s, pxy = fx["ecdsa_msg"][i], fx["ecdsa_sig"][i], fx["ecdsa_pubxy"][i]
        u1, u2, d, rpn = F.ecdsa_scalars(m, s, pxy, known)
        trig = S.ns_trigger(u1, u2, d, rpn and kind == 0)
        k = fx["ecdsa_pub33"][i] if kind == 0 else pxy
        out.append(Special(f"group.{label}#{i}", kind, m, k, s, fx[f"ref_verdict_{kind}"][i], "exact" if trig else "group", d))
    # a sample of the adversarial fixture (all valid): scalars that steer the ladder and the comb into rare branches
    from tests.test_group_emul import adversarial_items
    for i, (k_, m, k, s, u1, u2, d, rpn) in enumerate(adversarial_items(every=211)):
        if k_ == kind:
            cls = "exact" if S.ns_trigger(u1, u2, d, rpn) else "valid"
            out.append(Special(f"adversarial#{211 * (i // 2)}", kind, m, k, s, 1, cls, d))
    # the reference's ECDSA edge cases whose r has the second candidate r + n (and the ones around them)
    for i, c in enumerate(json.load(open(os.path.join(GOLDEN, "ecdsa_edge_cases.json")))):
        s = np.frombuffer(bytes.fromhex(c["sig64"]), np.uint8)
        r = _int(s[:32])
        if not 0 < r < P - N:
            continue
        conv = ecc.pubkey_convert(bytes.fromhex(c["pub33"]))
        k = np.frombuffer(conv[0] if kind == 0 else conv[1], np.uint8)
        cls = "exact" if kind == 0 and 0 < _int(s[32:]) <= N // 2 else ("valid" if c["expected"] else "invalid")
        d = 1 if c["pub33"] == "02" + "%064x" % ecc.GX else None
        out.append(Special(f"edge.{c['name']}", kind, bytes.fromhex(c["msg32"]), k, s, c["expected"], cls, d))
    return tuple(out)


def _bip340_encoding(key, sig):
    """the encoding check of BIP-340 batch verification (batch.cuh sb_prepare): r, px < p, s < n, both lift"""
    r, s, px = _int(sig[:32]), _int(sig[32:]), _int(key)
    return r < P and s < N and px < P and _is_x(r) and _is_x(px)


@functools.lru_cache(maxsize=None)
def bip340_catalogue():
    sk = BASE_D.to_bytes(32, "big")
    sig, x = ecc.schnorr_sign(sk, BASE_MSG)
    msg, sig, x = np.frombuffer(BASE_MSG, np.uint8), np.frombuffer(sig, np.uint8), np.frombuffer(x, np.uint8)
    raw = [("sig.r>=p", msg, x, _with(sig, r=2**256 - 1), 0, "parse"),
           ("sig.s>=n", msg, x, _with(sig, s=N), 0, "parse"),
           ("sig.s=0", msg, x, _with(sig, s=0), 0, "exact"),  # u1 = 0: the comb sum is at infinity
           ("key.x>=p", msg, np.full(32, 0xFF, np.uint8), sig, 0, "parse"),
           ("key.x_off_curve", msg, _b32(_off_curve_x(2)), sig, 0, "key"),
           ("key.x=0", msg, _b32(0), sig, 0, "key")]  # lifts to a point of order 3: its R parks a zero Z
    fx = F.load()
    for i, label in enumerate(fx["bip340_label"]):
        m, k, s = fx["bip340_msg"][i], fx["bip340_xonly"][i], fx["bip340_sig"][i]
        u1, u2, d = F.bip340_scalars(m, k, s, F._int(fx["bip340_d"][i]))
        cls = "exact" if S.ns_trigger(u1, u2, d) else "group"
        raw.append((f"group.{label}#{i}", m, k, s, fx["ref_verdict_2"][i], cls))
    for c in json.load(open(os.path.join(GOLDEN, "bip340.json"))):
        s = np.frombuffer(bytes.fromhex(c["sig64"]), np.uint8)
        k = np.frombuffer(bytes.fromhex(c["xonly"]), np.uint8)
        raw.append((f"bip340.json[{c['index']}]", np.frombuffer(bytes.fromhex(c["msg32"]), np.uint8), k, s, c["expected"],
                    "valid" if c["expected"] else "invalid"))
    return tuple(Special(label, 2, m, k, s, w, cls, sb_encoding=_bip340_encoding(k, s)) for label, m, k, s, w, cls in raw)


def catalogue(kind):
    return ecdsa_catalogue(kind) if kind != 2 else bip340_catalogue()


# ---- backgrounds ---------------------------------------------------------------------------------------------------------
def flipped(n, seed):
    """seeded positions (about 25 %) whose message gets a flipped bit"""
    return np.random.default_rng(seed).random(n) < 0.25


def with_flips(bg, seed):
    """a background (msg, key, sig, want) with about 25 % of its messages flipped: those verdicts become 0"""
    msg, key, sig, want = (a.copy() for a in bg)
    f = flipped(msg.shape[0], seed)
    msg[f, 9] ^= 0x20
    want[f] = 0
    return msg, key, sig, want


@functools.lru_cache(maxsize=None)
def _signed(kind, d, distinct):
    """`distinct` messages signed with secret key d (tests/ecc.py): (msg, key, sig), read-only arrays"""
    sk = d.to_bytes(32, "big")
    msgs = [hashlib.sha256(b"isolation/bg/%d/%d" % (d % 2**64, j)).digest() for j in range(distinct)]
    if kind == 2:
        pairs = [ecc.schnorr_sign(sk, m) for m in msgs]
        sig, key = [p[0] for p in pairs], [p[1] for p in pairs]
    else:
        pub33, xy = ecc.pubkey_create(sk)
        key = [pub33 if kind == 0 else xy] * distinct
        sig = [ecc.ecdsa_sign(sk, m) for m in msgs]
    out = tuple(np.frombuffer(b"".join(v), np.uint8).reshape(distinct, -1) for v in (msgs, key, sig))
    for a in out:
        a.flags.writeable = False
    return out


def host_background(kind, n, distinct=128, keys=8):
    """n valid items signed by `keys` keys with tests/ecc.py, `distinct` different items tiled (every 32-item unit holds 32
    different ones): (msg, key, sig, want)"""
    parts = [_signed(kind, _h("bg-key", kind, j) % N, distinct // keys) for j in range(keys)]
    msg, key, sig = (np.concatenate([p[i] for p in parts]) for i in range(3))
    reps = -(-n // distinct)
    tile = lambda a: np.ascontiguousarray(np.tile(a, (reps, 1))[:n])
    return tile(msg), tile(key), tile(sig), np.ones(n, np.uint8)


def samekey_background(kind, d, n, distinct=16):
    """n valid items all signed with d, `distinct` messages tiled"""
    msg, key, sig = _signed(kind, d, distinct)
    reps = -(-n // distinct)
    tile = lambda a: np.ascontiguousarray(np.tile(a, (reps, 1))[:n])
    return tile(msg), tile(key), tile(sig), np.ones(n, np.uint8)


# ---- layouts -------------------------------------------------------------------------------------------------------------
def block_positions(blocks=64, size=64):
    """block b holds its special at offset b"""
    return np.arange(blocks) * size + np.arange(blocks)


def place(bg, n, placed):
    """a batch of the first n background items with specials put in: placed = {position: Special}.  Returns (msg, key,
    sig, want)."""
    msg, key, sig, want = (np.ascontiguousarray(a[:n]).copy() for a in bg)
    for pos, sp in placed.items():
        msg[pos], key[pos], sig[pos], want[pos] = sp.msg, sp.key, sp.sig, sp.want
    return msg, key, sig, want


def block_layout(bg, sp, blocks=64, size=64):
    pos = block_positions(blocks, size)
    return place(bg, blocks * size, {int(p): sp for p in pos})


def pair_layout(specials, n, seed, unit=16):
    """{position: Special}: in every `unit`-item unit of n items two specials of different classes at two different
    offsets, drawn with a seeded generator"""
    rng = np.random.default_rng(seed)
    placed = {}
    for u in range(n // unit):
        a = specials[int(rng.integers(len(specials)))]
        others = [s for s in specials if s.cls != a.cls]
        b = others[int(rng.integers(len(others)))]
        oa, ob = (int(v) for v in rng.choice(unit, size=2, replace=False))
        placed[u * unit + oa], placed[u * unit + ob] = a, b
    return placed


def full_unit_layout(specials, unit=32):
    """(n, {position: Special}): special k fills the whole unit 2k + 1, background units between them"""
    placed = {}
    for k, sp in enumerate(specials):
        for j in range(unit):
            placed[(2 * k + 1) * unit + j] = sp
    return (2 * len(specials) + 1) * unit, placed


def mismatch(got, want, placed, unit=64):
    """None when got == want, else one line per unit with a difference: the special(s) of that unit with their offsets,
    whether a special's own verdict is wrong, and every neighbour offset whose verdict changed"""
    got, want = np.asarray(got), np.asarray(want)
    bad = np.nonzero(got != want)[0]
    if not bad.size:
        return None
    lines = []
    for u in np.unique(bad // unit):
        lo = int(u) * unit
        here = {p - lo: sp.label for p, sp in placed.items() if lo <= p < lo + unit}
        own = sorted(int(i - lo) for i in bad if lo <= i < lo + unit and int(i - lo) in here)
        nb = sorted(int(i - lo) for i in bad if lo <= i < lo + unit and int(i - lo) not in here)
        lines.append(f"unit {u} (items {lo}..{lo + unit - 1}): specials {here}; own verdict wrong at {own}; "
                     f"neighbour verdicts changed at {nb}")
        if len(lines) >= 12:
            lines.append(f"... {bad.size} differing items in all")
            break
    return "\n".join(lines)


class Coverage:
    """(route, kind, label) -> offsets within the block at which the special was verified"""

    def __init__(self):
        self.seen = {}

    def add(self, route, sp, positions, size=64):
        self.seen.setdefault((route, sp.kind, sp.label), set()).update(int(p) % size for p in positions)

    def missing(self, routes_of_kind, specials_of_kind, offsets):
        """entries of the catalogue not placed at every offset on every route of their kind"""
        out = []
        for kind, routes in routes_of_kind.items():
            for route in routes:
                for sp in specials_of_kind[kind]:
                    got = self.seen.get((route, kind, sp.label), set())
                    if got != set(offsets):
                        out.append((route, kind, sp.label, len(got)))
        return out
