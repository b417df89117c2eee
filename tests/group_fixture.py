"""Signatures built to reach every reachable exceptional addition of every verification schedule (tests/group_schedule.py
says which ones exist and why the others do not), and the committed fixture made of them.

ECDSA: the signer controls u1, u2 and the key d, so each case picks (d, u1, u2) to meet its condition and signs with
adversarial.craft (exact=True keeps the scalars from being negated for low S; an addition that ends at infinity is signed
with an arbitrary r and so is invalid).  BIP-340: u2 = -e is a hash the signer cannot steer, but u1 = s is free and e does
not depend on s, so the conditions tying u1 to u2*d are met by choosing s after e.

Regenerate with `python -m tests.group_fixture` (deterministic; pure-Python curve arithmetic, about a minute)."""
import hashlib
import os

import numpy as np

from tests import adversarial as A
from tests import ecc
from tests import group_schedule as S

N = S.N
FIXTURE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "group_exceptional.npz")


def _h(*a):
    return int.from_bytes(hashlib.sha256(b"group/" + b"/".join(str(v).encode() for v in a)).digest(), "big")


def _row_target(u1, row, sign):
    """the residue u2*d must have so that the comb addition of `row` doubles (sign +1) or cancels (sign -1)"""
    gd = S.prepare_u1(u1)
    partial = sum(g * 2**(16 * i) for i, g in enumerate(gd[:row]))
    return (sign * gd[row] * 2**(16 * row) - partial) % N


def ecdsa_cases():
    """[(label, d, u1, u2, r_if_infinity)] before signing"""
    out = []
    w = S.window_candidates(0)
    for i in range(4):
        for u2, step, br in w:
            out.append((f"{step}.{br}", _h("wd", i) % N, _h("wu1", i) % N, u2, None))
    for i, u2 in enumerate(S.join1_candidates(limit=4)):
        out.append(("join1.double", _h("j1d", i) % N, _h("j1u1", i) % N, u2, None))
    for i in range(6):
        u1 = _h("cu1", i) % N
        gd = S.prepare_u1(u1)
        rows = [j for j, g in enumerate(gd) if g]
        for row in (rows[0], rows[len(rows) // 2], rows[-2], rows[-1]):
            for sign, br in ((1, "double"), (-1, "infinity")):
                out.append((f"comb.row{row}.{br}", None, u1, (_h("cu2", i, row, sign) % N) or 1,
                            (sign, row, _h("cr", i, row) % N)))
    for i in range(4):
        u2, d = _h("j2u2", i) % N, _h("j2d", i) % N
        out.append(("join2.double", d, u2 * d % N, u2, None))
        out.append(("join2.infinity", d, -u2 * d % N, u2, _h("j2r", i) % N))
        out.append(("join2.b_inf", d, 0, u2, None))
    # the r + n candidate (r < p - n) sends the compressed-key flows without the square root to the plain path
    for i in range(3):
        out.append(("r_plus_n", _h("rnd", i) % N, _h("rnu1", i) % N, _h("rnu2", i) % N, ("r", _h("rnr", i) % 2**120 + 1)))
    return out


def sign_ecdsa(label, d, u1, u2, extra):
    """one case -> (msg32, pub33, pubxy, sig64) or None when the low-S rule would negate the scalars"""
    r_inf = None
    if isinstance(extra, tuple) and extra[0] == "r":
        # an arbitrary small r: R's x is not r, so the signature is invalid, but the r + n flag is set
        Q = A.mul(d, A.G)
        r = extra[1]
        s = r * pow(u2, -1, N) % N
        if s > N // 2:
            return None
        m = u1 * s % N
        b = lambda v: np.frombuffer(v.to_bytes(32, "big"), dtype=np.uint8)
        return b(m).copy(), np.concatenate([np.array([2 + (Q[1] & 1)], np.uint8), b(Q[0])]), \
            np.concatenate([b(Q[0]), b(Q[1])]), np.concatenate([b(r), b(s)])
    if isinstance(extra, tuple):
        sign, row, r_inf = extra
        d = _row_target(u1, row, sign) * pow(u2, -1, N) % N
        if not d:
            return None
    elif extra is not None:
        r_inf = extra
    return A.craft(d, u1, u2, exact=True, r_if_infinity=r_inf)


def bip340_cases():
    """[(label, msg32, xonly32, sig64, d)]: d is the even-y secret key of the x-only key"""
    out = []
    for i in range(40):
        d0 = _h("bd", i) % N
        x, y = ecc.base_mult(d0)
        d = d0 if y % 2 == 0 else N - d0
        r = ecc.base_mult(_h("br", i) % N)[0]
        m = hashlib.sha256(b"group/bip340/%d" % i).digest()
        px = x.to_bytes(32, "big")
        e = int.from_bytes(ecc.tagged_hash("BIP0340/challenge", r.to_bytes(32, "big") + px + m), "big") % N
        T = (N - e) * d % N  # u2*d
        kind = i % 5
        if kind == 0:
            label, s = "join2.double", T
        elif kind == 1:
            label, s = "join2.infinity", (N - T) % N
        elif kind == 2:
            label, s = "join2.b_inf", 0
        else:
            # comb: the top row doubles when s - g*2^240 == g*2^240 - T with a small prefix below it
            g = (T + 2**239) >> 240
            s = (2 * g * 2**240 - T) % N
            label = "comb.row15.double"
            if kind == 4:
                label, s = "comb.infinity", (N - T) % N
        out.append((label, m, px, r.to_bytes(32, "big") + s.to_bytes(32, "big"), d))
    return out


def generate():
    rows = []
    for label, d, u1, u2, extra in ecdsa_cases():
        c = sign_ecdsa(label, d, u1, u2, extra)
        if c is not None:
            rows.append((label,) + c)
    b = bip340_cases()
    return dict(
        ecdsa_label=np.array([r[0] for r in rows]), ecdsa_msg=np.stack([r[1] for r in rows]),
        ecdsa_pub33=np.stack([r[2] for r in rows]), ecdsa_pubxy=np.stack([r[3] for r in rows]),
        ecdsa_sig=np.stack([r[4] for r in rows]),
        bip340_label=np.array([c[0] for c in b]),
        bip340_msg=np.stack([np.frombuffer(c[1], np.uint8) for c in b]),
        bip340_xonly=np.stack([np.frombuffer(c[2], np.uint8) for c in b]),
        bip340_sig=np.stack([np.frombuffer(c[3], np.uint8) for c in b]),
        bip340_d=np.stack([np.frombuffer(c[4].to_bytes(32, "big"), np.uint8) for c in b]))


def load():
    z = np.load(FIXTURE)
    return {k: z[k] for k in z.files}


def _int(b):
    return int.from_bytes(bytes(b), "big")


def ecdsa_scalars(msg, sig, pubxy, known_d):
    """(u1, u2, d, r_plus_n) of one ECDSA item; d looked up by the key's point among the known secret keys"""
    r, s, m = _int(sig[:32]), _int(sig[32:]), _int(msg) % N
    si = pow(s, -1, N)
    return m * si % N, r * si % N, known_d[(_int(pubxy[:32]), _int(pubxy[32:]))], r < S.P - N


def bip340_scalars(msg, xonly, sig, d):
    r, s = sig[:32], _int(sig[32:])
    e = int.from_bytes(ecc.tagged_hash("BIP0340/challenge", bytes(r) + bytes(xonly) + bytes(msg)), "big") % N
    return s, (N - e) % N, d


def ecdsa_keys(fx):
    """x coordinate -> d for every key of the fixture, recovered from the generator's deterministic choices"""
    out = {}
    for label, d, u1, u2, extra in ecdsa_cases():
        if isinstance(extra, tuple) and extra[0] != "r":
            sign, row, _ = extra
            d = _row_target(u1, row, sign) * pow(u2, -1, N) % N
        if d:
            out[ecc.base_mult(d)] = d
    return out


def reference_verdicts(fx):
    """the reference's verdicts (oracle/_ref) per kind, stored with the fixture for the GPU tests"""
    from tests import util
    ref = util.load_ref()
    return {f"ref_verdict_{kind}": util.ref_verify(ref, kind, msg, key, sig)
            for kind, msg, key, sig in ((0, fx["ecdsa_msg"], fx["ecdsa_pub33"], fx["ecdsa_sig"]),
                                        (1, fx["ecdsa_msg"], fx["ecdsa_pubxy"], fx["ecdsa_sig"]),
                                        (2, fx["bip340_msg"], fx["bip340_xonly"], fx["bip340_sig"]))}


if __name__ == "__main__":
    fx = generate()
    fx.update(reference_verdicts(fx))
    np.savez_compressed(FIXTURE, **fx)
    print("wrote", FIXTURE, len(fx["ecdsa_label"]), "ECDSA and", len(fx["bip340_label"]), "BIP-340 cases")
