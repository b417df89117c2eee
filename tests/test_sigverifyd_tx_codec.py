"""CPU: the verifier subdaemon's transaction messages (sigverifyd_tx / sigverifyd_tx_reply).  The generated C codec
(lightning_b200/csrc/sigverifyd_wiregen.h, through tests/host_emul/wire_shim_tx.c) and the generated Python codec
(lightning_b200/sigverifyd_wire.py) must agree byte for byte in both directions, and both must refuse truncated and
over-long frames, counts that do not match the bytes that follow, and the wrong message type."""
import ctypes
import os
import struct
import subprocess

import numpy as np
import pytest

from lightning_b200 import sigverifyd_wire as W

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RID = 0x0102030405060708
U32_ARRAYS = ["version", "locktime", "sequence", "sighash_type", "prev_index", "flags"]
LEN_ARRAYS = ["script_len", "outputs_len", "prevouts_len", "sequences_len"]
# the per-transaction arrays in wire order, with their element size
ARRAYS = [(f, 4) for f in U32_ARRAYS] + [("prev_txid", 32), ("input_amount", 8), ("output_amount", 8)] + \
         [(f, 4) for f in LEN_ARRAYS]


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("wire") / "libwireshim_tx.so")
    subprocess.check_call(["gcc", "-O2", "-shared", "-fPIC", "-Wall", "-Wextra", "-Werror", "-o", so,
                           os.path.join(ROOT, "tests", "host_emul", "wire_shim_tx.c")])
    lib = ctypes.CDLL(so)
    lib.shim_towire_tx.restype = ctypes.c_size_t
    lib.shim_towire_tx.argtypes = [ctypes.c_char_p, ctypes.c_size_t, ctypes.c_uint64, ctypes.c_uint8, ctypes.c_uint32,
                                   ctypes.c_char_p, ctypes.c_uint32, ctypes.POINTER(ctypes.c_char_p), ctypes.c_uint32,
                                   ctypes.c_char_p, ctypes.c_uint8]
    lib.shim_towire_tx_reply.restype = ctypes.c_size_t
    lib.shim_towire_tx_reply.argtypes = [ctypes.c_char_p, ctypes.c_size_t, ctypes.c_uint64, ctypes.c_uint32, ctypes.c_char_p,
                                         ctypes.c_uint32, ctypes.c_char_p]
    for f in (lib.shim_fromwire_tx, lib.shim_fromwire_tx_reply):
        f.argtypes = [ctypes.c_char_p, ctypes.c_size_t, ctypes.POINTER(ctypes.c_uint64), ctypes.c_void_p, ctypes.c_void_p]
    return lib


def _be(vals, size):
    return b"".join(int(v).to_bytes(size, "big") for v in vals)


def _request(rng, n, kind, want):
    """a request of n transactions with random field values (the codec does not care what they mean)"""
    ks = 33 if kind == 0 else 64
    req = dict(req_id=RID, kind=kind, keylen=ks, key=rng.integers(0, 256, size=ks, dtype=np.uint8).tobytes(), n=n)
    for f in U32_ARRAYS:
        req[f] = [int(x) for x in rng.integers(0, 2**32, size=n, dtype=np.uint64)]
    req["prev_txid"] = rng.integers(0, 256, size=32 * n, dtype=np.uint8).tobytes()
    for f in ("input_amount", "output_amount"):
        req[f] = [int(x) for x in rng.integers(0, 2**63, size=n, dtype=np.uint64)] if n else []
    for f in LEN_ARRAYS:
        req[f] = [int(x) for x in rng.integers(0, 300, size=n)]
    if n:
        req["script_len"][0] = 70_000  # one long span
    total = sum(sum(req[f]) for f in LEN_ARRAYS)
    req.update(bloblen=total, blob=rng.integers(0, 256, size=total, dtype=np.uint8).tobytes(),
               sigs=rng.integers(0, 256, size=64 * n, dtype=np.uint8).tobytes(), want_sighash=want)
    return req


def _wire_view(req):
    """the request as both decoders return it: integer arrays as their big-endian bytes"""
    out = dict(req)
    for f, size in ARRAYS:
        if f != "prev_txid":
            out[f] = _be(req[f], size)
    return out


def _c_encode(shim, req, cap):
    arrays = [_wire_view(req)[f] for f, _ in ARRAYS] + [req["sigs"]]
    arr = (ctypes.c_char_p * 14)(*arrays)
    out = ctypes.create_string_buffer(max(cap, 1))
    ln = shim.shim_towire_tx(out, cap, RID, req["kind"], req["keylen"], req["key"], req["n"], arr, req["bloblen"],
                             req["blob"], req["want_sighash"])
    return out.raw[:ln] if ln else None


def _c_decode_request(shim, body):
    rid, sc, offs = ctypes.c_uint64(), (ctypes.c_uint32 * 5)(), (ctypes.c_size_t * 16)()
    if not shim.shim_fromwire_tx(body, len(body), ctypes.byref(rid), sc, offs):
        return None
    kind, keylen, n, bloblen, want = list(sc)
    o = list(offs)
    out = dict(req_id=rid.value, kind=kind, keylen=keylen, key=body[o[0]:o[0] + keylen], n=n)
    for k, (f, size) in enumerate(ARRAYS):
        out[f] = body[o[1 + k]:o[1 + k] + size * n]
    out.update(bloblen=bloblen, blob=body[o[14]:o[14] + bloblen], sigs=body[o[15]:o[15] + 64 * n], want_sighash=want)
    return out


def _c_decode_reply(shim, body):
    rid, sc, offs = ctypes.c_uint64(), (ctypes.c_uint32 * 2)(), (ctypes.c_size_t * 2)()
    if not shim.shim_fromwire_tx_reply(body, len(body), ctypes.byref(rid), sc, offs):
        return None
    n, nsh = list(sc)
    return dict(req_id=rid.value, n=n, verdicts=body[offs[0]:offs[0] + n], nsighash=nsh,
                sighashes=body[offs[1]:offs[1] + 32 * nsh])


def _py_decodes_as(body, name):
    try:
        return W.decode(body)[0] == name
    except (AssertionError, KeyError, IndexError, struct.error):
        return False


@pytest.mark.parametrize("n", [0, 1, 3, 483])
@pytest.mark.parametrize("kind", [0, 1], ids=["ecdsa33", "ecdsa_xy"])
@pytest.mark.parametrize("want", [0, 1], ids=["no_sighash", "want_sighash"])
def test_request_codecs_agree(shim, n, kind, want):
    rng = np.random.default_rng(n * 4 + kind * 2 + want)
    req = _request(rng, n, kind, want)
    frame = W.encode("sigverifyd_tx", **req)
    body = frame[4:]
    assert int.from_bytes(frame[:4], "big") == len(body) and body[:2] == (3005).to_bytes(2, "big")
    per_tx = 6 * 4 + 32 + 2 * 8 + 4 * 4 + 64
    assert len(body) == 2 + 8 + 1 + 4 + req["keylen"] + 4 + per_tx * n + 4 + req["bloblen"] + 1
    assert _c_encode(shim, req, len(body) + 16) == body
    assert _c_encode(shim, req, len(body) - 1) is None  # does not fit: nothing written
    assert _c_decode_request(shim, body) == _wire_view(req)
    assert W.decode(body) == ("sigverifyd_tx", _wire_view(req))
    # truncated anywhere, one byte too many, a count one larger or smaller than the bytes that follow: refused by both
    ks = req["keylen"]
    n_at = 2 + 8 + 1 + 4 + ks
    bl_at = n_at + 4 + (per_tx - 64) * n
    bad = [body[:k] for k in sorted({2, 9, 11, 14, n_at + 2, bl_at + 2, len(body) // 2, len(body) - 1})] + [body + b"\0"]
    bad.append(body[:11] + (ks + 1).to_bytes(4, "big") + body[15:])
    bad.append(body[:n_at] + (n + 1).to_bytes(4, "big") + body[n_at + 4:])
    if n:
        bad.append(body[:n_at] + (n - 1).to_bytes(4, "big") + body[n_at + 4:])
    bad.append(body[:bl_at] + (req["bloblen"] + 1).to_bytes(4, "big") + body[bl_at + 4:])
    if req["bloblen"]:
        bad.append(body[:bl_at] + (req["bloblen"] - 1).to_bytes(4, "big") + body[bl_at + 4:])
    for b in bad:
        assert _c_decode_request(shim, b) is None, len(b)
        assert not _py_decodes_as(b, "sigverifyd_tx"), len(b)


@pytest.mark.parametrize("n", [0, 1, 7, 484, 65_536])
@pytest.mark.parametrize("want", [0, 1], ids=["no_sighash", "want_sighash"])
def test_reply_codecs_agree(shim, n, want):
    rng = np.random.default_rng(n + want)
    verdicts = bytes(rng.integers(0, 2, size=n).astype(np.uint8))
    nsh = n if want else 0
    sh = rng.integers(0, 256, size=32 * nsh, dtype=np.uint8).tobytes()
    rep = dict(req_id=RID, n=n, verdicts=verdicts, nsighash=nsh, sighashes=sh)
    body = W.encode("sigverifyd_tx_reply", **rep)[4:]
    assert body[:2] == (3105).to_bytes(2, "big") and len(body) == 2 + 8 + 4 + n + 4 + 32 * nsh
    out = ctypes.create_string_buffer(len(body) + 16)
    ln = shim.shim_towire_tx_reply(out, len(out), RID, n, verdicts, nsh, sh)
    assert ln == len(body) and out.raw[:ln] == body
    assert shim.shim_towire_tx_reply(out, len(body) - 1, RID, n, verdicts, nsh, sh) == 0
    assert _c_decode_reply(shim, body) == rep
    assert W.decode(body) == ("sigverifyd_tx_reply", rep)
    bad = [body[:k] for k in sorted({2, 10, 13, len(body) - 1})] + [body + b"\0"]
    bad.append(body[:10] + (n + 1).to_bytes(4, "big") + body[14:])
    sh_at = 14 + n
    bad.append(body[:sh_at] + (nsh + 1).to_bytes(4, "big") + body[sh_at + 4:])
    if nsh:
        bad.append(body[:sh_at] + (nsh - 1).to_bytes(4, "big") + body[sh_at + 4:])
    for b in bad:
        assert _c_decode_reply(shim, b) is None, len(b)
        assert not _py_decodes_as(b, "sigverifyd_tx_reply"), len(b)


def test_wrong_type_is_refused(shim):
    req = W.encode("sigverifyd_tx", **_request(np.random.default_rng(3), 2, 1, 1))[4:]
    rep = W.encode("sigverifyd_tx_reply", req_id=RID, n=2, verdicts=b"\1\0", nsighash=0, sighashes=b"")[4:]
    for other in (3001, 3004, 3105):
        b = other.to_bytes(2, "big") + req[2:]
        assert _c_decode_request(shim, b) is None and not _py_decodes_as(b, "sigverifyd_tx")
    for other in (3005, 3101, 3104):
        b = other.to_bytes(2, "big") + rep[2:]
        assert _c_decode_reply(shim, b) is None and not _py_decodes_as(b, "sigverifyd_tx_reply")
    assert _c_decode_request(shim, rep) is None and _c_decode_reply(shim, req) is None
