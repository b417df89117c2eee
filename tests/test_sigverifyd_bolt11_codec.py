"""CPU: the verifier subdaemon's BOLT11 messages (sigverifyd_bolt11 / sigverifyd_bolt11_reply).  The generated C codec
(lightning_b200/csrc/sigverifyd_wiregen.h, through tests/host_emul/wire_shim_bolt11.c) and the generated Python codec
(lightning_b200/sigverifyd_wire.py) must agree byte for byte in both directions, and both must refuse truncated frames,
counts that do not match the bytes that follow and a message of another type."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from lightning_b200 import sigverifyd_wire as W

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RID = 0x0807060504030201


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("wire") / "libwireshim_bolt11.so")
    subprocess.check_call(["gcc", "-O2", "-shared", "-fPIC", "-Wall", "-Wextra", "-Werror", "-o", so,
                           os.path.join(ROOT, "tests", "host_emul", "wire_shim_bolt11.c")])
    lib = ctypes.CDLL(so)
    lib.shim_towire_bolt11.restype = ctypes.c_size_t
    lib.shim_towire_bolt11.argtypes = [ctypes.c_char_p, ctypes.c_size_t, ctypes.c_uint64, ctypes.c_uint32, ctypes.c_char_p,
                                       ctypes.c_uint32, ctypes.c_char_p]
    lib.shim_towire_bolt11_reply.restype = ctypes.c_size_t
    lib.shim_towire_bolt11_reply.argtypes = [ctypes.c_char_p, ctypes.c_size_t, ctypes.c_uint64, ctypes.c_uint32,
                                             ctypes.c_char_p, ctypes.c_char_p]
    for f in (lib.shim_fromwire_bolt11, lib.shim_fromwire_bolt11_reply):
        f.argtypes = [ctypes.c_char_p, ctypes.c_size_t, ctypes.POINTER(ctypes.c_uint64), ctypes.c_void_p, ctypes.c_void_p]
    return lib


def _invoice(rng, size, nul_at=None):
    """size printable bytes (lower-case bech32 letters and digits), with a NUL at nul_at if given"""
    s = bytearray(rng.choice(list(b"lnbc1qpzry9x8gf2tvdw0s3jn54khce6mua7l"), size=size).astype(np.uint8).tobytes())
    if nul_at is not None:
        s[nul_at] = 0
    return bytes(s)


def _request(strings):
    blob = b"".join(strings)
    return dict(req_id=RID, n=len(strings), lens=[len(s) for s in strings], bloblen=len(blob), blob=blob)


def _c_decode_request(shim, body):
    rid, sc, offs = ctypes.c_uint64(), (ctypes.c_uint32 * 2)(), (ctypes.c_size_t * 2)()
    if not shim.shim_fromwire_bolt11(body, len(body), ctypes.byref(rid), sc, offs):
        return None
    n, bloblen = list(sc)
    return dict(req_id=rid.value, n=n, lens=[int.from_bytes(body[offs[0] + 4 * i:offs[0] + 4 * i + 4], "big") for i in range(n)],
                bloblen=bloblen, blob=body[offs[1]:offs[1] + bloblen])


def _c_decode_reply(shim, body):
    rid, sc, offs = ctypes.c_uint64(), (ctypes.c_uint32 * 1)(), (ctypes.c_size_t * 2)()
    if not shim.shim_fromwire_bolt11_reply(body, len(body), ctypes.byref(rid), sc, offs):
        return None
    n = sc[0]
    return dict(req_id=rid.value, n=n, status=body[offs[0]:offs[0] + n], node_ids=body[offs[1]:offs[1] + 33 * n])


def _py_decodes(body):
    try:
        W.decode(body)
        return True
    except AssertionError:
        return False


CASES = {
    "n0": [],
    "one": [(300, None)],
    "empty_string": [(0, None)],
    "embedded_nul": [(120, 40), (64, 0), (90, 89)],
    "long_route_hints": [(2_400, None), (7, None), (0, None), (500, 250)],
}


@pytest.mark.parametrize("case", list(CASES))
def test_request_codecs_agree(shim, case):
    rng = np.random.default_rng(len(CASES[case]) * 7 + len(case))
    strings = [_invoice(rng, size, nul) for size, nul in CASES[case]]
    req = _request(strings)
    frame = W.encode("sigverifyd_bolt11", **req)
    body = frame[4:]
    assert int.from_bytes(frame[:4], "big") == len(body) and body[:2] == (3013).to_bytes(2, "big")
    assert len(body) == 2 + 8 + 4 + 4 * len(strings) + 4 + len(req["blob"])
    out = ctypes.create_string_buffer(len(body) + 16)
    lens_be = b"".join(len(s).to_bytes(4, "big") for s in strings)
    ln = shim.shim_towire_bolt11(out, len(out), RID, len(strings), lens_be, len(req["blob"]), req["blob"])
    assert ln == len(body) and out.raw[:ln] == body
    assert shim.shim_towire_bolt11(out, len(body) - 1, RID, len(strings), lens_be, len(req["blob"]), req["blob"]) == 0
    assert _c_decode_request(shim, body) == req  # the NUL bytes travel inside the blob
    name, vals = W.decode(body)
    assert name == "sigverifyd_bolt11" and vals == dict(req, lens=lens_be)
    # truncated anywhere, one byte too many, a count one larger or smaller than the bytes that follow: refused by both
    n = len(strings)
    bad = [body[:k] for k in sorted({2, 9, 11, 13, len(body) // 2, len(body) - 1})] + [body + b"\0"]
    bad.append(body[:10] + (n + 1).to_bytes(4, "big") + body[14:])
    if n:
        bad.append(body[:10] + (n - 1).to_bytes(4, "big") + body[14:])
    bl_at = 14 + 4 * n
    bad.append(body[:bl_at] + (len(req["blob"]) + 1).to_bytes(4, "big") + body[bl_at + 4:])
    if req["blob"]:
        bad.append(body[:bl_at] + (len(req["blob"]) - 1).to_bytes(4, "big") + body[bl_at + 4:])
    for b in bad:
        assert _c_decode_request(shim, b) is None, len(b)
        assert not _py_decodes(b), len(b)


@pytest.mark.parametrize("n", [0, 1, 9, 30_000])
def test_reply_codecs_agree(shim, n):
    rng = np.random.default_rng(n + 1)
    status = bytes(rng.choice([0, 1, 255], size=n).astype(np.uint8))
    nodes = b"".join(rng.integers(0, 256, size=33, dtype=np.uint8).tobytes() if s == 1 else bytes(33) for s in status)
    rep = dict(req_id=RID, n=n, status=status, node_ids=nodes)
    body = W.encode("sigverifyd_bolt11_reply", **rep)[4:]
    assert body[:2] == (3113).to_bytes(2, "big") and len(body) == 2 + 8 + 4 + n + 33 * n
    out = ctypes.create_string_buffer(len(body) + 16)
    ln = shim.shim_towire_bolt11_reply(out, len(out), RID, n, status, nodes)
    assert ln == len(body) and out.raw[:ln] == body
    assert shim.shim_towire_bolt11_reply(out, len(body) - 1, RID, n, status, nodes) == 0
    assert _c_decode_reply(shim, body) == rep
    assert W.decode(body) == ("sigverifyd_bolt11_reply", rep)
    bad = [body[:k] for k in sorted({2, 10, 13, len(body) - 1})] + [body + b"\0"]
    bad.append(body[:10] + (n + 1).to_bytes(4, "big") + body[14:])
    if n:
        bad.append(body[:10] + (n - 1).to_bytes(4, "big") + body[14:])
    for b in bad:
        assert _c_decode_reply(shim, b) is None, len(b)
        assert not _py_decodes(b), len(b)


def test_wrong_type_is_refused(shim):
    rng = np.random.default_rng(3)
    body = W.encode("sigverifyd_bolt11", **_request([_invoice(rng, 40)]))[4:]
    # the same fields under the sha256d type (the identical layout) and a reply type: neither parses as a request
    assert _c_decode_request(shim, (3006).to_bytes(2, "big") + body[2:]) is None
    assert _c_decode_request(shim, (3113).to_bytes(2, "big") + body[2:]) is None
    assert _c_decode_reply(shim, body) is None
    rep = W.encode("sigverifyd_bolt11_reply", req_id=1, n=1, status=b"\x01", node_ids=bytes(33))[4:]
    assert _c_decode_request(shim, rep) is None
    assert _c_decode_reply(shim, (3104).to_bytes(2, "big") + rep[2:]) is None
