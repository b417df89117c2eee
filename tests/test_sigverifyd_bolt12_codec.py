"""CPU: the verifier subdaemon's BOLT12 messages (sigverifyd_bolt12 / sigverifyd_bolt12_reply).  The generated C codec
(lightning_b200/csrc/sigverifyd_wiregen.h, through tests/host_emul/wire_shim_bolt12.c) and the generated Python codec
(lightning_b200/sigverifyd_wire.py) must agree byte for byte in both directions, and both must refuse truncated frames
and counts that do not match the bytes that follow."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from lightning_b200 import sigverifyd_wire as W

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RID = 0x0102030405060708


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("wire") / "libwireshim_bolt12.so")
    subprocess.check_call(["gcc", "-O2", "-shared", "-fPIC", "-Wall", "-Wextra", "-Werror", "-o", so,
                           os.path.join(ROOT, "tests", "host_emul", "wire_shim_bolt12.c")])
    lib = ctypes.CDLL(so)
    lib.shim_towire_bolt12.restype = ctypes.c_size_t
    lib.shim_towire_bolt12.argtypes = [ctypes.c_char_p, ctypes.c_size_t, ctypes.c_uint64, ctypes.c_uint16, ctypes.c_char_p,
                                       ctypes.c_uint16, ctypes.c_char_p, ctypes.c_uint32, ctypes.c_char_p, ctypes.c_uint32,
                                       ctypes.c_char_p, ctypes.c_char_p, ctypes.c_char_p, ctypes.c_uint8]
    lib.shim_towire_bolt12_reply.restype = ctypes.c_size_t
    lib.shim_towire_bolt12_reply.argtypes = [ctypes.c_char_p, ctypes.c_size_t, ctypes.c_uint64, ctypes.c_uint32,
                                             ctypes.c_char_p, ctypes.c_uint32, ctypes.c_char_p]
    for f in (lib.shim_fromwire_bolt12, lib.shim_fromwire_bolt12_reply):
        f.argtypes = [ctypes.c_char_p, ctypes.c_size_t, ctypes.POINTER(ctypes.c_uint64), ctypes.c_void_p, ctypes.c_void_p]
    return lib


def _request(rng, lens, want):
    n = len(lens)
    blob = rng.integers(0, 256, size=sum(lens), dtype=np.uint8).tobytes()
    xonly = rng.integers(0, 256, size=32 * n, dtype=np.uint8).tobytes()
    sigs = rng.integers(0, 256, size=64 * n, dtype=np.uint8).tobytes()
    return dict(req_id=RID, mnlen=15, messagename=b"invoice_request", fnlen=9, fieldname=b"signature", n=n, lens=lens,
                bloblen=len(blob), blob=blob, xonly=xonly, sigs=sigs, want_sighash=want)


def _c_decode_request(shim, body):
    rid, sc, offs = ctypes.c_uint64(), (ctypes.c_uint32 * 5)(), (ctypes.c_size_t * 6)()
    if not shim.shim_fromwire_bolt12(body, len(body), ctypes.byref(rid), sc, offs):
        return None
    mnlen, fnlen, n, bloblen, want = list(sc)
    o = list(offs)
    return dict(req_id=rid.value, mnlen=mnlen, messagename=body[o[0]:o[0] + mnlen], fnlen=fnlen,
                fieldname=body[o[1]:o[1] + fnlen], n=n,
                lens=[int.from_bytes(body[o[2] + 4 * i:o[2] + 4 * i + 4], "big") for i in range(n)], bloblen=bloblen,
                blob=body[o[3]:o[3] + bloblen], xonly=body[o[4]:o[4] + 32 * n], sigs=body[o[5]:o[5] + 64 * n],
                want_sighash=want)


def _c_decode_reply(shim, body):
    rid, sc, offs = ctypes.c_uint64(), (ctypes.c_uint32 * 2)(), (ctypes.c_size_t * 2)()
    if not shim.shim_fromwire_bolt12_reply(body, len(body), ctypes.byref(rid), sc, offs):
        return None
    n, nsh = list(sc)
    return dict(req_id=rid.value, n=n, status=body[offs[0]:offs[0] + n], nsighash=nsh,
                sighashes=body[offs[1]:offs[1] + 32 * nsh])


def _py_decodes(body):
    try:
        W.decode(body)
        return True
    except AssertionError:
        return False


@pytest.mark.parametrize("lens", [[], [0], [0, 300, 0], [20_001], [5, 20_500, 1, 0, 77]],
                         ids=["n0", "empty_stream", "empty_among_others", "long_stream", "mixed"])
@pytest.mark.parametrize("want", [0, 1], ids=["no_sighash", "want_sighash"])
def test_request_codecs_agree(shim, lens, want):
    rng = np.random.default_rng(len(lens) * 10 + want)
    req = _request(rng, lens, want)
    frame = W.encode("sigverifyd_bolt12", **req)
    body = frame[4:]
    assert int.from_bytes(frame[:4], "big") == len(body) and body[:2] == (3004).to_bytes(2, "big")
    out = ctypes.create_string_buffer(len(body) + 16)
    lens_be = b"".join(x.to_bytes(4, "big") for x in lens)
    ln = shim.shim_towire_bolt12(out, len(out), RID, 15, b"invoice_request", 9, b"signature", len(lens), lens_be,
                                 len(req["blob"]), req["blob"], req["xonly"], req["sigs"], want)
    assert ln == len(body) and out.raw[:ln] == body
    assert shim.shim_towire_bolt12(out, len(body) - 1, RID, 15, b"invoice_request", 9, b"signature", len(lens), lens_be,
                                   len(req["blob"]), req["blob"], req["xonly"], req["sigs"], want) == 0  # does not fit
    assert _c_decode_request(shim, body) == req
    name, vals = W.decode(body)
    assert name == "sigverifyd_bolt12"
    assert vals == dict(req, lens=lens_be)
    # truncated anywhere, one byte too many, a count one larger or smaller than the bytes that follow: refused by both
    n = len(lens)
    n_at = 2 + 8 + 2 + 15 + 2 + 9
    bad = [body[:k] for k in sorted({2, 9, 11, n_at + 2, len(body) // 2, len(body) - 1})] + [body + b"\0"]
    bad.append(body[:n_at] + (n + 1).to_bytes(4, "big") + body[n_at + 4:])
    if n:
        bad.append(body[:n_at] + (n - 1).to_bytes(4, "big") + body[n_at + 4:])
    bl_at = n_at + 4 + 4 * n
    bad.append(body[:bl_at] + (len(req["blob"]) + 1).to_bytes(4, "big") + body[bl_at + 4:])
    bad.append(body[:2 + 8] + (16).to_bytes(2, "big") + body[12:])  # messagename length past its bytes
    for b in bad:
        assert _c_decode_request(shim, b) is None, len(b)
        assert not _py_decodes(b), len(b)


@pytest.mark.parametrize("n", [0, 1, 7, 25_000])
@pytest.mark.parametrize("want", [0, 1], ids=["no_sighash", "want_sighash"])
def test_reply_codecs_agree(shim, n, want):
    rng = np.random.default_rng(n + want)
    status = bytes(rng.choice([0, 1, 255], size=n).astype(np.uint8))
    nsh = n if want else 0
    sh = rng.integers(0, 256, size=32 * nsh, dtype=np.uint8).tobytes()
    rep = dict(req_id=RID, n=n, status=status, nsighash=nsh, sighashes=sh)
    body = W.encode("sigverifyd_bolt12_reply", **rep)[4:]
    assert body[:2] == (3104).to_bytes(2, "big") and len(body) == 2 + 8 + 4 + n + 4 + 32 * nsh
    out = ctypes.create_string_buffer(len(body) + 16)
    ln = shim.shim_towire_bolt12_reply(out, len(out), RID, n, status, nsh, sh)
    assert ln == len(body) and out.raw[:ln] == body
    assert _c_decode_reply(shim, body) == rep
    assert W.decode(body) == ("sigverifyd_bolt12_reply", rep)
    bad = [body[:k] for k in sorted({2, 10, 13, len(body) - 1})] + [body + b"\0"]
    bad.append(body[:10] + (n + 1).to_bytes(4, "big") + body[14:])
    sh_at = 14 + n
    bad.append(body[:sh_at] + (nsh + 1).to_bytes(4, "big") + body[sh_at + 4:])
    if nsh:
        bad.append(body[:sh_at] + (nsh - 1).to_bytes(4, "big") + body[sh_at + 4:])
    for b in bad:
        assert _c_decode_reply(shim, b) is None, len(b)
        assert not _py_decodes(b), len(b)


def test_wrong_type_is_refused(shim):
    body = W.encode("sigverifyd_bolt12", **_request(np.random.default_rng(3), [4], 1))[4:]
    assert _c_decode_request(shim, (3001).to_bytes(2, "big") + body[2:]) is None
    assert _c_decode_reply(shim, body) is None
