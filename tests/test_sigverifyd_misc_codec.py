"""CPU: the verifier subdaemon's sha256_double and pubkey_from_der messages (sigverifyd_sha256d / _reply, sigverifyd_pubkey
/ _reply).  The generated C codec (lightning_b200/csrc/sigverifyd_wiregen.h, through tests/host_emul/wire_shim_misc.c) and
the generated Python codec (lightning_b200/sigverifyd_wire.py) must agree byte for byte in both directions, including
n = 0 and empty buffers, and both must refuse truncated and over-long frames, counts that do not match the bytes that
follow, and the wrong message type."""
import ctypes
import os
import struct
import subprocess

import numpy as np
import pytest

from lightning_b200 import sigverifyd_wire as W

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RID = 0x0102030405060708
NUM = {"sigverifyd_sha256d": 3006, "sigverifyd_sha256d_reply": 3106, "sigverifyd_pubkey": 3007,
       "sigverifyd_pubkey_reply": 3107}


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("wire") / "libwireshim_misc.so")
    subprocess.check_call(["gcc", "-O2", "-shared", "-fPIC", "-Wall", "-Wextra", "-Werror", "-o", so,
                           os.path.join(ROOT, "tests", "host_emul", "wire_shim_misc.c")])
    lib = ctypes.CDLL(so)
    u8p, sz = ctypes.c_char_p, ctypes.c_size_t
    lib.shim_towire_sha256d.argtypes = [u8p, sz, ctypes.c_uint64, ctypes.c_uint32, u8p, ctypes.c_uint32, u8p]
    lib.shim_towire_sha256d_reply.argtypes = [u8p, sz, ctypes.c_uint64, ctypes.c_uint32, u8p]
    lib.shim_towire_pubkey.argtypes = [u8p, sz, ctypes.c_uint64, ctypes.c_uint32, u8p]
    lib.shim_towire_pubkey_reply.argtypes = [u8p, sz, ctypes.c_uint64, ctypes.c_uint32, u8p, u8p]
    for name in NUM:
        short = name[len("sigverifyd_"):]
        getattr(lib, "shim_towire_" + short).restype = sz
        getattr(lib, "shim_fromwire_" + short).argtypes = [u8p, sz, ctypes.POINTER(ctypes.c_uint64), ctypes.c_void_p,
                                                           ctypes.c_void_p]
    return lib


def _rand(rng, n):
    return rng.integers(0, 256, size=n, dtype=np.uint8).tobytes()


def _message(name, rng, n):
    """the fields of one message with n items (random bytes: the codec does not care what they mean)"""
    if name == "sigverifyd_sha256d":
        # every SHA-256 padding boundary, empty buffers among them, and one long buffer
        lens = [int(x) for x in rng.choice([0, 1, 55, 56, 63, 64, 119, 120, 174], size=n)]
        if n > 2:
            lens[1] = 70_000
        return dict(req_id=RID, n=n, lens=b"".join(x.to_bytes(4, "big") for x in lens), bloblen=sum(lens),
                    blob=_rand(rng, sum(lens)))
    if name == "sigverifyd_sha256d_reply":
        return dict(req_id=RID, n=n, hashes=_rand(rng, 32 * n))
    if name == "sigverifyd_pubkey":
        return dict(req_id=RID, n=n, keys=_rand(rng, 33 * n))
    ok = rng.integers(0, 2, size=n).astype(np.uint8)
    xy = np.frombuffer(_rand(rng, 64 * n), np.uint8).reshape(n, 64) * ok[:, None]
    return dict(req_id=RID, n=n, ok=ok.tobytes(), xy=xy.tobytes())


def _c_encode(shim, name, m, cap):
    out = ctypes.create_string_buffer(max(cap, 1))
    short = name[len("sigverifyd_"):]
    args = {"sha256d": ("lens", "bloblen", "blob"), "sha256d_reply": ("hashes",), "pubkey": ("keys",),
            "pubkey_reply": ("ok", "xy")}[short]
    ln = getattr(shim, "shim_towire_" + short)(out, cap, m["req_id"], m["n"], *[m[a] for a in args])
    return out.raw[:ln] if ln else None


def _c_decode(shim, name, body):
    short = name[len("sigverifyd_"):]
    rid, sc, offs = ctypes.c_uint64(), (ctypes.c_uint32 * 2)(), (ctypes.c_size_t * 2)()
    if not getattr(shim, "shim_fromwire_" + short)(body, len(body), ctypes.byref(rid), sc, offs):
        return None
    n = sc[0]
    out = dict(req_id=rid.value, n=n)
    if short == "sha256d":
        out.update(lens=body[offs[0]:offs[0] + 4 * n], bloblen=sc[1], blob=body[offs[1]:offs[1] + sc[1]])
    elif short == "sha256d_reply":
        out["hashes"] = body[offs[0]:offs[0] + 32 * n]
    elif short == "pubkey":
        out["keys"] = body[offs[0]:offs[0] + 33 * n]
    else:
        out.update(ok=body[offs[0]:offs[0] + n], xy=body[offs[1]:offs[1] + 64 * n])
    return out


def _py_decodes_as(body, name):
    try:
        return W.decode(body)[0] == name
    except (AssertionError, KeyError, IndexError, struct.error):
        return False


def _length(name, m):
    n = m["n"]
    if name == "sigverifyd_sha256d":
        return 2 + 8 + 4 + 4 * n + 4 + m["bloblen"]
    return 2 + 8 + 4 + {"sigverifyd_sha256d_reply": 32, "sigverifyd_pubkey": 33, "sigverifyd_pubkey_reply": 65}[name] * n


@pytest.mark.parametrize("n", [0, 1, 2, 9, 483, 65_536])
@pytest.mark.parametrize("name", list(NUM))
def test_codecs_agree(shim, name, n):
    rng = np.random.default_rng(n * 7 + NUM[name])
    m = _message(name, rng, n)
    frame = W.encode(name, **m)
    body = frame[4:]
    assert int.from_bytes(frame[:4], "big") == len(body) == _length(name, m)
    assert body[:2] == NUM[name].to_bytes(2, "big") and body[2:10] == RID.to_bytes(8, "big")
    assert _c_encode(shim, name, m, len(body) + 16) == body
    assert _c_encode(shim, name, m, len(body) - 1) is None  # does not fit: nothing written
    assert _c_decode(shim, name, body) == m
    assert W.decode(body) == (name, m)
    # truncated anywhere, one byte too many, a count one larger or smaller than the bytes that follow: refused by both
    bad = [body[:k] for k in sorted({0, 1, 2, 9, 11, 13, len(body) // 2, len(body) - 1})] + [body + b"\0"]
    bad.append(body[:10] + (n + 1).to_bytes(4, "big") + body[14:])
    if n:
        bad.append(body[:10] + (n - 1).to_bytes(4, "big") + body[14:])
    if name == "sigverifyd_sha256d":
        bl_at = 14 + 4 * n
        bad.append(body[:bl_at] + (m["bloblen"] + 1).to_bytes(4, "big") + body[bl_at + 4:])
        if m["bloblen"]:
            bad.append(body[:bl_at] + (m["bloblen"] - 1).to_bytes(4, "big") + body[bl_at + 4:])
    for b in bad:
        assert _c_decode(shim, name, b) is None, len(b)
        assert not _py_decodes_as(b, name), len(b)


def test_empty_buffers(shim):
    """a request of empty buffers only: bloblen 0 and no blob bytes, n span lengths of 0"""
    m = dict(req_id=RID, n=3, lens=bytes(12), bloblen=0, blob=b"")
    body = W.encode("sigverifyd_sha256d", **m)[4:]
    assert body == (3006).to_bytes(2, "big") + RID.to_bytes(8, "big") + (3).to_bytes(4, "big") + bytes(12) + bytes(4)
    assert _c_encode(shim, "sigverifyd_sha256d", m, 64) == body
    assert _c_decode(shim, "sigverifyd_sha256d", body) == m


def test_wrong_type_is_refused(shim):
    rng = np.random.default_rng(5)
    bodies = {name: W.encode(name, **_message(name, rng, 3))[4:] for name in NUM}
    others = [3001, 3004, 3005, 3101, 3105, 3199] + list(NUM.values())
    for name, body in bodies.items():
        for other in others:
            if other == NUM[name]:
                continue
            b = other.to_bytes(2, "big") + body[2:]
            assert _c_decode(shim, name, b) is None and not _py_decodes_as(b, name), (name, other)
        for o in NUM:
            if o != name:
                assert _c_decode(shim, o, body) is None, (name, o)
