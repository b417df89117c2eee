"""CPU: the verifier subdaemon's gossip burst messages (sigverifyd_gossip_burst / _reply).  The generated C codec
(lightning_b200/csrc/sigverifyd_wiregen.h, through tests/host_emul/wire_shim_burst.c) and the generated Python codec
(lightning_b200/sigverifyd_wire.py) must agree byte for byte in both directions, including n = 0, and both must refuse
truncated and over-long frames, counts that do not match the bytes that follow, and the wrong message type."""
import ctypes
import os
import struct
import subprocess

import numpy as np
import pytest

from lightning_b200 import sigverifyd_wire as W

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RID = 0x0102030405060708
NUM = {"sigverifyd_gossip_burst": 3008, "sigverifyd_gossip_burst_reply": 3108}


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("wire") / "libwireshim_burst.so")
    subprocess.check_call(["gcc", "-O2", "-shared", "-fPIC", "-Wall", "-Wextra", "-Werror", "-o", so,
                           os.path.join(ROOT, "tests", "host_emul", "wire_shim_burst.c")])
    lib = ctypes.CDLL(so)
    u8p, sz, u32 = ctypes.c_char_p, ctypes.c_size_t, ctypes.c_uint32
    lib.shim_towire_gossip_burst.argtypes = [u8p, sz, ctypes.c_uint64, u8p, u32, u8p, u8p, u8p, u32, u8p]
    lib.shim_towire_gossip_burst_reply.argtypes = [u8p, sz, ctypes.c_uint64, u32, u8p]
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
    if name == "sigverifyd_gossip_burst":
        lens = [int(x) for x in rng.choice([0, 1, 138, 430, 1000], size=n)]
        return dict(req_id=RID, chain_hash=_rand(rng, 32), n=n, lens=b"".join(x.to_bytes(4, "big") for x in lens),
                    signer_kind=rng.integers(0, 3, size=n, dtype=np.uint8).tobytes(), signers=_rand(rng, 33 * n),
                    bloblen=sum(lens), blob=_rand(rng, sum(lens)))
    return dict(req_id=RID, n=n, status=rng.choice(np.array([0, 1, 2, 3, 4, 5, 252, 253, 254, 255], np.uint8), size=n).tobytes())


def _c_encode(shim, name, m, cap):
    out = ctypes.create_string_buffer(max(cap, 1))
    if name == "sigverifyd_gossip_burst":
        ln = shim.shim_towire_gossip_burst(out, cap, m["req_id"], m["chain_hash"], m["n"], m["lens"], m["signer_kind"],
                                           m["signers"], m["bloblen"], m["blob"])
    else:
        ln = shim.shim_towire_gossip_burst_reply(out, cap, m["req_id"], m["n"], m["status"])
    return out.raw[:ln] if ln else None


def _c_decode(shim, name, body):
    short = name[len("sigverifyd_"):]
    rid, sc, offs = ctypes.c_uint64(), (ctypes.c_uint32 * 2)(), (ctypes.c_size_t * 5)()
    if not getattr(shim, "shim_fromwire_" + short)(body, len(body), ctypes.byref(rid), sc, offs):
        return None
    n = sc[0]
    if short == "gossip_burst":
        return dict(req_id=rid.value, chain_hash=body[offs[0]:offs[0] + 32], n=n, lens=body[offs[1]:offs[1] + 4 * n],
                    signer_kind=body[offs[2]:offs[2] + n], signers=body[offs[3]:offs[3] + 33 * n], bloblen=sc[1],
                    blob=body[offs[4]:offs[4] + sc[1]])
    return dict(req_id=rid.value, n=n, status=body[offs[0]:offs[0] + n])


def _py_decodes_as(body, name):
    try:
        return W.decode(body)[0] == name
    except (AssertionError, KeyError, IndexError, struct.error):
        return False


def _length(name, m):
    n = m["n"]
    if name == "sigverifyd_gossip_burst":
        return 2 + 8 + 32 + 4 + 4 * n + n + 33 * n + 4 + m["bloblen"]
    return 2 + 8 + 4 + n


@pytest.mark.parametrize("n", [0, 1, 2, 9, 483, 20_000])
@pytest.mark.parametrize("name", list(NUM))
def test_codecs_agree(shim, name, n):
    rng = np.random.default_rng(n * 11 + NUM[name])
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
    n_at = 42 if name == "sigverifyd_gossip_burst" else 10
    bad = [body[:k] for k in sorted({0, 1, 2, 9, 11, 13, 41, 45, len(body) // 2, len(body) - 1}) if k < len(body)]
    bad.append(body + b"\0")
    bad.append(body[:n_at] + (n + 1).to_bytes(4, "big") + body[n_at + 4:])
    if n:
        bad.append(body[:n_at] + (n - 1).to_bytes(4, "big") + body[n_at + 4:])
    if name == "sigverifyd_gossip_burst":
        bl_at = 46 + 38 * n
        bad.append(body[:bl_at] + (m["bloblen"] + 1).to_bytes(4, "big") + body[bl_at + 4:])
        if m["bloblen"]:
            bad.append(body[:bl_at] + (m["bloblen"] - 1).to_bytes(4, "big") + body[bl_at + 4:])
    for b in bad:
        assert _c_decode(shim, name, b) is None, len(b)
        assert not _py_decodes_as(b, name), len(b)


def test_wrong_type_is_refused(shim):
    rng = np.random.default_rng(5)
    bodies = {name: W.encode(name, **_message(name, rng, 3))[4:] for name in NUM}
    others = [3001, 3002, 3004, 3005, 3006, 3007, 3102, 3199] + list(NUM.values())
    for name, body in bodies.items():
        for other in others:
            if other == NUM[name]:
                continue
            b = other.to_bytes(2, "big") + body[2:]
            assert _c_decode(shim, name, b) is None and not _py_decodes_as(b, name), (name, other)
        for o in NUM:
            if o != name:
                assert _c_decode(shim, o, body) is None, (name, o)


def test_existing_messages_unchanged():
    """adding the burst messages leaves every other message's number and fields as they were"""
    assert W.MSGS["sigverifyd_gossip"] == (3002, [("req_id", "u64", None), ("n", "u32", None), ("lens", "u32", "n"),
                                                  ("signers", "node_id", "n"), ("bloblen", "u32", None),
                                                  ("blob", "byte", "bloblen")])
    assert W.MSGS["sigverifyd_gossip_burst"][0] == 3008 and W.MSGS["sigverifyd_gossip_burst_reply"][0] == 3108
