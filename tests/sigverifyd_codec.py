"""The verifier subdaemon's wire codec for the CPU tests: the generated C codec (lightning_b200/csrc/sigverifyd_wiregen.h)
reached through a ctypes shim generated from the schema (sigverifyd_wire.MSGS), the layout of every message pinned by
literals independently of the CSV, and the checks every codec test makes: both encoders give the same bytes, both
decoders read them back, and both decoders refuse truncated, over-long, miscounted and retyped frames (CLN's fromwire_*
contract)."""
import ctypes
import os
import struct
import subprocess

from lightning_b200 import sigverifyd_wire as W

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WIREGEN = os.path.join(ROOT, "lightning_b200", "csrc", "sigverifyd_wiregen.h")
CT = {"u8": "uint8_t", "u16": "uint16_t", "u32": "uint32_t", "u64": "uint64_t"}

# every message's type number and body length, the per-item lengths written out by hand
LAYOUT = {
    "sigverifyd_verify": (3001, lambda m: 2 + 8 + 1 + 4 + 32 * m["n"] + 4 + m["keylen"] + 64 * m["n"]),
    "sigverifyd_verify_reply": (3101, lambda m: 2 + 8 + 4 + m["n"]),
    "sigverifyd_gossip": (3002, lambda m: 2 + 8 + 4 + 4 * m["n"] + 33 * m["n"] + 4 + m["bloblen"]),
    "sigverifyd_gossip_reply": (3102, lambda m: 2 + 8 + 4 + m["n"]),
    "sigverifyd_stats": (3003, lambda m: 2 + 8),
    "sigverifyd_stats_reply": (3103, lambda m: 2 + 8 + 3 * 8 + 4),
    "sigverifyd_bolt12": (3004, lambda m: 2 + 8 + 2 + m["mnlen"] + 2 + m["fnlen"] + 4 + 4 * m["n"] + 4 + m["bloblen"] +
                          32 * m["n"] + 64 * m["n"] + 1),
    "sigverifyd_bolt12_reply": (3104, lambda m: 2 + 8 + 4 + m["n"] + 4 + 32 * m["nsighash"]),
    "sigverifyd_tx": (3005, lambda m: 2 + 8 + 1 + 4 + m["keylen"] + 4 + (6 * 4 + 32 + 2 * 8 + 4 * 4 + 64) * m["n"] + 4 +
                      m["bloblen"] + 1),
    "sigverifyd_tx_reply": (3105, lambda m: 2 + 8 + 4 + m["n"] + 4 + 32 * m["nsighash"]),
    "sigverifyd_sha256d": (3006, lambda m: 2 + 8 + 4 + 4 * m["n"] + 4 + m["bloblen"]),
    "sigverifyd_sha256d_reply": (3106, lambda m: 2 + 8 + 4 + 32 * m["n"]),
    "sigverifyd_pubkey": (3007, lambda m: 2 + 8 + 4 + 33 * m["n"]),
    "sigverifyd_pubkey_reply": (3107, lambda m: 2 + 8 + 4 + 65 * m["n"]),
    "sigverifyd_gossip_burst": (3008, lambda m: 2 + 8 + 32 + 4 + 4 * m["n"] + m["n"] + 33 * m["n"] + 4 + m["bloblen"]),
    "sigverifyd_gossip_burst_reply": (3108, lambda m: 2 + 8 + 4 + m["n"]),
    "sigverifyd_fee_grind": (3009, lambda m: 2 + 8 + 1 + 4 + m["keylen"] + 5 * 4 + 32 + 8 + 4 + m["script_len"] + 4 +
                             m["out_script_len"] + 64 + 8 + 4 + 4),
    "sigverifyd_fee_grind_reply": (3109, lambda m: 2 + 8 + 1 + 4 + 8),
    "sigverifyd_gossip_store_prune": (3010, lambda m: 2 + 8 + 1 + 32 + 8),
    "sigverifyd_gossip_store_prune_reply": (3110, lambda m: 2 + 8 + 3 * 4 + 12 * 8),
    "sigverifyd_gossip_store_repair": (3011, lambda m: 2 + 8 + 1 + 32 + 8),
    "sigverifyd_gossip_store_repair_reply": (3111, lambda m: 2 + 8 + 3 * 4 + 13 * 8),
    "sigverifyd_gossip_store_salvage": (3012, lambda m: 2 + 8 + 1 + 32 + 8),
    "sigverifyd_gossip_store_salvage_reply": (3112, lambda m: 2 + 8 + 3 * 4 + 19 * 8),
    "sigverifyd_bolt11": (3013, lambda m: 2 + 8 + 4 + 4 * m["n"] + 4 + m["bloblen"]),
    "sigverifyd_bolt11_reply": (3113, lambda m: 2 + 8 + 4 + m["n"] + 33 * m["n"]),
    "sigverifyd_error": (3199, lambda m: 2 + 8 + 4),
}


def fields(name):
    return W.MSGS[name][1]


def scalar(ftype, count):
    return not count and ftype in W.INT


def size(ftype):
    return W.INT.get(ftype) or W.BLOB[ftype]


# ---- the C codec through a shim generated from the schema ------------------------------------------------------------
def shim_source():
    """per message: shim_towire_<msg>(out, cap, ints, ptrs) and shim_fromwire_<msg>(p, len, ints, offs), where ints are
    the scalar integer fields in CSV order and ptrs / offs the fixed blobs and arrays in CSV order"""
    o = ['#include "%s"' % WIREGEN]
    for name in W.MSGS:
        ints = [f for f, t, c in fields(name) if scalar(t, c)]
        ptrs = [f for f, t, c in fields(name) if not scalar(t, c)]
        args = ["(%s)ints[%d]" % (CT[t], ints.index(f)) if scalar(t, c) else "ptrs[%d]" % ptrs.index(f)
                for f, t, c in fields(name)]
        o.append(f"size_t shim_towire_{name}(uint8_t *out, size_t cap, const uint64_t *ints, const uint8_t *const *ptrs) {{")
        o.append(f"    (void)ptrs;\n    return towire_{name}(out, cap, {', '.join(args)});\n}}")
        o.append(f"int shim_fromwire_{name}(const uint8_t *p, size_t len, uint64_t *ints, size_t *offs) {{")
        o.append(f"    struct {name} m;\n    (void)offs;\n    if (!fromwire_{name}(p, len, &m)) return 0;")
        o += [f"    ints[{k}] = m.{f};" for k, f in enumerate(ints)]
        o += [f"    offs[{k}] = (size_t)(m.{f} - p);" for k, f in enumerate(ptrs)]
        o.append("    return 1;\n}")
    return "\n".join(o) + "\n"


def build_shim(d):
    """the shim, compiled into the directory d and loaded"""
    (d / "shim.c").write_text(shim_source())
    r = subprocess.run(["gcc", "-O2", "-shared", "-fPIC", "-Wall", "-Wextra", "-Werror", str(d / "shim.c"), "-o",
                        str(d / "libshim.so")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    lib = ctypes.CDLL(str(d / "libshim.so"))
    for name in W.MSGS:
        t = getattr(lib, "shim_towire_" + name)
        t.restype = ctypes.c_size_t
        t.argtypes = [ctypes.c_char_p, ctypes.c_size_t, ctypes.POINTER(ctypes.c_uint64), ctypes.POINTER(ctypes.c_char_p)]
        f = getattr(lib, "shim_fromwire_" + name)
        f.restype = ctypes.c_int
        f.argtypes = [ctypes.c_char_p, ctypes.c_size_t, ctypes.POINTER(ctypes.c_uint64), ctypes.POINTER(ctypes.c_size_t)]
    return lib


def c_encode(shim, name, m, cap):
    """towire_<msg>'s bytes into a buffer of cap bytes, None if it wrote nothing"""
    ints = [m[f] for f, t, c in fields(name) if scalar(t, c)]
    ptrs = [m[f] for f, t, c in fields(name) if not scalar(t, c)]
    out = ctypes.create_string_buffer(max(cap, 1))
    n = getattr(shim, "shim_towire_" + name)(out, cap, (ctypes.c_uint64 * len(ints))(*ints),
                                              (ctypes.c_char_p * max(len(ptrs), 1))(*ptrs))
    return out.raw[:n] if n else None


def c_decode(shim, name, body):
    """fromwire_<msg>'s fields (each view as the bytes it spans), None if it refuses the body"""
    fs = fields(name)
    ints = (ctypes.c_uint64 * len(fs))()
    offs = (ctypes.c_size_t * len(fs))()
    if not getattr(shim, "shim_fromwire_" + name)(body, len(body), ints, offs):
        return None
    out, i, k = {}, 0, 0
    for f, t, c in fs:
        if scalar(t, c):
            out[f] = ints[i]
            i += 1
        else:
            n = out[c] * size(t) if c else size(t)
            out[f] = body[offs[k]:offs[k] + n]
            k += 1
    return out


def py_decodes_as(body, name):
    try:
        return W.decode(body)[0] == name
    except (AssertionError, KeyError, struct.error):
        return False


# ---- the checks ------------------------------------------------------------------------------------------------------
def wire_view(name, m):
    """the fields of m as both decoders return them: blobs and arrays as their bytes, integer arrays big-endian"""
    out = {}
    for f, t, c in fields(name):
        v = m[f]
        if scalar(t, c):
            out[f] = int(v)
        elif c and t in W.INT and not isinstance(v, (bytes, bytearray)):
            out[f] = b"".join(int(x).to_bytes(size(t), "big") for x in v)
        else:
            out[f] = bytes(v)
    return out


def agree(shim, name, m):
    """both encoders give the pinned layout byte for byte; towire into one byte too few writes nothing; both decoders
    read back every field.  Returns the message body."""
    m = wire_view(name, m)
    frame = W.encode(name, **m)
    body = frame[4:]
    num, length = LAYOUT[name]
    assert int.from_bytes(frame[:4], "big") == len(body) == length(m)
    assert body[:2] == num.to_bytes(2, "big") and body[2:10] == m["req_id"].to_bytes(8, "big")
    assert c_encode(shim, name, m, len(body) + 16) == body
    assert c_encode(shim, name, m, len(body) - 1) is None
    assert c_decode(shim, name, body) == m
    assert W.decode(body) == (name, m)
    return body


def refused(shim, name, m):
    """truncated at every field boundary and one byte inside each field, one byte too long, each count one more or one
    less than the bytes that follow: refused by both decoders"""
    m = wire_view(name, m)
    body = W.encode(name, **m)[4:]
    cuts, at = {0, 1}, 2
    bad = [body + b"\0"]
    for f, t, c in fields(name):
        n = m[c] * size(t) if c else size(t)
        cuts.add(at)
        if n > 1:
            cuts.add(at + 1)
        if any(c2 == f for _, _, c2 in fields(name)):
            for v in (m[f] - 1, m[f] + 1):
                if 0 <= v < 2 ** (8 * n):
                    bad.append(body[:at] + v.to_bytes(n, "big") + body[at + n:])
        at += n
    assert at == len(body)
    bad += [body[:k] for k in sorted(cuts) if k < len(body)]
    for b in bad:
        assert c_decode(shim, name, b) is None, len(b)
        assert not py_decodes_as(b, name), len(b)


def wrong_type_refused(shim, name, m):
    """the body under every other message number: the C decoder refuses it, the Python one does not read it as name"""
    body = W.encode(name, **wire_view(name, m))[4:]
    for other in W.BY_NUM:
        if other != LAYOUT[name][0]:
            b = other.to_bytes(2, "big") + body[2:]
            assert c_decode(shim, name, b) is None, (name, other)
            assert not py_decodes_as(b, name), (name, other)
