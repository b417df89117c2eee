"""Python model of sv_salvage_gossip_store_host (the rule in include/cln_sigverify.h): the sound records of a
gossip_store, and the walk that restores each damaged header whose record resumes where its checksum says, or bridges the
span with deleted filler records.  The candidate filter runs in numpy; each candidate's checksum is computed in Python
and memoised by a digest of the record's bytes (at most 2^20 entries, 16 bytes each), so a tiled store costs about
one copy of its records."""
import bisect
import hashlib
import struct

import numpy as np

from tests.gossip_store import COMPLETED, DELETED, ENDED, HDR, crc32c

KNOWN = (256, 257, 258, 4101, 4103, 4105, 4106, 4107)
GAP, PIECE = 14, HDR + 65535
RESTORED, BRIDGED = 1, 2
FIELDS = ("breaks", "restored", "bridged", "bridged_bytes", "fillers", "sound")

_CRC = {}  # record digest -> checksum matches: a tiled store repeats its records and most random candidates
_CRC_MAX = 1 << 20


def _crc_ok(rec):
    key = hashlib.blake2b(rec, digest_size=16).digest()
    if key not in _CRC:
        if len(_CRC) >= _CRC_MAX:
            _CRC.clear()
        ln, crc, ts = struct.unpack(">HII", rec[2:12])
        _CRC[key] = crc32c(ts, rec[HDR:HDR + ln]) == crc
    return _CRC[key]


def candidates(store):
    """offsets o >= 1 with COMPLETED, 2 <= len, o + 12 + len <= len(store) and a known type, ascending"""
    n = len(store)
    if n < 1 + HDR + 2:
        return []
    a = np.frombuffer(store, np.uint8)
    typ = (a[1 + HDR:n - 1].astype(np.uint16) << 8) | a[2 + HDR:n]  # type at offset o = 1 + index
    o = np.nonzero(np.isin(typ, KNOWN))[0].astype(np.int64) + 1
    flags = (a[o].astype(np.int64) << 8) | a[o + 1]
    ln = (a[o + 2].astype(np.int64) << 8) | a[o + 3]
    keep = (flags & COMPLETED != 0) & (ln >= 2) & (o + HDR + ln <= n)
    return [int(x) for x in o[keep]]


def sound_offsets(store):
    """the sorted offsets of the sound records: candidates whose checksum matches"""
    out = []
    for o in candidates(store):
        ln = struct.unpack(">H", store[o + 2:o + 4])[0]
        if _crc_ok(bytes(store[o:o + HDR + ln])):
            out.append(o)
    return out


def pieces(span):
    """the filler sizes of a bridge of span bytes"""
    k = -(-span // PIECE)
    return [span // k + (i < span % k) for i in range(k)]


def _bridged(s, t, q):
    """[t, q) already holds the fillers a bridge of it writes"""
    p = t
    for size in pieces(q - t):
        if struct.unpack(">HH", s[p:p + 4]) != (DELETED | COMPLETED, size - HDR):
            return False
        p += size
    return True


def salvage(store, sound=None):
    """-> (salvaged bytes, [(t, q, RESTORED or BRIDGED)], summary dict)"""
    if store[0] >> 5:
        raise ValueError("major version")
    sound = sound_offsets(store) if sound is None else sound
    ss = set(sound)
    s = bytearray(store)
    acts, sm = [], dict.fromkeys(FIELDS, 0)
    sm["sound"] = len(sound)
    t = 1
    while t + HDR < len(s):
        flags, ln = struct.unpack(">HH", s[t:t + 4])
        if t in ss:
            if not flags & DELETED and struct.unpack(">H", s[t + HDR:t + HDR + 2])[0] == ENDED:
                break
            t += HDR + ln
            continue
        if flags & COMPLETED and t + HDR + ln in ss:
            t += HDR + ln
            continue
        k = bisect.bisect_left(sound, t + GAP)
        if k == len(sound):
            break
        q = sound[k]
        n = q - t - HDR
        if _bridged(s, t, q):  # salvaged before: fillers are never sound
            t = q
            continue
        sm["breaks"] += 1
        ts, crc = struct.unpack(">I", s[t + 8:t + 12])[0], struct.unpack(">I", s[t + 4:t + 8])[0]
        if n <= 0xFFFF and crc32c(ts, bytes(s[t + HDR:q])) == crc:
            struct.pack_into(">HH", s, t, flags | COMPLETED, n)
            sm["restored"] += 1
            acts.append((t, q, RESTORED))
        else:
            p = t
            for size in pieces(q - t):
                struct.pack_into(">HH", s, p, DELETED | COMPLETED, size - HDR)
                p += size
            sm["bridged"] += 1
            sm["bridged_bytes"] += q - t
            sm["fillers"] += len(pieces(q - t))
            acts.append((t, q, BRIDGED))
        t = q
    return bytes(s), acts, sm
