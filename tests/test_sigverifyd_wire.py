"""CPU: the verifier subdaemon's wire codec over the whole schema, every message of sigverifyd_wire.csv
(tests/sigverifyd_codec.py holds the checks).  For each message, instances built from the schema: every count at 0, 1, a
few values and a large one; integers 0, at their maximum and anywhere in their range."""
import numpy as np
import pytest

from lightning_b200 import sigverifyd_wire as W
from tests import sigverifyd_codec as codec

CASES = ["empty", "single", "few_a", "few_b", "few_c", "large"]


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    return codec.build_shim(tmp_path_factory.mktemp("wire"))


def _rand(rng, n):
    return rng.integers(0, 256, size=n, dtype=np.uint8).tobytes()


def _be(vals, size):
    return b"".join(int(v).to_bytes(size, "big") for v in vals)


def _sha256d(m, rng):
    """buffers at every SHA-256 padding boundary, empty ones among them, and one of 70,000 bytes"""
    lens = [int(x) for x in rng.choice([0, 1, 55, 56, 63, 64, 119, 120, 174], size=m["n"])]
    if m["n"] > 2:
        lens[1] = 70_000
    m.update(lens=_be(lens, 4), bloblen=sum(lens), blob=_rand(rng, sum(lens)))


def _bolt11(m, rng):
    """invoice-like strings, a tenth of them with a NUL inside (the codec carries every byte)"""
    strings = []
    for _ in range(m["n"]):
        s = bytearray(rng.choice(list(b"lnbc1qpzry9x8gf2tvdw0s3jn54khce6mua7l"), size=int(rng.integers(0, 400)))
                      .astype(np.uint8).tobytes())
        if s and rng.random() < 0.1:
            s[int(rng.integers(0, len(s)))] = 0
        strings.append(bytes(s))
    m.update(lens=_be(map(len, strings), 4), bloblen=sum(map(len, strings)), blob=b"".join(strings))


def _pubkey_reply(m, rng):
    """xy zeroed where ok is 0"""
    ok = rng.integers(0, 2, size=m["n"]).astype(np.uint8)
    xy = np.frombuffer(m["xy"], np.uint8).reshape(m["n"], 64) * ok[:, None]
    m.update(ok=ok.tobytes(), xy=xy.tobytes())


RULES = {"sigverifyd_sha256d": _sha256d, "sigverifyd_bolt11": _bolt11, "sigverifyd_pubkey_reply": _pubkey_reply}
LARGE = {"sigverifyd_bolt11": 30_000, "sigverifyd_bolt11_reply": 30_000}  # items of the large case; else 65,536


def instance(name, case):
    """the fields of one message: counts 0 (empty), 1 (single), a few, or large; the other integers 0 (empty), their
    maximum (single) or anywhere in their range; random bytes in every blob and array"""
    rng = np.random.default_rng([list(W.MSGS).index(name), CASES.index(case)])
    fields = codec.fields(name)
    counts = {c for _, _, c in fields if c}
    m = {}
    for f, t, c in fields:
        bits = 8 * W.INT.get(t, 0)
        if c:
            m[f] = _rand(rng, m[c] * codec.size(t))
        elif t in W.BLOB:
            m[f] = _rand(rng, W.BLOB[t])
        elif f in counts:
            m[f] = {"empty": 0, "single": 1, "large": min(LARGE.get(name, 65_536), 2**bits - 1)}.get(
                case, int(rng.choice([2, 3, 9, 33, 483])))
        else:
            m[f] = {"empty": 0, "single": 2**bits - 1}.get(case, int(rng.integers(0, 2**bits, dtype=np.uint64)))
    if name in RULES:
        RULES[name](m, rng)
    return m


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("name", list(W.MSGS))
def test_codecs_agree(shim, name, case):
    codec.agree(shim, name, instance(name, case))


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("name", list(W.MSGS))
def test_refusals(shim, name, case):
    m = instance(name, case)
    codec.refused(shim, name, m)
    codec.wrong_type_refused(shim, name, m)


def test_layout_covers_the_schema():
    """every message of the CSV has its pins in tests/sigverifyd_codec.py, and no pin is left without its message"""
    assert set(codec.LAYOUT) == set(W.MSGS)
