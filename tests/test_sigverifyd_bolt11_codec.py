"""CPU: the verifier subdaemon's BOLT11 messages (sigverifyd_bolt11 / sigverifyd_bolt11_reply) at the shapes the feature
sends: invoice strings with NULs inside, empty strings, long route hints and 30,000 replies.  The generated C codec and the
generated Python codec must agree byte for byte in both directions, and both must refuse truncated frames, counts that
do not match the bytes that follow and a message of another type (tests/sigverifyd_codec.py)."""
import numpy as np
import pytest

from tests import sigverifyd_codec as codec

RID = 0x0807060504030201


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    return codec.build_shim(tmp_path_factory.mktemp("wire"))


def _invoice(rng, size, nul_at=None):
    """size printable bytes (lower-case bech32 letters and digits), with a NUL at nul_at if given"""
    s = bytearray(rng.choice(list(b"lnbc1qpzry9x8gf2tvdw0s3jn54khce6mua7l"), size=size).astype(np.uint8).tobytes())
    if nul_at is not None:
        s[nul_at] = 0
    return bytes(s)


def _request(strings):
    blob = b"".join(strings)
    return dict(req_id=RID, n=len(strings), lens=[len(s) for s in strings], bloblen=len(blob), blob=blob)


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
    req = _request([_invoice(rng, size, nul) for size, nul in CASES[case]])
    codec.agree(shim, "sigverifyd_bolt11", req)  # the NUL bytes travel inside the blob
    codec.refused(shim, "sigverifyd_bolt11", req)


@pytest.mark.parametrize("n", [0, 1, 9, 30_000])
def test_reply_codecs_agree(shim, n):
    rng = np.random.default_rng(n + 1)
    status = bytes(rng.choice([0, 1, 255], size=n).astype(np.uint8))
    nodes = b"".join(rng.integers(0, 256, size=33, dtype=np.uint8).tobytes() if s == 1 else bytes(33) for s in status)
    rep = dict(req_id=RID, n=n, status=status, node_ids=nodes)
    codec.agree(shim, "sigverifyd_bolt11_reply", rep)
    codec.refused(shim, "sigverifyd_bolt11_reply", rep)


def test_wrong_type_is_refused(shim):
    """among the others, the request under the sha256d type (the identical layout) and under its reply's"""
    rng = np.random.default_rng(3)
    codec.wrong_type_refused(shim, "sigverifyd_bolt11", _request([_invoice(rng, 40)]))
    codec.wrong_type_refused(shim, "sigverifyd_bolt11_reply", dict(req_id=1, n=1, status=b"\x01", node_ids=bytes(33)))
