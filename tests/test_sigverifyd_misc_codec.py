"""CPU: the verifier subdaemon's sha256_double and pubkey_from_der messages (sigverifyd_sha256d / _reply, sigverifyd_pubkey
/ _reply) at the shapes the features send, n = 0 to 65,536 with every SHA-256 padding length and a 70,000-byte buffer.
The generated C codec and the generated Python codec must agree byte for byte in both directions, including n = 0 and
empty buffers, and both must refuse truncated and over-long frames, counts that do not match the bytes that follow, and
the wrong message type (tests/sigverifyd_codec.py)."""
import numpy as np
import pytest

from tests import sigverifyd_codec as codec

RID = 0x0102030405060708
NUM = {"sigverifyd_sha256d": 3006, "sigverifyd_sha256d_reply": 3106, "sigverifyd_pubkey": 3007,
       "sigverifyd_pubkey_reply": 3107}


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    return codec.build_shim(tmp_path_factory.mktemp("wire"))


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


@pytest.mark.parametrize("n", [0, 1, 2, 9, 483, 65_536])
@pytest.mark.parametrize("name", list(NUM))
def test_codecs_agree(shim, name, n):
    m = _message(name, np.random.default_rng(n * 7 + NUM[name]), n)
    codec.agree(shim, name, m)
    codec.refused(shim, name, m)


def test_empty_buffers(shim):
    """a request of empty buffers only: bloblen 0 and no blob bytes, n span lengths of 0"""
    m = dict(req_id=RID, n=3, lens=bytes(12), bloblen=0, blob=b"")
    body = codec.agree(shim, "sigverifyd_sha256d", m)
    assert body == (3006).to_bytes(2, "big") + RID.to_bytes(8, "big") + (3).to_bytes(4, "big") + bytes(12) + bytes(4)


def test_wrong_type_is_refused(shim):
    rng = np.random.default_rng(5)
    for name in NUM:
        codec.wrong_type_refused(shim, name, _message(name, rng, 3))
