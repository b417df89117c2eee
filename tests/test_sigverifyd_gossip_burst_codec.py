"""CPU: the verifier subdaemon's gossip burst messages (sigverifyd_gossip_burst / _reply) at the shapes the feature sends,
n = 0 to 20,000.  The generated C codec and the generated Python codec must agree byte for byte in both directions, and
both must refuse truncated and over-long frames, counts that do not match the bytes that follow, and the wrong message
type (tests/sigverifyd_codec.py)."""
import numpy as np
import pytest

from lightning_b200 import sigverifyd_wire as W
from tests import sigverifyd_codec as codec

RID = 0x0102030405060708
NUM = {"sigverifyd_gossip_burst": 3008, "sigverifyd_gossip_burst_reply": 3108}


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    return codec.build_shim(tmp_path_factory.mktemp("wire"))


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


@pytest.mark.parametrize("n", [0, 1, 2, 9, 483, 20_000])
@pytest.mark.parametrize("name", list(NUM))
def test_codecs_agree(shim, name, n):
    m = _message(name, np.random.default_rng(n * 11 + NUM[name]), n)
    codec.agree(shim, name, m)
    codec.refused(shim, name, m)


def test_wrong_type_is_refused(shim):
    rng = np.random.default_rng(5)
    for name in NUM:
        codec.wrong_type_refused(shim, name, _message(name, rng, 3))


def test_existing_messages_unchanged():
    """adding the burst messages leaves every other message's number and fields as they were"""
    assert W.MSGS["sigverifyd_gossip"] == (3002, [("req_id", "u64", None), ("n", "u32", None), ("lens", "u32", "n"),
                                                  ("signers", "node_id", "n"), ("bloblen", "u32", None),
                                                  ("blob", "byte", "bloblen")])
    assert W.MSGS["sigverifyd_gossip_burst"][0] == 3008 and W.MSGS["sigverifyd_gossip_burst_reply"][0] == 3108
