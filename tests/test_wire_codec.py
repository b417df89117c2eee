"""CPU: the verifier subdaemon's wire codec.  The C side (lightning_b200/csrc/sigverifyd_wiregen.h) and the Python side
(lightning_b200/sigverifyd_wire.py) are both generated from sigverifyd_wire.csv by tools/gen_wire.py; the committed files
must be what the generator makes of the CSV, and the two sides must agree byte for byte and refuse truncated, over-long
and wrongly-typed messages (CLN's fromwire_* contract, checked by tests/sigverifyd_codec.py)."""
import importlib.util
import os

import numpy as np
import pytest

from tests import sigverifyd_codec as codec

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    return codec.build_shim(tmp_path_factory.mktemp("wire"))


def test_generated_header_is_current():
    """the committed generated files are what tools/gen_wire.py makes of the committed CSV (nothing is written)"""
    spec = importlib.util.spec_from_file_location("gen_wire", os.path.join(ROOT, "tools", "gen_wire.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    msgs = gen.parse(gen.CSV)
    assert open(codec.WIREGEN).read() == gen.gen_c(msgs)
    assert open(os.path.join(ROOT, "lightning_b200", "sigverifyd_wire.py")).read() == gen.gen_py(msgs)


def test_c_and_python_codecs_agree(shim):
    rng = np.random.default_rng(1)
    for n, kind, ks in ((0, 0, 33), (1, 0, 33), (3, 1, 64), (483, 2, 32)):
        h, k, s = (rng.integers(0, 256, size=n * w, dtype=np.uint8).tobytes() for w in (32, ks, 64))
        m = dict(req_id=0x1122334455667788, kind=kind, n=n, hashes=h, keylen=n * ks, keys=k, sigs=s)
        codec.agree(shim, "sigverifyd_verify", m)
        codec.refused(shim, "sigverifyd_verify", m)
        codec.wrong_type_refused(shim, "sigverifyd_verify", m)
    for name, m in (("sigverifyd_verify_reply", dict(req_id=7, n=5, verdicts=bytes([1, 0, 1, 1, 0]))),
                    ("sigverifyd_stats_reply", dict(req_id=9, requests=10, launches=3, signatures=2**40, max_coalesced=4))):
        codec.agree(shim, name, m)
        codec.refused(shim, name, m)
    lens = [300, 5, 140]
    blob = rng.integers(0, 256, size=sum(lens), dtype=np.uint8).tobytes()
    sg = rng.integers(0, 256, size=33 * 3, dtype=np.uint8).tobytes()
    m = dict(req_id=1, n=3, lens=lens, signers=sg, bloblen=len(blob), blob=blob)
    codec.agree(shim, "sigverifyd_gossip", m)
    codec.refused(shim, "sigverifyd_gossip", m)
