"""GPU: sv_verify_gossip_store_host against Core Lightning's own gossmap.c (see tests/test_gossmap.py), on both
verification paths: the crafted stores with every prefix that ends after a channel_update, the fixture, its seeded
mutations and the fixture tiled x53."""
import pytest

from tests.test_gossmap import Tally, compare, crafted_stores, mutations, oracle
from tests.test_gossip_store_host import load_fixture
from tests.test_gpu_gossip_store import run

pytestmark = pytest.mark.gpu


def each_path(engine, body):
    small = engine.small_max()
    try:
        for sm in (small, 0):  # the latency path where a store is small enough, then always the throughput kernels
            engine.set_small_max(sm)
            body()
    finally:
        engine.set_small_max(small)


def test_crafted_vs_gossmap(engine):
    o = oracle()
    t = Tally()

    def body():
        for st in crafted_stores():
            compare(o, st, lambda s: run(engine, s), t, prefixes=True)
    each_path(engine, body)
    t.report("engine")
    assert t.positions >= 300


def test_fixture_mutations_tiled_vs_gossmap(engine):
    o = oracle()
    t = Tally()
    fx = load_fixture()
    stores = [fx] + mutations() + [fx[:1] + fx[1:] * 53]

    def body():
        for st in stores:
            compare(o, st, lambda s: run(engine, s), t)
    each_path(engine, body)
    t.report("engine")
    assert t.stores >= 2 * 200
