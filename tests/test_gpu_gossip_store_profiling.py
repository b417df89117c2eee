"""GPU: the gossip_store audit and prune in profiling mode.  The funding calls on stores that hold no gossip message
return normally, and on the fixture every split the timing getters report (sv_get_last_gossip_store_timing,
sv_get_last_gossip_prune_timing, sv_get_last_gossip_funding_timing) covers its work and fits inside the call."""
import struct
import time

import pytest

from tests import gossip_store as gs
from tests import gossip_store_funding as gf
from tests.test_gossip_store_host import load_fixture
from tests.test_gpu_gossip_burst import TESTNET
from tests.test_gpu_gossip_store_funding import funding_table

pytestmark = pytest.mark.gpu


@pytest.fixture
def profiling(engine):
    engine.set_profiling(True)
    yield engine
    engine.set_profiling(False)


def test_funding_on_stores_without_messages(profiling):
    fx = load_fixture()
    ft = funding_table(gf.table_of_store(fx))
    amount = gs.record(struct.pack(">HQ", gs.CHANNEL_AMOUNT, 1000))
    for store in (fx[:1], fx[:1] + amount):
        n = len(gs.walk(store)[0])
        _, _, _, _, s, _, fs = profiling.verify_gossip_store(store, TESTNET, funding=ft)
        assert s["records"] == n and fs["checked"] == 0
        _, _, s, _, fs = profiling.prune_gossip_store(store, TESTNET, funding=ft)
        assert s["records"] == n and s["pruned"] == 0 and fs["checked"] == 0
        assert len(profiling.last_gossip_funding_timing()) == 2


def _timed(call):
    call()  # warm-up
    t = time.perf_counter()
    call()
    return (time.perf_counter() - t) * 1e3


def test_splits_cover_their_work_and_fit_the_call(profiling):
    # one announcement without its funding output: the prune's flag write has deletions to write
    store, t = gf.fixture_cases(load_fixture())["no_txout"]
    ft = funding_table(t)
    # the audit: walk, H2D, checksums, the rest; the funding step's staging comes before them and its kernel after
    wall = _timed(lambda: profiling.verify_gossip_store(store, TESTNET, funding=ft))
    split, (stage, kernel) = profiling.last_gossip_store_timing(), profiling.last_gossip_funding_timing()
    assert len(split) == 4 and min(split) > 0 and stage > 0 and kernel > 0, (split, stage, kernel)
    assert sum(split) + stage + kernel <= wall, (split, stage, kernel, wall)
    # the prune: walk, first round, second round (the funding kernel runs inside it), flag write
    wall = _timed(lambda: profiling.prune_gossip_store(store, TESTNET, funding=ft))
    split, (stage, kernel) = profiling.last_gossip_prune_timing(), profiling.last_gossip_funding_timing()
    assert len(split) == 4 and min(split) > 0 and stage > 0 and kernel > 0, (split, stage, kernel)
    assert sum(split) + stage <= wall and kernel <= split[2], (split, stage, kernel, wall)
