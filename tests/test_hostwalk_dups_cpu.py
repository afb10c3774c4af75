"""The duplicate statistics of the level-synchronous host walk (tests/native/hostwalk_dups.cpp): the walk is walk_bfs's
(same verdict, same configurations), and its per-level counts add up."""
import pytest

import hostwalk
import hostwalk_dups
from jepsen_tigerbeetle_b200 import history as H
from jepsen_tigerbeetle_b200 import synth


def bank():
    return H.make_model(H.MODEL_BANK, accounts=range(1, 9))


@pytest.mark.parametrize("model,spec", [
    ("bank", synth.SynthSpec("bank", 400, 8, 2, tau_think_ns=5e6, stale_read=True)),
    ("bank", synth.SynthSpec("bank", 300, 8, 3, tau_think_ns=5e6, stale_read=False)),
    ("cas-register", synth.SynthSpec("cas-register", 300, 10, 4, tau_think_ns=5e6, stale_read=True, n_values=5)),
])
def test_counts_add_up_and_match_walk_bfs(model, spec):
    h = synth.generate(spec)
    m = bank() if model == "bank" else H.make_model(H.MODEL_CAS_REGISTER)
    windows = (4, 32, 256)
    d = hostwalk_dups.walk_dups(h, m, windows=windows, eager_reads=False)
    b = hostwalk.walk_bfs(h, m, eager_reads=False, width_cap=20000)
    assert d["valid"] == b["valid"]
    assert d["configs"] == b["configs"]
    assert d["levels"] == b["levels"]
    assert sum(r["new"] for r in d["rows"]) == d["configs"]
    assert [r["new"] for r in d["rows"]] == b["widths"]
    for lv, r in enumerate(d["rows"]):
        if lv + 1 < len(d["rows"]):
            assert d["rows"][lv + 1]["parents"] == r["new"]
        # every duplicate within a block is a duplicate within the level: children = new + level duplicates
        assert r["new"] <= r["children"]
        prev = 0
        for w in windows:   # a larger block sees every duplicate a smaller aligned block inside it sees
            assert prev <= r["dups"][w] <= r["children"] - r["new"]
            prev = r["dups"][w]
    assert any(r["dups"][32] > 0 for r in d["rows"])


def test_budget_stops_the_walk():
    h = synth.generate(synth.SynthSpec("bank", 400, 8, 2, tau_think_ns=5e6, stale_read=True))
    d = hostwalk_dups.walk_dups(h, bank(), windows=(32,), max_configs=1000)
    assert d["valid"] == H.UNKNOWN
    assert 1000 <= d["configs"] < 1000 + 400 * 64


def test_bad_windows_are_refused():
    h = synth.generate(synth.SynthSpec("bank", 50, 4, 1))
    with pytest.raises(RuntimeError):
        hostwalk_dups.walk_dups(h, bank(), windows=(32, 0))
    with pytest.raises(RuntimeError):
        hostwalk_dups.walk_dups(h, bank(), windows=(1, 2, 4, 8, 16))
