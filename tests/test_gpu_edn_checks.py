"""GPU tier: K19, the host checks of a ledger compose on a stored history.edn, against the same checkers on
edn.read_history's op maps (full result dicts) and against the Python model of the summary."""
import numpy as np
import pytest

import edn_checks_model as M
from jepsen_tigerbeetle_b200 import checker as CK
from jepsen_tigerbeetle_b200 import edn, stored, synth

CHECKERS = (CK.UnexpectedOps, CK.LookupAllInvokedTransfers, CK.FinalReads, CK.Stats)


def _same_summary(g, m):
    """The device summary against the model's: counts, the flagged ops' ordinals, spans, times, indices, suspect bits,
    and the same partition into classes."""
    for name in ("n_ops", "n_client", "n_ok", "n_fail", "n_info", "n_open", "n_final_reads", "n_final_lookups",
                 "n_read_classes", "n_lookup_classes", "n_invoked", "n_suspect"):
        assert g[name] == m[name], name
    assert (g["last"] is None) == (m["last"] is None)
    fields = ["op", "begin", "end", "time", "index", "has_time", "has_index", "first", "suspect"]
    if g["last"] is not None:
        assert all(g["last"][f] == m["last"][f] for f in fields[:-2])
    for kind in ("open", "fails", "final_reads", "final_lookups"):
        a, b = np.sort(g[kind], order="op"), np.sort(m[kind], order="op")
        for f in fields:
            assert np.array_equal(a[f], b[f]), (kind, f)
        pairs = set(zip(a["cls"].tolist(), b["cls"].tolist()))
        assert len(pairs) == len({x for x, _ in pairs}) == len({y for _, y in pairs}), kind


def _check(ctx, data, where="", model=True):
    h = CK.StoredLedgerHistory(data, ctx=ctx)
    ops = edn.read_history(data.decode())
    for c in CHECKERS:
        assert c().check({}, h) == c().check({}, ops), (where, c.__name__)
    s = h.checks()
    assert s is not None, (where, h._checks["refused"])
    if model:
        _same_summary(s, M.summarize(data))
    return s


@pytest.mark.gpu
@pytest.mark.parametrize("p_info", [0.0, 0.02])
@pytest.mark.parametrize("p_lookup", [0.0, 0.05])
@pytest.mark.parametrize("seed", [1, 2, 3])
def test_generated_histories(gpu_ctx, p_info, p_lookup, seed):
    spec = synth.SynthSpec("bank", 2000, 16, seed, p_info=p_info, tau_think_ns=10e6, final_reads=True)
    ops = stored.generate_ledger_ops(spec, p_lookup=p_lookup, nemesis_every=53)
    for vector in (False, True):
        _check(gpu_ctx, stored.write_edn(ops, vector=vector), where=(p_info, p_lookup, seed, vector))


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(M.HAND_CASES))
def test_hand_cases(gpu_ctx, name):
    _check(gpu_ctx, M.HAND_CASES[name], where=name)


@pytest.mark.gpu
def test_large_final_lookups(gpu_ctx):
    """Final lookups of 2 * 10^4 records each: complete, missing a single id, reversed, complete again."""
    recs = [["l-t", i, {"debit-acct": 1 + i % 7, "credit-acct": 2 + i % 5, "amount": 1 + i % 9}]
            for i in range(1, 20_001)]
    ops = [dict(type="invoke", process=0, f="txn", value=[["t", i, r[2]] for i, r in enumerate(recs, 1)], index=0,
                time=1),
           dict(type="ok", process=0, f="txn", value=[["t", i, r[2]] for i, r in enumerate(recs, 1)], index=1, time=2)]
    for p, v in enumerate((recs, recs[:10_000] + recs[10_001:], recs[::-1], recs), 1):
        ops += [dict(type="invoke", process=p, f="txn", value=[["l-t", 1, None]], index=2 * p, time=2 * p,
                     **{"final?": True}),
                dict(type="ok", process=p, f="txn", value=v, index=2 * p + 1, time=2 * p + 1, **{"final?": True})]
    s = _check(gpu_ctx, stored.write_edn(ops), model=False)
    assert s["n_invoked"] == 20_000 and s["n_lookup_classes"] == 3
    assert s["final_lookups"]["suspect"].tolist() == [0, 1, 0, 0]


@pytest.mark.gpu
@pytest.mark.parametrize("p_info", [0.0, 0.02])
def test_ledger_checker_never_parses_in_python(gpu_ctx, monkeypatch, p_info):
    spec = synth.SynthSpec("bank", 1000, 8, 3, p_info=p_info, tau_think_ns=10e6, final_reads=True)
    data = stored.write_edn(stored.generate_ledger_ops(spec, p_lookup=0.05, nemesis_every=41))
    expect = CK.ledger_checker(ctx=gpu_ctx, linear=False).check({}, edn.read_history(data.decode()))
    calls = []
    real = edn.read_history
    monkeypatch.setattr(edn, "read_history", lambda *a, **k: calls.append(1) or real(*a, **k))
    r = CK.ledger_checker(ctx=gpu_ctx, linear=False).check({}, CK.StoredLedgerHistory(data, ctx=gpu_ctx))
    assert calls == []
    assert not any(op.parsed for op in r["lookup-transfers"].get("suspect-final-lookups", []))
    assert _strip(r) == _strip(expect) and calls == []


def _strip(r):
    if isinstance(r, dict):
        return {k: _strip(v) for k, v in r.items() if not k.startswith("seconds")}
    if isinstance(r, list):
        return [_strip(v) for v in r]
    return r


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(M.REFUSED_CASES))
def test_refusals_fall_back(gpu_ctx, monkeypatch, name):
    data = M.REFUSED_CASES[name]
    expect = [c().check({}, edn.read_history(data.decode())) for c in CHECKERS]
    calls = []
    real = edn.read_history
    monkeypatch.setattr(edn, "read_history", lambda *a, **k: calls.append(1) or real(*a, **k))
    h = CK.StoredLedgerHistory(data, ctx=gpu_ctx)
    assert [c().check({}, h) for c in CHECKERS] == expect
    assert h.checks() is None and h._checks["refused"]["reason"]
    assert len(calls) == 1
    _check(gpu_ctx, M.HAND_CASES["valid finals"])   # the context still reads another history
