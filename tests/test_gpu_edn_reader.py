"""GPU tier: K18, the device reader of stored ledger histories, against edn.read_history + flatten_ops."""
import numpy as np
import pytest

from jepsen_tigerbeetle_b200 import checker as CK
from jepsen_tigerbeetle_b200 import edn, stored, synth
from jepsen_tigerbeetle_b200 import history as H
from jepsen_tigerbeetle_b200.native import NativeError

FORMS = ("bank", "ledger-counters", "ledger-lookups")
ARRAYS = ("type", "f", "flags", "process", "index", "time_ns", "a", "b", "c", "payload_off", "payload_len", "payload",
          "shard_off", "key_ids")

LEDGER_EDN = """
[{:type :invoke, :f :txn, :value [[:t 1 {:debit-acct 1, :credit-acct 2, :amount 3N}]], :process 0, :time 10, :index 0}
 {:type :ok, :f :txn, :value [[:t 1 {:debit-acct 1, :credit-acct 2, :amount 3}]], :process 0, :time 20, :index 1}
 #jepsen.history.Op{:type :invoke, :f :txn, :value [[:r 1 nil] [:r 2 nil]], :process 1, :time 30, :index 2}
 {:type :ok, :f :txn, :value [[:r 1 {:credits-posted 0, :debits-posted 3}] [:r 2 {:credits-posted 3, :debits-posted 0}]], :process 1, :time 40, :index 3}
 {:type :invoke, :f :txn, :value [[:l-t nil nil]], :process 2, :time 50, :index 4}
 {:type :ok, :f :txn, :value [[:l-t 1 {}]], :process 2, :time 60, :index 5}]
"""


def _python(text, form):
    return H.flatten_ops(edn.read_history(text if isinstance(text, str) else text.decode()), form)


def _same(g, p, where=""):
    for name in ARRAYS:
        x, y = getattr(g, name), getattr(p, name)
        assert x.dtype == y.dtype and np.array_equal(x, y), (where, name, x[:20], y[:20])
    if "multi_transfer_txns" in p.meta:
        assert g.meta["multi_transfer_txns"] == p.meta["multi_transfer_txns"], where


def _check(ctx, text, forms=FORMS, where=""):
    data = text.encode() if isinstance(text, str) else text
    for form in forms:
        try:
            p = _python(data, form)
        except Exception:   # noqa: BLE001 - the device must refuse whatever the Python path refuses
            with pytest.raises(NativeError):
                ctx.read_ledger_edn(data, form)
            continue
        _same(ctx.read_ledger_edn(data, form), p, (where, form))


def _ok_after(ctx):
    """the context still reads a history after an error"""
    _same(ctx.read_ledger_edn(LEDGER_EDN.encode(), "bank"), _python(LEDGER_EDN, "bank"))


@pytest.mark.gpu
def test_ledger_fixture(gpu_ctx):
    _check(gpu_ctx, LEDGER_EDN)
    _check(gpu_ctx, LEDGER_EDN.strip()[1:-1])          # the same ops, one per line
    _check(gpu_ctx, "")                                # an empty history


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
@pytest.mark.parametrize("mutation", ["lost_transfer", "phantom_record", "inflated_read"])
def test_mutations(gpu_ctx, mutation):
    spec = synth.SynthSpec("bank", 2000, 16, 1, p_info=0.02, tau_think_ns=10e6, final_reads=True)
    _check(gpu_ctx, stored.write_edn(stored.generate_ledger_ops(spec, **{mutation: True})), where=mutation)


def _line(**kw):
    return stored.op_line(kw)


T = lambda i, d=1, c=2, a=3: ["t", i, {"debit-acct": d, "credit-acct": c, "amount": a}]   # noqa: E731


@pytest.mark.gpu
def test_hand_cases(gpu_ctx):
    cases = {
        "empty ok lookup": [dict(type="invoke", process=0, f="txn", value=[["l-t", 5, None]], index=0, time=1),
                            dict(type="ok", process=0, f="txn", value=[], index=1, time=2),
                            dict(type="invoke", process=1, f="txn", value=[["r", 1, None]], index=2, time=3),
                            dict(type="ok", process=1, f="txn", value=[], index=3, time=4),
                            dict(type="invoke", process=0, f="txn", value=[["l-t", 5, None]], index=4, time=5),
                            dict(type="ok", process=0, f="txn", value=None, index=5, time=6)],
        "multi-transfer txn": [dict(type="invoke", process=0, f="txn", value=[T(1), T(2, 3, 4, 5), T(3)], index=0,
                                    time=1),
                               dict(type="ok", process=0, f="txn", value=[T(1), T(2, 3, 4, 5), T(3)], index=1, time=2)],
        "int64 bounds": [dict(type="invoke", process=0, f="txn", value=[T(-(1 << 63)), T((1 << 63) - 1)], index=0,
                              time=-(1 << 63)),
                         dict(type="invoke", process=1, f="txn", value=[["r", 1, None]], index=1, time=(1 << 63) - 1),
                         dict(type="ok", process=1, f="txn",
                              value=[["r", 1, {"debits-posted": (1 << 63) - 1, "credits-posted": -(1 << 63)}]],
                              index=2, time=3),
                         dict(type="invoke", process=2, f="txn", value=[["l-t", 1, None]], index=3, time=4),
                         dict(type="ok", process=2, f="txn", value=[["l-t", -(1 << 63), {"debit-acct": -(1 << 31),
                              "credit-acct": (1 << 31) - 1, "amount": 0}]], index=4, time=5)],
        "nil amounts": [dict(type="invoke", process=1, f="txn", value=[["r", 1, None], ["r", 2, None]], index=0, time=1),
                        dict(type="ok", process=1, f="txn", value=[["r", 1, None],
                             ["r", 2, {"debits-posted": None, "credits-posted": 4}]], index=1, time=2)],
        "no index or time": [dict(type="info", process="nemesis", f="start", value=None),
                             dict(type="invoke", process=0, f="txn", value=[T(1)]),
                             dict(type="ok", process=0, f="txn", value=[T(1)], **{"final?": True})],
    }
    for name, ops in cases.items():
        _check(gpu_ctx, stored.write_edn(ops), where=name)
    # what flatten_ops makes of truthy and empty values: :final? by truthiness; an empty map, set, string, false or 0 as
    # the value of an :ok lookup (the pending tag), [] or {} as the value of an :ok read; tagged values read through
    inv_l = '{:type :invoke, :f :txn, :value [[:l-t 1 nil]], :process 0, :index 0}\n'
    inv_r = '{:type :invoke, :f :txn, :value [[:r 1 nil]], :process 1, :index 2}\n'
    for final in (":yes", '"x"', '""', "[1]", "[]", "#{}", "{:a 1}", "0", "-0", "7N", "nil", "false", "#inst \"t\""):
        _check(gpu_ctx, inv_l + '{:type :ok, :f :txn, :value [], :process 0, :index 1, :final? %s}' % final,
               where=("final?", final))
    for value in ("{}", "#{}", '""', "false", "0", "nil", "[]", "()"):
        _check(gpu_ctx, inv_l + '{:type :ok, :f :txn, :value %s, :process 0, :index 1}' % value, where=("lookup", value))
        _check(gpu_ctx, inv_r + '{:type :ok, :f :txn, :value %s, :process 1, :index 3}' % value, where=("read", value))
    _check(gpu_ctx, '{:type :invoke, :f :txn, :value [[:t 1 #x.y{:debit-acct 1, :credit-acct 2, :amount #z 3}]], '
                    ':process 0, :time #t 5}\n' + inv_r
                    + '{:type :ok, :f :txn, :value [[:r 1 #m{:debits-posted 4, :credits-posted #n 5}]], :process 1}',
           where="tagged")
    # nemesis strings holding ], }, " and \\, and CRLF line ends
    ops = stored.generate_ledger_ops(synth.SynthSpec("bank", 200, 4, 1, tau_think_ns=10e6, final_reads=True),
                                     nemesis_every=3)
    _check(gpu_ctx, stored.write_edn(ops, newline="\r\n"), where="crlf")
    _check(gpu_ctx, '{:type :info, :process :nemesis, :f :kill, :value "a ] } \\" \\\\ b", :n #{1 [2]}}\n'
                    + _line(type="invoke", process=0, f="txn", value=[T(1)]), where="strings")


@pytest.mark.gpu
def test_one_final_lookup_of_1e5_records(gpu_ctx):
    recs = [["l-t", i, {"debit-acct": 1 + i % 7, "credit-acct": 2 + i % 5, "amount": 1 + i % 9}]
            for i in range(1, 100_001)]
    ops = [dict(type="invoke", process=0, f="txn", value=[["l-t", 1, None]], index=0, time=1, **{"final?": True}),
           dict(type="ok", process=0, f="txn", value=recs, index=1, time=2, **{"final?": True})]
    _check(gpu_ctx, stored.write_edn(ops), forms=("ledger-lookups",))


ERRORS = {
    "f other than txn": '{:type :invoke, :f :write, :value [[:r 1 nil]], :process 0}',
    "unknown micro-op": '{:type :invoke, :f :txn, :value [[:x 1 nil]], :process 0}',
    "txn without micro-ops": '{:type :invoke, :f :txn, :value [], :process 0}',
    "account outside [0, 2^30)": '{:type :ok, :f :txn, :value [[:r 1073741824 {:debits-posted 1}]], :process 0}',
    "negative account": '{:type :ok, :f :txn, :value [[:r -1 {:debits-posted 1}]], :process 0}',
    "transfer without id": '{:type :invoke, :f :txn, :value [[:t nil {:debit-acct 1, :credit-acct 2, :amount 3}]], '
                           ':process 0}',
    "id outside int64": '{:type :invoke, :f :txn, :value [[:t 9223372036854775808 {:debit-acct 1, :credit-acct 2, '
                        ':amount 3}]], :process 0}',
    "counter outside int64": '{:type :ok, :f :txn, :value [[:r 1 {:debits-posted -9223372036854775809}]], :process 0}',
    "amount outside int32": '{:type :invoke, :f :txn, :value [[:t 1 {:debit-acct 1, :credit-acct 2, '
                            ':amount 2147483648}]], :process 0}',
    "index outside int32": '{:type :invoke, :f :txn, :value [[:r 1 nil]], :process 0, :index 2147483648}',
    "process outside int32": '{:type :invoke, :f :txn, :value [[:r 1 nil]], :process -2147483649}',
    "balance outside int32": '{:type :ok, :f :txn, :value [[:r 1 {:debits-posted 0, :credits-posted 2147483648}]], '
                             ':process 0}',
    "empty ok lookup without a pending invoke": '{:type :ok, :f :txn, :value [], :process 0}',
    "unknown type": '{:type :done, :f :txn, :value [[:r 1 nil]], :process 0}',
    "comment": '; a comment\n{:type :invoke, :f :txn, :value [[:r 1 nil]], :process 0}',
    "discard": '#_ {:a 1} {:type :invoke, :f :txn, :value [[:r 1 nil]], :process 0}',
    "character literal": '{:type :invoke, :f :txn, :value [[:r 1 nil]], :process 0, :c \\a}',
    "float": '{:type :invoke, :f :txn, :value [[:r 1 nil]], :process 0, :time 1.5}',
    "mismatched brackets": '{:type :invoke, :f :txn, :value [[:r 1 nil]), :process 0}',
    "unterminated string": '{:type :invoke, :f :txn, :value [[:r 1 nil]], :process 0, :s "abc}',
    "not a map": '[1 2] {:type :invoke, :f :txn, :value [[:r 1 nil]], :process 0}',
    "transfer completion with a nil value": '{:type :invoke, :f :txn, :value [[:t 1 {:debit-acct 1, :credit-acct 2, '
                                            ':amount 3}]], :process 0}\n{:type :info, :f :txn, :value nil, :process 0}',
    "transfer completion with an empty value": '{:type :invoke, :f :txn, :value [[:t 1 {:debit-acct 1, :credit-acct 2, '
                                               ':amount 3}]], :process 0}\n{:type :ok, :f :txn, :value [], :process 0}',
    "ok read with a nil value": '{:type :invoke, :f :txn, :value [[:r 1 nil]], :process 0}\n'
                                '{:type :ok, :f :txn, :value nil, :process 0}',
    "ok read with a false value": '{:type :invoke, :f :txn, :value [[:r 1 nil]], :process 0}\n'
                                  '{:type :ok, :f :txn, :value false, :process 0}',
    "odd op map": '{:type}',
    "odd op map ending in a key": '{:type :invoke, :f :txn, :value [[:r 1 nil]], :a 1 :process}',
    "odd op map before another op": '{:type :invoke, :process}\n{:type :invoke, :f :txn, :value [[:r 1 nil]], :process 0}',
}
PYTHON_ACCEPTS = {"comment", "discard", "character literal", "float"}   # EDN outside the store's subset


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(ERRORS))
def test_errors(gpu_ctx, name):
    """rc < 0 wherever the Python path raises (and on EDN outside the store's subset), the history otherwise; the
    context reads the next history either way."""
    data = ERRORS[name].encode()
    refused = 0
    for form in FORMS:
        try:
            p = _python(data, form)
        except Exception:   # noqa: BLE001
            p = None
        if p is None or name in PYTHON_ACCEPTS:
            with pytest.raises(NativeError, match="history.edn"):
                gpu_ctx.read_ledger_edn(data, form)
            refused += 1
        else:
            _same(gpu_ctx.read_ledger_edn(data, form), p, (name, form))
        _ok_after(gpu_ctx)
    assert refused >= 1, name


@pytest.mark.gpu
def test_empty_ok_lookup_in_the_bank_forms(gpu_ctx):
    text = ('{:type :invoke, :f :txn, :value [[:l-t 1 nil]], :process 0}\n'
            '{:type :ok, :f :txn, :value [], :process 0}\n').encode()
    for form in ("bank", "ledger-counters"):
        with pytest.raises(IndexError):
            _python(text, form)
        with pytest.raises(NativeError):
            gpu_ctx.read_ledger_edn(text, form)
    _check(gpu_ctx, text, forms=("ledger-lookups",))


@pytest.mark.gpu
def test_checks_agree_on_the_device_form(gpu_ctx):
    spec = synth.SynthSpec("bank", 2000, 16, 2, p_info=0.02, tau_think_ns=10e6, final_reads=True)
    data = stored.write_edn(stored.generate_ledger_ops(spec, p_lookup=0.05))
    m = H.make_model(H.MODEL_BANK, accounts=range(1, 9))
    for g, p in [(gpu_ctx.read_ledger_edn(data, f), _python(data, f)) for f in FORMS]:
        form = p.meta["model"]
        if form == "bank":
            assert gpu_ctx.check_bank_totals(g, m, 0) | {"seconds": 0, "seconds_kernel": 0} == \
                gpu_ctx.check_bank_totals(p, m, 0) | {"seconds": 0, "seconds_kernel": 0}
            continue
        calls = [gpu_ctx.check_monotonic_keys, gpu_ctx.check_counter_bounds]
        if form == "ledger-lookups":
            calls += [gpu_ctx.check_transfer_placement, gpu_ctx.check_lookup_witness]
        for call in calls:
            x, y = call(g), call(p)
            for r in (x, y):
                r.pop("seconds_kernel"), r.pop("seconds_total")
            assert x == y, call.__name__


@pytest.mark.gpu
def test_ledger_checker_on_a_stored_history(gpu_ctx):
    spec = synth.SynthSpec("bank", 1000, 8, 3, p_info=0.02, tau_think_ns=10e6, final_reads=True)
    data = stored.write_edn(stored.generate_ledger_ops(spec, p_lookup=0.05, nemesis_every=41))
    c = CK.ledger_checker(ctx=gpu_ctx, linear=False, monotonic=True, counter_bounds=True, transfer_lookups=True,
                          transfer_placement=True, lookup_witness=True)

    def strip(r):
        if isinstance(r, dict):
            return {k: strip(v) for k, v in r.items() if not k.startswith("seconds")}
        if isinstance(r, list):
            return [strip(v) for v in r]
        return r
    a = c.check({}, CK.StoredLedgerHistory(data, ctx=gpu_ctx))
    b = c.check({}, edn.read_history(data.decode()))
    assert strip(a) == strip(b)


@pytest.mark.gpu
def test_input_above_2_pow_31_bytes(gpu_ctx):
    """A small history's lines repeated with fresh indices past 2^31 bytes: checked on the counts and a sample of
    events, not through the Python reader."""
    spec = synth.SynthSpec("bank", 400, 8, 1, p_info=0.02, tau_think_ns=10e6, final_reads=True)
    ops = stored.generate_ledger_ops(spec, p_lookup=0.05)
    small = _python(stored.write_edn(ops), "ledger-lookups")
    n_ops = len(ops)
    width = 10   # :index written with a fixed width, so every copy of the block has the same length
    lines = [stored.op_line({**op, "index": 0}).replace(":index 0", ":index %0" + str(width) + "d") for op in ops]
    block = ("\n".join(lines) + "\n")
    copies = (1 << 31) // len(block % tuple(range(n_ops))) + 2
    assert copies * n_ops < (1 << 31)
    parts = []
    for k in range(copies):
        parts.append((block % tuple(range(k * n_ops, (k + 1) * n_ops))).encode())
    data = b"".join(parts)
    del parts
    assert len(data) > (1 << 31)
    g = gpu_ctx.read_ledger_edn(data, "ledger-lookups")
    ne, npl = small.n_events, small.payload.shape[0]
    assert g.n_events == copies * ne and g.payload.shape[0] == copies * npl
    for k in (0, 1, copies // 2, copies - 1):
        sl = slice(k * ne, (k + 1) * ne)
        for name in ("type", "f", "flags", "process", "time_ns", "a", "b", "c", "payload_len"):
            assert np.array_equal(getattr(g, name)[sl], getattr(small, name)), (k, name)
        assert np.array_equal(g.index[sl], small.index + k * n_ops)
        assert np.array_equal(g.payload_off[sl], small.payload_off + k * npl)
        assert np.array_equal(g.payload[k * npl:(k + 1) * npl], small.payload)
