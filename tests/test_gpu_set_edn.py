"""GPU tier: K20, the device reader of stored set-full histories, against edn.read_history(independent=True) +
flatten_ops(..., "set"), and the set-full workload checker on a StoredSetHistory."""
import numpy as np
import pytest

from jepsen_tigerbeetle_b200 import checker as CK
from jepsen_tigerbeetle_b200 import edn, stored, synth
from jepsen_tigerbeetle_b200 import history as H
from jepsen_tigerbeetle_b200.native import Context, NativeError

ARRAYS = ("type", "f", "flags", "process", "index", "time_ns", "a", "b", "c", "payload_off", "payload_len", "payload",
          "shard_off", "key_ids")

SET_EDN = """
[{:type :invoke, :f :add, :value [1 9], :process 0, :time 10, :index 0}
 {:type :invoke, :f :read, :value [2 nil], :process 1, :time 11, :index 1}
 {:type :ok, :f :add, :value [1 9], :process 0, :time 20, :index 2}
 #jepsen.history.Op{:type :ok, :f :read, :value [2 #{12 10 11}], :process 1, :time 30, :index 3}
 {:type :info, :f :start, :value nil, :process :nemesis, :time 31}
 {:type :invoke, :f :add, :value [2 13], :process 0, :time 40, :index 4}
 {:type :info, :f :add, :value [2 13], :process 0, :time 50, :index 5, :error :timeout}
 {:type :invoke, :f :read, :value [1 nil], :process 1, :time 60, :index 6, :final? true}
 {:type :ok, :f :read, :value [1 #{9}], :process 1, :time 70, :index 7, :final? true}]
"""


@pytest.fixture(scope="module")
def ctx():
    c = Context(device=0)
    yield c
    c.close()


def _python(data):
    return H.flatten_ops(edn.read_history(data if isinstance(data, str) else data.decode(), independent=True), "set")


def _same(g, p, where=""):
    for name in ARRAYS:
        x, y = getattr(g, name), getattr(p, name)
        assert x.dtype == y.dtype and np.array_equal(x, y), (where, name, x[:20], y[:20])
    assert g.meta == p.meta, where


def _check(ctx, text, where=""):
    data = text.encode() if isinstance(text, str) else text
    try:
        p = _python(data)
    except Exception:   # noqa: BLE001 - the device must refuse whatever the Python path refuses
        with pytest.raises(NativeError, match="history.edn"):
            ctx.read_set_edn(data)
        return None
    g = ctx.read_set_edn(data)
    _same(g, p, where)
    return g


def _ok_after(ctx):
    """the context still reads a history after an error"""
    _same(ctx.read_set_edn(SET_EDN.encode()), _python(SET_EDN))


@pytest.mark.gpu
def test_set_fixture(ctx):
    g = _check(ctx, SET_EDN)
    assert g.key_ids.tolist() == [1, 2] and g.payload.tolist() == [9, 10, 11, 12]
    _check(ctx, SET_EDN.strip()[1:-1])   # the same ops, one per line
    g = _check(ctx, "")                  # an empty history: one empty shard, key id -1
    assert g.shard_off.tolist() == [0, 0] and g.key_ids.tolist() == [-1]


@pytest.mark.gpu
@pytest.mark.parametrize("n_keys", [1, 8, 64])
@pytest.mark.parametrize("p_info", [0.0, 0.01])
@pytest.mark.parametrize("seed", [1, 2, 3])
def test_generated_histories(ctx, n_keys, p_info, seed):
    h = synth.config_c4(seed=seed, n_keys=n_keys, p_info=p_info, n_ops=3000 if n_keys > 1 else 1500)
    ops = stored.set_ops(h, nemesis_every=97)
    for vector, newline in ((False, "\n"), (True, "\n"), (False, "\r\n")):
        g = _check(ctx, stored.write_edn(ops, vector=vector, newline=newline), where=(seed, p_info, n_keys, vector))
        assert g is not None and g.n_shards == n_keys


def _line(**kw):
    return stored.op_line(kw)


@pytest.mark.gpu
def test_hand_cases(ctx):
    inv = '{:type :invoke, :f :read, :value [1 nil], :process 1, :index 0, :time 1}\n'
    cases = {
        "nil nil add-ok": inv + '{:type :invoke, :f :add, :value [3 5], :process 0, :index 1, :time 2}\n'
                                '{:type :ok, :f :add, :value [nil nil], :process 0, :index 2, :time 3}\n'
                                '{:type :ok, :f :add, :value [3 nil], :process 0, :index 3, :time 4}\n'
                                '{:type :ok, :f :add, :value nil, :process 0, :index 4, :time 5}',
        "empty sets": inv + '{:type :ok, :f :read, :value [1 #{}], :process 1, :index 1, :time 2}\n'
                            '{:type :ok, :f :read, :value [2 #{ }], :process 1, :index 2, :time 3}\n'
                            '{:type :ok, :f :read, :value [3 []], :process 1, :index 3, :time 4}',
        "unsorted sets": inv + '{:type :ok, :f :read, :value [1 #{5 3 9 -2 7 100 0}], :process 1, :index 1}\n'
                               '{:type :ok, :f :read, :value [1 #{41,40 , 39}], :process 1, :index 2}',
        "vectors and lists": inv + '{:type :ok, :f :read, :value [1 [5 3 5 3]], :process 1, :index 1}\n'
                                   '{:type :ok, :f :read, :value [2 (9 9 1)], :process 1, :index 2}\n'
                                   '{:type :ok, :f :read, :value (3 [2 1]), :process 1, :index 3}\n'
                                   '{:type :ok, :f :read, :value [4 4 4], :process 1, :index 4}\n'
                                   '{:type :ok, :f :read, :value [7], :process 1, :index 5}\n'
                                   '{:type :ok, :f :read, :value [], :process 1, :index 6}',
        "unkeyed last": '{:type :ok, :f :read, :value #{3 4}, :process 1, :index 0}\n'
                        '{:type :ok, :f :read, :value [-1 #{1}], :process 1, :index 1}\n'
                        '{:type :invoke, :f :add, :value 5, :process 2, :index 2}\n'
                        '{:type :invoke, :f :read, :value nil, :process 3, :index 3}\n'
                        '{:type :invoke, :f :read, :process 3, :index 4}\n'
                        '{:type :ok, :f :read, :value [nil #{2}], :process 3, :index 5}\n'
                        '{:type :invoke, :f :add, :value [-2 6], :process 2, :index 6}\n'
                        '{:type :invoke, :f :add, :value [nil 7], :process 2, :index 7}\n'
                        '{:type :ok, :f :read, :value (5 6 7), :process 1, :index 8}',
        "bounds": '{:type :invoke, :f :add, :value [9223372036854775807 2147483647], :process 0, :index 2147483647, '
                  ':time 9223372036854775807}\n'
                  '{:type :invoke, :f :add, :value [-9223372036854775808 -2147483648], :process -2147483648, '
                  ':index -2147483648, :time -9223372036854775808}\n'
                  '{:type :ok, :f :read, :value [0 #{-2147483648 2147483647 0}], :process 2147483647, :index 0}\n'
                  '{:type :ok, :f :read, :value [9223372036854775807N [2147483647N -1]], :process 1, :index 1}',
        "no index or time": '{:type :info, :process :nemesis, :f :start, :value nil}\n'
                            '{:type :invoke, :f :add, :value [1 2], :process 0}\n'
                            '{:type :ok, :f :add, :value [1 2], :process 0, :final? true}\n'
                            '{:type :invoke, :f :read, :value [1 nil], :process 0, :time 5}\n'
                            '{:type :ok, :f :read, :value [1 #{2}], :process 0, :index 9}',
        "tagged": '#jepsen.history.Op {:type :ok, :f :read, :value #t [1 #s #{#x 5 3N}], :process #p 1, :index #i 0}\n'
                  '{:type :invoke, :f :add, :value #t (2 #v 8), :process 0, :time #inst 4}',
        "strings": '{:type :info, :process :nemesis, :f :kill, :value "a ] } \\" \\\\ b", :n #{1 [2]}}\n'
                   '{:type :ok, :f :read, :value [1 #{1 2}], :process 0, :note "[3 #{4}]", :index 1}',
    }
    for name, text in cases.items():
        assert _check(ctx, text, where=name) is not None, name
    for final in (":yes", '"x"', '""', "[1]", "[]", "#{}", "{:a 1}", "0", "-0", "7N", "nil", "false", "#inst \"t\""):
        g = _check(ctx, inv + '{:type :ok, :f :read, :value [1 #{2}], :process 1, :index 1, :final? %s}' % final,
                   where=("final?", final))
        assert g is not None


@pytest.mark.gpu
def test_one_read_of_1e6_members(ctx):
    ids = np.random.default_rng(5).permutation(1_000_000) - 500_000
    text = ('{:type :invoke, :f :read, :value [3 nil], :process 0, :index 0, :final? true}\n'
            '{:type :ok, :f :read, :value [3 #{%s}], :process 0, :index 1, :final? true}\n'
            '{:type :ok, :f :read, :value [4 [%s]], :process 1, :index 2}\n'
            % (" ".join(map(str, ids)), " ".join(map(str, ids))))
    g = _check(ctx, text)
    assert g.payload_len.tolist() == [-1, 1_000_000, 1_000_000]
    assert np.array_equal(g.payload[:1_000_000], np.sort(ids)) and np.array_equal(g.payload[1_000_000:], ids)


ERRORS = {
    "f other than add or read": '{:type :invoke, :f :write, :value [1 2], :process 0}',
    "no f": '{:type :invoke, :value [1 2], :process 0}',
    "keyword key": '{:type :invoke, :f :add, :value [:a 2], :process 0}',
    "vector key": '{:type :invoke, :f :add, :value [[1] 2], :process 0}',
    "mixed keys": '{:type :invoke, :f :add, :value [1 2], :process 0}\n{:type :invoke, :f :add, :value ["k" 3], '
                  ':process 0}',
    "key outside int64": '{:type :invoke, :f :add, :value [9223372036854775808 2], :process 0}',
    "add outside int32": '{:type :invoke, :f :add, :value [1 2147483648], :process 0}',
    "add below int32": '{:type :invoke, :f :add, :value [1 -2147483649], :process 0}',
    "add keyword": '{:type :invoke, :f :add, :value [1 :x], :process 0}',
    "add set": '{:type :invoke, :f :add, :value [1 #{1}], :process 0}',
    "add vector": '{:type :invoke, :f :add, :value [1 2 3], :process 0}',
    "member outside int32": '{:type :ok, :f :read, :value [1 #{2147483648}], :process 0}',
    "member nil": '{:type :ok, :f :read, :value [1 #{nil}], :process 0}',
    "member keyword": '{:type :ok, :f :read, :value [1 [:a]], :process 0}',
    "member vector": '{:type :ok, :f :read, :value [1 #{[1 2]}], :process 0}',
    "read of an integer": '{:type :ok, :f :read, :value [1 5], :process 0}',
    "read of true": '{:type :ok, :f :read, :value true, :process 0}',
    "index outside int32": '{:type :invoke, :f :add, :value [1 2], :process 0, :index 2147483648}',
    "process outside int32": '{:type :invoke, :f :add, :value [1 2], :process 2147483648}',
    "time outside int64": '{:type :invoke, :f :add, :value [1 2], :process 0, :time 9223372036854775808}',
    "time nil": '{:type :invoke, :f :add, :value [1 2], :process 0, :time nil}',
    "unknown type": '{:type :done, :f :add, :value [1 2], :process 0}',
    "odd op map": '{:type :invoke, :f :add, :value [1 2], :process}',
    "not a map": '[1 2] {:type :invoke, :f :add, :value [1 2], :process 0}',
    "mismatched brackets": '{:type :invoke, :f :add, :value [1 2), :process 0}',
    # EDN outside the store's subset, and shapes the store never writes that the Python path accepts
    "comment": '; c\n{:type :invoke, :f :add, :value [1 2], :process 0}',
    "float": '{:type :invoke, :f :add, :value [1 2.0], :process 0}',
    "boolean key": '{:type :invoke, :f :add, :value [true 2], :process 0}',
    "string add": '{:type :invoke, :f :add, :value [1 "7"], :process 0}',
    "map read": '{:type :ok, :f :read, :value [1 {}], :process 0}',
    "string read": '{:type :ok, :f :read, :value [1 "12"], :process 0}',
    "repeated set member": '{:type :ok, :f :read, :value [1 #{2 3 2}], :process 0}',
    "boolean member": '{:type :ok, :f :read, :value [1 [true]], :process 0}',
    "dropped add with an index outside int32": '{:type :ok, :f :add, :value [1 nil], :process 0, :index 2147483648}',
}
PYTHON_ACCEPTS = {"comment", "float", "boolean key", "string add", "map read", "string read", "repeated set member",
                  "boolean member", "dropped add with an index outside int32"}


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(ERRORS))
def test_errors(ctx, name):
    """rc < 0 wherever the Python path raises, and on the known refusals; the context reads the next history either
    way."""
    data = ERRORS[name].encode()
    try:
        _python(data)
        accepted = True
    except Exception:   # noqa: BLE001
        accepted = False
    assert accepted == (name in PYTHON_ACCEPTS), name
    with pytest.raises(NativeError, match="history.edn"):
        ctx.read_set_edn(data)
    _ok_after(ctx)


def _strip(r):
    if isinstance(r, dict):
        return {k: _strip(v) for k, v in r.items() if not str(k).startswith("seconds")}
    if isinstance(r, list):
        return [_strip(v) for v in r]
    return r


@pytest.mark.gpu
@pytest.mark.parametrize("p_info", [0.0, 0.01])
@pytest.mark.parametrize("poisoned", [False, True])
def test_workload_checker_on_a_stored_history(ctx, poisoned, p_info):
    """The whole result map equals the Python path's.  set-full is INVALID on the poisoned key only; with p_info 0
    (no :info add that never took effect, which read-all-invoked-adds flags) so is the whole check."""
    # seeds where poison_c4's two dropped ids are :lost (at these sizes it depends on the seed)
    h = synth.config_c4(seed=3 if p_info == 0 else 4, n_keys=8, n_ops=12000, p_info=p_info)
    if poisoned:
        h = synth.poison_c4(h)
    data = stored.write_edn(stored.set_ops(h, nemesis_every=101))
    c = CK.set_full_workload_checker(ctx=ctx)
    stored_history = CK.StoredSetHistory(data, ctx=ctx)
    a = c.check({}, stored_history)
    assert stored_history._ops is None   # read on the device, never parsed in Python
    b = c.check({}, edn.read_history(data.decode(), independent=True))
    assert _strip(a) == _strip(b)
    poison = [int(h.key_ids[5])] if poisoned else []
    assert [k for k, r in a["results"].items() if r["set-full"]["valid?"] is not True] == poison
    if p_info == 0:
        assert a["failures"] == poison and a["valid?"] is (not poisoned)


@pytest.mark.gpu
def test_stored_set_history_api(ctx):
    data = SET_EDN.encode()
    s = CK.StoredSetHistory(data, ctx=ctx)
    assert s.flat() is s.flat("set")
    _same(s.flat(), _python(data))
    _same(edn.read_set_flat(data, ctx=ctx), _python(data))
    assert list(s) == edn.read_history(SET_EDN, independent=True) and len(s) == 9
    assert s[0]["value"] == (1, 9)
    with pytest.raises(ValueError):
        s.flat("bank")
    assert CK._flat(s, "set") is s.flat()
    with pytest.raises(ValueError, match="unknown :f"):
        CK._flat(s, "register")   # any other model flattens the op maps, and :add is not a register op


@pytest.mark.gpu
def test_stored_set_history_falls_back_where_the_device_refuses(ctx):
    """A known refusal (a repeated set member) is flattened from the op maps; a file the Python path rejects raises."""
    data = (SET_EDN.strip()[1:-1] + '\n{:type :ok, :f :read, :value [2 #{11 11}], :process 1, :index 8}').encode()
    s = CK.StoredSetHistory(data, ctx=ctx)
    _same(s.flat(), _python(data))
    assert "repeated member" in s.refused
    c = CK.set_full_workload_checker(ctx=ctx)
    assert _strip(c.check({}, CK.StoredSetHistory(data, ctx=ctx))) == _strip(c.check({}, list(s)))
    bad = CK.StoredSetHistory(ERRORS["add outside int32"].encode(), ctx=ctx)
    with pytest.raises(OverflowError):
        bad.flat()
    assert "int32" in bad.refused
    _ok_after(ctx)

