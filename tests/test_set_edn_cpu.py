"""CPU tier for K20 (the device reader of stored set-full histories): the set-full op maps `stored.set_ops` writes
read back through edn.read_history(independent=True) + flatten_ops, the binding, and the kernels compiled for
sm_90a."""
import os
import shutil
import subprocess

import numpy as np
import pytest

from jepsen_tigerbeetle_b200 import checker as CK
from jepsen_tigerbeetle_b200 import edn, native, stored, synth
from jepsen_tigerbeetle_b200 import history as H

CSRC = os.path.join(os.path.dirname(__file__), "..", "jepsen_tigerbeetle_b200", "csrc")

HISTORIES = {
    "c1": lambda: synth.config_c1(seed=1),
    "c4 K=1": lambda: synth.config_c4(seed=2, n_keys=1, n_ops=800),
    "c4 K=8": lambda: synth.config_c4(seed=3, n_keys=8, n_ops=2000),
    "c4 K=64": lambda: synth.config_c4(seed=4, n_keys=64, n_ops=3000),
    "c4 K=8 poisoned": lambda: synth.poison_c4(synth.config_c4(seed=5, n_keys=8, n_ops=3000)),
}


def _expect(h):
    """h as flatten_ops spells it: the payload packed, adds without a payload (-1) and reads with a = 0"""
    r = h.select_shards(range(h.n_shards))
    add = r.f == H.F_ADD
    r.payload_len = np.where(add, -1, r.payload_len).astype(np.int32)
    r.a = np.where(add, r.a, 0).astype(np.int32)
    return r


@pytest.mark.parametrize("vector", [False, True])
@pytest.mark.parametrize("tagged", [False, True])
@pytest.mark.parametrize("name", sorted(HISTORIES))
def test_set_ops_round_trip(name, vector, tagged):
    h = HISTORIES[name]()
    ops = stored.set_ops(h, nemesis_every=13)
    assert any(op["process"] == "nemesis" for op in ops)
    text = stored.write_edn(ops, vector=vector, tagged=tagged).decode()
    assert edn.read_history(text, independent=True) == ops
    f, r = H.flatten_ops(edn.read_history(text, independent=True), "set"), _expect(h)
    for arr in ("type", "f", "flags", "process", "index", "time_ns", "a", "b", "c", "payload_len", "payload",
                "shard_off", "key_ids"):
        assert np.array_equal(getattr(f, arr), getattr(r, arr)), arr
    reads = r.payload_len >= 0
    assert np.array_equal(f.payload_off[reads], r.payload_off[reads])


def test_set_ops_shapes():
    """the op shapes of workloads/set_full.clj: [k id] adds, [k nil] read invokes, [k #{...}] :ok reads, :final? reads"""
    ops = stored.generate_set_ops(synth.SynthSpec("set", 200, 4, 1, p_info=0.1, n_keys=2, final_reads=True))
    kinds = {(op["f"], op["type"], type(op["value"][1]).__name__) for op in ops}
    assert {("add", "invoke", "int"), ("read", "invoke", "NoneType"), ("read", "ok", "frozenset")} <= kinds
    assert all(isinstance(op["value"], tuple) and op["value"][0] in (1, 2) for op in ops)
    assert any(op.get("final?") for op in ops) and any(op.get("error") == "timeout" for op in ops)
    assert stored.op_line(ops[0], tagged=False).startswith("{:index 0, :time ")
    with pytest.raises(ValueError):
        stored.generate_set_ops(synth.SynthSpec("bank", 10, 2, 1))


def test_stored_set_history_reads_op_maps_as_tuples():
    text = '{:type :ok, :f :read, :value [3 #{2 1}], :process 0, :index 0}\n'
    s = CK.StoredSetHistory(text.encode())
    assert s[0]["value"] == (3, frozenset({1, 2})) and len(s) == 1
    assert CK.StoredLedgerHistory(text.encode())[0]["value"] == [3, frozenset({1, 2})]


def test_binding_exists():
    assert "jtb_read_set_edn" in native.EXPORTS and "jtb_set_edn.cuh" in native._DEPS
    assert callable(getattr(native.Context, "read_set_edn"))
    assert native.lib().jtb_read_set_edn is not None


NEW_KERNELS = ("set_op_kernel", "set_item_kernel", "set_event_kernel", "set_member_kernel", "set_key_kernel",
               "set_order_kernel", "set_write_events_kernel", "set_sort_key_kernel", "set_repeat_kernel")


@pytest.mark.skipif(shutil.which("nvcc") is None, reason="needs nvcc")
def test_kernels_compile_for_sm_90a_without_spills(tmp_path):
    src = tmp_path / "set_edn.cu"
    src.write_text('#include "%s/jtb_set_edn.cuh"\n' % os.path.abspath(CSRC))
    out = subprocess.run(["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v",
                          "-c", str(src), "-o", str(tmp_path / "set_edn.o")], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr[-4000:]
    props = {}   # the reader's own kernels (jtb::set_*, and the partition's jtb::pt_*): their "Function properties"
    lines = out.stderr.splitlines()
    for i, line in enumerate(lines):
        if "Function properties for _ZN3jtb" in line and ("set_" in line or "pt_" in line) and i + 1 < len(lines):
            props[line.split()[-1]] = lines[i + 1]
    for k in NEW_KERNELS + ("pt_init", "pt_heads", "pt_emit"):
        assert any(k in name for name in props), k
    assert all(" 0 bytes spill stores" in v for v in props.values()), props
