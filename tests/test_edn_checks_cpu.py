"""CPU tier for K19 (the host checks of a ledger compose on a stored history.edn): the ABI image of the new structs,
the kernels compiled for sm_90a, `StoredOp`, and the host assembly of the four checkers' results from a summary, fed
by the Python model in edn_checks_model.py."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import edn_checks_model as M
from jepsen_tigerbeetle_b200 import abi, edn, stored, synth
from jepsen_tigerbeetle_b200 import checker as CK

CSRC = os.path.join(os.path.dirname(__file__), "..", "jepsen_tigerbeetle_b200", "csrc")


def test_abi_image_of_the_edn_checks():
    from jepsen_tigerbeetle_b200 import native
    lib = native.lib()
    assert lib.jtb_struct_size(34) == ctypes.sizeof(abi.CEdnChecks)
    assert lib.jtb_struct_size(29) == lib.jtb_struct_size(32) == -1
    assert np.dtype(abi.EDN_FLAG_DTYPE).itemsize == ctypes.sizeof(abi.CEdnFlag) == 56
    assert [f for f, *_ in abi.EDN_FLAG_DTYPE] == [f for f, _ in abi.CEdnFlag._fields_]


@pytest.mark.skipif(shutil.which("nvcc") is None, reason="needs nvcc")
def test_kernels_compile_for_sm_90a_without_spills(tmp_path):
    src = tmp_path / "edn_checks.cu"
    src.write_text('#include "%s/jtb_edn_checks.cuh"\n' % os.path.abspath(CSRC))
    out = subprocess.run(["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v",
                          "-c", str(src), "-o", str(tmp_path / "edn_checks.o")], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr[-4000:]
    props = {}   # K19's own kernels (jtb::ec_*): spill stores from their "Function properties" entry
    lines = out.stderr.splitlines()
    for i, line in enumerate(lines):
        if re.search(r"Function properties for _ZN3jtb\d+ec_", line) and i + 1 < len(lines):
            props[line.split()[-1]] = lines[i + 1]
    for k in ("ec_item_kernel", "ec_op_digest_kernel", "ec_confirm_kernel", "ec_slot_kernel", "ec_suspect_kernel",
              "ec_record_kernel"):
        assert any(k in name for name in props), k
    assert len(props) >= 9 and all(" 0 bytes spill stores" in v for v in props.values()), props


@pytest.mark.parametrize("vector,tagged,newline", [(False, True, "\n"), (True, True, "\n"), (False, False, "\r\n"),
                                                   (True, False, "\r\n")])
def test_stored_op_parses_when_read(vector, tagged, newline):
    spec = synth.SynthSpec("bank", 300, 4, 1, p_info=0.02, tau_think_ns=10e6, final_reads=True)
    ops = stored.generate_ledger_ops(spec, p_lookup=0.05, nemesis_every=7)
    data = stored.write_edn(ops, vector=vector, tagged=tagged, newline=newline)
    spans = M.op_spans(data)
    assert len(spans) == len(ops)
    lazy = [CK.StoredOp(data, b, e) for b, e in spans]
    assert not any(op.parsed for op in lazy)
    repr(lazy[0])
    assert not lazy[0].parsed
    assert lazy == edn.read_history(data.decode()) and all(op.parsed for op in lazy)
    assert CK.StoredOp(data, *spans[3]) != ops[4]


@pytest.mark.parametrize("name", sorted(M.HAND_CASES))
def test_assembly_reproduces_the_checkers(name):
    data = M.HAND_CASES[name]
    ops = edn.read_history(data.decode())
    s = M.summarize(data)
    for c in (CK.UnexpectedOps, CK.LookupAllInvokedTransfers, CK.FinalReads):
        assert c.from_summary(s, data) == c().check({}, ops), c.__name__
    assert CK.Stats.from_summary(s) == CK.Stats().check({}, ops)


@pytest.mark.parametrize("p_info", [0.0, 0.02])
def test_assembly_on_generated_histories(p_info):
    spec = synth.SynthSpec("bank", 600, 8, 2, p_info=p_info, tau_think_ns=10e6, final_reads=True)
    data = stored.write_edn(stored.generate_ledger_ops(spec, p_lookup=0.05, nemesis_every=17))
    ops = edn.read_history(data.decode())
    s = M.summarize(data)
    for c in (CK.UnexpectedOps, CK.LookupAllInvokedTransfers, CK.FinalReads):
        assert c.from_summary(s, data) == c().check({}, ops), c.__name__
    assert CK.Stats.from_summary(s) == CK.Stats().check({}, ops)


def test_unequal_final_values_parse_one_op_per_class():
    data = M.HAND_CASES["unequal final reads and lookups"]
    s = M.summarize(data)
    parsed = []
    real = CK.StoredOp._map
    try:
        CK.StoredOp._map = lambda self: parsed.append(self._begin) or real(self)
        r = CK.FinalReads.from_summary(s, data)
    finally:
        CK.StoredOp._map = real
    assert len(r["unequal-final-reads"]) == s["n_read_classes"] == 3
    assert len(r["unequal-final-lookups"]) == s["n_lookup_classes"] == 3
    assert len(set(parsed)) == 6
    bad = dict(s, n_read_classes=2)   # a summary whose classes do not match the values trips the assertion
    with pytest.raises(AssertionError):
        CK.FinalReads.from_summary(bad, data)
