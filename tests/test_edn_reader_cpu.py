"""CPU tier for K18 (the device reader of stored ledger histories): the EDN writer and the ledger op-map generator it
is tested with, the witness re-checkers on the generator's histories, the ABI image of the new struct, and the kernels
compiled for sm_90a."""
import ctypes
import os
import shutil
import subprocess

import pytest

import mono_oracle as M
from jepsen_tigerbeetle_b200 import abi, edn, stored, synth
from jepsen_tigerbeetle_b200 import history as H
from lookup_witness import verify as verify_lookups
from serial_witness import verify as verify_serial

CSRC = os.path.join(os.path.dirname(__file__), "..", "jepsen_tigerbeetle_b200", "csrc")


def _spec(seed, p_info=0.02, n=600):
    return synth.SynthSpec("bank", n, 8, seed, p_info=p_info, tau_think_ns=10e6, final_reads=True)


@pytest.mark.parametrize("vector", [False, True])
@pytest.mark.parametrize("tagged", [False, True])
def test_writer_round_trips_through_read_history(vector, tagged):
    ops = stored.generate_ledger_ops(_spec(1), p_lookup=0.05, nemesis_every=7)
    assert any(op["process"] == "nemesis" for op in ops)
    assert edn.read_history(stored.write_edn(ops, vector=vector, tagged=tagged).decode()) == ops


def test_writer_writes_the_store_format():
    op = {"type": "ok", "f": "txn", "value": [["t", 1, {"debit-acct": 1, "credit-acct": 2, "amount": 3}]],
          "process": 0, "index": 7, "time": 9, "node": "n1 b", "final?": True}
    assert stored.op_line(op) == ('#jepsen.history.Op{:index 7, :time 9, :type :ok, :process 0, :f :txn, '
                                  ':value [[:t 1 {:debit-acct 1, :credit-acct 2, :amount 3}]], :node "n1 b", '
                                  ':final? true}')
    assert stored.write_edn([op, op], newline="\r\n").count(b"\r\n") == 2


def test_generated_ops_flatten_to_the_generated_history():
    """flatten_ops of the generator's op maps gives synth's ledger-lookups history: the same events, payloads of the
    reads and lookups, and transfer records."""
    for seed, p_lookup in ((1, 0.0), (2, 0.05)):
        h = synth.generate_ledger_lookups(_spec(seed), p_lookup=p_lookup)
        f = H.flatten_ops(stored.ledger_ops(h, nemesis_every=11), "ledger-lookups")
        for name in ("type", "f", "flags", "process", "index", "time_ns"):
            assert (getattr(f, name) == getattr(h, name)).all(), name
        has = h.payload_len > 0
        assert (f.payload_len[has] == h.payload_len[has]).all()
        tr = h.f == H.F_TRANSFER
        assert (f.a[tr] == h.a[tr]).all() and (f.b[tr] == h.b[tr]).all() and (f.c[tr] == h.c[tr]).all()
        assert sorted(f.payload.tolist()) == sorted(h.payload.tolist())


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_generated_histories_pass_the_witness_rechecks(seed):
    """Where the oracle proves a generated history (read back from its EDN), the independent verifiers accept the
    proof."""
    ops = stored.generate_ledger_ops(_spec(seed), p_lookup=0.05, nemesis_every=13)
    h = H.flatten_ops(edn.read_history(stored.write_edn(ops).decode()), "ledger-lookups")
    sw = M.check_serial_witness(h)
    verify_serial(h, sw)
    lk = M.check_lookup_witness(h)
    verify_lookups(h, lk)
    assert lk["valid"] == H.VALID and lk["n_lookups_placed"] > 0


def test_abi_image_of_the_edn_history():
    from jepsen_tigerbeetle_b200 import native
    lib = native.lib()
    assert lib.jtb_struct_size(33) == ctypes.sizeof(abi.CEdnHistory)
    assert lib.jtb_struct_size(29) == lib.jtb_struct_size(32) == -1
    assert abi.FORMS == {"bank": 0, "ledger-counters": 1, "ledger-lookups": 2}


@pytest.mark.skipif(shutil.which("nvcc") is None, reason="needs nvcc")
def test_kernels_compile_for_sm_90a_without_spills(tmp_path):
    src = tmp_path / "edn.cu"
    src.write_text('#include "%s/jtb_edn.cuh"\n' % os.path.abspath(CSRC))
    out = subprocess.run(["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v",
                          "-c", str(src), "-o", str(tmp_path / "edn.o")], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr[-4000:]
    props = {}   # the reader's own kernels (jtb::edn_*): spill stores from their "Function properties" entry
    lines = out.stderr.splitlines()
    for i, line in enumerate(lines):
        if "Function properties for _ZN3jtb" in line and "edn_" in line and i + 1 < len(lines):
            props[line.split()[-1]] = lines[i + 1]
    for k in ("edn_byte_check_kernel", "edn_op_kernel", "edn_item_kernel", "edn_contrib_kernel",
              "edn_write_payload_kernel"):
        assert any(k in name for name in props), k
    assert len(props) >= 15 and all(" 0 bytes spill stores" in v for v in props.values()), props
