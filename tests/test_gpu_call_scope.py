"""A device allocation that a call is refused ends with that call.  The CUDA runtime also keeps a refused cudaMalloc
as the thread's last error; a call that left it there made the next, unrelated call on the thread fail at its own
cudaGetLastError() check with a stale "out of memory".  Each case has a call refused its first large allocation, then
runs a monotonic-key check on the same context, which must succeed and equal the oracle."""
import ctypes as C

import numpy as np
import pytest

import mono_oracle as M
from jepsen_tigerbeetle_b200 import abi, native, synth
from jepsen_tigerbeetle_b200 import history as H

pytestmark = pytest.mark.gpu

HUGE = 1 << 40   # elements: no device holds them, so the allocation is refused before anything is copied


def refused_call(ctx, path):
    """rc and message of a call whose payload (or input arrays) claim HUGE elements.  The history has no events, so
    nothing reads the small host buffer that stands in for those arrays."""
    L = native.lib()
    word = np.zeros(4, dtype=np.int64)
    h = H.CHistory()
    h.payload = word.ctypes.data
    h.n_payload = HUGE
    if path == "bank_totals":
        model, res = H.make_model(H.MODEL_BANK, accounts=range(1, 9)), abi.CBankResult()
        rc = L.jtb_check_bank_totals(ctx._h, C.addressof(h), C.addressof(model), C.c_int64(0), C.addressof(res))
    elif path == "set_full":
        out = abi.CSetFullOut()
        rc = L.jtb_check_set_full(ctx._h, C.addressof(h), 1, C.addressof(out))
    else:
        p = C.c_void_p(word.ctypes.data)
        rc = L.jtb_ledger_balances(C.c_void_p(ctx._h), C.c_int64(HUGE), p, p, p)
    return rc, ctx._err()


@pytest.mark.parametrize("path", ["bank_totals", "set_full", "ledger_balances"])
def test_refused_allocation_does_not_fail_the_next_call(path):
    h = synth.generate_ledger_counters(synth.SynthSpec("bank", 2000, 16, 1, tau_think_ns=10e6))
    with native.Context(device=0) as ctx:
        rc, msg = refused_call(ctx, path)
        assert rc == -1 and "out of" in msg, (rc, msg)
        g, o = ctx.check_monotonic_keys(h), M.check_monotonic_keys(h, M.MONO_GRAPH)
        assert g["valid"] == H.VALID
        assert (g["valid"], g["shards"]) == (o["valid"], o["shards"])
