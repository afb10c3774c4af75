"""H100-native history checker for Jepsen-style tests (drop-in for the checker hot path of
nurturenature/jepsen-tigerbeetle).  See DESIGN.md.  The compute path is the CUDA library
`libjtb_check.so` (csrc/); there is no CPU fallback."""
from . import abi, history, synth  # noqa: F401

__version__ = "0.1.0"
