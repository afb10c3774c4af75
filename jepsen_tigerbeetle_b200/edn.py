"""Minimal EDN reader for stored Jepsen histories (`store/<test>/<time>/history.edn`).

SURVEY §8(f) N1: lets real histories recorded by the reference (op shapes of
src/tigerbeetle/workloads/set_full.clj:29-31,114-134 and workloads/ledger.clj:40-78) be re-checked on the
GPU without a JVM.  Supports the EDN subset Jepsen writes: nil/true/false, integers (incl. `N`), floats,
strings, keywords, symbols, vectors, lists, maps, sets, `#_` discard, `;` comments, commas, and tagged
literals (`#jepsen.history.Op{...}`, `#inst "..."`: the tag is dropped, the value kept).

Keywords become plain strings without the colon (`:invoke` -> "invoke"); maps -> dict, vectors/lists ->
list, sets -> frozenset.  `read_history` yields the op maps `history.flatten_ops` consumes.
"""
from __future__ import annotations

from typing import Any, Iterable, Iterator

_WS = set(" \t\r\n,")
_DELIM = set("()[]{}\"; \t\r\n,")


class EDNError(ValueError):
    pass


class _Reader:
    def __init__(self, text: str) -> None:
        self.s = text
        self.i = 0
        self.n = len(text)

    def skip(self) -> None:
        s, n = self.s, self.n
        while self.i < n:
            c = s[self.i]
            if c in _WS:
                self.i += 1
            elif c == ";":
                while self.i < n and s[self.i] != "\n":
                    self.i += 1
            elif c == "#" and self.i + 1 < n and s[self.i + 1] == "_":
                self.i += 2
                self.read()  # discard next form
            else:
                return

    def at_end(self) -> bool:
        self.skip()
        return self.i >= self.n

    def read(self) -> Any:
        self.skip()
        if self.i >= self.n:
            raise EDNError("unexpected end of input")
        c = self.s[self.i]
        if c == "{":
            self.i += 1
            items = self._seq("}")
            if len(items) % 2:
                raise EDNError("map with odd number of forms")
            return {_hashable(items[k]): items[k + 1] for k in range(0, len(items), 2)}
        if c == "[":
            self.i += 1
            return self._seq("]")
        if c == "(":
            self.i += 1
            return self._seq(")")
        if c == '"':
            return self._string()
        if c == "#":
            if self.i + 1 < self.n and self.s[self.i + 1] == "{":
                self.i += 2
                return frozenset(_hashable(x) for x in self._seq("}"))
            # tagged literal: drop the tag, keep the value
            self.i += 1
            self._token()
            return self.read()
        if c == "\\":
            self.i += 1
            tok = self._token()
            return {"newline": "\n", "space": " ", "tab": "\t", "return": "\r"}.get(tok, tok)
        tok = self._token()
        return _atom(tok)

    def _seq(self, close: str) -> list:
        out = []
        while True:
            self.skip()
            if self.i >= self.n:
                raise EDNError(f"missing {close!r}")
            if self.s[self.i] == close:
                self.i += 1
                return out
            out.append(self.read())

    def _string(self) -> str:
        self.i += 1
        out = []
        s = self.s
        while self.i < self.n:
            c = s[self.i]
            if c == '"':
                self.i += 1
                return "".join(out)
            if c == "\\":
                self.i += 1
                e = s[self.i]
                out.append({"n": "\n", "t": "\t", "r": "\r", '"': '"', "\\": "\\"}.get(e, e))
            else:
                out.append(c)
            self.i += 1
        raise EDNError("unterminated string")

    def _token(self) -> str:
        j = self.i
        s, n = self.s, self.n
        while j < n and s[j] not in _DELIM:
            j += 1
        if j == self.i:
            raise EDNError(f"unexpected character {s[self.i]!r} at {self.i}")
        tok = s[self.i:j]
        self.i = j
        return tok


def _hashable(x: Any) -> Any:
    if isinstance(x, list):
        return tuple(_hashable(y) for y in x)
    if isinstance(x, dict):
        return tuple(sorted((k, _hashable(v)) for k, v in x.items()))
    return x


def _atom(tok: str) -> Any:
    if tok == "nil":
        return None
    if tok == "true":
        return True
    if tok == "false":
        return False
    if tok[0] == ":":
        return tok[1:]
    c = tok[0]
    if c.isdigit() or (c in "+-" and len(tok) > 1 and tok[1].isdigit()):
        t = tok[:-1] if tok[-1] in "NM" else tok
        try:
            return int(t)
        except ValueError:
            return float(t)
    return tok  # symbol


def loads(text: str) -> Any:
    """Parse one EDN form."""
    r = _Reader(text)
    v = r.read()
    if not r.at_end():
        raise EDNError("trailing forms; use loads_all")
    return v


def loads_all(text: str) -> Iterator[Any]:
    """Parse every top-level form (Jepsen writes one op map per line)."""
    r = _Reader(text)
    while not r.at_end():
        yield r.read()


def _tuplify(op: dict, independent: bool) -> dict:
    v = op.get("value")
    if independent and isinstance(v, list) and len(v) == 2:
        op = dict(op)
        op["value"] = (v[0], v[1])  # jepsen.independent/tuple prints as a 2-vector
    return op


def read_history(text_or_lines: str | Iterable[str], independent: bool = False) -> list[dict]:
    """history.edn -> list of op maps (client and nemesis ops alike; the flattener ignores non-integer
    :process).  independent=True turns 2-vector :value fields into (key, value) tuples, as the set-full
    workload writes them (set_full.clj:31,44,116,134)."""
    text = text_or_lines if isinstance(text_or_lines, str) else "\n".join(text_or_lines)
    forms = list(loads_all(text))
    if len(forms) == 1 and isinstance(forms[0], list):
        forms = forms[0]  # a single vector of ops
    ops = []
    for f in forms:
        if not isinstance(f, dict):
            raise EDNError("history entries must be maps")
        ops.append(_tuplify(f, independent))
    return ops


def read_ledger_flat(path, form: str, ctx=None):
    """history.edn (a path or its bytes) -> the FlatHistory flatten_ops(read_history(text), form) makes, for the ledger
    forms "bank", "ledger-counters" and "ledger-lookups", read on the GPU (K18, `Context.read_ledger_edn`).  ctx: a
    native.Context to use; None opens one on device 0 for this call."""
    from . import native
    if ctx is not None:
        return ctx.read_ledger_edn(path, form)
    with native.Context(device=0) as c:
        return c.read_ledger_edn(path, form)


def read_set_flat(path, ctx=None):
    """history.edn (a path or its bytes) of a set-full test -> the FlatHistory
    flatten_ops(read_history(text, independent=True), "set") makes, one shard per key, read on the GPU (K20,
    `Context.read_set_edn`).  ctx: a native.Context to use; None opens one on device 0 for this call."""
    from . import native
    if ctx is not None:
        return ctx.read_set_edn(path)
    with native.Context(device=0) as c:
        return c.read_set_edn(path)
