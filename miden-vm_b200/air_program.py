"""Builder for the AIR constraint op-list consumed by `mdn_air.program` (include/miden_b200.h).

The reference evaluates `LiftedAir::eval(builder)` -- generic Rust -- at every quotient-domain point
(crates/lifted-stark/src/prover/constraints/mod.rs:233).  A C-ABI backend cannot call that, so the
host lowers `eval` once into a DAG over the leaf/op vocabulary the reference itself enumerates in
crates/ace-codegen/src/dag/lower.rs:109-210 and ships it as a flat list.  This module is the
host-side constructor of that list (what the Rust shim's `SymbolicAirBuilder` capture would emit);
`dummy_miden_air` restates crates/lifted-stark/src/testing/airs/miden.rs:57-62.
"""
from __future__ import annotations

import numpy as np

P = 0xFFFFFFFF00000001
MAGIC = 0x5249414D

OP_MAIN, OP_AUX, OP_PUBLIC, OP_CHALLENGE, OP_AUX_VALUE = 0, 1, 2, 3, 4
OP_IS_FIRST, OP_IS_LAST, OP_IS_TRANSITION, OP_CONST, OP_EXT_CONST = 5, 6, 7, 8, 9
OP_ADD, OP_SUB, OP_MUL, OP_NEG, OP_PERIODIC, OP_PREPROCESSED = 10, 11, 12, 13, 14, 15


class Expr:
    __slots__ = ("b", "id")

    def __init__(self, b: "ProgramBuilder", id_: int):
        self.b, self.id = b, id_

    def _bin(self, op, other):
        if not isinstance(other, Expr):
            other = self.b.const(int(other))
        return self.b._node(op, self.id, other.id)

    def __add__(self, o): return self._bin(OP_ADD, o)
    def __sub__(self, o): return self._bin(OP_SUB, o)
    def __mul__(self, o): return self._bin(OP_MUL, o)
    def __neg__(self): return self.b._node(OP_NEG, self.id, 0)


class ProgramBuilder:
    """Mirrors the builder surface an AIR sees (main/aux windows, selectors, public values,
    randomness, permutation values, assert_zero / assert_zero_ext)."""

    def __init__(self):
        self.nodes: list[tuple[int, int, int]] = []
        self.constraints: list[int] = []
        self.consts: list[int] = []

    def _node(self, op, a=0, b=0) -> Expr:
        self.nodes.append((op, a, b))
        return Expr(self, len(self.nodes) - 1)

    def main(self, offset: int, col: int) -> Expr: return self._node(OP_MAIN, offset, col)
    def aux(self, offset: int, col: int) -> Expr: return self._node(OP_AUX, offset, col)
    def public(self, i: int) -> Expr: return self._node(OP_PUBLIC, i)
    def challenge(self, i: int) -> Expr: return self._node(OP_CHALLENGE, i)
    def aux_value(self, i: int) -> Expr: return self._node(OP_AUX_VALUE, i)
    def is_first_row(self) -> Expr: return self._node(OP_IS_FIRST)
    def is_last_row(self) -> Expr: return self._node(OP_IS_LAST)
    def is_transition(self) -> Expr: return self._node(OP_IS_TRANSITION)
    def periodic(self, col: int) -> Expr: return self._node(OP_PERIODIC, col)
    def preprocessed(self, offset: int, col: int) -> Expr: return self._node(OP_PREPROCESSED, offset, col)

    def const(self, v: int) -> Expr:
        self.consts.append(v % P)
        return self._node(OP_CONST, len(self.consts) - 1)

    def ext_const(self, c0: int, c1: int) -> Expr:
        self.consts += [c0 % P, c1 % P]
        return self._node(OP_EXT_CONST, len(self.consts) - 2)

    def assert_zero(self, e: Expr): self.constraints.append(e.id)
    assert_zero_ext = assert_zero

    def serialize(self) -> np.ndarray:
        w = [MAGIC, 1, len(self.nodes), len(self.constraints), len(self.consts)]
        for n in self.nodes:
            w += list(n)
        w += self.constraints
        for c in self.consts:
            w += [c & 0xFFFFFFFF, c >> 32]
        return np.array(w, dtype=np.uint32)


LOOKUP_MAGIC = 0x504B4C4D
NO_FLAG = 0xFFFFFFFF


class LookupProgramBuilder(ProgramBuilder):
    """Host-side lowering of `LookupAir::eval` (air/src/lookup/builder.rs) for the device aux build: the node
    surface a `LookupBuilder` exposes (main window, preprocessed window `preprocessed(offset, col)` -- the AIR must
    declare preprocessed columns --, periodic values, challenges alpha = challenge(0) and beta = challenge(1),
    constants) and one record per interaction -- `insert(column, flag, multiplicity,
    denominator)` is `LookupGroup::insert` / `LookupBatch::insert` after `LookupMessage::encode`.

    With `num_registers` > 0 the program also builds register columns after the LogUp ones (a version-2 program, as
    the uint chiplets' Schwartz-Zippel columns): aux column num_columns + i is register i, 0 on row 0 and
    `update(i, expr)` evaluated on row r at row r + 1.  `register(i)` is register i's row-r value, readable by updates
    only, and every update must be affine in the registers."""

    def __init__(self, num_columns: int, num_registers: int = 0):
        super().__init__()
        self.num_columns = num_columns
        self.num_registers = num_registers
        self.updates: list[int | None] = [None] * num_registers
        self.interactions: list[tuple[int, int, int, int]] = []
        # mutual-exclusion annotation of every interaction (mdn_check_trace_balance): NO_FLAG, or group << 16 | site
        self.sites: list[int] = []
        self._groups = [0] * num_columns       # next group index per column (the reference's group_idx)
        self._group = None                     # (column, group index, cached, next site) of the open group
        self._batch_site = None
        # fold annotation of every interaction (mdn_check_lookup_folds): 3 opens a group, 1 an insert / batch, 0 continues a batch
        self.marks: list[int] = []
        self._opens = 3                        # what the next insert opens

    class _Scope:
        def __init__(self, enter, leave):
            self._enter, self._leave = enter, leave

        def __enter__(self):
            return self._enter()

        def __exit__(self, *exc):
            self._leave()

    def group(self, column: int, cached: bool = False):
        """`with b.group(c, cached)`: the inserts inside belong to the next group of column c (`LookupColumn::group`, or
        `group_with_cached_encoding` when cached: then every insert / batch inside is one mutual-exclusion site)."""
        def enter():
            assert self._group is None, "groups do not nest"
            self._group = [column, self._groups[column], cached, 0]
            self._groups[column] += 1
            self._opens = 3
            return self._group[1]

        def leave():
            self._group = None
            self._opens = 3
        return self._Scope(enter, leave)

    def batch(self):
        """`with b.batch()`: the inserts inside are one `LookupGroup::batch` call (they share its flag): one site."""
        def enter():
            assert self._group is not None and self._batch_site is None
            self._batch_site = self._new_site()
            self._opens |= 1

        def leave():
            self._batch_site = None
            self._opens |= 1
        return self._Scope(enter, leave)

    def _new_site(self):
        g = self._group
        site = g[3]
        g[3] += 1
        return site

    def mutex_sites(self) -> np.ndarray:
        """One word per interaction for mdn_check_trace_balance: 0xFFFFFFFF outside a cached-encoding group, else
        (group index within its column) << 16 | site."""
        return np.array(self.sites, dtype=np.uint32)

    def fold_marks(self) -> np.ndarray:
        """One word per interaction for mdn_check_lookup_folds: 3 when it opens a group (an insert outside `group` is a
        group of its own), 1 when it opens an insert or batch in the open group, 0 when it continues the open batch."""
        return np.array(self.marks, dtype=np.uint32)

    def bus_prefix(self, bus: int, max_message_width: int) -> Expr:
        """`Challenges::new`: bus_prefix[i] = alpha + (i + 1) * beta^W (air/src/lookup/challenges.rs)."""
        beta = self.challenge(1)
        g = beta
        for _ in range(max_message_width - 1):
            g = g * beta
        return self.challenge(0) + g * self.const(bus + 1)

    def encode(self, bus: int, max_message_width: int, elems) -> Expr:
        """`Challenges::encode`: bus_prefix[bus] + sum_i beta^i * elems[i]."""
        acc = self.bus_prefix(bus, max_message_width)
        bp = None
        for i, e in enumerate(elems):
            bp = self.const(1) if i == 0 else (self.challenge(1) if i == 1 else bp * self.challenge(1))
            acc = acc + (e if i == 0 else bp * e)
        return acc

    def insert(self, column: int, flag, multiplicity: Expr, denominator: Expr):
        self.interactions.append((column, NO_FLAG if flag is None else flag.id, multiplicity.id, denominator.id))
        g = self._group
        self.marks.append(self._opens)
        self._opens = 3 if g is None else (0 if self._batch_site is not None else 1)
        if g is None or not g[2]:
            self.sites.append(NO_FLAG)
            return
        assert g[0] == column, "an insert belongs to its group's column"
        site = self._batch_site if self._batch_site is not None else self._new_site()
        self.sites.append((g[1] << 16) | site)

    def register(self, i: int) -> Expr:
        """Register i's value on the current row (the AUX leaf of aux column num_columns + i, offset 0)."""
        return self._node(OP_AUX, 0, self.num_columns + i)

    def update(self, i: int, e: Expr):
        """Register i on the next row = `e` evaluated on the current row."""
        self.updates[i] = e.id

    def assert_zero(self, e):  # pragma: no cover - a lookup description emits no constraints
        raise TypeError("LookupBuilder has no assert_* surface")

    def serialize(self) -> np.ndarray:
        """Version 1 without registers; version 2 (an update node per register after the interactions) with them."""
        if self.num_registers:
            assert None not in self.updates, "every register needs an update"
            w = [LOOKUP_MAGIC, 2, len(self.nodes), len(self.interactions), len(self.consts), self.num_registers]
        else:
            w = [LOOKUP_MAGIC, 1, len(self.nodes), len(self.interactions), len(self.consts)]
        for n in self.nodes:
            w += list(n)
        for it in self.interactions:
            w += list(it)
        w += self.updates
        for c in self.consts:
            w += [c & 0xFFFFFFFF, c >> 32]
        return np.array(w, dtype=np.uint32)


def dummy_miden_air() -> np.ndarray:
    """`local[0] * local[1] * ... * local[8] == 0` (testing/airs/miden.rs:57-62): degree 9, so
    log_quotient_degree = 3.  The fold starts from ONE exactly like the reference's `fold`."""
    b = ProgramBuilder()
    acc = b.const(1)
    for j in range(9):
        acc = acc * b.main(0, j)
    b.assert_zero(acc)
    return b.serialize()
