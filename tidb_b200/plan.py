"""Descriptor builders: the information executorBuilder hands to the operators.

JoinPlan mirrors what buildHashJoinV2FromChildExecs passes to HashJoinV2Exec
(pkg/executor/builder.go:1771-1931: child schemas, key column indices, LUsed/RUsed, JoinType,
RightAsBuildSide, Build/ProbeFilter); AggPlan mirrors buildHashAggFromChildExec
(builder.go:2106-2181: GroupByItems, AggFuncDescs).  Both render to the C-ABI structs of
include/tidbgpu.h.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field
from typing import List, Optional, Sequence, Tuple

from . import abi


UNSPECIFIED_LENGTH = -1   # types.UnspecifiedLength


@dataclass
class FieldType:
    """types.FieldType reduced to what the path needs: MySQL type code + flag bits, GetFlen() / GetDecimal() (the
    precision and scale of a DECIMAL column; -1 = not given) and GetCollate() (the MySQL collation id of a string column)."""
    tp: int = abi.TYPE_LONGLONG
    flag: int = 0
    flen: int = UNSPECIFIED_LENGTH
    decimal: int = UNSPECIFIED_LENGTH
    collation: int = abi.COLLATION_UTF8MB4_BIN

    @property
    def not_null(self) -> bool:
        return bool(self.flag & abi.FLAG_NOT_NULL)

    @property
    def unsigned(self) -> bool:
        return bool(self.flag & abi.FLAG_UNSIGNED)


def _i32(vals: Sequence[int]):
    return (C.c_int32 * max(len(vals), 1))(*vals)


def _u32(vals: Sequence[int]):
    return (C.c_uint32 * max(len(vals), 1))(*vals)


@dataclass
class FilterItem:
    """One CNF item `col OP const` / `col OP col` (tg_filter_item).  is_decimal: a DECIMAL item of tg_vec_filter_ex over
    40-byte MyDecimal cell columns, whose constant is the 40-byte cell const_cell (Constant.Value.GetMysqlDecimal()).
    is_string: a STRING item of tg_vec_filter_ex2 over var-length string columns: str_kind abi.STR_CMP compares with
    rhs_col or the constant const_bytes, abi.STR_LIKE / STR_NOT_LIKE match the pattern const_bytes with `escape`, under
    the MySQL collation id `collation`."""
    op: int
    lhs_col: int
    rhs_col: int = -1
    is_real: bool = False
    lhs_unsigned: bool = False
    const_i64: int = 0
    const_f64: float = 0.0
    rhs_unsigned: bool = False
    is_decimal: bool = False
    const_cell: Optional[bytes] = None
    is_string: bool = False
    const_bytes: Optional[bytes] = None
    collation: int = abi.COLLATION_UTF8MB4_BIN
    str_kind: int = abi.STR_CMP
    escape: int = ord("\\")

    def to_struct(self) -> abi.TgFilterItem:
        s = abi.TgFilterItem()
        s.op, s.lhs_col, s.rhs_col = self.op, self.lhs_col, self.rhs_col
        kind = abi.FILTER_STRING if self.is_string else (abi.FILTER_DECIMAL if self.is_decimal else int(self.is_real))
        s.is_real, s.lhs_unsigned = kind, int(self.lhs_unsigned)
        s.rhs_unsigned = int(self.rhs_unsigned)
        s.const_i64, s.const_f64 = self.const_i64, self.const_f64
        return s


def filter_array(items: Sequence[FilterItem]):
    arr = (abi.TgFilterItem * max(len(items), 1))()
    for i, it in enumerate(items):
        arr[i] = it.to_struct()
    return arr


def dec_const_array(items: Sequence[FilterItem]):
    """tg_vec_filter_ex's dec_consts: 40 bytes per item, item i's constant cell at byte 40 * i (zeros where an item has
    none); None when no item has a constant cell"""
    if not any(it.const_cell is not None for it in items):
        return None
    buf = bytearray(40 * len(items))
    for i, it in enumerate(items):
        if it.const_cell is not None:
            assert len(it.const_cell) == 40, "a DECIMAL constant is one 40-byte MyDecimal cell"
            buf[40 * i:40 * i + 40] = bytes(it.const_cell)
    return (C.c_uint8 * len(buf)).from_buffer(buf)


def str_arg_array(items: Sequence[FilterItem]):
    """tg_vec_filter_ex2's str_args: one tg_str_arg per item (zeros for the items that are not STRING); None when no item
    is STRING.  The constant and pattern buffers are kept alive on the array (`_keep`)."""
    if not any(it.is_string for it in items):
        return None
    arr = (abi.TgStrArg * len(items))()
    arr._keep = []
    for i, it in enumerate(items):
        if not it.is_string:
            continue
        b = bytes(it.const_bytes or b"")
        buf = (C.c_uint8 * max(len(b), 1)).from_buffer_copy(b.ljust(1, b"\0"))
        arr._keep.append(buf)
        arr[i].bytes = C.cast(buf, C.c_void_p) if b else None
        arr[i].len, arr[i].collation, arr[i].kind, arr[i].escape = len(b), it.collation, it.str_kind, it.escape
    return arr


@dataclass
class OtherCond:
    """One CNF item of HashJoinV2Exec.OtherCondition: `side.col OP side.col` (or a constant with rhs_side = -1) over the
    joined row; side 0 = left child, 1 = right child (tg_other_item)."""
    op: int
    lhs_side: int
    lhs_col: int
    rhs_side: int = -1
    rhs_col: int = -1
    is_real: bool = False
    lhs_unsigned: bool = False
    rhs_unsigned: bool = False
    const_i64: int = 0
    const_f64: float = 0.0

    def to_struct(self) -> abi.TgOtherItem:
        s = abi.TgOtherItem()
        s.op, s.is_real = self.op, int(self.is_real)
        s.lhs_side, s.lhs_col, s.rhs_side, s.rhs_col = self.lhs_side, self.lhs_col, self.rhs_side, self.rhs_col
        s.lhs_unsigned, s.rhs_unsigned = int(self.lhs_unsigned), int(self.rhs_unsigned)
        s.const_i64, s.const_f64 = self.const_i64, self.const_f64
        return s


@dataclass
class JoinPlan:
    join_type: int
    left_types: List[FieldType]
    right_types: List[FieldType]
    left_keys: List[int]
    right_keys: List[int]
    build_is_right: bool = True
    lused: Optional[List[int]] = None      # None = all columns (Go nil)
    rused: Optional[List[int]] = None
    build_filter: List[FilterItem] = field(default_factory=list)
    probe_filter: List[FilterItem] = field(default_factory=list)
    device: int = 0
    stream: int = 0
    load_factor: float = 0.0
    other_cond: List[OtherCond] = field(default_factory=list)

    def out_schema(self) -> List[FieldType]:
        lu = self.lused if self.lused is not None else list(range(len(self.left_types)))
        ru = self.rused if self.rused is not None else list(range(len(self.right_types)))
        out = [self.left_types[i] for i in lu] + [self.right_types[i] for i in ru]
        if self.join_type in (abi.JOIN_LEFT_OUTER_SEMI, abi.JOIN_ANTI_LEFT_OUTER_SEMI):
            out.append(FieldType(abi.TYPE_LONGLONG, 0))
        return out

    def to_struct(self) -> Tuple[abi.TgJoinDesc, list]:
        keep = []
        d = abi.TgJoinDesc()
        d.join_type = self.join_type
        d.build_is_right = int(self.build_is_right)
        d.n_left_cols, d.n_right_cols = len(self.left_types), len(self.right_types)
        for name, vals, mk in (("left_types", [t.tp for t in self.left_types], _i32),
                               ("left_flags", [t.flag for t in self.left_types], _u32),
                               ("right_types", [t.tp for t in self.right_types], _i32),
                               ("right_flags", [t.flag for t in self.right_types], _u32),
                               ("left_key_idx", self.left_keys, _i32),
                               ("right_key_idx", self.right_keys, _i32)):
            arr = mk(vals)
            keep.append(arr)
            setattr(d, name, arr)
        d.nkeys = len(self.left_keys)
        if self.lused is None:
            d.n_lused = -1
        else:
            arr = _i32(self.lused); keep.append(arr); d.lused = arr; d.n_lused = len(self.lused)
        if self.rused is None:
            d.n_rused = -1
        else:
            arr = _i32(self.rused); keep.append(arr); d.rused = arr; d.n_rused = len(self.rused)
        d.n_build_filter, d.n_probe_filter = len(self.build_filter), len(self.probe_filter)
        if self.build_filter:
            arr = filter_array(self.build_filter); keep.append(arr); d.build_filter = arr
        if self.probe_filter:
            arr = filter_array(self.probe_filter); keep.append(arr); d.probe_filter = arr
        d.device = self.device
        d.stream = self.stream or None
        d.load_factor = self.load_factor
        d.n_other_cond = len(self.other_cond)
        if self.other_cond:
            arr = (abi.TgOtherItem * len(self.other_cond))(*[o.to_struct() for o in self.other_cond]); keep.append(arr); d.other_cond = arr
        return d, keep


@dataclass
class AggFunc:
    name: int
    arg_col: int = -1
    arg_type: int = abi.TYPE_LONGLONG
    arg_flag: int = 0
    mode: int = abi.AGGMODE_COMPLETE
    arg_col2: int = -1
    arg_expr: int = 0          # abi.ARGEXPR_*: the argument as arg_col * arg_col2 / arg_col * (arg_const - arg_col2)
    arg_const: float = 0.0
    ret_type: int = 0          # AggFuncDesc.RetTp.GetType(): abi.TYPE_NEWDECIMAL = exact DECIMAL SUM / AVG of an integer
                               # column, or SUM / AVG / MIN / MAX of a DECIMAL column
    ret_frac: int = 0          # AggFuncDesc.RetTp.GetDecimal()
    distinct: bool = False     # AggFuncDesc.HasDistinct: COUNT / SUM / AVG of the distinct values (tg_agg_desc_ex2)


@dataclass
class AggPlan:
    col_types: List[FieldType]
    group_by: List[int]
    funcs: List[AggFunc]
    device: int = 0
    stream: int = 0
    expected_groups: int = 0

    def to_struct(self) -> Tuple[abi.TgAggDesc, list]:
        keep = []
        d = abi.TgAggDesc()
        d.n_cols, d.n_group_by = len(self.col_types), len(self.group_by)
        a = _i32([t.tp for t in self.col_types]); keep.append(a); d.col_types = a
        a = _u32([t.flag for t in self.col_types]); keep.append(a); d.col_flags = a
        a = _i32(self.group_by); keep.append(a); d.group_by_cols = a
        fa = (abi.TgAggFunc * max(len(self.funcs), 1))()
        for i, f in enumerate(self.funcs):
            fa[i].name, fa[i].mode, fa[i].arg_col = f.name, f.mode, f.arg_col
            fa[i].arg_type, fa[i].arg_flag, fa[i].arg_col2 = f.arg_type, f.arg_flag, f.arg_col2
            fa[i].arg_expr, fa[i].arg_const = f.arg_expr, f.arg_const
            fa[i].ret_type, fa[i].ret_frac = f.ret_type, f.ret_frac
        keep.append(fa)
        d.funcs = fa
        d.n_funcs = len(self.funcs)
        d.device = self.device
        d.stream = self.stream or None
        d.expected_groups = self.expected_groups
        return d, keep

    def to_struct_ex(self) -> Tuple[abi.TgAggDescEx, list]:
        """tg_agg_desc_ex: to_struct() plus the precision and scale of every child column"""
        d, keep = self.to_struct()
        ex = abi.TgAggDescEx()
        ex.base = d
        a = _i32([t.flen for t in self.col_types]); keep.append(a); ex.col_flen = a
        a = _i32([t.decimal for t in self.col_types]); keep.append(a); ex.col_decimal = a
        return ex, keep

    def to_struct_ex2(self) -> Tuple[abi.TgAggDescEx2, list]:
        """tg_agg_desc_ex2: to_struct_ex() plus HasDistinct per function (NULL when no function has it)"""
        ex, keep = self.to_struct_ex()
        d = abi.TgAggDescEx2()
        d.ex = ex
        if any(f.distinct for f in self.funcs):
            a = (C.c_uint8 * len(self.funcs))(*[int(f.distinct) for f in self.funcs]); keep.append(a); d.has_distinct = a
        return d, keep

    def to_struct_ex3(self) -> Tuple[abi.TgAggDescEx3, list]:
        """tg_agg_desc_ex3: to_struct_ex2() plus the collation id of every child column"""
        ex2, keep = self.to_struct_ex2()
        d = abi.TgAggDescEx3()
        d.ex2 = ex2
        a = _i32([t.collation for t in self.col_types]); keep.append(a); d.col_collation = a
        return d, keep

    def string_results(self) -> List[bool]:
        """per function: its result is a string column (FIRSTROW of a string column)"""
        return [f.name == abi.AGG_FIRSTROW and f.arg_col >= 0 and self.col_types[f.arg_col].tp in abi.STRING_TYPES for f in self.funcs]


# ---------------------------------------------------------------------------------------------------------------
# Scalar expressions for ProjectionExec (expression.Expression reduced to what the VecEval kernels offload)
# ---------------------------------------------------------------------------------------------------------------
class Expr:
    def ret_type(self, schema: Sequence[FieldType]) -> FieldType:
        raise NotImplementedError


@dataclass
class ColRef(Expr):
    """expression.Column: passed through (EvaluatorSuite swaps plain column references, evaluator.go:128)"""
    idx: int

    def ret_type(self, schema):
        return schema[self.idx]


@dataclass
class Const(Expr):
    """expression.Constant: handed to the kernels as a scalar (the reference materialises a column, vectorized.go:23).
    cell: a DECIMAL constant, its 40-byte MyDecimal cell (value is then not used).  bytes_value: a string constant (or
    a LIKE pattern), its bytes."""
    value: float = 0
    is_real: bool = False
    cell: Optional[bytes] = None
    bytes_value: Optional[bytes] = None

    def ret_type(self, schema):
        if self.bytes_value is not None:
            return FieldType(abi.TYPE_VARSTRING, abi.FLAG_NOT_NULL)
        if self.cell is not None:
            return FieldType(abi.TYPE_NEWDECIMAL, abi.FLAG_NOT_NULL)
        return FieldType(abi.TYPE_DOUBLE if self.is_real else abi.TYPE_LONGLONG, abi.FLAG_NOT_NULL)


@dataclass
class ScalarFunc(Expr):
    """builtinArithmetic{Plus,Minus,Multiply}{Int,Real}Sig / builtin{LT,LE,GT,GE,EQ,NE}{Int,Real,Decimal}Sig over two
    arguments (kind "arith": op = abi.ARITH_*, kind "cmp": op = abi.CMP_*); the right argument may be a Const.
    is_decimal (kind "cmp" only): both arguments are DECIMAL (cell columns; a Const with a cell).
    is_string (kind "cmp"): both arguments are strings (var-length columns; a Const with bytes_value), compared under the
    MySQL collation id `collation`.  Kind "like": builtinLikeSig, the first argument LIKE the Const pattern (bytes_value)
    with `escape`, under `collation`."""
    kind: str
    op: int
    args: Tuple[Expr, Expr]
    is_real: bool = False
    a_unsigned: bool = False
    b_unsigned: bool = False
    is_decimal: bool = False
    is_string: bool = False
    collation: int = abi.COLLATION_UTF8MB4_BIN
    escape: int = ord("\\")

    def ret_type(self, schema):
        if self.kind == "arith" and self.is_real:
            return FieldType(abi.TYPE_DOUBLE, 0)
        if self.kind == "arith" and (self.a_unsigned or self.b_unsigned):
            # integer +, - and * are UNSIGNED when either argument is (builtin_arithmetic.go:207, :378, :583)
            return FieldType(abi.TYPE_LONGLONG, abi.FLAG_UNSIGNED)
        return FieldType(abi.TYPE_LONGLONG, 0)
