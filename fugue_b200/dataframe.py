"""Host-side DataFrame types mirroring the reference's interface.

* ``DataFrame`` / ``LocalDataFrame``    fugue/dataframe/dataframe.py:29-299
* ``ArrowDataFrame`` / ``PandasDataFrame`` / ``ArrayDataFrame``
                                       fugue/dataframe/{arrow,pandas,array}_dataframe.py
  (all three are thin constructors over one pyarrow-backed local frame here)
* ``B200DataFrame``                    the engine's own frame: a ``B200Table`` in HBM,
  ``is_local == False`` so ``transform()`` hands back the device table
  (fugue/workflow/api.py:184) and ``as_local()`` is the explicit D2H.
* ``df_eq``                            fugue/dataframe/utils.py:24-94 (_df_eq)
"""
from typing import Any, Dict, Iterable, List, Optional

import pandas as pd
import pyarrow as pa

from .schema import Schema


class FugueDataFrameOperationError(Exception):
    pass


class FugueDatasetEmptyError(Exception):
    pass


class DataFrame:
    def __init__(self, schema: Any = None):
        self._schema = schema if isinstance(schema, Schema) else Schema(schema)
        self._metadata: Optional[Dict[str, Any]] = None

    # ---- Dataset (fugue/dataset/dataset.py:14-110) -------------------------------------
    @property
    def metadata(self) -> Dict[str, Any]:
        if self._metadata is None:
            self._metadata = {}
        return self._metadata

    @property
    def has_metadata(self) -> bool:
        return self._metadata is not None and len(self._metadata) > 0

    def reset_metadata(self, metadata: Any) -> None:
        self._metadata = dict(metadata) if metadata is not None else None

    @property
    def schema(self) -> Schema:
        return self._schema

    @property
    def columns(self) -> List[str]:
        return self._schema.names

    # ---- abstract ---------------------------------------------------------------------
    @property
    def native(self) -> Any:  # pragma: no cover
        raise NotImplementedError

    @property
    def is_local(self) -> bool:  # pragma: no cover
        raise NotImplementedError

    @property
    def is_bounded(self) -> bool:
        return True

    @property
    def num_partitions(self) -> int:
        return 1

    @property
    def empty(self) -> bool:
        return self.count() == 0

    def count(self) -> int:  # pragma: no cover
        raise NotImplementedError

    def as_arrow(self, type_safe: bool = False) -> pa.Table:  # pragma: no cover
        raise NotImplementedError

    # ---- derived ----------------------------------------------------------------------
    def as_local(self) -> "LocalDataFrame":
        return self.as_local_bounded()

    def as_local_bounded(self) -> "LocalDataFrame":
        res = ArrowDataFrame(self.as_arrow(), self.schema)
        if self.has_metadata:
            res.reset_metadata(self.metadata)
        return res

    def as_pandas(self) -> pd.DataFrame:
        return self.as_arrow().to_pandas()

    def as_array(self, columns: Optional[List[str]] = None, type_safe: bool = False) -> List[List[Any]]:
        t = self.as_arrow()
        if columns is not None:
            t = t.select(columns)
        cols = [c.to_pylist() for c in t.columns]
        return [list(r) for r in zip(*cols)] if cols else []

    def as_array_iterable(self, columns: Optional[List[str]] = None, type_safe: bool = False) -> Iterable[List[Any]]:
        return iter(self.as_array(columns, type_safe))

    def as_dicts(self, columns: Optional[List[str]] = None) -> List[Dict[str, Any]]:
        names = columns or self.columns
        return [dict(zip(names, r)) for r in self.as_array(columns)]

    def peek_array(self) -> List[Any]:
        if self.empty:
            raise FugueDatasetEmptyError("dataframe is empty")
        return self.head(1).as_array()[0]

    def peek_dict(self) -> Dict[str, Any]:
        return dict(zip(self.columns, self.peek_array()))

    def head(self, n: int, columns: Optional[List[str]] = None) -> "LocalDataFrame":
        t = self.as_arrow().slice(0, n)
        if columns is not None:
            t = t.select(columns)
        return ArrowDataFrame(t)

    def __getitem__(self, columns: List[Any]) -> "DataFrame":
        for c in columns:
            if c not in self._schema:
                raise FugueDataFrameOperationError(f"{c} not in {self._schema}")
        if len(columns) == 0:
            raise FugueDataFrameOperationError("must select at least one column")
        return self._select_cols(columns)

    def drop(self, columns: List[str]) -> "DataFrame":
        for c in columns:
            if c not in self._schema:
                raise FugueDataFrameOperationError(f"{c} not in {self._schema}")
        if len(columns) >= len(self._schema):
            raise FugueDataFrameOperationError("can't drop all columns")
        return self._select_cols([c for c in self.columns if c not in set(columns)])

    def _select_cols(self, columns: List[Any]) -> "DataFrame":  # pragma: no cover
        raise NotImplementedError

    def rename(self, columns: Dict[str, str]) -> "DataFrame":  # pragma: no cover
        raise NotImplementedError

    def native_as_df(self) -> Any:
        """The underlying dataframe object (fugue/dataframe/dataframe.py ``native_as_df``)."""
        return self.native

    def as_dict_iterable(self, columns: Optional[List[str]] = None) -> Iterable[Dict[str, Any]]:
        return iter(self.as_dicts(columns))

    def _altered_schema(self, columns: Any) -> Optional[Schema]:
        """Schema after ``alter_columns(columns)``; None when nothing changes
        (fugue/dataframe/dataframe.py ``alter_columns``: ``columns`` must be a subset of the schema)."""
        sub = Schema(columns)
        for f in sub.fields:
            if f.name not in self._schema:
                raise FugueDataFrameOperationError(f"{f.name} not in {self._schema}")
        new = self._schema.alter(sub)
        return None if new == self._schema else new

    def alter_columns(self, columns: Any) -> "DataFrame":
        """Change column data types; column order is kept."""
        new = self._altered_schema(columns)
        if new is None:
            return self
        try:
            return ArrowDataFrame(_cast_table(self.as_arrow(), new))
        except (pa.ArrowInvalid, pa.ArrowNotImplementedError) as e:
            raise FugueDataFrameOperationError(str(e)) from e

    def show(self, n: int = 10, with_count: bool = False, title: Optional[str] = None) -> None:
        """Print the first ``n`` rows (fugue/dataset/dataset.py:86-102, display of
        fugue/dataframe/dataframe_iterable_dataframe / DataFrameDisplay): title, schema line, rows,
        optionally the total count, then the metadata if there is any."""
        lines: List[str] = []
        if title:
            lines.append(str(title))
        lines.append(f"{type(self).__name__}")
        lines.append(str(self.schema))
        head = self.head(n).as_array()
        lines.extend(str(r) for r in head)
        if len(head) == 0:
            lines.append("(empty)")
        if with_count:
            lines.append(f"Total count: {self.count()}")
        if self.has_metadata:
            lines.append(f"Metadata: {self.metadata}")
        print("\n".join(lines))

    def get_info_str(self) -> str:
        """One JSON line: schema, type, metadata (fugue/dataframe/dataframe.py ``get_info_str``)."""
        import json

        return json.dumps({"schema": str(self.schema), "type": f"{type(self).__module__}.{type(self).__name__}",
                           "metadata": self.metadata if self.has_metadata else {}})

    def __repr__(self) -> str:
        return f"{type(self).__name__}({self.schema})"

    def _repr_html_(self) -> str:
        import html

        return html.escape(repr(self))

    def __copy__(self) -> "DataFrame":
        return self

    def __deepcopy__(self, memo: Any) -> "DataFrame":
        return self


class LocalDataFrame(DataFrame):
    @property
    def is_local(self) -> bool:
        return True

    def as_local_bounded(self) -> "LocalDataFrame":
        return self


_TRUE_WORDS, _FALSE_WORDS = ("true", "t", "yes", "1"), ("false", "f", "no", "0")


def _clean_cell(v: Any, tp: pa.DataType) -> Any:
    """One row value -> what ``pa.array`` takes for ``tp``.  Rows are untyped Python data in the reference
    (``ArrayDataFrame`` keeps them as given and converts on ``as_array(type_safe=True)``,
    fugue/dataframe/array_dataframe.py + triad's type-safe converters); this frame is typed at construction,
    so the same conversions run here:

    * pandas' missing markers (NaT, NA) and float NaN in a numeric / temporal column are NULL
      (fugue_test/dataframe_suite.py:179-196);
    * text into a numeric / boolean / temporal column is parsed, numbers into a text column are written with
      ``str``, a float into an integer column is truncated (tests/fugue/dataframe/test_array_dataframe.py:25-60,
      106-140);
    * nested values may come as JSON text; struct keys the type does not name are dropped, missing ones are
      NULL, members are converted recursively (:86-96)."""
    if v is None or v is pd.NaT or v is pd.NA:
        return None
    if pa.types.is_timestamp(tp) or pa.types.is_date(tp):
        if isinstance(v, str):
            v = pd.Timestamp(v)
        if isinstance(v, pd.Timestamp):
            v = v.to_pydatetime()
        if pa.types.is_date(tp) and hasattr(v, "date") and callable(v.date):
            v = v.date()
        return v
    if pa.types.is_floating(tp) or pa.types.is_integer(tp):
        if isinstance(v, str):
            v = float(v) if pa.types.is_floating(tp) or not v.strip().lstrip("+-").isdigit() else int(v)
        if isinstance(v, float) and v != v:
            return None
        if pa.types.is_integer(tp) and not isinstance(v, (int, bool)):
            return int(v)          # truncation, like a C cast
        return v
    if pa.types.is_boolean(tp):
        if isinstance(v, str):
            w = v.strip().lower()
            if w not in _TRUE_WORDS + _FALSE_WORDS:
                raise ValueError(f"{v!r} is not a boolean")
            return w in _TRUE_WORDS
        return bool(v)
    if pa.types.is_string(tp) or pa.types.is_large_string(tp):
        return v if isinstance(v, str) else (v.decode() if isinstance(v, bytes) else str(v))
    if pa.types.is_list(tp) or pa.types.is_large_list(tp):
        if isinstance(v, str):
            import json

            v = json.loads(v)
        return [_clean_cell(x, tp.value_type) for x in v] if isinstance(v, (list, tuple)) else v
    if pa.types.is_struct(tp):
        if isinstance(v, str):
            import json

            v = json.loads(v)
        if isinstance(v, dict):   # keys the type does not name are dropped
            return {tp.field(i).name: _clean_cell(v.get(tp.field(i).name), tp.field(i).type)
                    for i in range(tp.num_fields)}
    return v


def _rows_to_arrow(rows: Any, schema: Schema) -> pa.Table:
    rows = list(rows) if rows is not None else []
    ncol = len(schema)
    cols: List[List[Any]] = [[] for _ in range(ncol)]
    for r in rows:
        r = list(r)
        assert len(r) == ncol, f"row {r} doesn't match schema {schema}"
        for i in range(ncol):
            cols[i].append(r[i])
    arrays = [pa.array([_clean_cell(v, tp) for v in vals], type=tp) for vals, tp in zip(cols, schema.types)]
    return pa.Table.from_arrays(arrays, schema=schema.pa_schema)


def _cast_table(t: pa.Table, new: Schema) -> pa.Table:
    """``alter_columns`` on a host table, column by column, with the string forms the reference's suites pin
    (fugue_test/dataframe_suite.py:296-420): a datetime becomes ``YYYY-MM-DD HH:MM:SS`` (fractional seconds
    only when there are any), everything else is the Arrow cast (unsafe: double -> int truncates)."""
    import pyarrow.compute as pc

    cols = []
    for name, tp in zip(new.names, new.types):
        c = t.column(name)
        if c.type != tp and pa.types.is_timestamp(c.type) and (pa.types.is_string(tp) or pa.types.is_large_string(tp)):
            whole = c.cast(pa.timestamp("s", c.type.tz), safe=False)
            if whole.cast(c.type).equals(c):
                c = whole
            c = pc.strftime(c, format="%Y-%m-%d %H:%M:%S").cast(tp)
        elif c.type != tp and pa.types.is_floating(c.type) and (pa.types.is_string(tp) or pa.types.is_large_string(tp)):
            # Python's float text ("1.0", "1.1"), what the reference's pandas / python casts write
            c = pa.chunked_array([pa.array([None if x is None else str(x) for x in c.to_pylist()], type=tp)])
        elif c.type != tp:
            c = c.cast(tp, safe=False)
        cols.append(c)
    return pa.Table.from_arrays(cols, schema=new.pa_schema)


class ArrowDataFrame(LocalDataFrame):
    """pyarrow-backed local bounded frame (fugue/dataframe/arrow_dataframe.py:45-200)."""

    def __init__(self, df: Any = None, schema: Any = None):
        if df is None:
            sch = Schema(schema)
            self._native = _rows_to_arrow([], sch)
        elif isinstance(df, pa.Table):
            if schema is not None:
                sch = Schema(schema)
                if Schema(df.schema) != sch:
                    df = df.select(sch.names).cast(sch.pa_schema) if set(sch.names) <= set(df.schema.names) \
                        else df.rename_columns(sch.names).cast(sch.pa_schema)
            else:
                sch = Schema(df.schema)
            self._native = df
        elif isinstance(df, (pd.DataFrame, pd.Series)):
            if isinstance(df, pd.Series):
                df = df.to_frame()
            if schema is None:
                t = pa.Table.from_pandas(df, preserve_index=False)
                if any(pa.types.is_large_string(f.type) for f in t.schema):
                    # pandas 3 string columns arrive as large_string; Fugue's "str" is pa.string()
                    t = t.cast(pa.schema([pa.field(f.name, pa.string()) if pa.types.is_large_string(f.type) else f
                                          for f in t.schema]))
                sch = Schema(t.schema)
            else:
                sch = Schema(schema)
                try:   # one pass when pandas' dtypes already fit the schema
                    t = pa.Table.from_pandas(df[sch.names], schema=sch.pa_schema, preserve_index=False, safe=False)
                except (pa.ArrowInvalid, pa.ArrowTypeError):
                    # otherwise: the natural Arrow types first, then the casts of alter_columns (int -> "1")
                    t = _cast_table(pa.Table.from_pandas(df[sch.names], preserve_index=False), sch)
            self._native = t
        elif isinstance(df, DataFrame):
            t = df.as_arrow()
            if isinstance(schema, (list, tuple)) and all(isinstance(x, str) and ":" not in x for x in schema):
                sch = df.schema.extract(list(schema))        # a list of names: projection
            else:
                sch = Schema(schema) if schema is not None else df.schema
            if Schema(t.schema) != sch:
                missing = [n for n in sch.names if n not in t.schema.names]
                if missing:
                    raise FugueDataFrameOperationError(f"{missing} not in {Schema(t.schema)}")
                t = _cast_table(t.select(sch.names), sch)
            self._native = t
        elif isinstance(df, (list, tuple)) or hasattr(df, "__iter__"):
            if schema is None:
                raise FugueDataFrameOperationError("schema is required to build a dataframe from rows")
            sch = Schema(schema)
            self._native = _rows_to_arrow(df, sch)
        else:
            raise ValueError(f"{type(df)} is not supported")
        super().__init__(sch)

    @property
    def native(self) -> pa.Table:
        return self._native

    def count(self) -> int:
        return self._native.num_rows

    def as_arrow(self, type_safe: bool = False) -> pa.Table:
        return self._native

    def _select_cols(self, columns: List[Any]) -> "DataFrame":
        return ArrowDataFrame(self._native.select(columns))

    def rename(self, columns: Dict[str, str]) -> "DataFrame":
        try:
            sch = self.schema.rename(columns)
        except Exception as e:
            raise FugueDataFrameOperationError(str(e)) from e
        return ArrowDataFrame(self._native.rename_columns(sch.names))


class PandasDataFrame(ArrowDataFrame):
    """Constructor-compatible with fugue/dataframe/pandas_dataframe.py:38-95."""

    def __init__(self, df: Any = None, schema: Any = None, pandas_df_wrapper: bool = False):
        super().__init__(df, schema)


class ArrayDataFrame(ArrowDataFrame):
    """Constructor-compatible with fugue/dataframe/array_dataframe.py (rows + schema)."""

    def __init__(self, df: Any = None, schema: Any = None):
        super().__init__([] if df is None else df, schema)


class B200DataFrame(DataFrame):
    """A ``B200Table`` in HBM behind the reference's DataFrame interface."""

    def __init__(self, table: Any, schema: Any = None):
        from .table import B200Table

        if isinstance(table, B200DataFrame):
            table = table.native
        if not isinstance(table, B200Table):
            raise ValueError(f"B200DataFrame wraps a B200Table, got {type(table)}")
        if schema is not None and Schema(schema) != table.schema:
            sch = Schema(schema)
            if sch.names != table.schema.names:
                if len(sch) != len(table.schema):
                    raise FugueDataFrameOperationError(f"{sch} doesn't match {table.schema}")
                table = table.rename(dict(zip(table.schema.names, sch.names)))
            if sch != table.schema:
                raise FugueDataFrameOperationError(
                    f"device table of {table.schema} can't be viewed as {sch}; cast on the host first")
        self._table = table
        super().__init__(table.schema)

    @property
    def native(self) -> Any:
        return self._table

    def native_as_df(self) -> Any:
        return self._table

    @property
    def is_local(self) -> bool:
        return False

    @property
    def num_partitions(self) -> int:
        return self._table.num_partitions

    def count(self) -> int:
        return self._table.num_rows

    @property
    def empty(self) -> bool:
        return self._table.num_rows == 0

    def as_arrow(self, type_safe: bool = False) -> pa.Table:
        return self._table.to_arrow()

    def peek_array(self) -> List[Any]:
        if self.empty:
            raise FugueDatasetEmptyError("dataframe is empty")
        return ArrowDataFrame(self._table.slice(0, 1).to_arrow()).as_array()[0]

    def head(self, n: int, columns: Optional[List[str]] = None) -> LocalDataFrame:
        t = self._table.slice(0, min(n, self._table.num_rows))
        if columns is not None:
            t = t.select(columns)
        return ArrowDataFrame(t.to_arrow())

    def _select_cols(self, columns: List[Any]) -> DataFrame:
        return B200DataFrame(self._table.select(columns))

    def alter_columns(self, columns: Any) -> DataFrame:
        """Casts run on the device (one fb_eval_expr program), casts from strings to numbers, bools, dates and
        timestamps included (K13), and casts of those to strings (K14: the text the host frames write, formatted once
        per distinct value).  Casts to the types the device does not parse to, and to strings from types it does not
        format (a timestamp in a time zone other than UTC, decimal ...), go through the host."""
        new = self._altered_schema(columns)
        if new is None:
            return self
        from . import expr as X
        from .column import col
        from .strings import StringParseError

        try:
            exprs = [col(n) if tp == self._schema[n].type else col(n).cast(tp) for n, tp in zip(new.names, new.types)]
            return B200DataFrame(X.project(self._table, exprs))
        except NotImplementedError:
            from .table import B200Table

            host = super().alter_columns(columns).as_arrow()
            return B200DataFrame(B200Table.from_arrow(host, self._table.device))
        except StringParseError as e:  # a string that does not parse, as the host path reports it
            raise FugueDataFrameOperationError(str(e)) from e

    def rename(self, columns: Dict[str, str]) -> DataFrame:
        try:
            return B200DataFrame(self._table.rename(columns))
        except Exception as e:
            raise FugueDataFrameOperationError(str(e)) from e


def as_fugue_df(df: Any, schema: Any = None) -> DataFrame:
    """fugue/dataframe/api.py ``as_fugue_df`` for the types this package knows."""
    from .table import B200Table

    if isinstance(df, DataFrame):
        return df
    if isinstance(df, B200Table):
        return B200DataFrame(df, schema)
    if isinstance(df, (pa.Table, pd.DataFrame)):
        return ArrowDataFrame(df, schema)
    if isinstance(df, (list, tuple)) or hasattr(df, "__iter__"):
        return ArrayDataFrame(df, schema)
    raise NotImplementedError(f"no conversion of {type(df)} to a Fugue DataFrame")  # fugue/dataframe/api.py


def df_eq(df: Any, data: Any, schema: Any = None, digits: int = 8, check_order: bool = False,
          check_schema: bool = True, check_content: bool = True, throw: bool = False) -> bool:
    """Order-insensitive multiset equality with abs tol 10**-digits
    (fugue/dataframe/utils.py:24-94)."""
    df1 = as_fugue_df(df).as_local_bounded()
    df2 = as_fugue_df(data, schema).as_local_bounded()
    try:
        assert df1.count() == df2.count(), f"count mismatch {df1.count()}, {df2.count()}"
        assert not check_schema or df1.schema == df2.schema, \
            f"schema mismatch {df1.schema}, {df2.schema}"
        if not check_content:
            return True
        d1, d2 = df1.as_pandas(), df2.as_pandas()
        d2.columns = d1.columns
        if not check_order:
            d1 = d1.sort_values(list(d1.columns))
            d2 = d2.sort_values(list(d2.columns))
        d1 = d1.reset_index(drop=True)
        d2 = d2.reset_index(drop=True)
        pd.testing.assert_frame_equal(d1, d2, rtol=0, atol=10 ** (-digits), check_dtype=False,
                                      check_exact=False)
        return True
    except AssertionError:
        if throw:
            raise
        return False
