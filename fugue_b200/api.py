"""Functional API with the reference's names: ``transform``, ``engine_context``,
``make_execution_engine``, ``as_fugue_engine_df``, ``repartition`` ...

Mirrors
  * ``fa.transform``            fugue/workflow/api.py:34-184
  * ``fa.engine_context``       fugue/execution/api.py:21-50
  * ``make_execution_engine``   fugue/execution/factory.py:237-339
  * function -> transformer     fugue/extensions/transformer/convert.py:328-385, 576-594
                                fugue/dataframe/function_wrapper.py:49-148
The reference builds a two-task DAG (adagio) around one ``map_dataframe`` call; that
driver-side plumbing is O(1) and is collapsed into a direct call here (SURVEY.md 3.1).
"""
import collections.abc
import inspect
import re
from typing import Any, Callable, Dict, Iterable, Iterator, List, Optional, get_args, get_origin, get_type_hints

import pandas as pd
import pyarrow as pa

from .dataframe import (ArrayDataFrame, ArrowDataFrame, B200DataFrame, DataFrame, LocalDataFrame,
                        PandasDataFrame, as_fugue_df)
from .execution_engine import B200ExecutionEngine, assert_or_throw
from .lifecycle import (EngineLifecycle, FugueInvalidOperation, clear_global_engine, register_global_conf,  # noqa: F401
                        try_get_context_engine)
from .lifecycle import get_current_conf as _context_conf
from .partition import PartitionCursor, PartitionSpec
from .schema import Schema
from .table import B200Table

_ENGINE_FACTORIES: Dict[str, Callable[..., Any]] = {}
_SQL_ENGINE_FACTORIES: Dict[str, Callable[..., Any]] = {}


def _register(table: Dict[str, Callable[..., Any]], name: str, func: Callable[..., Any], on_dup: str) -> None:
    if name in table and on_dup == "ignore":
        return
    if name in table and on_dup == "throw":
        raise KeyError(f"{name} is already registered")
    table[name] = func


def register_execution_engine(name: str, func: Callable[..., Any], on_dup: str = "overwrite") -> None:
    """fugue/execution/factory.py:18-88 (name registration only): ``func(conf, **kwargs) -> engine``."""
    _register(_ENGINE_FACTORIES, name, func, on_dup)


def register_sql_engine(name: str, func: Callable[..., Any], on_dup: str = "overwrite") -> None:
    """fugue/execution/factory.py:132-170: ``func(execution_engine, **kwargs) -> sql engine``."""
    _register(_SQL_ENGINE_FACTORIES, name, func, on_dup)


register_execution_engine("b200", lambda conf, **kw: B200ExecutionEngine(conf, **kw))
register_sql_engine("b200", lambda engine, **kw: engine.create_default_sql_engine())


def infer_execution_engine(objs: Optional[List[Any]]) -> Any:
    """Which engine the inputs ask for (fugue/execution/factory.py:401-447): device tables / frames -> "b200"."""
    for o in objs or []:
        if isinstance(o, (B200Table, B200DataFrame)):
            return "b200"
    return None


def make_sql_engine(engine: Any, execution_engine: Any, **kwargs: Any) -> Any:
    """fugue/execution/factory.py:342-398: None -> the engine's default, a registered name, a type (called with
    the execution engine) or a ready instance."""
    if engine is None or engine == "":
        return execution_engine.create_default_sql_engine()
    if isinstance(engine, str):
        assert_or_throw(engine in _SQL_ENGINE_FACTORIES, lambda: ValueError(
            f"{engine!r} is not a registered SQL engine (this package provides 'b200')"))
        return _SQL_ENGINE_FACTORIES[engine](execution_engine, **kwargs)
    if isinstance(engine, type):
        return engine(execution_engine, **kwargs)
    return engine


def make_execution_engine(engine: Any = None, conf: Any = None, infer_by: Optional[List[Any]] = None,
                          **kwargs: Any) -> Any:
    """Engine resolution of fugue/execution/factory.py:237-339.  ``engine`` None: the context engine, else the
    global engine, else what ``infer_by`` asks for, else a new "b200" engine.  Otherwise a registered name, an
    engine type, an engine instance, or a pair ``(engine, sql_engine)``.  ``conf`` and ``kwargs`` end up in the
    engine's conf in every case."""
    if engine is None or engine == "":
        engine = try_get_context_engine()
        if engine is None:
            engine = infer_execution_engine(infer_by)
        if engine is None:
            engine = "b200"
    if isinstance(engine, tuple):
        assert_or_throw(len(engine) == 2, lambda: ValueError(f"(engine, sql_engine) expected, got {engine}"))
        result = make_execution_engine(engine[0], conf, **kwargs)
        result._sql_engine = make_sql_engine(engine[1], result)
        return result
    if isinstance(engine, EngineLifecycle):
        result = engine
    elif isinstance(engine, str):
        assert_or_throw(engine in _ENGINE_FACTORIES, lambda: ValueError(
            f"{engine!r} is not a registered execution engine (this package provides 'b200')"))
        result = _ENGINE_FACTORIES[engine](conf, **kwargs)
    elif isinstance(engine, type) and issubclass(engine, EngineLifecycle):
        result = engine(conf, **kwargs)
    else:
        raise TypeError(f"{engine} can't be converted to an execution engine")
    if conf:
        result.conf.update(dict(conf))
    if kwargs:
        result.conf.update(kwargs)
    return result


def engine_context(engine: Any = None, engine_conf: Any = None, infer_by: Any = None) -> Any:
    """``with fa.engine_context(...) as e`` (fugue/execution/api.py:21-50): the engine becomes the context
    engine; leaving its last context stops it."""
    return make_execution_engine(engine, engine_conf, infer_by=infer_by).as_context()


def set_global_engine(engine: Any, engine_conf: Any = None) -> Any:
    assert_or_throw(engine is not None, ValueError("engine must be specified"))
    return make_execution_engine(engine, engine_conf).set_global()


def get_context_engine() -> Any:
    """The context (else global) engine; an error when there is none (fugue/execution/api.py:95-102)."""
    engine = try_get_context_engine()
    if engine is None:
        raise FugueInvalidOperation("No global/context engine is set")
    return engine


def as_fugue_engine_df(engine: B200ExecutionEngine, df: Any, schema: Any = None) -> DataFrame:
    """fugue/execution/api.py:124-142."""
    return engine.to_df(df, schema)


def repartition(df: Any, partition: Any, engine: Any = None, engine_conf: Any = None,
                as_fugue: bool = False) -> Any:
    e = make_execution_engine(engine, engine_conf)
    res = e.repartition(e.to_df(df), PartitionSpec(partition))
    return res if as_fugue or isinstance(df, DataFrame) else res.native


# ----------------------------------------------------------------------------------------
class FugueWorkflowCompileValidationError(Exception):
    """fugue/exceptions.py: a validation rule that does not need data was violated."""


class FugueWorkflowRuntimeValidationError(Exception):
    """fugue/exceptions.py: a validation rule on the input data (its schema) was violated."""


# function wrapper: decides how the user function sees a partition
# ----------------------------------------------------------------------------------------
class _FuncAsTransformer:
    """What ``_to_transformer(using, schema)`` builds in the reference
    (extensions/transformer/convert.py:328-385): validates the signature, resolves the output
    schema and adapts LocalDataFrame <-> the annotated types."""

    def __init__(self, func: Callable, schema: Any, params: Optional[Dict[str, Any]]):
        assert_or_throw(callable(func), lambda: TypeError(f"{func} is not callable"))
        self._func = func
        self._params = dict(params or {})
        sig = inspect.signature(func)
        try:
            hints = get_type_hints(func)
        except Exception:
            hints = {}
        names = list(sig.parameters)
        assert_or_throw(len(names) >= 1, lambda: TypeError("transformer needs a dataframe parameter"))
        self._df_param = names[0]
        self._in_kind = self._kind(hints.get(names[0], sig.parameters[names[0]].annotation))
        self._out_kind = self._kind(hints.get("return", sig.return_annotation))
        assert_or_throw(self._in_kind is not None, lambda: TypeError(
            f"first parameter of {func.__name__} must be annotated with B200Table, pd.DataFrame, "
            "pa.Table, List[List[Any]], Iterable[List[Any]], List[Dict[str, Any]] or a Fugue DataFrame"))
        self._wants_cursor = [n for n in names[1:] if hints.get(n, None) is PartitionCursor]
        self._schema_expr = schema if schema is not None else self._schema_from_comment(func)
        self._rules = self._rules_from_comment(func)
        assert_or_throw(self._schema_expr is not None, lambda: ValueError(
            "schema is required (argument or a '# schema:' comment above the function)"))

    @staticmethod
    def _comment_hint(func: Callable, key: str) -> Optional[str]:
        """The ``# <key>: ...`` line of the comment block directly above the function
        (fugue/_utils/interfaceless.py:9-40): the LOWEST matching line wins, anything after a second ``#`` on
        that line is a remark.  None when there is no such line, "" when it is empty."""
        try:
            block = inspect.getcomments(func) or ""
        except Exception:
            return None
        hint = re.compile(r"^\s*#\s*" + re.escape(key) + r"\s*:([^#]*)")
        for line in reversed(block.splitlines()):
            m = hint.match(line)
            if m is not None:
                return m.group(1).strip()
        return None

    @staticmethod
    def _schema_from_comment(func: Callable) -> Optional[str]:
        text = _FuncAsTransformer._comment_hint(func, "schema")
        assert_or_throw(text != "", SyntaxError("incorrect schema annotation"))   # interfaceless.py:43-66
        return text

    @staticmethod
    def _rules_from_comment(func: Callable) -> Dict[str, Any]:
        """Validation rules written as comment hints above the function (fugue/extensions/_utils.py:36-81):
        ``partitionby_has / partitionby_is`` (key names), ``presort_has / presort_is`` (presort expressions),
        ``input_has`` (column names, optionally ``name:type``), ``input_is`` (a schema)."""
        from .partition import parse_presort_exp

        rules: Dict[str, Any] = {}
        for key in ("partitionby_has", "partitionby_is", "presort_has", "presort_is", "input_has", "input_is"):
            text = _FuncAsTransformer._comment_hint(func, key)
            if text is None:
                continue
            assert_or_throw(text != "", lambda: SyntaxError(f"{key} can't be empty"))
            if key.startswith("partitionby"):
                rules[key] = PartitionSpec(by=[x.strip() for x in text.split(",")]).partition_by
            elif key.startswith("presort"):
                rules[key] = list(parse_presort_exp(text).items())
            elif key == "input_has":
                rules[key] = text.replace(" ", "").split(",")
            else:
                rules[key] = str(Schema(text))
        return rules

    def validate_on_compile(self, spec: PartitionSpec) -> None:
        """What can be checked before any data is seen: the partitioning the call asks for against the
        function's ``partitionby_* / presort_*`` rules (fugue/extensions/_utils.py:84-129)."""
        def fail(msg: str) -> Any:
            return lambda: FugueWorkflowCompileValidationError(msg)

        for key, want in self._rules.items():
            if key.startswith("partitionby"):
                for k in want:
                    assert_or_throw(k in spec.partition_by, fail(f"required partition key {k} is not in {spec}"))
                if key == "partitionby_is":
                    assert_or_throw(len(want) == len(spec.partition_by), fail(f"{want} does not match {spec}"))
            elif key.startswith("presort"):
                have = spec.presort
                for k, asc in want:
                    assert_or_throw(k in have, fail(f"required presort key {k} is not in presort of {spec}"))
                    assert_or_throw(have[k] == asc, fail(f"order of {k} doesn't match presort of {spec}"))
                if key == "presort_is":
                    assert_or_throw(want == list(have.items()), fail(f"{want} does not match presort of {spec}"))

    @property
    def has_input_rules(self) -> bool:
        return any(k.startswith("input_") for k in self._rules)

    def validate_on_runtime(self, schema: Schema) -> None:
        """``input_has / input_is`` against the schema of the actual input (fugue/extensions/_utils.py:132-150)."""
        for key, want in self._rules.items():
            if key == "input_has":
                for c in want:
                    assert_or_throw(c in schema, lambda: FugueWorkflowRuntimeValidationError(
                        f"required column {c} is not in {schema}"))
            elif key == "input_is":
                assert_or_throw(schema == want, lambda: FugueWorkflowRuntimeValidationError(
                    f"{want} does not match {schema}"))

    @staticmethod
    def _kind(tp: Any) -> Optional[str]:
        if tp is inspect.Parameter.empty or tp is None:
            return None
        if tp is B200Table:
            return "b200"
        if tp is pd.DataFrame:
            return "pandas"
        if tp is pa.Table:
            return "pyarrow"
        if inspect.isclass(tp) and issubclass(tp, DataFrame):
            return "fugue"
        # generic annotations (function_wrapper.py:330-516: _ListListParam, _IterableListParam, _ListDictParam,
        # _IterableDictParam, _IterablePandasParam, _IterableArrowParam): outer container, then the element
        origin, args = get_origin(tp), get_args(tp)
        lazy = origin in (collections.abc.Iterable, collections.abc.Iterator, collections.abc.Generator)
        if lazy and args and args[0] is pd.DataFrame:
            return "pandas_iter"
        if lazy and args and args[0] is pa.Table:
            return "pyarrow_iter"
        s = str(tp)
        if "Dict" in s or "dict" in s:
            return "dicts"
        if "List" in s or "list" in s or "Iterable" in s or "Iterator" in s:
            return "array"
        return None

    def get_format_hint(self) -> Optional[str]:
        """Preferred hand-off format: the input annotation's, else the return annotation's
        (function_wrapper.py:150-160).  Only an INPUT typed ``B200Table`` makes the map engine hand over whole
        device partitions, so "b200" is never derived from the return type."""
        hints = {"b200": "b200", "pandas": "pandas", "pandas_iter": "pandas", "pyarrow": "pyarrow",
                 "pyarrow_iter": "pyarrow"}
        if self._in_kind in hints:
            return hints[self._in_kind]
        out = hints.get(self._out_kind or "")
        return None if out == "b200" else out

    def get_output_schema(self, df: DataFrame) -> Schema:
        if isinstance(self._schema_expr, Schema):
            return self._schema_expr
        return df.schema.transform(self._schema_expr)

    def _to_input(self, df: DataFrame) -> Any:
        k = self._in_kind
        if k == "b200":
            assert_or_throw(isinstance(df, B200DataFrame), lambda: TypeError(
                "a B200Table-typed function can only run on the b200 engine"))
            return df.native
        if k == "pandas":
            return df.as_pandas()
        if k == "pyarrow":
            return df.as_arrow()
        if k == "pandas_iter":   # one chunk: a logical partition is materialised as a whole here
            return iter([df.as_pandas()])
        if k == "pyarrow_iter":
            return iter([df.as_arrow()])
        if k == "array":
            return df.as_array(type_safe=True)
        if k == "dicts":
            return df.as_dicts()
        return df

    def _to_output(self, out: Any, schema: Schema) -> DataFrame:
        if isinstance(out, B200Table):
            return B200DataFrame(out)  # map_dataframe asserts the schema (native_execution_engine.py:149-153)
        if isinstance(out, DataFrame):
            return out
        if isinstance(out, (pd.DataFrame, pa.Table)):
            return ArrowDataFrame(out, schema)
        if out is None:
            return ArrowDataFrame(None, schema)
        if isinstance(out, dict):   # Dict[str, Any]: ONE output row (function_wrapper.py:254-262)
            out = [out]
        out = list(out)
        if out and all(isinstance(x, pd.DataFrame) for x in out):   # Iterable[pd.DataFrame]: chunks of the result
            frames = [x for x in out if x.shape[0] > 0]
            return ArrowDataFrame(pd.concat(frames, ignore_index=True) if frames else None, schema)
        if out and all(isinstance(x, pa.Table) for x in out):
            tables = [x for x in out if x.num_rows > 0]
            return ArrowDataFrame(pa.concat_tables(tables) if tables else None, schema)
        if out and isinstance(out[0], dict):
            out = [[r.get(n) for n in schema.names] for r in out]
        return ArrayDataFrame(out, schema)

    def make_runner(self, output_schema: Schema, ignore_errors: List[type], discard_output: bool = False
                    ) -> Callable[[PartitionCursor, DataFrame], DataFrame]:
        def run(cursor: PartitionCursor, df: DataFrame) -> DataFrame:
            kw = dict(self._params)
            for n in self._wants_cursor:
                kw[n] = cursor
            try:
                out = self._func(self._to_input(df), **kw)
                if discard_output:           # output transformer: only the side effects count
                    if inspect.isgenerator(out):
                        for _ in out:
                            pass
                    return ArrowDataFrame(None, output_schema)
                return self._to_output(out, output_schema)
            except tuple(ignore_errors) if ignore_errors else ():  # processors.py:330-338
                return ArrowDataFrame(None, output_schema)

        from .colmap import ColumnMap

        # a declarative map: the map engine may fuse it into the partition kernels (K4)
        run.column_map = self._func if isinstance(self._func, ColumnMap) else None  # type: ignore
        return run


def transform(
    df: Any,
    using: Any,
    schema: Any = None,
    params: Any = None,
    partition: Any = None,
    callback: Any = None,
    ignore_errors: Optional[List[Any]] = None,
    persist: bool = False,
    as_local: bool = False,
    save_path: Optional[str] = None,
    checkpoint: bool = False,
    engine: Any = None,
    engine_conf: Any = None,
    as_fugue: bool = False,
) -> Any:
    """``fa.transform`` (fugue/workflow/api.py:34-184) on the B200 engine.

    ``using`` may be typed on ``B200Table`` (runs once per device table, vectorised over the
    logical partitions - the GPU hot path), or on pandas / arrow / lists (called once per
    logical partition on the host after the device partitioned the table).
    """
    assert_or_throw(callback is None, NotImplementedError("callback (RPC) is out of scope"))
    # fugue/workflow/api.py:16-31: only parquet paths are accepted for a path input / save_path
    for what, pth in (("df", df if isinstance(df, str) else None), ("save_path", save_path)):
        assert_or_throw(pth is None or (isinstance(pth, str) and pth.lower().endswith(".parquet")),
                        lambda: ValueError(f"fugue transform can only load / save parquet file paths ({what}={pth})"))
    e = make_execution_engine(engine, engine_conf, infer_by=[df])
    fugue_in = isinstance(df, DataFrame)      # decides the return type: a path or a native object in -> native out
    if isinstance(df, str):
        df = e.load_df(df, format_hint="parquet")
    tf = _FuncAsTransformer(using, schema, params)
    spec = PartitionSpec(partition)
    tf.validate_on_compile(spec)
    if tf.has_input_rules:     # needs the input schema: only then is a native input looked at here
        tf.validate_on_runtime(get_schema(df))
    res: Optional[DataFrame] = None
    from .colmap import ColumnMap

    windowed = isinstance(using, ColumnMap) and using.has_window  # needs the sort of map_dataframe
    if as_local and tf.get_format_hint() == "b200" and not isinstance(df, (B200DataFrame, B200Table)) \
            and not windowed:
        # host input, host output, device function: overlap H2D / partition (/ exchange) / D2H column by column
        from .streaming import streaming_transform

        ldf = as_fugue_df(df)
        out_schema = tf.get_output_schema(ldf)
        run = tf.make_runner(out_schema, list(ignore_errors or []))
        res = e.streaming_transform(ldf, run, out_schema, spec) if e.is_distributed \
            else streaming_transform(e, ldf, run, out_schema, spec)
    if res is None:
        edf = e.to_df(df)
        out_schema = tf.get_output_schema(edf)
        runner = tf.make_runner(out_schema, list(ignore_errors or []))
        res = e.map_engine.map_dataframe(edf, runner, out_schema, spec,
                                         map_func_format_hint=tf.get_format_hint())
    if persist:
        res = e.persist(res)
    # save_path / checkpoint (fugue/workflow/api.py:100-120, fugue/workflow/_checkpoint.py:38-128): a strong,
    # non-deterministic file checkpoint = save as parquet, continue from the file
    if checkpoint or save_path is not None:
        target = save_path
        if target is None:
            import os
            import uuid

            root = e.conf.get("fugue.workflow.checkpoint.path", "")
            assert_or_throw(root != "", ValueError(
                "fugue.workflow.checkpoint.path is not set (needed for checkpoint=True without save_path)"))
            os.makedirs(root, exist_ok=True)
            target = os.path.join(root, uuid.uuid4().hex + ".parquet")
        e.save_df(res, target, format_hint="parquet", mode="overwrite")
        if not checkpoint:
            return save_path
        res = e.load_df(target, format_hint="parquet")
    res = e.convert_yield_dataframe(res, as_local)
    if as_fugue or fugue_in:
        return res
    return res.as_pandas() if res.is_local else res.native


OUTPUT_TRANSFORMER_DUMMY_SCHEMA = "__output_no_data__:int"   # fugue/extensions/transformer/constants.py:1


def out_transform(df: Any, using: Any, params: Any = None, partition: Any = None, callback: Any = None,
                  ignore_errors: Optional[List[Any]] = None, engine: Any = None, engine_conf: Any = None) -> None:
    """``fa.out_transform`` (fugue/workflow/api.py:187-250): run ``using`` on every partition for its side effects,
    eagerly, returning nothing.  As in the reference (``_FuncAsOutputTransformer``, convert.py:386-403) the
    function's result is dropped and every call hands an empty frame of a dummy schema back to the map engine."""
    assert_or_throw(callback is None, NotImplementedError("callback (RPC) is out of scope"))
    assert_or_throw(not isinstance(df, str) or df.lower().endswith(".parquet"),
                    lambda: ValueError(f"fugue transform can only load parquet file paths (df={df})"))
    e = make_execution_engine(engine, engine_conf, infer_by=[df])
    if isinstance(df, str):
        df = e.load_df(df, format_hint="parquet")
    tf = _FuncAsTransformer(using, OUTPUT_TRANSFORMER_DUMMY_SCHEMA, params)
    tf.validate_on_compile(PartitionSpec(partition))
    if tf.has_input_rules:
        tf.validate_on_runtime(get_schema(df))
    out_schema = Schema(OUTPUT_TRANSFORMER_DUMMY_SCHEMA)
    inner = tf.make_runner(out_schema, list(ignore_errors or []), discard_output=True)
    e.map_engine.map_dataframe(e.to_df(df), inner, out_schema, PartitionSpec(partition),
                               map_func_format_hint=tf.get_format_hint())


def _finish(e: Any, df: Any, res: DataFrame, as_fugue: bool, as_local: bool) -> Any:
    res = e.convert_yield_dataframe(res, as_local)
    if as_fugue or isinstance(df, DataFrame):
        return res
    return res.as_pandas() if res.is_local else res.native


def aggregate(df: Any, partition_by: Any = None, engine: Any = None, engine_conf: Any = None,
              as_fugue: bool = False, as_local: bool = False, **agg_kwcols: Any) -> Any:
    """``fa.aggregate`` (fugue/execution/api.py:1175-1232):
    ``aggregate(df, "key", s=f.sum(col("v0")), c=f.count(all_cols()))``."""
    from .column import ColumnExpr, lit

    cols = [v.alias(k) if isinstance(v, ColumnExpr) else lit(v).alias(k) for k, v in agg_kwcols.items()]
    e = make_execution_engine(engine, engine_conf, infer_by=[df])
    spec = None if partition_by is None else PartitionSpec(by=partition_by)
    return _finish(e, df, e.aggregate(e.to_df(df), spec, cols), as_fugue, as_local)


def select(df: Any, *columns: Any, where: Any = None, having: Any = None, distinct: bool = False,
           engine: Any = None, engine_conf: Any = None, as_fugue: bool = False, as_local: bool = False) -> Any:
    """``fa.select`` (fugue/execution/api.py:975-1057): SQL SELECT over one dataframe written with
    column expressions; strings are column names."""
    from .column import SelectColumns, col

    cols = SelectColumns(*[col(x) if isinstance(x, str) else x for x in columns], arg_distinct=distinct)
    e = make_execution_engine(engine, engine_conf, infer_by=[df])
    return _finish(e, df, e.select(e.to_df(df), cols, where=where, having=having), as_fugue, as_local)


def filter(df: Any, condition: Any, engine: Any = None, engine_conf: Any = None,  # noqa: A001
           as_fugue: bool = False, as_local: bool = False) -> Any:
    """``fa.filter`` (fugue/execution/api.py:1060-1102)."""
    e = make_execution_engine(engine, engine_conf, infer_by=[df])
    return _finish(e, df, e.filter(e.to_df(df), condition), as_fugue, as_local)


def assign(df: Any, engine: Any = None, engine_conf: Any = None, as_fugue: bool = False,
           as_local: bool = False, **columns: Any) -> Any:
    """``fa.assign`` (fugue/execution/api.py:1105-1172): ``assign(df, x=1, c=col("b") + 1)``."""
    from .column import ColumnExpr, lit

    cols = [v.alias(k) if isinstance(v, ColumnExpr) else lit(v).alias(k) for k, v in columns.items()]
    e = make_execution_engine(engine, engine_conf, infer_by=[df])
    return _finish(e, df, e.assign(e.to_df(df), cols), as_fugue, as_local)


def join(df1: Any, df2: Any, *dfs: Any, how: str, on: Optional[Iterable[str]] = None, engine: Any = None,
         engine_conf: Any = None, as_fugue: bool = False, as_local: bool = False) -> Any:
    """``fa.join`` (fugue/execution/api.py:541-588): joins two or more dataframes left to right."""
    e = make_execution_engine(engine, engine_conf, infer_by=[df1, df2, *dfs])
    res: DataFrame = e.join(e.to_df(df1), e.to_df(df2), how=how, on=None if on is None else list(on))
    for odf in dfs:
        res = e.join(res, e.to_df(odf), how=how, on=None if on is None else list(on))
    res = e.convert_yield_dataframe(res, as_local)
    if as_fugue or any(isinstance(x, DataFrame) for x in (df1, df2, *dfs)):
        return res
    return res.as_pandas() if res.is_local else res.native


def asof_join(df1: Any, df2: Any, on: Optional[Iterable[str]], asof: str, how: str = "inner",
              direction: str = "backward", allow_exact_matches: bool = True, tolerance: Any = None, engine: Any = None,
              engine_conf: Any = None, as_fugue: bool = False, as_local: bool = False) -> Any:
    """As-of join of two dataframes with ``pandas.merge_asof`` semantics (``B200ExecutionEngine.asof_join``):
    ``on`` are the equality keys (None: the common columns but ``asof``; empty: one group), ``asof`` the column
    matched by the latest (``direction="backward"``), next (``"forward"``) or nearest value."""
    e = make_execution_engine(engine, engine_conf, infer_by=[df1, df2])
    res: DataFrame = e.asof_join(e.to_df(df1), e.to_df(df2), on=None if on is None else list(on), asof=asof, how=how,
                                 direction=direction, allow_exact_matches=allow_exact_matches, tolerance=tolerance)
    res = e.convert_yield_dataframe(res, as_local)
    if as_fugue or any(isinstance(x, DataFrame) for x in (df1, df2)):
        return res
    return res.as_pandas() if res.is_local else res.native


def range_join(df1: Any, df2: Any, on: Optional[Iterable[str]], at: str, start: str, end: str, how: str = "inner",
               closed: str = "both", engine: Any = None, engine_conf: Any = None, as_fugue: bool = False,
               as_local: bool = False) -> Any:
    """Range join of two dataframes (``B200ExecutionEngine.range_join``): every row of ``df1`` with every row of
    ``df2`` of equal ``on`` key (None: the common columns but ``at``; empty: one group) whose interval
    [``start``, ``end``] holds its ``at`` value; ``closed`` ("both", "left", "right", "neither") says which
    ends belong to the interval."""
    e = make_execution_engine(engine, engine_conf, infer_by=[df1, df2])
    res: DataFrame = e.range_join(e.to_df(df1), e.to_df(df2), on=None if on is None else list(on), at=at,
                                  start=start, end=end, how=how, closed=closed)
    res = e.convert_yield_dataframe(res, as_local)
    if as_fugue or any(isinstance(x, DataFrame) for x in (df1, df2)):
        return res
    return res.as_pandas() if res.is_local else res.native


def inner_join(df1: Any, df2: Any, *dfs: Any, **kwargs: Any) -> Any:
    return join(df1, df2, *dfs, how="inner", **kwargs)


def semi_join(df1: Any, df2: Any, *dfs: Any, **kwargs: Any) -> Any:
    return join(df1, df2, *dfs, how="semi", **kwargs)


def anti_join(df1: Any, df2: Any, *dfs: Any, **kwargs: Any) -> Any:
    return join(df1, df2, *dfs, how="anti", **kwargs)


def left_outer_join(df1: Any, df2: Any, *dfs: Any, **kwargs: Any) -> Any:
    return join(df1, df2, *dfs, how="left_outer", **kwargs)


def right_outer_join(df1: Any, df2: Any, *dfs: Any, **kwargs: Any) -> Any:
    return join(df1, df2, *dfs, how="right_outer", **kwargs)


def full_outer_join(df1: Any, df2: Any, *dfs: Any, **kwargs: Any) -> Any:
    return join(df1, df2, *dfs, how="full_outer", **kwargs)


def cross_join(df1: Any, df2: Any, *dfs: Any, **kwargs: Any) -> Any:
    return join(df1, df2, *dfs, how="cross", **kwargs)


def raw_sql(*statements: Any, engine: Any = None, engine_conf: Any = None, as_fugue: bool = False,
            as_local: bool = False) -> Any:
    """``fa.raw_sql`` (fugue/sql/api.py): strings and dataframes interleaved, e.g.
    ``fa.raw_sql("SELECT key, SUM(v0) AS s, COUNT(*) AS c FROM", df, "GROUP BY key")``."""
    from .column import ColumnExpr, has_bare_window, to_sql
    from .sql import StructuredRawSQL

    e = make_execution_engine(engine, engine_conf, infer_by=[s for s in statements
                                                             if not isinstance(s, (str, ColumnExpr))])
    dfs: Dict[str, Any] = {}
    pieces = []
    for s in statements:
        assert_or_throw(not has_bare_window(s), lambda: NotImplementedError(
            f"{s}: a window function without PARTITION BY / ORDER BY has no SQL form; give it "
            "over(partition_by=.., order_by=..), or use it in a ColumnMap of fa.transform"))
        if isinstance(s, str):
            pieces.append((False, s))
        elif isinstance(s, ColumnExpr):  # an expression piece: its SQL text
            pieces.append((False, to_sql(s)))
        else:
            name = f"_{len(dfs)}"
            dfs[name] = e.to_df(s)
            pieces.append((True, name))
    res: DataFrame = e.sql_engine.select(dfs, StructuredRawSQL(pieces))
    res = e.convert_yield_dataframe(res, as_local)
    if as_fugue or any(isinstance(s, DataFrame) for s in statements):
        return res
    return res.as_pandas() if res.is_local else res.native


def _run_engine_function(name: str, dfs: List[Any], engine: Any, engine_conf: Any, as_fugue: bool,
                         as_local: bool, **kwargs: Any) -> Any:
    """fugue/execution/api.py:145-179 (run_engine_function)."""
    e = make_execution_engine(engine, engine_conf, infer_by=dfs)
    fn = getattr(e, name)
    res = fn(e.to_df(dfs[0]), **kwargs) if len(dfs) == 1 else fn(e.to_df(dfs[0]), e.to_df(dfs[1]), **kwargs)
    for odf in dfs[2:]:
        res = fn(res, e.to_df(odf), **kwargs)
    res = e.convert_yield_dataframe(res, as_local)
    if as_fugue or any(isinstance(x, DataFrame) for x in dfs):
        return res
    return res.as_pandas() if res.is_local else res.native


def union(df1: Any, df2: Any, *dfs: Any, distinct: bool = True, engine: Any = None, engine_conf: Any = None,
          as_fugue: bool = False, as_local: bool = False) -> Any:
    return _run_engine_function("union", [df1, df2, *dfs], engine, engine_conf, as_fugue, as_local, distinct=distinct)


def subtract(df1: Any, df2: Any, *dfs: Any, distinct: bool = True, engine: Any = None, engine_conf: Any = None,
             as_fugue: bool = False, as_local: bool = False) -> Any:
    return _run_engine_function("subtract", [df1, df2, *dfs], engine, engine_conf, as_fugue, as_local,
                                distinct=distinct)


def intersect(df1: Any, df2: Any, *dfs: Any, distinct: bool = True, engine: Any = None, engine_conf: Any = None,
              as_fugue: bool = False, as_local: bool = False) -> Any:
    return _run_engine_function("intersect", [df1, df2, *dfs], engine, engine_conf, as_fugue, as_local,
                                distinct=distinct)


def distinct(df: Any, engine: Any = None, engine_conf: Any = None, as_fugue: bool = False,
             as_local: bool = False) -> Any:
    return _run_engine_function("distinct", [df], engine, engine_conf, as_fugue, as_local)


def dropna(df: Any, how: str = "any", thresh: Optional[int] = None, subset: Optional[List[str]] = None,
           engine: Any = None, engine_conf: Any = None, as_fugue: bool = False, as_local: bool = False) -> Any:
    return _run_engine_function("dropna", [df], engine, engine_conf, as_fugue, as_local, how=how, thresh=thresh,
                                subset=subset)


def fillna(df: Any, value: Any, subset: Optional[List[str]] = None, engine: Any = None, engine_conf: Any = None,
           as_fugue: bool = False, as_local: bool = False) -> Any:
    return _run_engine_function("fillna", [df], engine, engine_conf, as_fugue, as_local, value=value, subset=subset)


def sample(df: Any, n: Optional[int] = None, frac: Optional[float] = None, replace: bool = False,
           seed: Optional[int] = None, engine: Any = None, engine_conf: Any = None, as_fugue: bool = False,
           as_local: bool = False) -> Any:
    return _run_engine_function("sample", [df], engine, engine_conf, as_fugue, as_local, n=n, frac=frac,
                                replace=replace, seed=seed)


def load(path: Any, format_hint: Any = None, columns: Any = None, engine: Any = None, engine_conf: Any = None,
         as_fugue: bool = False, **kwargs: Any) -> Any:
    e = make_execution_engine(engine, engine_conf)
    res = e.load_df(path, format_hint=format_hint, columns=columns, **kwargs)
    return res if as_fugue else res.native


def save(df: Any, path: str, format_hint: Any = None, mode: str = "overwrite", engine: Any = None,
         engine_conf: Any = None, **kwargs: Any) -> None:
    e = make_execution_engine(engine, engine_conf, infer_by=[df])
    e.save_df(e.to_df(df), path, format_hint=format_hint, mode=mode, **kwargs)


def take(df: Any, n: int, presort: Any = None, na_position: str = "last", partition: Any = None,
         engine: Any = None, engine_conf: Any = None, as_fugue: bool = False, as_local: bool = False) -> Any:
    """``fa.take`` (fugue/execution/api.py): first n rows (per partition key group) after sorting."""
    return _run_engine_function("take", [df], engine, engine_conf, as_fugue, as_local, n=n, presort=presort,
                                na_position=na_position,
                                partition_spec=None if partition is None else PartitionSpec(partition))


# ---------------------------------------------------------------------------------------------
# dataframe / dataset utilities of ``fugue.api`` (fugue/dataframe/api.py, fugue/dataset/api.py):
# thin functional wrappers over the DataFrame interface, accepting anything ``as_fugue_df`` knows
# ---------------------------------------------------------------------------------------------
def _convert_df(input_df: Any, output: DataFrame, as_fugue: bool) -> Any:
    """Return type rule of fugue/dataframe/api.py ``_convert_df``: a Fugue DataFrame when asked for or
    when the input was one, otherwise the same kind of native object as the input."""
    import pandas as pd
    import pyarrow as pa

    if as_fugue or isinstance(input_df, DataFrame):
        return output
    if isinstance(input_df, pd.DataFrame):
        return output.as_pandas()
    if isinstance(input_df, pa.Table):
        return output.as_arrow()
    return output.native_as_df()


def is_df(df: Any) -> bool:
    import pandas as pd
    import pyarrow as pa

    from .table import B200Table

    return isinstance(df, (DataFrame, pd.DataFrame, pa.Table, B200Table))


def show(df: Any, n: int = 10, with_count: bool = False, title: Optional[str] = None) -> None:
    """``fa.show`` (fugue/dataset/api.py:18-35)."""
    as_fugue_df(df).show(n=n, with_count=with_count, title=title)


def get_native_as_df(df: Any) -> Any:
    assert_or_throw(is_df(df), lambda: NotImplementedError(f"{type(df)} is not a dataframe"))
    return df.native_as_df() if isinstance(df, DataFrame) else df


def get_schema(df: Any) -> Any:
    return as_fugue_df(df).schema


def get_column_names(df: Any) -> List[Any]:
    return as_fugue_df(df).columns


def as_pandas(df: Any) -> Any:
    return as_fugue_df(df).as_pandas()


def as_arrow(df: Any) -> Any:
    return as_fugue_df(df).as_arrow()


def as_array(df: Any, columns: Optional[List[str]] = None, type_safe: bool = False) -> List[Any]:
    return as_fugue_df(df).as_array(columns, type_safe)


def as_array_iterable(df: Any, columns: Optional[List[str]] = None, type_safe: bool = False) -> Iterable[Any]:
    return as_fugue_df(df).as_array_iterable(columns, type_safe)


def as_dicts(df: Any, columns: Optional[List[str]] = None) -> List[Dict[str, Any]]:
    return as_fugue_df(df).as_dicts(columns)


def as_dict_iterable(df: Any, columns: Optional[List[str]] = None) -> Iterable[Dict[str, Any]]:
    return as_fugue_df(df).as_dict_iterable(columns)


def peek_array(df: Any) -> List[Any]:
    return as_fugue_df(df).peek_array()


def peek_dict(df: Any) -> Dict[str, Any]:
    return as_fugue_df(df).peek_dict()


def head(df: Any, n: int, columns: Optional[List[str]] = None, as_fugue: bool = False) -> Any:
    return _convert_df(df, as_fugue_df(df).head(n, columns), as_fugue)


def alter_columns(df: Any, columns: Any, as_fugue: bool = False) -> Any:
    return _convert_df(df, as_fugue_df(df).alter_columns(columns), as_fugue)


def drop_columns(df: Any, columns: List[str], as_fugue: bool = False) -> Any:
    return _convert_df(df, as_fugue_df(df).drop(columns), as_fugue)


def select_columns(df: Any, columns: List[Any], as_fugue: bool = False) -> Any:
    return _convert_df(df, as_fugue_df(df)[columns], as_fugue)


def rename(df: Any, columns: Dict[str, Any], as_fugue: bool = False) -> Any:
    if len(columns) == 0:
        return df
    return _convert_df(df, as_fugue_df(df).rename(columns), as_fugue)


def as_local(df: Any) -> Any:
    assert_or_throw(is_df(df), lambda: NotImplementedError(f"{type(df)} can't be converted to a local dataset"))
    return _convert_df(df, as_fugue_df(df).as_local(), False)


def as_local_bounded(df: Any) -> Any:
    assert_or_throw(is_df(df), lambda: NotImplementedError(
        f"{type(df)} can't be converted to a local bounded dataset"))  # fugue/dataset/api.py:47-55
    return _convert_df(df, as_fugue_df(df).as_local_bounded(), False)


def is_local(df: Any) -> bool:
    return as_fugue_df(df).is_local


def is_bounded(df: Any) -> bool:
    return as_fugue_df(df).is_bounded


def is_empty(df: Any) -> bool:
    return as_fugue_df(df).empty


def count(df: Any) -> int:
    return as_fugue_df(df).count()


def get_num_partitions(df: Any) -> int:
    return as_fugue_df(df).num_partitions


def get_current_parallelism(engine: Any = None, engine_conf: Any = None) -> int:
    """``fa.get_current_parallelism`` (fugue/execution/api.py): number of GPUs behind the engine."""
    return make_execution_engine(engine, engine_conf).get_current_parallelism()


def get_current_conf(engine: Any = None, engine_conf: Any = None) -> Dict[str, Any]:
    """Conf of the context / global engine, else the registered global conf (fugue/execution/api.py:104-111);
    with an explicit ``engine``: that engine's conf."""
    if engine is None and engine_conf is None:
        return _context_conf()
    return make_execution_engine(engine, engine_conf).conf


def persist(df: Any, lazy: bool = False, engine: Any = None, engine_conf: Any = None, as_fugue: bool = False,
            as_local: bool = False, **kwargs: Any) -> Any:
    """``fa.persist``: on this engine = keep the table resident in HBM."""
    e = make_execution_engine(engine, engine_conf, infer_by=[df])
    return _finish(e, df, e.persist(e.to_df(df), lazy=lazy, **kwargs), as_fugue, as_local)


def broadcast(df: Any, engine: Any = None, engine_conf: Any = None, as_fugue: bool = False,
              as_local: bool = False) -> Any:
    e = make_execution_engine(engine, engine_conf, infer_by=[df])
    return _finish(e, df, e.broadcast(e.to_df(df)), as_fugue, as_local)


def run_engine_function(func: Any, engine: Any = None, engine_conf: Any = None, as_fugue: bool = False,
                        as_local: bool = False, infer_by: Optional[List[Any]] = None) -> Any:
    """``fa.run_engine_function`` (fugue/execution/api.py:145-179): run ``func(engine)`` in the engine's
    context and convert a dataframe result the way every ``fa.*`` function does."""
    e = make_execution_engine(engine, engine_conf, infer_by=infer_by)
    with engine_context(e):
        res = func(e)
    if isinstance(res, DataFrame):
        res = e.convert_yield_dataframe(res, as_local)
        if as_fugue or any(isinstance(x, DataFrame) for x in (infer_by or [])):
            return res
        return res.as_pandas() if res.is_local else res.native
    return res
