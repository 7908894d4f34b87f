"""CPU oracle for the buffer stage's data path — TEST INFRASTRUCTURE (see oracle/__init__.py).

Only the *data* semantics are restated (what a drained window contains and in which row order); the
trigger logic (timers, capacity) is host code tested directly against the reference's own tests.
  memory buffer      : drain oldest-first, concat            buffer/memory.rs:106-138,155
  window buffers     : per input drain newest-first, concat per input, then concat across inputs in
                       first-seen input order, or JoinOperation                 buffer/window.rs:99-190
  JoinOperation      : json-decode each input's __value__, require every configured input, run the SQL
                                                                                 buffer/join.rs:62-146
Every concatenation is arrow-rs `concat_batches(schema, batches)` with the schema of one chosen batch (concat_batches
below); each drain names which batch, as its call site does.
"""
from __future__ import annotations

from typing import Optional

import pyarrow as pa

from .json_oracle import json_to_arrow
from .sql_oracle import OracleError, sql_join

MERGE = "Merge batches failed: "  # Error::Process(format!("Merge batches failed: {}", e)), memory.rs:131 and the others


def concat_batches(schema: pa.Schema, batches: list[pa.RecordBatch]) -> pa.RecordBatch:
    """arrow-rs 55 `arrow::compute::concat_batches(&schema, &batches)` followed by the call sites' map_err.

    Columns are matched by position; names, types and nullability come from `schema`, whatever the members call them.
    A member column of another type fails (kind Process; the text is arrow-rs's and not restated).  The result is built
    with RecordBatch::try_new, which fails when a non-nullable field holds NULLs: the message below is arrow-array's
    (record_batch.rs, try_new_impl).  No batches give an empty batch; no fields give a batch of the summed rows."""
    if len(schema) == 0:
        n = sum(b.num_rows for b in batches)
        return pa.RecordBatch.from_struct_array(pa.array([{}] * n, pa.struct([])))
    if not batches:
        return pa.RecordBatch.from_arrays([pa.array([], f.type) for f in schema], schema=schema)
    cols = []
    for i, f in enumerate(schema):
        parts = []
        for b in batches:
            if b.num_columns != len(schema) or b.column(i).type != f.type:
                raise OracleError("Process", MERGE + "Invalid argument error: column types must match schema types")
            parts.append(b.column(i))
        col = pa.concat_arrays(parts)
        if not f.nullable and col.null_count > 0:
            raise OracleError("Process", MERGE + f"Invalid argument error: Column '{f.name}' is declared as non-nullable "
                                                 "but contains null values")
        cols.append(col)
    return pa.RecordBatch.from_arrays(cols, schema=schema)


def concat(batches: list[pa.RecordBatch]) -> pa.RecordBatch:
    """concat_batches with the first batch's schema: every call site takes the schema of messages[0]."""
    return concat_batches(batches[0].schema, batches)


def memory_drain(writes: list[pa.RecordBatch]) -> pa.RecordBatch:
    return concat(list(writes))  # FIFO: the oldest batch gives the schema


def window_drain(writes: list[tuple[Optional[str], pa.RecordBatch]], join: Optional[dict] = None, input_names=()) -> pa.RecordBatch:
    order, queues = [], {}
    for name, rb in writes:
        name = name or ""
        if name not in queues:
            queues[name] = []
            order.append(name)
        queues[name].insert(0, rb)  # push_front
    per_input = [(n, concat(queues[n])) for n in order]  # pop_front ⇒ newest first: the newest batch gives the schema
    if join is None:
        return concat([b for _, b in per_input])  # the first input's merged batch gives the schema
    tables = {}
    for n, b in per_input:
        decoded = json_to_arrow(b, join.get("value_field") or "__value__")
        if n:
            tables[n] = decoded
    if not all(n in tables for n in input_names):
        return pa.RecordBatch.from_arrays([], schema=pa.schema([]))
    return sql_join(tables, join["query"])


def sliding_windows(writes: list[pa.RecordBatch], window_size: int, slide_size: int) -> list[pa.RecordBatch]:
    """SlidingWindow::process_slide repeated until fewer than window_size batches remain
    (buffer/sliding_window.rs:104-158): a window is the first window_size queued batches concatenated in
    arrival order; then slide_size batches leave the front of the queue.  PARITY: the reference asserts
    only that a window is produced (sliding_window.rs:396-418) — contents unpinned."""
    q = list(writes)
    out = []
    while len(q) >= window_size:
        out.append(concat(q[:window_size]))  # the oldest batch of the window gives the schema
        del q[:slide_size]
    return out


def batch_processor(writes: list[pa.RecordBatch], count: int) -> list[pa.RecordBatch]:
    """BatchProcessor::process by count only (processor/batch.rs:95-116): every `count`-th message returns
    the concatenation of the held ones.  batch.rs:170-186 pins `batch.len() == 2` for count = 2."""
    out, held = [], []
    for rb in writes:
        held.append(rb)
        if len(held) >= count:
            out.append(concat(held))  # the oldest held batch gives the schema (batch.rs:80-82)
            held = []
    return out
