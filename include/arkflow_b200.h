/*
 * arkflow_b200.h — C ABI of libarkflow_b200.so (H100 / sm_90a)
 *
 * Drop-in boundary for ArkFlow's per-batch processor stage.  The reference has NO C ABI on this
 * path: the boundary is two Rust traits resolved through a string-keyed registry
 *   trait Processor { async fn process(&self, MessageBatchRef) -> Result<ProcessResult, Error>; close }
 *       crates/arkflow-core/src/processor/mod.rs:32-79
 *   trait Buffer    { write / read / flush / close }
 *       crates/arkflow-core/src/buffer/mod.rs:26-47
 * A ~150-line Rust shim (INTEGRATION.md) implements those traits by calling the entry points
 * below; data crosses as Arrow C Data Interface structs, the same mechanism the reference already
 * uses toward Python (crates/arkflow-plugin/src/processor/python.rs:52,67).
 *
 * Conventions
 *   - every function returns an ark_status; on non-zero, ark_last_error() (thread-local) holds
 *     the message that the shim wraps into the reference's Error::{Config,Process,…} variant.
 *   - `in` arrays are *moved* into the callee (Arrow C Data Interface semantics: the callee calls
 *     in->release when it is done).  Callee-allocated `out` arrays are released by the caller.
 *   - ProcessResult::None (reference: sql.rs:211-213, empty input batch) is signalled by
 *     out->release == NULL with status ARK_OK.
 *   - all entry points are thread-safe and re-entrant: `process` is called from `thread_num`
 *     concurrent tokio workers in the reference (crates/arkflow-core/src/stream/mod.rs:117-126).
 *   - host variants take host buffers (copies to/from HBM happen inside the call);
 *     *_device variants take/return ArrowDeviceArray with device_type == ARROW_DEVICE_CUDA whose
 *     buffer pointers are device pointers of the current CUDA device (batches stay resident in
 *     HBM between processors).
 */
#ifndef ARKFLOW_B200_H
#define ARKFLOW_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- Arrow C Data Interface (https://arrow.apache.org/docs/format/CDataInterface.html) ---- */
#ifndef ARROW_C_DATA_INTERFACE
#define ARROW_C_DATA_INTERFACE
#define ARROW_FLAG_DICTIONARY_ORDERED 1
#define ARROW_FLAG_NULLABLE 2
#define ARROW_FLAG_MAP_KEYS_SORTED 4
struct ArrowSchema {
  const char* format;
  const char* name;
  const char* metadata;
  int64_t flags;
  int64_t n_children;
  struct ArrowSchema** children;
  struct ArrowSchema* dictionary;
  void (*release)(struct ArrowSchema*);
  void* private_data;
};
struct ArrowArray {
  int64_t length;
  int64_t null_count;
  int64_t offset;
  int64_t n_buffers;
  int64_t n_children;
  const void** buffers;
  struct ArrowArray** children;
  struct ArrowArray* dictionary;
  void (*release)(struct ArrowArray*);
  void* private_data;
};
#endif

#ifndef ARROW_C_DEVICE_DATA_INTERFACE
#define ARROW_C_DEVICE_DATA_INTERFACE
typedef int32_t ArrowDeviceType;
#define ARROW_DEVICE_CPU 1
#define ARROW_DEVICE_CUDA 2
#define ARROW_DEVICE_CUDA_HOST 3
struct ArrowDeviceArray {
  struct ArrowArray array;
  int64_t device_id;
  ArrowDeviceType device_type;
  void* sync_event; /* cudaEvent_t* or NULL (NULL: data is ready) */
  int64_t reserved[3];
};
#endif

/* ---- status codes → reference Error variants (crates/arkflow-core/src/lib.rs:66-110) ---- */
typedef enum ark_status {
  ARK_OK = 0,
  ARK_ERR_CONFIG = 1,      /* Error::Config(msg)         e.g. sql.rs:235-239 missing configuration   */
  ARK_ERR_PROCESS = 2,     /* Error::Process(msg)        e.g. sql.rs:92-98,120-147                   */
  ARK_ERR_UNSUPPORTED = 3, /* SQL outside the GPU subset: the shim may fall back to DataFusion      */
  ARK_ERR_SERIALIZATION = 4, /* Error::Serialization   (serde_json::from_value `?`, sql.rs:240)      */
  ARK_ERR_CUDA = 5,        /* CUDA runtime failure (no reference analogue) → Error::Process          */
  ARK_ERR_EOF = 6          /* Error::EOF (buffer closed and drained)                                 */
} ark_status;

typedef struct ark_proc ark_proc_t; /* a built Processor (sql / json_to_arrow / arrow_to_json / protobuf_to_arrow / arrow_to_protobuf) */
typedef struct ark_buf ark_buf_t;   /* a built Buffer (memory / session_window / tumbling_window / sliding_window) */
typedef struct ark_batcher ark_batcher_t; /* a built `batch` processor                                  */
typedef struct ark_dist ark_dist_t; /* one rank's end of the device-side GROUP BY exchange              */
typedef struct ark_input ark_input_t; /* a built Input (`generate`, `file`) that produces batches in HBM   */

/* ---- library ---- */
/* Bind the calling process to CUDA device `device` (-1: keep current) and warm the pools.
 * Replaces nothing in the reference (it has no device); called once from the shim's init(). */
int ark_b200_init(int device);
int ark_b200_device_count(int* out_count);
const char* ark_b200_version(void);
const char* ark_last_error(void); /* thread-local, valid until the next call on this thread */

/* ---- `sql` processor: replaces SqlProcessorBuilder::build / SqlProcessor::{new,process,close}
 *      crates/arkflow-plugin/src/processor/sql.rs:227-243, 68-105, 208-225 ---- */
/* config_json = the processor's flattened YAML as JSON: {"query": "...", "table_name": "flow"?,
 * "temporary_list": [{"name","table_name","key"}]?, "temporaries_resolved": true?} — the shim owns
 * Resource.temporary: it checks each name (sql.rs:70-86: "Temporary X not found"), sets
 * temporaries_resolved, evaluates the keys with ark_expr_evaluate and registers what Temporary::get
 * returns through ark_sql_process_tables.
 * NULL config → ARK_ERR_CONFIG ("Batch processor configuration is missing", sql.rs:235-239);
 * unparsable SQL → ARK_ERR_PROCESS ("SQL query error: …", sql.rs:92-98) at construction. */
int ark_sql_create(const char* config_json, ark_proc_t** out);
/* One RecordBatch (struct array + schema) in, one out.  Replaces SqlProcessor::process
 * (sql.rs:209-220) + execute_query (sql.rs:108-149). */
int ark_sql_process(ark_proc_t* p, struct ArrowArray* in, struct ArrowSchema* in_schema,
                    struct ArrowArray* out, struct ArrowSchema* out_schema);
int ark_sql_process_device(ark_proc_t* p, struct ArrowDeviceArray* in, struct ArrowSchema* in_schema,
                           struct ArrowDeviceArray* out, struct ArrowSchema* out_schema);
/* Multi-table form used by the window buffers' JoinOperation (buffer/join.rs:62-132): table i is
 * registered under names[i] before the query runs. */
int ark_sql_process_tables(ark_proc_t* p, int n_tables, const char* const* names,
                           struct ArrowArray* ins, struct ArrowSchema* in_schemas,
                           struct ArrowArray* out, struct ArrowSchema* out_schema);
int ark_sql_process_tables_device(ark_proc_t* p, int n_tables, const char* const* names,
                                  struct ArrowDeviceArray* ins, struct ArrowSchema* in_schemas,
                                  struct ArrowDeviceArray* out, struct ArrowSchema* out_schema);

/* ---- `json_to_arrow` / `arrow_to_json` processors: replace Json{ToArrow,…}ProcessorBuilder::build
 *      and ::process, crates/arkflow-plugin/src/processor/json.rs:115-152, 48-61, 78-113 ---- */
/* config_json: {"value_field": "__value__"?, "fields_to_include": ["a","b"]?}; NULL → ARK_ERR_CONFIG */
int ark_json_to_arrow_create(const char* config_json, ark_proc_t** out);
int ark_json_to_arrow_process(ark_proc_t* p, struct ArrowArray* in, struct ArrowSchema* in_schema,
                              struct ArrowArray* out, struct ArrowSchema* out_schema);
int ark_json_to_arrow_process_device(ark_proc_t* p, struct ArrowDeviceArray* in,
                                     struct ArrowSchema* in_schema, struct ArrowDeviceArray* out,
                                     struct ArrowSchema* out_schema);
int ark_arrow_to_json_create(const char* config_json, ark_proc_t** out);
int ark_arrow_to_json_process(ark_proc_t* p, struct ArrowArray* in, struct ArrowSchema* in_schema,
                              struct ArrowArray* out, struct ArrowSchema* out_schema);
int ark_arrow_to_json_process_device(ark_proc_t* p, struct ArrowDeviceArray* in,
                                     struct ArrowSchema* in_schema, struct ArrowDeviceArray* out,
                                     struct ArrowSchema* out_schema);

/* ---- `protobuf_to_arrow` / `arrow_to_protobuf` processors: replace {ProtobufToArrow,ArrowToProtobuf}
 *      ProcessorBuilder::build, ProtobufProcessor::{new,process} and the conversions they call,
 *      crates/arkflow-plugin/src/processor/protobuf.rs:197-232, 71-148 and
 *      crates/arkflow-plugin/src/component/protobuf.rs:41-339 ---- */
/* config_json: {"proto_inputs": ["dir", …], "proto_includes": ["dir", …]?, "message_type": "pkg.Msg",
 * "value_field": "__value__"? (protobuf_to_arrow), "fields_to_include": ["a", …]? (arrow_to_protobuf)}.
 * Deliberate deviation: the keys are read flat, the shape the reference's documentation
 * (docs/docs/components/2-processors/protobuf.md) and examples/protobuf_example.yaml use; the reference's
 * ArrowToProtobufProcessorConfig nests them under `c` (protobuf.rs:165-169, no #[serde(flatten)]) and so
 * rejects its own documented shape with "missing field `c`".
 * Every `*.proto` file directly inside each proto_inputs directory is parsed (imports resolved against
 * proto_includes, default proto_inputs) on the host, without a CUDA device.  NULL config → ARK_ERR_CONFIG
 * ("ProtobufToArrow processor configuration is missing" / "ArrowToProtobuf …"); a missing or mistyped key →
 * ARK_ERR_SERIALIZATION; no .proto file → ARK_ERR_CONFIG ("No proto files found in the specified paths…");
 * a parse or type-resolution error → ARK_ERR_CONFIG ("Failed to parse the proto file: …"); an unknown
 * message → ARK_ERR_CONFIG ("The message type could not be found: <name>").
 * An empty batch gives no output (ProcessResult::None, protobuf.rs:101-103); a batch of only NULL payloads gives zero
 * rows with the message's columns (the reference panics there).  Library limits, not reference behaviour:
 * protobuf_to_arrow of a message with more than 64 fields, and arrow_to_protobuf encoding more than 64 fields, return
 * ARK_ERR_UNSUPPORTED; an output string / binary column of 2 GiB or more returns ARK_ERR_PROCESS.  protobuf_to_arrow decodes the
 * Binary column `value_field` into one non-nullable column per message field; arrow_to_protobuf appends a
 * non-null Binary `__value__` column to the input.  Error rules: csrc/protobuf.cu. */
int ark_protobuf_to_arrow_create(const char* config_json, ark_proc_t** out);
int ark_protobuf_to_arrow_process(ark_proc_t* p, struct ArrowArray* in, struct ArrowSchema* in_schema,
                                  struct ArrowArray* out, struct ArrowSchema* out_schema);
int ark_protobuf_to_arrow_process_device(ark_proc_t* p, struct ArrowDeviceArray* in,
                                         struct ArrowSchema* in_schema, struct ArrowDeviceArray* out,
                                         struct ArrowSchema* out_schema);
int ark_arrow_to_protobuf_create(const char* config_json, ark_proc_t** out);
int ark_arrow_to_protobuf_process(ark_proc_t* p, struct ArrowArray* in, struct ArrowSchema* in_schema,
                                  struct ArrowArray* out, struct ArrowSchema* out_schema);
int ark_arrow_to_protobuf_process_device(ark_proc_t* p, struct ArrowDeviceArray* in,
                                         struct ArrowSchema* in_schema, struct ArrowDeviceArray* out,
                                         struct ArrowSchema* out_schema);

/* ---- expr::evaluate_expr: replaces crates/arkflow-plugin/src/expr/mod.rs:92-122 (the key expression
 *      of a `temporary_list` entry, processor/sql.rs:151-186) ---- */
/* Parses `expr` as ONE SQL scalar expression against the batch schema and evaluates it on the device.
 * The result is a one-column batch: as many rows as the input (ColumnarValue::Array), or ONE row with
 * *is_scalar = 1 when the expression references no column (ColumnarValue::Scalar).  Parsed expressions
 * are cached by text (EXPR_CACHE, expr/mod.rs:27-28).  Errors → ARK_ERR_PROCESS / ARK_ERR_UNSUPPORTED. */
int ark_expr_evaluate(const char* expr, struct ArrowArray* in, struct ArrowSchema* in_schema,
                      struct ArrowArray* out, struct ArrowSchema* out_schema, int* is_scalar);
int ark_expr_evaluate_device(const char* expr, struct ArrowDeviceArray* in, struct ArrowSchema* in_schema,
                             struct ArrowDeviceArray* out, struct ArrowSchema* out_schema, int* is_scalar);

/* Processor::close (sql.rs:222-224, json.rs:63-65) and drop. */
int ark_proc_close(ark_proc_t* p);
void ark_proc_destroy(ark_proc_t* p);

/* ---- concat_batches: replaces arrow::compute::concat_batches at
 *      buffer/memory.rs:130, buffer/window.rs:131,159, sql.rs:146, component/json.rs:54 ---- */
int ark_concat_batches(int n, struct ArrowArray* ins, struct ArrowSchema* in_schemas,
                       struct ArrowArray* out, struct ArrowSchema* out_schema);
int ark_concat_batches_device(int n, struct ArrowDeviceArray* ins, struct ArrowSchema* in_schemas,
                              struct ArrowDeviceArray* out, struct ArrowSchema* out_schema);

/* ---- buffers: replace {Memory,SessionWindow,TumblingWindow}BufferBuilder::build and
 *      Buffer::{write,read,flush,close}: buffer/memory.rs:142-237, session_window.rs:97-159,
 *      tumbling_window.rs:90-145, window.rs:99-190 ---- */
/* kind: "memory" | "session_window" | "tumbling_window" | "sliding_window" (buffer/sliding_window.rs:
 * 52-238, builder checks :255-270); config_json = the buffer's YAML as JSON
 * ({"capacity":N,"timeout":"1s"} | {"gap":"1s","join":{...}?} | {"interval":"1s","join":{...}?} |
 *  {"window_size":N,"interval":"1s","slide_size":M});
 * input_names_json: JSON array of the input names Resource.input_names held at build time
 * (multiple_inputs.rs:133-142), or NULL. */
int ark_buffer_create(const char* kind, const char* config_json, const char* input_names_json,
                      ark_buf_t** out);
/* input_name: MessageBatch::get_input_name() or NULL; ack_token: opaque id the shim maps back to
 * its Arc<dyn Ack> (returned from read as a list). */
int ark_buffer_write(ark_buf_t* b, struct ArrowArray* in, struct ArrowSchema* in_schema,
                     const char* input_name, uint64_t ack_token);
/* Blocks like Buffer::read.  status ARK_OK with out->release==NULL ⇒ Ok(None) (closed & empty).
 * acks: caller-provided array of capacity acks_cap; *n_acks receives the number of tokens whose
 * batches were merged into `out` (VecAck, window.rs:124-139 / ArrayAck, memory.rs:121-137). */
int ark_buffer_read(ark_buf_t* b, struct ArrowArray* out, struct ArrowSchema* out_schema,
                    uint64_t* acks, int64_t acks_cap, int64_t* n_acks);
/* The same write / read for batches that already are / shall stay in HBM (nothing is copied). */
int ark_buffer_write_device(ark_buf_t* b, struct ArrowDeviceArray* in, struct ArrowSchema* in_schema,
                            const char* input_name, uint64_t ack_token);
int ark_buffer_read_device(ark_buf_t* b, struct ArrowDeviceArray* out, struct ArrowSchema* out_schema,
                           uint64_t* acks, int64_t acks_cap, int64_t* n_acks);
int ark_buffer_flush(ark_buf_t* b);
int ark_buffer_close(ark_buf_t* b);
void ark_buffer_destroy(ark_buf_t* b);

/* ---- `batch` processor: replaces BatchProcessorBuilder::build and BatchProcessor::{process,flush,close},
 *      crates/arkflow-plugin/src/processor/batch.rs:126-143, 95-124, 72-92 ---- */
/* config_json: {"count": N, "timeout_ms": T}; NULL → ARK_ERR_CONFIG ("Batch processor configuration is
 * missing", batch.rs:135-139).  process() keeps the batch in HBM; when `count` batches are held or
 * `timeout_ms` has passed since the last flush it returns their concatenation (ProcessResult::Single),
 * otherwise out->release stays NULL (ProcessResult::None). */
int ark_batch_create(const char* config_json, ark_batcher_t** out);
int ark_batch_process(ark_batcher_t* b, struct ArrowArray* in, struct ArrowSchema* in_schema,
                      struct ArrowArray* out, struct ArrowSchema* out_schema);
int ark_batch_flush(ark_batcher_t* b, struct ArrowArray* out, struct ArrowSchema* out_schema);
int ark_batch_close(ark_batcher_t* b);
void ark_batch_destroy(ark_batcher_t* b);

/* ---- multi-GPU GROUP BY / JOIN building blocks (device-resident; SURVEY.md §8(e)).  The
 *      exchange between them is the caller's NCCL all-to-all or the peer-memory pull below; nothing like this exists in the
 *      reference (DataFusion's RepartitionExec(Hash) is in-process). ---- */
/* Partial aggregate of one local batch → (keys, partial states) batch, hash-partitioned into
 * n_parts contiguous row ranges; part_rows[n_parts] receives the row count of each range. */
int ark_sql_partial_aggregate_device(ark_proc_t* p, struct ArrowDeviceArray* in,
                                     struct ArrowSchema* in_schema, int n_parts,
                                     struct ArrowDeviceArray* out, struct ArrowSchema* out_schema,
                                     int64_t* part_rows);
/* Merge partial-state batches (as produced above, possibly from several ranks) into the final
 * result of the query. */
int ark_sql_final_aggregate_device(ark_proc_t* p, struct ArrowDeviceArray* in,
                                   struct ArrowSchema* in_schema, struct ArrowDeviceArray* out,
                                   struct ArrowSchema* out_schema);
/* Hash-partition the rows of a batch on column key_column into n_parts contiguous ranges
 * (RepartitionExec(Hash) stand-in for the join repartition). */
int ark_hash_partition_device(struct ArrowDeviceArray* in, struct ArrowSchema* in_schema,
                              const char* key_column, int n_parts, struct ArrowDeviceArray* out,
                              struct ArrowSchema* out_schema, int64_t* part_rows);

/* ---- the same exchange over peer memory instead of NCCL (csrc/ipc_exchange.cu; one node, one process per
 *      GPU).  ark_ipc_export_device describes a device batch as CUDA IPC handles (blob: header + one record
 *      per column; query the size with blob_cap = 0, status ARK_ERR_PROCESS and *blob_size set); the caller
 *      all-gathers the blobs and the partition row counts, and every rank pulls its slices of all sources
 *      with ark_ipc_concat_slices_device: ONE segmented-copy launch reads the peers' buffers over NVLink and
 *      lays the rows out as one local batch (sources in order).  The exporter keeps its batch alive until
 *      every reader is done (a barrier in the caller). ---- */
int ark_ipc_export_device(struct ArrowDeviceArray* in, struct ArrowSchema* in_schema, uint8_t* blob,
                          int64_t blob_cap, int64_t* blob_size);
int ark_ipc_concat_slices_device(int n_src, const uint8_t* const* blobs, const int64_t* blob_sizes,
                                 const int64_t* row0, const int64_t* n_rows,
                                 struct ArrowDeviceArray* out, struct ArrowSchema* out_schema);

/* ---- the GROUP BY exchange as device code (csrc/group_exchange.cu; one node, one process — or context — per GPU).
 *      Replaces the host-orchestrated sequence partial_aggregate → export → all-gather → pull → final_aggregate
 *      for keys that fit a table slot (Utf8/Binary up to 12 bytes, Int64, Boolean, NULL): the kernel that scans
 *      the partial hash table PUSHES each group's {key, accumulators} slot over NVLink into the owner rank's receive
 *      region, signals with a system-scope release store, and the owner's merge kernel consumes the records of
 *      every source as soon as their flags arrive — no NCCL call, no host round trip and no staging copy on the
 *      data path (DataFusion's AggregateExec(Partial) → RepartitionExec(Hash) → AggregateExec(FinalPartitioned),
 *      reached in-process from crates/arkflow-plugin/src/processor/sql.rs:126-129).
 *
 *      Set-up, once per process: ark_dist_create allocates this rank's comm buffer (header + 2 × world receive
 *      regions of region_bytes: a region must hold the partial states one source sends this rank in one step,
 *      32 bytes per group for up to two accumulators); ark_dist_export describes it (CUDA IPC handle,
 *      ark_dist_handle_bytes() bytes); the caller gathers every rank's handle by any means (the harness uses one
 *      torch.distributed all_gather) and passes them, in rank order, to ark_dist_connect.
 *      Per batch, on every rank in the same order: ark_sql_group_by_exchange_device(in) → this rank's share of the
 *      groups (owners are disjoint: the concatenation over ranks is the full result).  The push and merge halves
 *      are also exported separately (several ranks driven from one thread in the tests).
 *      Returns ARK_ERR_UNSUPPORTED on EVERY rank alike when some rank met a key that cannot travel inline (longer
 *      than 12 bytes); the step is consumed and the caller falls back to the descriptor exchange above. ---- */
int ark_dist_create(int rank, int world, int64_t region_bytes, ark_dist_t** out);
int64_t ark_dist_handle_bytes(void);
int ark_dist_export(ark_dist_t* d, uint8_t* blob, int64_t blob_cap, int64_t* blob_size);
int ark_dist_connect(ark_dist_t* d, const uint8_t* blobs, int64_t blob_stride);
/* out4 = {steps issued, records received in the last step, groups owned after the last merge, region_bytes} */
int ark_dist_stats(ark_dist_t* d, int64_t* out4);
void ark_dist_destroy(ark_dist_t* d);
int ark_sql_group_by_exchange_device(ark_proc_t* p, ark_dist_t* d, struct ArrowDeviceArray* in,
                                     struct ArrowSchema* in_schema, struct ArrowDeviceArray* out,
                                     struct ArrowSchema* out_schema);
int ark_sql_group_by_push_device(ark_proc_t* p, ark_dist_t* d, struct ArrowDeviceArray* in,
                                 struct ArrowSchema* in_schema);
int ark_sql_group_by_merge_device(ark_proc_t* p, ark_dist_t* d, struct ArrowDeviceArray* out,
                                  struct ArrowSchema* out_schema);

/* ---- inputs that produce their batches on the device (csrc/inputs.cu).
 *      type "generate" ← `impl Input for GenerateInput`, crates/arkflow-plugin/src/input/generate.rs:59-96: config
 *        {context: string, interval: duration string, count?: usize, batch_size?: usize (default 1)}; read() yields
 *        batch_size clones of `context` as a non-null Binary column `__value__`, sleeps `interval` before every read
 *        but the first, and returns ARK_ERR_EOF once `count` is reached or the next batch would exceed it.
 *        NULL config → ARK_ERR_CONFIG "Generate input configuration is missing" (generate.rs:107-111).
 *      type "file" ← `impl Input for FileInput`, crates/arkflow-plugin/src/input/file.rs:395-455: config
 *        {input_type: {type: "json" | "csv", path}, query?: {query, table?}, batch_size?}; connect() loads the file into
 *        HBM and indexes its lines, read() decodes the next batch_size lines (NDJSON: json_to_arrow kernels; CSV:
 *        header + type inference over the first 1000 rows on the host, csv_parse_kernel) and applies the optional
 *        query; ARK_ERR_EOF at the end.  parquet / avro / arrow and remote stores → ARK_ERR_UNSUPPORTED.
 *      ark_input_read_device leaves the batch in HBM (feed it to ark_buffer_write_device / *_process_device). ---- */
int ark_input_create(const char* type, const char* config_json, ark_input_t** out);
int ark_input_connect(ark_input_t* in);
int ark_input_read(ark_input_t* in, struct ArrowArray* out, struct ArrowSchema* out_schema);
int ark_input_read_device(ark_input_t* in, struct ArrowDeviceArray* out, struct ArrowSchema* out_schema);
int ark_input_close(ark_input_t* in);
void ark_input_destroy(ark_input_t* in);

/* ---- synthetic input of schema S (SURVEY.md §8(d)), generated in HBM.  Bench/test support. ---- */
/* value_kind: 0 = Int64 uniform [0,20), 1 = Float64 20*u.  key_space K: sensor = "temp_%07d" % k.
 * row0: global index of the first row (so shards/batches are slices of one logical table). */
int ark_synth_batch_device(int64_t n_rows, int64_t row0, uint64_t seed, int value_kind,
                           int64_t key_space, struct ArrowDeviceArray* out,
                           struct ArrowSchema* out_schema);

/* ---- counters (bench.py's gpu_launches claim) ---- */
int64_t ark_kernel_launch_count(void); /* kernels of this library launched since load */
/* Device time (ms, CUDA events on the launching stream) and launches accumulated for kernel
 * `name` since the last reset; timing is off unless enabled. */
void ark_kernel_timing_enable(int on);
void ark_kernel_timing_reset(void);
int ark_kernel_timing_get(const char* name, double* total_ms, int64_t* launches);

/* The host copy used to stage pageable input buffers into pinned memory (csrc/host_copy.cpp; no reference counterpart — arrow-rs
 * buffers are handed to DataFusion in place).  kind: 0 memcpy, 1 AVX2 non-temporal, 2 AVX-512 non-temporal, -1 best the CPU has.
 * Exposed so that the copy can be tested without a GPU.  Returns the kind that was used. */
int ark_host_copy(void* dst, const void* src, int64_t n, int kind);

#ifdef __cplusplus
}
#endif
#endif /* ARKFLOW_B200_H */
