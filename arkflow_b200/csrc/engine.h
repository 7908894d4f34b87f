// engine.h — host-side processors: the C++ mirror of the reference's plugin objects for this path.
//   SqlProcessor        ← crates/arkflow-plugin/src/processor/sql.rs:59-225
//   JsonToArrow / ArrowToJson ← crates/arkflow-plugin/src/processor/json.rs:42-113
//   ProtobufToArrow / ArrowToProtobuf ← crates/arkflow-plugin/src/processor/protobuf.rs:33-244
#pragma once
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "batch.h"
#include "filter_project.cuh"
#include "plan.h"
#include "sql.h"

namespace ark {

// declared in batch.cu
const std::string& last_error_ref();
int64_t launch_count();
void timing_enable(int on);
void timing_reset();
bool timing_get(const char* name, double* ms, int64_t* n);
void resolve_varlen_extents(Batch& b, const std::vector<int>& col_idx, cudaStream_t stream);
void resolve_varlen_extents_many(std::vector<Column*>& cols, cudaStream_t stream);
Batch apply_concats(const Plan& plan, Batch& r, cudaStream_t stream);  // string_funcs.cu
Column format_int64_column(const Column& src, const std::string& name, cudaStream_t stream);  // string_funcs.cu

// kernels' host launchers
void launch_filter_project(const FpParams& P, int pred_kind, cudaStream_t stream);
void launch_utf8_validate(const int32_t* offsets, const uint8_t* data, const uint8_t* validity, int vbit0, int64_t n, int* bad, cudaStream_t stream);
const char* vm_error_text(int vm_error);  // arrow-arith / arrow-cast message of a VmError
void launch_pack_bits(const uint8_t* bytes, int64_t n, uint8_t* bitmap, unsigned long long* zeros, cudaStream_t stream);

struct Processor {
  virtual ~Processor() {}
  virtual const char* type() const = 0;
};

struct SqlProcessor : Processor {
  const char* type() const override { return "sql"; }
  std::string query_text;
  std::string table_name = "flow";  // DEFAULT_TABLE_NAME, sql.rs:38
  Query ast;

  // config_json as documented at ark_sql_create
  static std::unique_ptr<SqlProcessor> from_config(const char* config_json);

  // plan cache: one bound plan per distinct input schema (SURVEY.md appendix D.2)
  std::shared_ptr<const Plan> plan_for(const std::vector<Field>& fields);
  // the aggregate plan most recently bound by this processor (the final merge sees only partial states)
  std::shared_ptr<const Plan> last_aggregate_plan();
  std::shared_ptr<const Plan> join_plan_for(const std::vector<std::string>& names,
                                            const std::vector<std::vector<Field>>& tables);

  // Runs the bound plan on an HBM-resident batch.  `in` must contain the plan's used columns.
  Batch execute(const Plan& plan, Batch& in, cudaStream_t stream);

 private:
  std::mutex mu_;
  std::map<std::string, std::shared_ptr<const Plan>> plans_;
  std::shared_ptr<const Plan> last_agg_;
};

Batch run_filter_project(const Plan& plan, Batch& in, cudaStream_t stream);
Batch run_aggregate(const Plan& plan, Batch& in, cudaStream_t stream);
Batch run_join(const Plan& plan, Batch& left, Batch& right, cudaStream_t stream);
Batch run_partial_aggregate(const Plan& plan, Batch& in, int n_parts, std::vector<int64_t>& part_rows, cudaStream_t stream);
Batch run_final_aggregate(const Plan& plan, Batch& partial, cudaStream_t stream);
struct DistCtx;  // group_exchange.h
void run_group_by_push(const Plan& plan, Batch& in, DistCtx& d, cudaStream_t stream);
bool run_group_by_merge(const Plan& plan, DistCtx& d, Batch& out, cudaStream_t stream);
std::unique_ptr<Processor> make_json_to_arrow(const char* config_json);
const std::string& json_to_arrow_value_field(const Processor& p);
std::unique_ptr<Processor> make_json_to_arrow_for_sample(const std::vector<std::string>& sample_records);  // schema fixed by the sample (file input)
Batch json_to_arrow_device(const Processor& proc, Batch& in, cudaStream_t stream);
Batch hash_partition(Batch& in, const std::string& key_column, int n_parts, std::vector<int64_t>& part_rows, cudaStream_t stream);
Column take_column(const Column& src, const unsigned int* idx, int64_t n, const std::string& name, cudaStream_t stream, bool may_miss = false);
struct TakeSpec { const Column* src; int side; std::string name; bool may_miss; };  // side: which index array (0 | 1)
std::vector<Column> take_columns(const std::vector<TakeSpec>& specs, const unsigned int* idx0, const unsigned int* idx1, int64_t n, cudaStream_t stream);
std::unique_ptr<Processor> make_arrow_to_json(const char* config_json);
Batch arrow_to_json_device(const Processor& proc, Batch& in, cudaStream_t stream);
// `fields_to_include` kept none of a non-empty batch's columns (arrow_to_json, arrow_to_protobuf)
[[noreturn]] void fail_filtered_to_no_columns();
std::unique_ptr<Processor> make_protobuf_to_arrow(const char* config_json);
const std::string& protobuf_to_arrow_value_field(const Processor& p);
Batch protobuf_to_arrow_device(const Processor& proc, Batch& in, cudaStream_t stream);
std::unique_ptr<Processor> make_arrow_to_protobuf(const char* config_json);
Batch arrow_to_protobuf_device(const Processor& proc, Batch& in, cudaStream_t stream);
Batch concat_device(std::vector<Batch>& ins, cudaStream_t stream);
Batch synth_batch(int64_t n, int64_t row0, uint64_t seed, int value_kind, int64_t key_space, cudaStream_t stream);

}  // namespace ark
