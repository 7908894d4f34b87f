// plan.h — a Query bound to one concrete input schema: what DataFusion's
// statement_to_plan + optimiser + physical planner produce per batch in the reference
// (crates/arkflow-plugin/src/processor/sql.rs:188-204), produced here once per schema and cached.
#pragma once
#include <atomic>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "batch.h"
#include "sql.h"
#include "vm.h"

namespace ark {

// One value the row kernels can produce for a selected row.
struct ValueSource {
  enum Kind { PassThrough, Computed } kind = PassThrough;
  int slot = -1;        // PassThrough: index into Plan::used_cols
  VmProgram prog{};     // Computed: result type = type
  DType type = DType::Null;
  bool nullable = true;
  bool validate_utf8 = false;  // CAST(Binary AS Utf8): arrow-cast rejects invalid UTF-8 (safe = false)
};

struct OutputCol {
  std::string name;
  ValueSource src;
};

struct SimplePredicate {  // `col <cmp> literal` on an Int64/Float64 column: the templated fast path
  bool enabled = false;
  int slot = 0;
  int cmp = 0;
  bool is_f64 = false;
  uint64_t constant = 0;  // raw bits of the literal (already coerced to the column's type)
};

enum class AggFunc { Sum, Count, CountStar, Avg, Min, Max };

struct AggSpec {
  AggFunc func = AggFunc::CountStar;
  ValueSource arg;          // unused for CountStar
  DType out_type = DType::Int64;
  std::string name;         // DataFusion display name, e.g. sum(flow.value)
};

struct PostItem {  // one item of the SELECT list of an aggregate query
  enum Kind { Key, Agg, Literal } kind = Key;
  int index = 0;            // key index / agg index
  DType lit_type = DType::Null;
  uint64_t lit_bits = 0;
  std::string lit_str;
  std::string name;
  bool cast_utf8 = false;   // Agg: CAST(<Int64 aggregate> AS STRING), e.g. cast(count(sensor) as string)
};

// concat(a, b, …) of Utf8 columns and string literals (datafusion-functions' ConcatFunc: NULL arguments
// count as empty strings, the result is never NULL).  Evaluated after the row kernels, on the surviving
// rows: its column arguments ride along as hidden PassThrough outputs.
struct ConcatPart {
  bool is_literal = false;
  std::string literal;
  int out_index = -1;   // index into Plan::outputs (visible or hidden)
  DType col_type = DType::Utf8;  // Utf8 bytes, or an Int64 / Boolean column rendered as arrow-cast does ("-12", "true")
};
struct ConcatItem {
  std::string name;
  std::vector<ConcatPart> parts;
  bool is_cast = false;  // CAST(col AS STRING): one part, NULL in ⇒ NULL out (concat() itself never yields NULL)
};
struct FinalItem {      // one column of the result, in SELECT order
  bool is_concat = false;
  int index = 0;        // Plan::outputs index, or Plan::concats index
};

// What the previous batch taught an aggregate plan about its table: sized per plan (two queries of different
// cardinality running side by side must not resize each other's tables).  Shared by the copies of a Plan.
struct AggHints {
  std::atomic<unsigned long long> capacity{1ull << 16};  // table slots to start with
  std::atomic<unsigned int> groups{0};                   // groups of the previous batch (0 = none yet)
  std::atomic<double> avg_key_len{-1.0};                 // bytes per var-len key of the previous batch (sizes the key staging)
  // Key dictionaries kept from batch to batch.  A stream asks the same GROUP BY of batch after batch over largely the
  // same keys (config 3: 10^10 rows, 10^6 sensors): the table's KEYS stay, only the accumulators are reset, so a batch
  // finds its groups with a plain load instead of claiming 10^6 slots with 128-bit CAS again.  A group belongs to a
  // batch's result iff its COUNT(*) accumulator is non-zero.  One table per concurrent caller (thread_num workers).
  struct CachedTable {
    BufferPtr table;
    unsigned long long capacity = 0, total_keys = 0;
    int n_acc = 0;
  };
  std::mutex cache_mu;
  std::vector<CachedTable> cache;
};

// The JSON path functions of datafusion-functions-json 0.47 (DESIGN.md §6).
enum class JsonFn : uint8_t { GetStr, GetInt, GetFloat, GetBool, GetJson, AsText, Contains, Length };

struct JsonPathElem {
  bool is_key = true;
  std::string key;     // an object key, matched against each key with its escapes decoded
  int64_t index = 0;   // an array index (>= 0)
};

// One distinct json_* call of the query.  The planner replaces it by a column appended after the input fields
// (input_fields[n_input_fields + i] for derived[i]); json_path.cu fills every derived column before the plan runs, so
// the row kernels and the aggregate only ever see ordinary columns.
struct DerivedCol {
  JsonFn fn = JsonFn::GetStr;
  int doc_col = -1;          // the input column holding the documents
  bool doc_cast = false;     // a Binary column read through CAST(.. AS STRING): invalid UTF-8 fails the query as the cast does
  std::vector<JsonPathElem> path;  // at most JSON_MAX_PATH elements
};
constexpr int JSON_MAX_PATH = 8;

struct Plan {
  enum Kind { FilterProject, Aggregate, Join } kind = FilterProject;
  std::vector<Field> input_fields;   // of table 0, then one per derived column
  size_t n_input_fields = 0;         // the batch's own columns
  std::vector<DerivedCol> derived;
  std::vector<int> used_cols;        // slot → input column index (kernels see only these)
  bool has_pred = false;
  VmProgram pred{};
  SimplePredicate simple;
  // FilterProject
  std::vector<OutputCol> outputs;
  bool identity = false;             // SELECT * with no WHERE: output = input, no kernel
  int64_t limit = -1;
  std::vector<ConcatItem> concats;   // empty ⇒ the result is `outputs` as is
  std::vector<FinalItem> final_items;
  // Aggregate
  std::vector<ValueSource> keys;     // group keys (PassThrough only)
  std::vector<std::string> key_names;
  std::vector<AggSpec> aggs;
  std::vector<PostItem> post;
  // HAVING, computed SELECT items or LIMIT: `post` is the group frame (every key, then every distinct aggregate call of
  // SELECT and HAVING) and this FilterProject plan over the frame yields the query's result (planner.cc, bind_stage).
  // Null for every other aggregate query, whose result is `post` itself.
  std::shared_ptr<const Plan> stage;
  std::shared_ptr<AggHints> hints = std::make_shared<AggHints>();
  std::shared_ptr<AggHints> final_hints = std::make_shared<AggHints>();  // table of the multi-GPU final merge
  // Join (two tables, inner equi-join)
  std::string left_table, right_table;
  std::vector<Field> right_fields;
  int left_key = -1, right_key = -1;     // column indices in each table
  int join_type = 0;                     // JoinClause::Type: 0 inner, 1 left outer, 2 right outer
  struct JoinOut { int side; int col; std::string name; };
  std::vector<JoinOut> join_out;
};

// Throws ARK_ERR_PROCESS ("Execution query error: …") for binding errors the reference would raise
// at plan time (unknown column/table, type errors) and ARK_ERR_UNSUPPORTED for constructs outside
// the GPU subset.  `json_functions`: the json_* calls bind (the sql processor and the file input's query register
// datafusion-functions-json; a bare SessionContext, as expression evaluation uses, does not).
Plan bind_query(const Query& q, const std::string& table_name, const std::vector<Field>& fields, bool json_functions = false);
Plan bind_join(const Query& q, const std::vector<std::string>& names,
               const std::vector<std::vector<Field>>& tables);

// DataFusion's `schema_name()` of an expression (result column naming).
std::string expr_display_name(const Expr& e, const std::string& table);

}  // namespace ark
