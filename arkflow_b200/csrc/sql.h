// sql.h — AST of the SQL subset the CUDA `sql` processor accepts.
//
// The reference hands the query string to DataFusion's parser once at build time
// (crates/arkflow-plugin/src/processor/sql.rs:91-98, sqlparser 0.55 generic dialect) and re-plans it
// per batch (sql.rs:188-204).  Here the string is parsed once into this AST; binding to a concrete
// input schema (plan.h) happens once per distinct schema and is cached.
#pragma once
#include <cstdint>
#include <memory>
#include <string>
#include <vector>

namespace ark {

// List / Struct: columns this library produces itself (json_to_arrow of nested values); never query operands.
// Int32 / UInt32 / UInt64 / Float32: only the protobuf codec produces and reads them (protobuf.cu); never query operands.
enum class DType : uint8_t { Null = 0, Bool = 1, Int64 = 2, Float64 = 3, Utf8 = 4, Binary = 5, List = 6, Struct = 7,
                             Int32 = 8, UInt32 = 9, UInt64 = 10, Float32 = 11 };
const char* dtype_name(DType t);         // DataFusion display name: Int64, Float64, Utf8, …
const char* dtype_arrow_format(DType t); // Arrow C format string: "l", "g", "u", "z", "b", "n"

struct Expr;
using ExprPtr = std::unique_ptr<Expr>;

struct Expr {
  enum Kind { Column, Literal, Binary, Unary, Func, Cast, IsNull, Star } kind = Literal;
  // Column
  std::string name;       // column or function name (functions lower-cased)
  std::string qualifier;  // table qualifier, may be empty
  // Literal
  DType lit_type = DType::Null;
  int64_t i64 = 0;
  double f64 = 0.0;
  bool b = false;
  std::string str;
  // Binary / Unary: op is one of + - * / % = != < <= > >= AND OR ; unary: NOT, NEG
  std::string op;
  std::vector<ExprPtr> args;
  // Cast
  DType cast_to = DType::Null;
  // IsNull
  bool negated = false;  // IS NOT NULL
  // Func
  bool distinct = false;
  bool star_arg = false;  // count(*)

  ExprPtr clone() const;
};

struct SelectItem {
  ExprPtr expr;           // null when is_star
  std::string alias;      // empty when none
  bool is_star = false;   // `*` or `t.*`
  std::string star_qualifier;
};

struct TableRef {
  std::string name;
  std::string alias;  // empty when none
  const std::string& visible() const { return alias.empty() ? name : alias; }
};

struct JoinClause {
  enum Type { Inner = 0, Left = 1, Right = 2 } type = Inner;  // LEFT / RIGHT [OUTER]: the other side's columns turn NULL
  TableRef table;
  ExprPtr on;
  std::vector<std::string> using_cols;
};

struct Query {
  std::vector<SelectItem> select;
  TableRef from;
  std::vector<JoinClause> joins;
  ExprPtr where;
  std::vector<ExprPtr> group_by;
  std::vector<ExprPtr> order_by;  // accepted only where it cannot change the result (one-row global aggregates)
  int64_t limit = -1;
};

// Throws ArkError(ARK_ERR_PROCESS, "SQL query error: …") on a syntax error (reference: sql.rs:92-98)
// and ArkError(ARK_ERR_UNSUPPORTED, …) for valid SQL outside the subset (ORDER BY, subqueries, …).
Query parse_sql(const std::string& sql);
// One scalar expression (DataFusion's parse_sql_expr); the same error classes as parse_sql.
ExprPtr parse_sql_expr(const std::string& text);

}  // namespace ark
