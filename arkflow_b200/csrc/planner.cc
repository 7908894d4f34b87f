// planner.cc — binds a parsed Query to an input schema and compiles its expressions to VmPrograms.
//
// Type coercion, result typing and result naming restate DataFusion 47 (third-party; reached from
// crates/arkflow-plugin/src/processor/sql.rs:197-203):
//   Int64 ∘ Float64 → Float64;  Int64 / Int64 → Int64;  comparisons → Boolean;
//   SUM(Int64) → Int64, SUM(Float64) → Float64, COUNT → Int64 (non-null), AVG → Float64,
//   MIN/MAX keep the argument type;  names: sum(flow.value), count(*), flow.value + Int64(1), alias.
#include <cmath>
#include <cstdio>

#include "common.h"
#include "plan.h"

namespace ark {

namespace {

[[noreturn]] void plan_error(const std::string& m) { fail(ARK_ERR_PROCESS, "Execution query error: " + m); }
[[noreturn]] void unsupported(const std::string& m) { fail(ARK_ERR_UNSUPPORTED, "SQL outside the GPU subset: " + m); }

bool is_numeric(DType t) { return t == DType::Int64 || t == DType::Float64; }
bool is_string(DType t) { return t == DType::Utf8 || t == DType::Binary; }
bool is_cmp_op(const std::string& op) { return op == "=" || op == "!=" || op == "<" || op == "<=" || op == ">" || op == ">="; }
bool is_arith_op(const std::string& op) { return op == "+" || op == "-" || op == "*" || op == "/" || op == "%"; }
int cmp_code(const std::string& op) {
  if (op == "=") return CMP_EQ;
  if (op == "!=") return CMP_NE;
  if (op == "<") return CMP_LT;
  if (op == "<=") return CMP_LE;
  if (op == ">") return CMP_GT;
  return CMP_GE;
}
int cmp_flip(int c) {
  switch (c) { case CMP_LT: return CMP_GT; case CMP_LE: return CMP_GE; case CMP_GT: return CMP_LT; case CMP_GE: return CMP_LE; default: return c; }
}

std::string fmt_f64(double v) {
  if (std::isnan(v)) return "NaN";
  if (std::isinf(v)) return v > 0 ? "inf" : "-inf";
  if (v == std::floor(v) && std::fabs(v) < 1e15) { char b[64]; snprintf(b, sizeof b, "%.0f", v); return b; }
  for (int prec = 1; prec <= 17; ++prec) {
    char b[64]; snprintf(b, sizeof b, "%.*g", prec, v);
    if (strtod(b, nullptr) == v) return b;
  }
  char b[64]; snprintf(b, sizeof b, "%.17g", v); return b;
}

struct Binder {
  std::string table;                 // visible table name (alias or name)
  const std::vector<Field>* fields;  // the input's fields, then the derived columns' (Plan::input_fields)
  size_t n_input = 0;                // fields the query can name
  std::vector<int>* used;            // slot → column index

  int resolve(const Expr& e) const {
    if (e.derived >= 0) return (int)n_input + e.derived;
    if (!e.qualifier.empty() && e.qualifier != table)
      plan_error("Schema error: No field named " + e.qualifier + "." + e.name + ".");
    for (size_t i = 0; i < n_input; ++i) if ((*fields)[i].name == e.name) return (int)i;
    std::string valid;
    for (size_t i = 0; i < n_input; ++i) { if (!valid.empty()) valid += ", "; valid += table + "." + (*fields)[i].name; }
    plan_error("Schema error: No field named " + e.name + ". Valid fields are " + valid + ".");
  }
  int slot_of(int col) const {
    for (size_t i = 0; i < used->size(); ++i) if ((*used)[i] == col) return (int)i;
    if ((int)used->size() >= MAX_COLS) unsupported("query references more than " + std::to_string(MAX_COLS) + " columns");
    const Field& f = (*fields)[col];
    if (f.type == DType::Null && f.format != "n") unsupported("column '" + f.name + "' has Arrow type '" + f.format + "'");
    used->push_back(col);
    return (int)used->size() - 1;
  }

  DType type_of(const Expr& e) const {
    switch (e.kind) {
      case Expr::Column: {
        const Field& f = (*fields)[resolve(e)];
        if (f.type == DType::Null && f.format != "n") unsupported("column '" + f.name + "' has Arrow type '" + f.format + "'");
        return f.type;
      }
      case Expr::Literal: return e.lit_type;
      case Expr::Binary: {
        DType l = type_of(*e.args[0]), r = type_of(*e.args[1]);
        if (e.op == "AND" || e.op == "OR") {
          if ((l != DType::Bool && l != DType::Null) || (r != DType::Bool && r != DType::Null))
            plan_error("Error during planning: Cannot infer common argument type for logical boolean operation " +
                       std::string(dtype_name(l)) + " " + e.op + " " + dtype_name(r));
          return DType::Bool;
        }
        if (is_cmp_op(e.op)) {
          bool ok = (is_numeric(l) || l == DType::Null) && (is_numeric(r) || r == DType::Null);
          ok = ok || (is_string(l) && is_string(r)) || (l == DType::Bool && r == DType::Bool);
          if (!ok) {
            if ((is_string(l) && is_numeric(r)) || (is_numeric(l) && is_string(r))) unsupported("string/number comparison coercion");
            plan_error("Error during planning: Cannot infer common argument type for comparison operation " +
                       std::string(dtype_name(l)) + " " + e.op + " " + dtype_name(r));
          }
          return DType::Bool;
        }
        if (is_arith_op(e.op)) {
          if (!(is_numeric(l) || l == DType::Null) || !(is_numeric(r) || r == DType::Null))
            plan_error("Error during planning: Cannot coerce arithmetic expression " + std::string(dtype_name(l)) + " " +
                       e.op + " " + dtype_name(r) + " to valid types");
          if (l == DType::Null && r == DType::Null) return DType::Int64;
          return (l == DType::Float64 || r == DType::Float64) ? DType::Float64 : DType::Int64;
        }
        unsupported("operator " + e.op);
      }
      case Expr::Unary: {
        DType t = type_of(*e.args[0]);
        if (e.op == "NOT") { if (t != DType::Bool && t != DType::Null) plan_error("Error during planning: NOT requires a boolean argument"); return DType::Bool; }
        if (!is_numeric(t)) plan_error("Error during planning: Negation only supports numeric types");
        return t;
      }
      case Expr::Cast: return e.cast_to;
      case Expr::IsNull: type_of(*e.args[0]); return DType::Bool;
      case Expr::Func: unsupported("scalar function " + e.name + "()");
      case Expr::Star: unsupported("* in expression");
    }
    return DType::Null;
  }

  bool nullable_of(const Expr& e) const {
    switch (e.kind) {
      case Expr::Column: return (*fields)[resolve(e)].nullable;
      case Expr::Literal: return e.lit_type == DType::Null;
      case Expr::IsNull: return false;
      default: { bool n = false; for (auto& a : e.args) n = n || nullable_of(*a); return n; }
    }
  }

  static void emit(VmProgram& p, uint8_t op, int dst, int a, int b, int32_t aux) {
    if (p.n_instr >= VM_MAX_INSTR) unsupported("expression too long");
    if (dst >= VM_MAX_REGS) unsupported("expression too deep");
    VmInstr& in = p.instr[p.n_instr++];
    in.op = op; in.dst = (uint8_t)dst; in.a = (uint8_t)a; in.b = (uint8_t)b; in.aux = aux;
  }
  static int add_const(VmProgram& p, uint64_t bits, int& n_consts) {
    if (n_consts >= VM_MAX_CONST) unsupported("too many constants in one expression");
    p.consts[n_consts] = bits;
    return n_consts++;
  }

  struct CompileState { int n_consts = 0; int n_str = 0; };

  void coerce(VmProgram& p, int reg, DType from, DType to) const {
    if (from == to || from == DType::Null) return;
    if (from == DType::Int64 && to == DType::Float64) emit(p, VM_I64_TO_F64, reg, reg, 0, 0);
    else if (from == DType::Float64 && to == DType::Int64) emit(p, VM_F64_TO_I64, reg, reg, 0, 0);
    else if (from == DType::Bool && to == DType::Int64) emit(p, VM_BOOL_TO_I64, reg, reg, 0, 0);
    else if (from == DType::Bool && to == DType::Float64) { emit(p, VM_BOOL_TO_I64, reg, reg, 0, 0); emit(p, VM_I64_TO_F64, reg, reg, 0, 0); }
    else if (from == DType::Int64 && to == DType::Bool) emit(p, VM_I64_TO_BOOL, reg, reg, 0, 0);
    else if (from == DType::Float64 && to == DType::Bool) emit(p, VM_F64_TO_BOOL, reg, reg, 0, 0);
    else unsupported(std::string("CAST from ") + dtype_name(from) + " to " + dtype_name(to));
  }

  // Emits code leaving the value of `e` in register `reg`; returns its type.
  DType compile(const Expr& e, VmProgram& p, int reg, CompileState& st) const {
    if (reg >= VM_MAX_REGS) unsupported("expression too deep");
    switch (e.kind) {
      case Expr::Column: {
        int col = resolve(e);
        DType t = (*fields)[col].type;
        int s = slot_of(col);
        if (t == DType::Int64) emit(p, VM_LOAD_I64, reg, s, 0, 0);
        else if (t == DType::Float64) emit(p, VM_LOAD_F64, reg, s, 0, 0);
        else if (t == DType::Bool) emit(p, VM_LOAD_BOOL, reg, s, 0, 0);
        else if (t == DType::Null) emit(p, VM_NULL, reg, 0, 0, 0);
        else unsupported("string column '" + e.name + "' used as a scalar value");
        return t;
      }
      case Expr::Literal: {
        if (e.lit_type == DType::Null) { emit(p, VM_NULL, reg, 0, 0, 0); return DType::Null; }
        uint64_t bits = 0;
        if (e.lit_type == DType::Int64) bits = (uint64_t)e.i64;
        else if (e.lit_type == DType::Float64) memcpy(&bits, &e.f64, 8);
        else if (e.lit_type == DType::Bool) bits = e.b ? 1 : 0;
        else unsupported("string literal used as a scalar value");
        emit(p, VM_CONST, reg, 0, 0, add_const(p, bits, st.n_consts));
        return e.lit_type;
      }
      case Expr::Binary: {
        DType lt = type_of(*e.args[0]), rt = type_of(*e.args[1]);
        type_of(e);  // raises the planning errors
        if (e.op == "AND" || e.op == "OR") {
          compile(*e.args[0], p, reg, st);
          compile(*e.args[1], p, reg + 1, st);
          emit(p, e.op == "AND" ? VM_AND : VM_OR, reg, reg, reg + 1, 0);
          return DType::Bool;
        }
        if (is_cmp_op(e.op) && is_string(lt) && is_string(rt)) {
          const Expr* l = e.args[0].get(); const Expr* r = e.args[1].get();
          int cmp = cmp_code(e.op);
          if (l->kind == Expr::Literal && r->kind == Expr::Column) { std::swap(l, r); cmp = cmp_flip(cmp); }
          if (l->kind == Expr::Column && r->kind == Expr::Literal) {
            if (st.n_str >= VM_MAX_STR_CONST || (int)r->str.size() > VM_STR_CONST_BYTES) unsupported("string literal too long / too many");
            int k = st.n_str++;
            p.str_len[k] = (int32_t)r->str.size();
            memcpy(p.str_bytes[k], r->str.data(), r->str.size());
            emit(p, VM_CMP_STR_CONST, reg, slot_of(resolve(*l)), k, cmp);
            return DType::Bool;
          }
          if (l->kind == Expr::Column && r->kind == Expr::Column) {
            emit(p, VM_CMP_STR_COL, reg, slot_of(resolve(*l)), slot_of(resolve(*r)), cmp);
            return DType::Bool;
          }
          unsupported("string comparison between computed expressions");
        }
        DType a = compile(*e.args[0], p, reg, st);
        DType b = compile(*e.args[1], p, reg + 1, st);
        if (is_cmp_op(e.op)) {
          if (a == DType::Bool && b == DType::Bool) { emit(p, VM_CMP_BOOL, reg, reg, reg + 1, cmp_code(e.op)); return DType::Bool; }
          DType common = (a == DType::Float64 || b == DType::Float64) ? DType::Float64 : DType::Int64;
          coerce(p, reg, a, common); coerce(p, reg + 1, b, common);
          emit(p, common == DType::Float64 ? VM_CMP_F64 : VM_CMP_I64, reg, reg, reg + 1, cmp_code(e.op));
          return DType::Bool;
        }
        DType common = (a == DType::Float64 || b == DType::Float64) ? DType::Float64 : DType::Int64;
        coerce(p, reg, a, common); coerce(p, reg + 1, b, common);
        uint8_t op;
        if (common == DType::Int64) op = e.op == "+" ? VM_ADD_I64 : e.op == "-" ? VM_SUB_I64 : e.op == "*" ? VM_MUL_I64 : e.op == "/" ? VM_DIV_I64 : VM_MOD_I64;
        else op = e.op == "+" ? VM_ADD_F64 : e.op == "-" ? VM_SUB_F64 : e.op == "*" ? VM_MUL_F64 : e.op == "/" ? VM_DIV_F64 : VM_MOD_F64;
        emit(p, op, reg, reg, reg + 1, 0);
        return common;
      }
      case Expr::Unary: {
        DType t = compile(*e.args[0], p, reg, st);
        type_of(e);
        if (e.op == "NOT") { emit(p, VM_NOT, reg, reg, 0, 0); return DType::Bool; }
        emit(p, t == DType::Float64 ? VM_NEG_F64 : VM_NEG_I64, reg, reg, 0, 0);
        return t;
      }
      case Expr::Cast: {
        DType from = type_of(*e.args[0]);
        if (is_string(e.cast_to) || is_string(from)) unsupported("CAST involving strings inside an expression");
        DType t = compile(*e.args[0], p, reg, st);
        coerce(p, reg, t, e.cast_to);
        return e.cast_to;
      }
      case Expr::IsNull: {
        const Expr& x = *e.args[0];
        if (x.kind == Expr::Column) {
          emit(p, e.negated ? VM_IS_NOT_NULL_COL : VM_IS_NULL_COL, reg, slot_of(resolve(x)), 0, 0);
          return DType::Bool;
        }
        compile(x, p, reg, st);
        emit(p, e.negated ? VM_IS_NOT_NULL : VM_IS_NULL, reg, reg, 0, 0);
        return DType::Bool;
      }
      case Expr::Func: unsupported("scalar function " + e.name + "()");
      case Expr::Star: unsupported("* in expression");
    }
    return DType::Null;
  }

  VmProgram compile_program(const Expr& e, DType* out_type) const {
    VmProgram p;
    memset(&p, 0, sizeof p);
    CompileState st;
    DType t = compile(e, p, 0, st);
    p.result_reg = 0;
    if (out_type) *out_type = t;
    return p;
  }

  ValueSource value_source(const Expr& e) const {
    ValueSource v;
    if (e.kind == Expr::Column) {
      int col = resolve(e);
      v.kind = ValueSource::PassThrough; v.slot = slot_of(col);
      v.type = (*fields)[col].type; v.nullable = (*fields)[col].nullable;
      return v;
    }
    if (e.kind == Expr::Cast && e.args[0]->kind == Expr::Column) {
      int col = resolve(*e.args[0]);
      DType from = (*fields)[col].type;
      if (from == e.cast_to || (from == DType::Utf8 && e.cast_to == DType::Binary)) {
        v.kind = ValueSource::PassThrough; v.slot = slot_of(col); v.type = e.cast_to; v.nullable = (*fields)[col].nullable;
        return v;
      }
      if (from == DType::Binary && e.cast_to == DType::Utf8) {
        v.kind = ValueSource::PassThrough; v.slot = slot_of(col); v.type = DType::Utf8; v.nullable = (*fields)[col].nullable;
        v.validate_utf8 = true;  // checked on the surviving rows by utf8_validate_kernel
        return v;
      }
    }
    DType t;
    v.kind = ValueSource::Computed;
    v.prog = compile_program(e, &t);
    if (t == DType::Null) unsupported("NULL-typed projection");
    v.type = t; v.nullable = nullable_of(e);
    return v;
  }
};

std::string display(const Expr& e, const std::string& table) {
  switch (e.kind) {
    case Expr::Column: return e.derived >= 0 ? e.name : (e.qualifier.empty() ? table : e.qualifier) + "." + e.name;
    case Expr::Literal:
      switch (e.lit_type) {
        case DType::Null: return "NULL";
        case DType::Int64: return "Int64(" + std::to_string(e.i64) + ")";
        case DType::Float64: return "Float64(" + fmt_f64(e.f64) + ")";
        case DType::Bool: return std::string("Boolean(") + (e.b ? "true" : "false") + ")";
        default: return "Utf8(\"" + e.str + "\")";
      }
    case Expr::Binary: return display(*e.args[0], table) + " " + e.op + " " + display(*e.args[1], table);
    case Expr::Unary: return e.op == "NOT" ? "NOT " + display(*e.args[0], table) : "(- " + display(*e.args[0], table) + ")";
    case Expr::Cast: return display(*e.args[0], table);
    case Expr::IsNull: return display(*e.args[0], table) + (e.negated ? " IS NOT NULL" : " IS NULL");
    case Expr::Func: {
      std::string s = e.name + "(";
      if (e.distinct) s += "DISTINCT ";
      if (e.star_arg) s += "*";
      for (size_t i = 0; i < e.args.size(); ++i) { if (i) s += ","; s += display(*e.args[i], table); }
      return s + ")";
    }
    case Expr::Star: return "*";
  }
  return "";
}

bool is_aggregate_name(const std::string& n) {
  return n == "sum" || n == "count" || n == "avg" || n == "mean" || n == "min" || n == "max";
}
bool contains_aggregate(const Expr& e) {
  if (e.kind == Expr::Func && is_aggregate_name(e.name)) return true;
  for (auto& a : e.args) if (contains_aggregate(*a)) return true;
  return false;
}

void detect_simple_predicate(const Expr& w, const Binder& b, Plan& plan) {
  if (w.kind != Expr::Binary || !is_cmp_op(w.op)) return;
  const Expr* l = w.args[0].get(); const Expr* r = w.args[1].get();
  int cmp = cmp_code(w.op);
  if (l->kind == Expr::Literal && r->kind == Expr::Column) { std::swap(l, r); cmp = cmp_flip(cmp); }
  if (l->kind != Expr::Column || r->kind != Expr::Literal) return;
  int col = b.resolve(*l);
  DType ct = (*b.fields)[col].type;
  SimplePredicate sp;
  if (ct == DType::Int64 && r->lit_type == DType::Int64) { sp.is_f64 = false; sp.constant = (uint64_t)r->i64; }
  else if (ct == DType::Float64 && (r->lit_type == DType::Int64 || r->lit_type == DType::Float64)) {
    double v = r->lit_type == DType::Int64 ? (double)r->i64 : r->f64;
    sp.is_f64 = true; memcpy(&sp.constant, &v, 8);
  } else return;
  sp.enabled = true; sp.cmp = cmp; sp.slot = b.slot_of(col);
  plan.simple = sp;
}

// One aggregate call: its function, argument and DataFusion name (sum(flow.value), count(*), avg for mean).
AggSpec bind_aggregate(const Expr& e, const Binder& b) {
  if (e.distinct) unsupported("aggregate DISTINCT");
  AggSpec a;
  std::string fn = e.name == "mean" ? "avg" : e.name;
  if (fn == "count") {
    if (e.star_arg || (e.args.size() == 1 && e.args[0]->kind == Expr::Literal && e.args[0]->lit_type != DType::Null)) {
      a.func = AggFunc::CountStar;
    } else {
      if (e.args.size() != 1) plan_error("Error during planning: count expects one argument");
      a.func = AggFunc::Count;
      a.arg = b.value_source(*e.args[0]);
    }
    a.out_type = DType::Int64;
  } else {
    if (e.star_arg || e.args.size() != 1) plan_error("Error during planning: " + fn + " expects one argument");
    if (contains_aggregate(*e.args[0])) plan_error("Error during planning: nested aggregates are not allowed");
    a.arg = b.value_source(*e.args[0]);
    if (!is_numeric(a.arg.type)) {
      if ((fn == "min" || fn == "max")) unsupported(fn + " over " + dtype_name(a.arg.type));
      plan_error("Error during planning: " + fn + " does not support " + dtype_name(a.arg.type));
    }
    if (fn == "sum") { a.func = AggFunc::Sum; a.out_type = a.arg.type; }
    else if (fn == "avg") { a.func = AggFunc::Avg; a.out_type = DType::Float64; }
    else if (fn == "min") { a.func = AggFunc::Min; a.out_type = a.arg.type; }
    else { a.func = AggFunc::Max; a.out_type = a.arg.type; }
  }
  ExprPtr named = e.clone();
  named->name = fn;
  a.name = display(*named, b.table);
  return a;
}

void bind_where(const Query& q, const Binder& b, Plan& plan) {
  if (!q.where) return;
  DType t = b.type_of(*q.where);
  if (t != DType::Bool && t != DType::Null)
    plan_error("Error during planning: Cannot create filter with non-boolean predicate '" + display(*q.where, b.table) + "' returning " + dtype_name(t));
  plan.has_pred = true;
  plan.pred = b.compile_program(*q.where, nullptr);
  detect_simple_predicate(*q.where, b, plan);
}

// ---- json_* calls → derived columns ----

bool json_fn_of(const std::string& n, JsonFn* fn) {
  static const std::pair<const char*, JsonFn> names[] = {
      {"json_get_str", JsonFn::GetStr}, {"json_get_int", JsonFn::GetInt}, {"json_get_float", JsonFn::GetFloat},
      {"json_get_bool", JsonFn::GetBool}, {"json_get_json", JsonFn::GetJson}, {"json_as_text", JsonFn::AsText},
      {"json_contains", JsonFn::Contains}, {"json_length", JsonFn::Length}};
  for (auto& p : names) if (n == p.first) { *fn = p.second; return true; }
  return false;
}

// json_length is UInt64 in datafusion-functions-json; it is Int64 here, the column type the plan reads (DESIGN.md §6).
DType json_result_type(JsonFn fn) {
  switch (fn) {
    case JsonFn::GetInt: case JsonFn::Length: return DType::Int64;
    case JsonFn::GetFloat: return DType::Float64;
    case JsonFn::GetBool: case JsonFn::Contains: return DType::Bool;
    default: return DType::Utf8;
  }
}

// Replaces every json_* call under `e` by a Column naming its derived column, one per distinct display name.
void rewrite_json(ExprPtr& e, const Binder& b, Plan& plan) {
  JsonFn fn;
  if (e->kind != Expr::Func || !json_fn_of(e->name, &fn)) {
    for (auto& a : e->args) rewrite_json(a, b, plan);
    return;
  }
  const std::string what = e->name + "()";
  if (e->distinct || e->star_arg || e->args.empty()) unsupported(what + " without a JSON document argument");
  if (e->args.size() > 1 + (size_t)JSON_MAX_PATH) unsupported(what + " with more than " + std::to_string(JSON_MAX_PATH) + " path elements");
  DerivedCol d;
  d.fn = fn;
  const Expr& doc = *e->args[0];
  const Expr* col = doc.kind == Expr::Column ? &doc
                  : doc.kind == Expr::Cast && doc.cast_to == DType::Utf8 && doc.args[0]->kind == Expr::Column ? doc.args[0].get()
                  : nullptr;
  const DType t = col && col->derived < 0 ? b.type_of(*col) : DType::Null;
  if (t != DType::Utf8 && !(t == DType::Binary && col != &doc))
    unsupported(what + ": the JSON document must be a Utf8 column or CAST(<Binary column> AS STRING)");
  d.doc_col = b.resolve(*col);
  d.doc_cast = t == DType::Binary;
  for (size_t i = 1; i < e->args.size(); ++i) {
    const Expr& a = *e->args[i];
    JsonPathElem pe;
    if (a.kind == Expr::Literal && a.lit_type == DType::Utf8) pe.key = a.str;
    else if (a.kind == Expr::Literal && a.lit_type == DType::Int64 && a.i64 >= 0) { pe.is_key = false; pe.index = a.i64; }
    else unsupported(what + ": a path element must be a string or non-negative integer literal");
    d.path.push_back(pe);
  }
  auto c = std::make_unique<Expr>();
  c->kind = Expr::Column;
  c->name = display(*e, b.table);
  for (size_t k = 0; k < plan.derived.size(); ++k)
    if (plan.input_fields[b.n_input + k].name == c->name) c->derived = (int)k;
  if (c->derived < 0) {
    c->derived = (int)plan.derived.size();
    const DType rt = json_result_type(fn);
    plan.derived.push_back(d);
    plan.input_fields.push_back(Field{c->name, rt, true, dtype_arrow_format(rt)});
  }
  e = std::move(c);
}

// A copy of `q` whose json_* calls are derived columns of `plan` (the parsed query serves every schema).
Query rewrite_json_calls(const Query& q, const Binder& b, Plan& plan) {
  auto take = [&](const ExprPtr& e) {
    ExprPtr c = e ? e->clone() : nullptr;
    if (c) rewrite_json(c, b, plan);
    return c;
  };
  Query r;
  r.from = q.from;
  r.limit = q.limit;
  for (auto& it : q.select) {
    SelectItem s;
    s.expr = take(it.expr); s.alias = it.alias; s.is_star = it.is_star; s.star_qualifier = it.star_qualifier;
    r.select.push_back(std::move(s));
  }
  r.where = take(q.where);
  for (auto& g : q.group_by) r.group_by.push_back(take(g));
  r.having = take(q.having);
  for (auto& o : q.order_by) r.order_by.push_back(take(o));
  return r;
}

Plan bind_single(const Query& q, Plan plan);

// ---- HAVING, computed items and LIMIT of an aggregate query: a FilterProject stage over the group frame ----
//
// DataFusion plans these as Aggregate → Filter → Projection → Limit.  The aggregate here emits a *frame*: every GROUP BY
// key, then every distinct aggregate call of SELECT and HAVING (plan.post / plan.aggs, hidden ones included).  SELECT
// and HAVING are rewritten so that each key and each aggregate call reads a frame column, and the rewritten query
// (WHERE = HAVING, the items, LIMIT) is bound by the single-table FilterProject binder into Plan::stage.  The frame's
// columns are all "derived" columns of the stage plan: a Column node that reads one carries its display name, so the
// stage's results are named as DataFusion names them (max(flow.value) - min(flow.value)).

// The aggregate SELECT lists that bind without a stage: keys, aggregates, CAST(<aggregate> AS STRING) and literals.
bool needs_stage(const Query& q) {
  if (q.having || q.limit >= 0) return true;
  for (auto& it : q.select) {
    if (it.is_star) continue;
    const Expr* e = it.expr.get();
    if (e->kind == Expr::Cast && e->cast_to == DType::Utf8 && e->args[0]->kind == Expr::Func && is_aggregate_name(e->args[0]->name)) continue;
    if ((e->kind == Expr::Func && is_aggregate_name(e->name)) || e->kind == Expr::Column || e->kind == Expr::Literal) continue;
    return true;
  }
  return false;
}

struct FrameRewriter {
  const Query& q;
  const Binder& b;
  const std::vector<std::string>& key_display;
  Plan& plan;
  std::vector<Field> fields;  // the frame's columns, in plan.post order

  static ExprPtr frame_column(const std::vector<Field>& fields, int index) {
    auto c = std::make_unique<Expr>();
    c->kind = Expr::Column;
    c->name = fields[index].name;
    c->derived = index;
    return c;
  }

  // Replaces every key and aggregate call under `e` by a frame column.  `clause` names the clause in the planning error
  // of a column that is neither; in HAVING, an unqualified column named as a SELECT alias stands for that item's
  // expression (datafusion-sql's resolve_aliases_to_exprs).
  void rewrite(ExprPtr& e, const char* clause, bool aliases) {
    if (e->kind == Expr::Func && is_aggregate_name(e->name)) {
      for (auto& a : e->args)
        if (contains_aggregate(*a)) plan_error("Error during planning: nested aggregates are not allowed");
      AggSpec a = bind_aggregate(*e, b);
      size_t k = 0;
      while (k < plan.aggs.size() && plan.aggs[k].name != a.name) ++k;
      if (k == plan.aggs.size()) {
        const bool is_count = a.func == AggFunc::Count || a.func == AggFunc::CountStar;
        PostItem pi;
        pi.kind = PostItem::Agg; pi.index = (int)k; pi.name = a.name;
        plan.post.push_back(pi);
        fields.push_back(Field{a.name, a.out_type, !is_count, dtype_arrow_format(a.out_type)});
        plan.aggs.push_back(std::move(a));
      }
      e = frame_column(fields, (int)(plan.keys.size() + k));
      return;
    }
    if (e->kind == Expr::Column) {
      if (aliases && e->qualifier.empty() && e->derived < 0)
        for (auto& it : q.select)
          if (!it.is_star && !it.alias.empty() && it.alias == e->name) {
            e = it.expr->clone();
            rewrite(e, clause, false);
            return;
          }
      const std::string d = display(*e, b.table);
      for (size_t k = 0; k < key_display.size(); ++k)
        if (key_display[k] == d) { e = frame_column(fields, (int)k); return; }
      b.resolve(*e);
      plan_error(std::string("Error during planning: Column in ") + clause +
                 " must be in GROUP BY or an aggregate function: While expanding wildcard, column \"" + e->name +
                 "\" must appear in the GROUP BY clause or must be part of an aggregate function");
    }
    for (auto& a : e->args) rewrite(a, clause, aliases);
  }
};

void bind_stage(const Query& q, const Binder& b, const std::vector<std::string>& key_display, Plan& plan) {
  FrameRewriter fr{q, b, key_display, plan, {}};
  for (size_t k = 0; k < plan.keys.size(); ++k) {
    PostItem pi;
    pi.kind = PostItem::Key; pi.index = (int)k; pi.name = key_display[k];
    plan.post.push_back(pi);
    fr.fields.push_back(Field{key_display[k], plan.keys[k].type, plan.keys[k].nullable, dtype_arrow_format(plan.keys[k].type)});
  }
  Query sq;
  sq.from = q.from;
  sq.limit = q.limit;
  for (auto& it : q.select) {
    if (it.is_star) plan_error("Error during planning: SELECT * is not valid with GROUP BY / aggregates");
    SelectItem s;
    s.expr = it.expr->clone();
    s.alias = it.alias;
    if (s.alias.empty() && s.expr->kind == Expr::Column) s.alias = s.expr->name;  // a bare key keeps its own name
    fr.rewrite(s.expr, "SELECT", false);
    sq.select.push_back(std::move(s));
  }
  if (q.having) {
    sq.where = q.having->clone();
    fr.rewrite(sq.where, "HAVING", true);
  }
  Plan stage;
  stage.input_fields = fr.fields;
  stage.n_input_fields = 0;  // every frame column is read through a derived Column node
  plan.stage = std::make_shared<Plan>(bind_single(sq, std::move(stage)));
}

}  // namespace

std::string expr_display_name(const Expr& e, const std::string& table) { return display(e, table); }

Plan bind_query(const Query& q, const std::string& table_name, const std::vector<Field>& fields, bool json_functions) {
  if (!q.joins.empty()) unsupported("JOIN in a single-table processor call");
  if (q.from.name != table_name)
    plan_error("Error during planning: table '" + q.from.name + "' not found");
  Plan plan;
  plan.input_fields = fields;
  plan.n_input_fields = fields.size();
  if (json_functions) {
    Binder b;
    b.table = q.from.visible(); b.fields = &plan.input_fields; b.n_input = fields.size(); b.used = &plan.used_cols;
    Query r = rewrite_json_calls(q, b, plan);
    if (!plan.derived.empty()) return bind_single(r, std::move(plan));
  }
  return bind_single(q, std::move(plan));
}

namespace {

Plan bind_single(const Query& q, Plan plan) {
  const std::vector<Field>& fields = plan.input_fields;
  plan.limit = q.limit;
  Binder b;
  b.table = q.from.visible(); b.fields = &fields; b.n_input = plan.n_input_fields; b.used = &plan.used_cols;

  bool has_agg = !q.group_by.empty();
  for (auto& it : q.select) if (!it.is_star && contains_aggregate(*it.expr)) has_agg = true;
  if (q.having && contains_aggregate(*q.having)) has_agg = true;
  if (q.where && contains_aggregate(*q.where))
    plan_error("Error during planning: Aggregate functions are not allowed in the WHERE clause");
  if (q.having && !has_agg)
    plan_error("Error during planning: HAVING clause references: " + display(*q.having, b.table) +
               " must appear in the GROUP BY clause or be used in an aggregate function");

  bind_where(q, b, plan);
  // ORDER BY is accepted only where it cannot change the result: a global aggregate yields exactly one row
  // (examples/protobuf_example.yaml orders such a query by one of its aliases)
  if (!q.order_by.empty() && (!has_agg || !q.group_by.empty())) unsupported("ORDER BY");

  if (!has_agg) {
    plan.kind = Plan::FilterProject;
    bool all_star = true;
    std::vector<std::pair<int, const SelectItem*>> concat_items;
    for (auto& it : q.select) {
      if (it.is_star) {
        if (!it.star_qualifier.empty() && it.star_qualifier != b.table)
          plan_error("Error during planning: Invalid qualifier " + it.star_qualifier);
        for (size_t c = 0; c < plan.n_input_fields; ++c) {
          const Field& f = fields[c];
          if (f.type == DType::Null && f.format != "n") unsupported("column '" + f.name + "' has Arrow type '" + f.format + "'");
          OutputCol oc; oc.name = f.name;
          oc.src.kind = ValueSource::PassThrough; oc.src.slot = b.slot_of((int)c); oc.src.type = f.type; oc.src.nullable = f.nullable;
          plan.outputs.push_back(oc);
        }
      } else if ((it.expr->kind == Expr::Func && it.expr->name == "concat") ||
                 (it.expr->kind == Expr::Cast && it.expr->cast_to == DType::Utf8 && it.expr->args[0]->kind == Expr::Column &&
                  (b.type_of(*it.expr->args[0]) == DType::Int64 || b.type_of(*it.expr->args[0]) == DType::Bool))) {
        all_star = false;
        concat_items.push_back({(int)plan.outputs.size(), &it});  // bound after the visible outputs
        OutputCol placeholder;
        placeholder.name = "\x01concat";
        plan.outputs.push_back(placeholder);
      } else {
        all_star = false;
        OutputCol oc;
        oc.src = b.value_source(*it.expr);
        oc.name = !it.alias.empty() ? it.alias : (it.expr->kind == Expr::Column ? it.expr->name : display(*it.expr, b.table));
        plan.outputs.push_back(oc);
      }
    }
    if (!concat_items.empty()) {
      // visible outputs keep their order; placeholders are dropped and the concat sources appended (hidden)
      std::vector<OutputCol> visible;
      std::vector<int> new_index(plan.outputs.size(), -1);
      for (size_t i = 0; i < plan.outputs.size(); ++i)
        if (plan.outputs[i].name != "\x01concat") { new_index[i] = (int)visible.size(); visible.push_back(plan.outputs[i]); }
      size_t next_concat = 0;
      for (size_t i = 0; i < plan.outputs.size(); ++i) {
        FinalItem fi;
        if (new_index[i] >= 0) { fi.index = new_index[i]; }
        else {
          const SelectItem& it = *concat_items[next_concat++].second;
          const Expr& e = *it.expr;
          if (e.distinct || e.star_arg || e.args.empty()) plan_error("Error during planning: concat expects at least one argument");
          ConcatItem ci;
          ci.is_cast = e.kind == Expr::Cast;  // CAST(<Int64 | Boolean column> AS STRING)
          ci.name = !it.alias.empty() ? it.alias : display(e, b.table);
          for (auto& a : e.args) {
            ConcatPart part;
            if (a->kind == Expr::Literal && a->lit_type == DType::Utf8) { part.is_literal = true; part.literal = a->str; }
            else if (a->kind == Expr::Literal && a->lit_type == DType::Null) { part.is_literal = true; }
            else if (a->kind == Expr::Column) {
              ValueSource v = b.value_source(*a);
              if (v.type != DType::Utf8 && v.type != DType::Int64 && v.type != DType::Bool)
                unsupported(std::string("concat() over a ") + dtype_name(v.type) + " argument");
              part.col_type = v.type;
              OutputCol hidden;
              hidden.name = "\x01src" + std::to_string(visible.size());
              hidden.src = v;
              part.out_index = (int)visible.size();
              visible.push_back(hidden);
            } else unsupported("concat() over a computed argument");
            ci.parts.push_back(part);
          }
          fi.is_concat = true; fi.index = (int)plan.concats.size();
          plan.concats.push_back(std::move(ci));
        }
        plan.final_items.push_back(fi);
      }
      plan.outputs = std::move(visible);
      all_star = false;
    }
    plan.identity = all_star && q.select.size() == 1 && !plan.has_pred && plan.limit < 0;
    return plan;
  }

  // ---- aggregate ----
  plan.kind = Plan::Aggregate;
  std::vector<std::string> key_display;
  for (auto& g : q.group_by) {
    if (g->kind != Expr::Column) unsupported("GROUP BY on a computed expression");
    ValueSource v = b.value_source(*g);
    if (v.type != DType::Int64 && v.type != DType::Utf8 && v.type != DType::Binary && v.type != DType::Bool)
      unsupported(std::string("GROUP BY key of type ") + dtype_name(v.type));
    plan.keys.push_back(v);
    plan.key_names.push_back(g->name);
    key_display.push_back(display(*g, b.table));
  }
  if (plan.keys.size() > 2) unsupported("more than two GROUP BY keys");
  if (needs_stage(q)) {
    bind_stage(q, b, key_display, plan);
    return plan;
  }
  for (auto& it : q.select) {
    if (it.is_star) plan_error("Error during planning: SELECT * is not valid with GROUP BY / aggregates");
    const Expr* ep = it.expr.get();
    PostItem pi;
    if (ep->kind == Expr::Cast && ep->cast_to == DType::Utf8 && ep->args[0]->kind == Expr::Func && is_aggregate_name(ep->args[0]->name)) {
      pi.cast_utf8 = true;  // CAST(<aggregate> AS STRING): the aggregate, rendered as decimal text afterwards
      ep = ep->args[0].get();
    }
    const Expr& e = *ep;
    if (e.kind == Expr::Func && is_aggregate_name(e.name)) {
      AggSpec a = bind_aggregate(e, b);
      if (pi.cast_utf8 && a.out_type != DType::Int64) unsupported(std::string("CAST(") + dtype_name(a.out_type) + " aggregate AS STRING)");
      pi.kind = PostItem::Agg; pi.index = (int)plan.aggs.size();
      pi.name = it.alias.empty() ? a.name : it.alias;
      plan.aggs.push_back(a);
    } else if (e.kind == Expr::Column) {
      std::string d = display(e, b.table);
      int k = -1;
      for (size_t i = 0; i < key_display.size(); ++i) if (key_display[i] == d) k = (int)i;
      if (k < 0) {
        b.resolve(e);
        plan_error("Error during planning: Column in SELECT must be in GROUP BY or an aggregate function: While expanding wildcard, column \"" +
                   e.name + "\" must appear in the GROUP BY clause or must be part of an aggregate function");
      }
      pi.kind = PostItem::Key; pi.index = k; pi.name = it.alias.empty() ? e.name : it.alias;
    } else if (e.kind == Expr::Literal) {
      pi.kind = PostItem::Literal; pi.lit_type = e.lit_type;
      if (e.lit_type == DType::Int64) pi.lit_bits = (uint64_t)e.i64;
      else if (e.lit_type == DType::Float64) memcpy(&pi.lit_bits, &e.f64, 8);
      else if (e.lit_type == DType::Bool) pi.lit_bits = e.b;
      else if (e.lit_type == DType::Utf8) pi.lit_str = e.str;
      else unsupported("NULL literal in an aggregate SELECT list");
      pi.name = it.alias.empty() ? display(e, b.table) : it.alias;
    } else {
      if (contains_aggregate(e)) unsupported("expression over aggregates: " + display(e, b.table));
      unsupported("computed non-aggregate expression in an aggregate SELECT list");
    }
    plan.post.push_back(pi);
  }
  return plan;
}

}  // namespace

Plan bind_join(const Query& q, const std::vector<std::string>& names, const std::vector<std::vector<Field>>& tables) {
  if (q.joins.size() != 1) {
    if (q.joins.empty() && names.size() >= 1) {
      // single-table query evaluated through the multi-table entry point (window.rs join with one input)
      for (size_t i = 0; i < names.size(); ++i)
        if (names[i] == q.from.name) return bind_query(q, names[i], tables[i]);
      plan_error("Error during planning: table '" + q.from.name + "' not found");
    }
    unsupported("more than one JOIN");
  }
  if (q.where) unsupported("WHERE on a join query");
  if (q.having) unsupported("HAVING on a join query");
  if (!q.group_by.empty()) unsupported("GROUP BY on a join query");
  if (q.limit >= 0) unsupported("LIMIT on a join query");
  auto find_table = [&](const std::string& n) -> int {
    for (size_t i = 0; i < names.size(); ++i) if (names[i] == n) return (int)i;
    plan_error("Error during planning: table '" + n + "' not found");
  };
  int lt = find_table(q.from.name), rt = find_table(q.joins[0].table.name);
  const std::string lvis = q.from.visible(), rvis = q.joins[0].table.visible();
  if (lvis == rvis) unsupported("self-join without distinct aliases");
  Plan plan;
  plan.kind = Plan::Join;
  plan.left_table = q.from.name; plan.right_table = q.joins[0].table.name;
  plan.input_fields = tables[lt]; plan.right_fields = tables[rt];
  auto find_col = [&](const std::vector<Field>& f, const std::string& n) -> int {
    for (size_t i = 0; i < f.size(); ++i) if (f[i].name == n) return (int)i;
    return -1;
  };
  const JoinClause& jc = q.joins[0];
  plan.join_type = (int)jc.type;
  if (!jc.using_cols.empty()) unsupported("JOIN … USING");
  const Expr* on = jc.on.get();
  if (!on || on->kind != Expr::Binary || on->op != "=" || on->args[0]->kind != Expr::Column || on->args[1]->kind != Expr::Column)
    unsupported("JOIN condition other than a single column equality");
  auto side_of = [&](const Expr& c, int* col) -> int {
    if (!c.qualifier.empty()) {
      if (c.qualifier == lvis) { *col = find_col(plan.input_fields, c.name); if (*col < 0) plan_error("Schema error: No field named " + c.qualifier + "." + c.name + "."); return 0; }
      if (c.qualifier == rvis) { *col = find_col(plan.right_fields, c.name); if (*col < 0) plan_error("Schema error: No field named " + c.qualifier + "." + c.name + "."); return 1; }
      plan_error("Schema error: No field named " + c.qualifier + "." + c.name + ".");
    }
    int l = find_col(plan.input_fields, c.name), r = find_col(plan.right_fields, c.name);
    if (l >= 0 && r >= 0) plan_error("Schema error: Ambiguous reference to unqualified field " + c.name);
    if (l >= 0) { *col = l; return 0; }
    if (r >= 0) { *col = r; return 1; }
    plan_error("Schema error: No field named " + c.name + ".");
  };
  int c0, c1;
  int s0 = side_of(*on->args[0], &c0), s1 = side_of(*on->args[1], &c1);
  if (s0 == s1) unsupported("JOIN condition does not relate the two tables");
  plan.left_key = s0 == 0 ? c0 : c1;
  plan.right_key = s0 == 0 ? c1 : c0;
  DType lk = plan.input_fields[plan.left_key].type, rk = plan.right_fields[plan.right_key].type;
  if (lk != rk || (lk != DType::Int64 && lk != DType::Utf8)) unsupported("join key types other than Int64=Int64 / Utf8=Utf8");
  auto add_all = [&](int side) {
    const auto& f = side == 0 ? plan.input_fields : plan.right_fields;
    for (size_t i = 0; i < f.size(); ++i) {
      if (f[i].type == DType::Null && f[i].format != "n") unsupported("column '" + f[i].name + "' has Arrow type '" + f[i].format + "'");
      plan.join_out.push_back({side, (int)i, f[i].name});
    }
  };
  for (auto& it : q.select) {
    if (it.is_star) {
      if (it.star_qualifier.empty()) { add_all(0); add_all(1); }
      else if (it.star_qualifier == lvis) add_all(0);
      else if (it.star_qualifier == rvis) add_all(1);
      else plan_error("Error during planning: Invalid qualifier " + it.star_qualifier);
    } else if (it.expr->kind == Expr::Column) {
      int col; int side = side_of(*it.expr, &col);
      plan.join_out.push_back({side, col, it.alias.empty() ? it.expr->name : it.alias});
    } else unsupported("computed expression in a join SELECT list");
  }
  return plan;
}

}  // namespace ark
