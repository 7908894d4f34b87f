// sql_parser.cc — hand-written tokenizer + recursive-descent parser for the SQL subset of sql.h.
//
// Stands in for DataFusion's `sql_to_statement` at crates/arkflow-plugin/src/processor/sql.rs:91-98.
// Behaviour kept from the reference: a syntax error is reported at construction time with the
// prefix "SQL query error: " (sql.rs:98); only a single SELECT statement is accepted, DDL/DML is
// rejected (the reference verifies this per batch with SQLOptions, sql.rs:192-201).
#include <algorithm>
#include <cctype>
#include <cerrno>
#include <cstdlib>
#include <cstring>

#include "common.h"
#include "sql.h"

namespace ark {

const char* dtype_name(DType t) {
  switch (t) {
    case DType::Null: return "Null";
    case DType::Bool: return "Boolean";
    case DType::Int64: return "Int64";
    case DType::Float64: return "Float64";
    case DType::Utf8: return "Utf8";
    case DType::Binary: return "Binary";
    case DType::List: return "List";
    case DType::Struct: return "Struct";
    case DType::Int32: return "Int32";
    case DType::UInt32: return "UInt32";
    case DType::UInt64: return "UInt64";
    case DType::Float32: return "Float32";
  }
  return "?";
}
const char* dtype_arrow_format(DType t) {
  switch (t) {
    case DType::Null: return "n";
    case DType::Bool: return "b";
    case DType::Int64: return "l";
    case DType::Float64: return "g";
    case DType::Utf8: return "u";
    case DType::Binary: return "z";
    case DType::List: return "+l";
    case DType::Struct: return "+s";
    case DType::Int32: return "i";
    case DType::UInt32: return "I";
    case DType::UInt64: return "L";
    case DType::Float32: return "f";
  }
  return "n";
}

ExprPtr Expr::clone() const {
  auto e = std::make_unique<Expr>();
  e->kind = kind; e->name = name; e->qualifier = qualifier; e->lit_type = lit_type; e->i64 = i64;
  e->f64 = f64; e->b = b; e->str = str; e->op = op; e->cast_to = cast_to; e->negated = negated;
  e->distinct = distinct; e->star_arg = star_arg; e->derived = derived;
  for (auto& a : args) e->args.push_back(a->clone());
  return e;
}

namespace {

enum class Tok { End, Ident, QuotedIdent, Number, String, Op, LParen, RParen, Comma, Dot, Star, Semicolon };

struct Token {
  Tok t = Tok::End;
  std::string text;   // identifier (lower-cased unless quoted), operator, number text, string body
  std::string upper;  // upper-cased identifier text for keyword matching
  size_t pos = 0;
};

[[noreturn]] void syntax(const std::string& msg) { fail(ARK_ERR_PROCESS, "SQL query error: " + msg); }
[[noreturn]] void unsupported(const std::string& msg) {
  fail(ARK_ERR_UNSUPPORTED, "SQL outside the GPU subset: " + msg);
}

std::vector<Token> tokenize(const std::string& s) {
  std::vector<Token> out;
  size_t i = 0, n = s.size();
  while (i < n) {
    char c = s[i];
    if (isspace((unsigned char)c)) { ++i; continue; }
    if (c == '-' && i + 1 < n && s[i + 1] == '-') {  // line comment
      while (i < n && s[i] != '\n') ++i;
      continue;
    }
    Token tk; tk.pos = i;
    if (isalpha((unsigned char)c) || c == '_') {
      size_t j = i;
      while (j < n && (isalnum((unsigned char)s[j]) || s[j] == '_')) ++j;
      tk.t = Tok::Ident;
      tk.text = s.substr(i, j - i);
      tk.upper = tk.text;
      for (auto& ch : tk.text) ch = (char)tolower((unsigned char)ch);   // DataFusion normalises idents
      for (auto& ch : tk.upper) ch = (char)toupper((unsigned char)ch);
      i = j;
    } else if (c == '"' || c == '`') {
      char q = c; size_t j = i + 1; std::string body;
      while (true) {
        if (j >= n) syntax("Unterminated quoted identifier at position " + std::to_string(i));
        if (s[j] == q) { if (j + 1 < n && s[j + 1] == q) { body += q; j += 2; continue; } break; }
        body += s[j++];
      }
      tk.t = Tok::QuotedIdent; tk.text = body; i = j + 1;
    } else if (c == '\'') {
      size_t j = i + 1; std::string body;
      while (true) {
        if (j >= n) syntax("Unterminated string literal at position " + std::to_string(i));
        if (s[j] == '\'') { if (j + 1 < n && s[j + 1] == '\'') { body += '\''; j += 2; continue; } break; }
        body += s[j++];
      }
      tk.t = Tok::String; tk.text = body; i = j + 1;
    } else if (isdigit((unsigned char)c) || (c == '.' && i + 1 < n && isdigit((unsigned char)s[i + 1]))) {
      size_t j = i; bool seen_e = false;
      while (j < n) {
        char d = s[j];
        if (isdigit((unsigned char)d) || d == '.') { ++j; continue; }
        if ((d == 'e' || d == 'E') && !seen_e && j + 1 < n &&
            (isdigit((unsigned char)s[j + 1]) || ((s[j + 1] == '+' || s[j + 1] == '-') && j + 2 < n && isdigit((unsigned char)s[j + 2])))) {
          seen_e = true; j += 2; continue;
        }
        break;
      }
      tk.t = Tok::Number; tk.text = s.substr(i, j - i); i = j;
    } else {
      auto two = [&](const char* op) { return i + 1 < n && s[i] == op[0] && s[i + 1] == op[1]; };
      if (two("<=") || two(">=") || two("<>") || two("!=") || two("==") || two("||")) {
        tk.t = Tok::Op; tk.text = s.substr(i, 2); i += 2;
        if (tk.text == "<>") tk.text = "!=";
        if (tk.text == "==") tk.text = "=";
      } else {
        switch (c) {
          case '(': tk.t = Tok::LParen; break;
          case ')': tk.t = Tok::RParen; break;
          case ',': tk.t = Tok::Comma; break;
          case '.': tk.t = Tok::Dot; break;
          case '*': tk.t = Tok::Star; break;
          case ';': tk.t = Tok::Semicolon; break;
          case '+': case '-': case '/': case '%': case '=': case '<': case '>':
            tk.t = Tok::Op; break;
          default:
            syntax(std::string("Unexpected character '") + c + "' at position " + std::to_string(i));
        }
        tk.text = std::string(1, c); ++i;
      }
    }
    out.push_back(std::move(tk));
  }
  Token e; e.t = Tok::End; e.pos = n; out.push_back(e);
  return out;
}

bool has_aggregate_call(const Expr& e) {
  if (e.kind == Expr::Func && (e.name == "sum" || e.name == "count" || e.name == "avg" || e.name == "mean" || e.name == "min" || e.name == "max")) return true;
  for (auto& a : e.args) if (has_aggregate_call(*a)) return true;
  return false;
}

struct Parser {
  std::vector<Token> toks;
  size_t p = 0;

  const Token& cur() const { return toks[p]; }
  const Token& peek(size_t k = 1) const { return toks[std::min(p + k, toks.size() - 1)]; }
  bool is_kw(const char* kw) const { return cur().t == Tok::Ident && cur().upper == kw; }
  bool peek_kw(size_t k, const char* kw) const { return peek(k).t == Tok::Ident && peek(k).upper == kw; }
  bool accept_kw(const char* kw) { if (is_kw(kw)) { ++p; return true; } return false; }
  void expect_kw(const char* kw) {
    if (!accept_kw(kw)) syntax(std::string("Expected ") + kw + ", found: " + describe());
  }
  bool accept(Tok t) { if (cur().t == t) { ++p; return true; } return false; }
  void expect(Tok t, const char* what) {
    if (!accept(t)) syntax(std::string("Expected ") + what + ", found: " + describe());
  }
  std::string describe() const {
    if (cur().t == Tok::End) return "EOF";
    return cur().text;
  }

  static bool reserved(const std::string& u) {
    static const char* kws[] = {"SELECT", "FROM", "WHERE", "GROUP", "BY", "HAVING", "ORDER", "LIMIT",
                                "JOIN", "INNER", "LEFT", "RIGHT", "FULL", "CROSS", "ON", "USING",
                                "AND", "OR", "NOT", "AS", "IS", "NULL", "UNION", "EXCEPT",
                                "INTERSECT", "OFFSET", "CASE", "WHEN", "THEN", "ELSE", "END",
                                "BETWEEN", "IN", "LIKE", "DISTINCT", "TRUE", "FALSE", "NATURAL"};
    for (auto k : kws) if (u == k) return true;
    return false;
  }

  std::string ident(const char* what) {
    if (cur().t == Tok::QuotedIdent) return toks[p++].text;
    if (cur().t == Tok::Ident && !reserved(cur().upper)) return toks[p++].text;
    syntax(std::string("Expected ") + what + ", found: " + describe());
  }

  Query parse_statement() {
    if (cur().t == Tok::Ident) {
      const std::string& u = cur().upper;
      if (u == "INSERT" || u == "UPDATE" || u == "DELETE" || u == "CREATE" || u == "DROP" ||
          u == "ALTER" || u == "SET" || u == "COPY" || u == "TRUNCATE") {
        // The reference rejects these per batch through SQLOptions (sql.rs:192-201); we reject at build.
        fail(ARK_ERR_PROCESS, "SQL query error: DDL/DML/statements are not allowed: " + cur().text);
      }
      if (u == "WITH" || u == "EXPLAIN" || u == "VALUES" || u == "SHOW" || u == "DESCRIBE")
        unsupported(u);
    }
    Query q = parse_select();
    while (accept(Tok::Semicolon)) {}
    if (cur().t != Tok::End) syntax("Expected end of statement, found: " + describe());
    return q;
  }

  Query parse_select() {
    Query q;
    expect_kw("SELECT");
    if (is_kw("DISTINCT")) unsupported("SELECT DISTINCT");
    if (accept_kw("ALL")) {}
    do { q.select.push_back(parse_select_item()); } while (accept(Tok::Comma));
    if (!accept_kw("FROM")) {
      if (cur().t == Tok::End || cur().t == Tok::Semicolon) unsupported("SELECT without FROM");
      syntax("Expected FROM, found: " + describe());
    }
    q.from = parse_table_ref();
    while (true) {
      if (accept(Tok::Comma)) unsupported("comma (cross) join");
      bool inner = false;
      JoinClause::Type jtype = JoinClause::Inner;
      if (is_kw("INNER")) { ++p; inner = true; }
      else if (is_kw("LEFT") || is_kw("RIGHT")) {  // LEFT [OUTER] JOIN / RIGHT [OUTER] JOIN
        jtype = is_kw("LEFT") ? JoinClause::Left : JoinClause::Right;
        ++p;
        accept_kw("OUTER");
        inner = true;  // JOIN must follow
      }
      if (is_kw("FULL") || is_kw("CROSS") || is_kw("NATURAL"))
        unsupported(cur().upper + " JOIN");
      if (accept_kw("JOIN")) {
        JoinClause j;
        j.type = jtype;
        j.table = parse_table_ref();
        if (accept_kw("ON")) {
          j.on = parse_expr();
        } else if (accept_kw("USING")) {
          expect(Tok::LParen, "(");
          do { j.using_cols.push_back(ident("column name")); } while (accept(Tok::Comma));
          expect(Tok::RParen, ")");
        } else {
          syntax("Expected ON or USING after JOIN, found: " + describe());
        }
        q.joins.push_back(std::move(j));
      } else {
        if (inner) syntax("Expected JOIN, found: " + describe());
        break;
      }
    }
    if (accept_kw("WHERE")) q.where = parse_expr();
    if (accept_kw("GROUP")) {
      expect_kw("BY");
      do { q.group_by.push_back(parse_expr()); } while (accept(Tok::Comma));
    }
    if (accept_kw("HAVING")) q.having = parse_expr();
    if (accept_kw("ORDER")) {
      expect_kw("BY");
      do {
        q.order_by.push_back(parse_expr());
        if (!accept_kw("ASC")) accept_kw("DESC");
        if (accept_kw("NULLS")) { if (!accept_kw("FIRST")) expect_kw("LAST"); }
      } while (accept(Tok::Comma));
    }
    if (is_kw("UNION") || is_kw("EXCEPT") || is_kw("INTERSECT")) unsupported(cur().upper);
    if (accept_kw("LIMIT")) {
      if (cur().t != Tok::Number) syntax("Expected a number after LIMIT, found: " + describe());
      q.limit = strtoll(cur().text.c_str(), nullptr, 10);
      ++p;
    }
    if (is_kw("OFFSET")) unsupported("OFFSET");
    if (!q.order_by.empty()) {
      // ORDER BY survives only where it cannot change the result: an aggregate query without GROUP BY has one row
      bool agg = false;
      for (auto& it : q.select) if (!it.is_star && has_aggregate_call(*it.expr)) agg = true;
      if (!agg || !q.group_by.empty()) unsupported("ORDER BY");
    }
    return q;
  }

  TableRef parse_table_ref() {
    if (cur().t == Tok::LParen) unsupported("subquery in FROM");
    TableRef t;
    t.name = ident("table name");
    while (accept(Tok::Dot)) t.name = ident("table name");  // schema.table → keep last part
    if (accept_kw("AS")) t.alias = ident("table alias");
    else if (cur().t == Tok::QuotedIdent || (cur().t == Tok::Ident && !reserved(cur().upper)))
      t.alias = ident("table alias");
    return t;
  }

  SelectItem parse_select_item() {
    SelectItem it;
    if (accept(Tok::Star)) { it.is_star = true; return it; }
    if ((cur().t == Tok::Ident || cur().t == Tok::QuotedIdent) && peek(1).t == Tok::Dot && peek(2).t == Tok::Star) {
      it.is_star = true; it.star_qualifier = cur().text; p += 3; return it;
    }
    it.expr = parse_expr();
    if (accept_kw("AS")) it.alias = ident("alias");
    else if (cur().t == Tok::QuotedIdent || (cur().t == Tok::Ident && !reserved(cur().upper)))
      it.alias = ident("alias");
    return it;
  }

  static ExprPtr mk_binary(const std::string& op, ExprPtr l, ExprPtr r) {
    auto e = std::make_unique<Expr>();
    e->kind = Expr::Binary; e->op = op;
    e->args.push_back(std::move(l)); e->args.push_back(std::move(r));
    return e;
  }

  ExprPtr parse_expr() { return parse_or(); }
  ExprPtr parse_or() {
    auto l = parse_and();
    while (accept_kw("OR")) l = mk_binary("OR", std::move(l), parse_and());
    return l;
  }
  ExprPtr parse_and() {
    auto l = parse_not();
    while (accept_kw("AND")) l = mk_binary("AND", std::move(l), parse_not());
    return l;
  }
  ExprPtr parse_not() {
    if (accept_kw("NOT")) {
      auto e = std::make_unique<Expr>();
      e->kind = Expr::Unary; e->op = "NOT"; e->args.push_back(parse_not());
      return e;
    }
    return parse_cmp();
  }
  ExprPtr parse_cmp() {
    auto l = parse_add();
    while (true) {
      if (cur().t == Tok::Op && (cur().text == "=" || cur().text == "!=" || cur().text == "<" ||
                                 cur().text == "<=" || cur().text == ">" || cur().text == ">=")) {
        std::string op = toks[p++].text;
        l = mk_binary(op, std::move(l), parse_add());
      } else if (is_kw("IS")) {
        ++p;
        bool neg = accept_kw("NOT");
        if (accept_kw("NULL")) {
          auto e = std::make_unique<Expr>();
          e->kind = Expr::IsNull; e->negated = neg; e->args.push_back(std::move(l));
          l = std::move(e);
        } else {
          unsupported("IS [NOT] TRUE/FALSE/DISTINCT FROM");
        }
      } else if (is_kw("BETWEEN") || is_kw("IN") || is_kw("LIKE") || is_kw("ILIKE") ||
                 (is_kw("NOT") && (peek_kw(1, "BETWEEN") || peek_kw(1, "IN") || peek_kw(1, "LIKE")))) {
        unsupported(cur().upper);
      } else {
        break;
      }
    }
    return l;
  }
  ExprPtr parse_add() {
    auto l = parse_mul();
    while (cur().t == Tok::Op && (cur().text == "+" || cur().text == "-")) {
      std::string op = toks[p++].text;
      l = mk_binary(op, std::move(l), parse_mul());
    }
    if (cur().t == Tok::Op && cur().text == "||") unsupported("string concatenation ||");
    return l;
  }
  ExprPtr parse_mul() {
    auto l = parse_unary();
    while (true) {
      if (cur().t == Tok::Star) { ++p; l = mk_binary("*", std::move(l), parse_unary()); }
      else if (cur().t == Tok::Op && (cur().text == "/" || cur().text == "%")) {
        std::string op = toks[p++].text;
        l = mk_binary(op, std::move(l), parse_unary());
      } else break;
    }
    return l;
  }
  ExprPtr parse_unary() {
    if (cur().t == Tok::Op && cur().text == "-") {
      ++p;
      auto inner = parse_unary();
      if (inner->kind == Expr::Literal && inner->lit_type == DType::Int64) {
        inner->i64 = (int64_t)(0 - (uint64_t)inner->i64); return inner;
      }
      if (inner->kind == Expr::Literal && inner->lit_type == DType::Float64) { inner->f64 = -inner->f64; return inner; }
      auto e = std::make_unique<Expr>();
      e->kind = Expr::Unary; e->op = "NEG"; e->args.push_back(std::move(inner));
      return e;
    }
    if (cur().t == Tok::Op && cur().text == "+") { ++p; return parse_unary(); }
    return parse_primary();
  }

  DType parse_type_name() {
    if (cur().t != Tok::Ident) syntax("Expected a data type, found: " + describe());
    std::string u = toks[p++].upper;
    if (u == "DOUBLE") { accept_kw("PRECISION"); return DType::Float64; }
    if (u == "FLOAT8" || u == "REAL8") return DType::Float64;
    if (u == "BIGINT" || u == "INT8") return DType::Int64;
    if (u == "BOOLEAN" || u == "BOOL") return DType::Bool;
    if (u == "STRING" || u == "TEXT" || u == "VARCHAR" || u == "CHAR") {
      if (accept(Tok::LParen)) { while (cur().t != Tok::RParen && cur().t != Tok::End) ++p; expect(Tok::RParen, ")"); }
      return DType::Utf8;
    }
    if (u == "BYTEA" || u == "BINARY" || u == "VARBINARY") return DType::Binary;
    unsupported("CAST to " + u);
  }

  ExprPtr parse_primary() {
    const Token& t = cur();
    if (t.t == Tok::LParen) {
      ++p;
      if (is_kw("SELECT")) unsupported("scalar subquery");
      auto e = parse_expr();
      expect(Tok::RParen, ")");
      return e;
    }
    if (t.t == Tok::Number) {
      auto e = std::make_unique<Expr>();
      e->kind = Expr::Literal;
      bool is_float = t.text.find_first_of(".eE") != std::string::npos;
      if (!is_float) {
        errno = 0;
        char* endp = nullptr;
        long long v = strtoll(t.text.c_str(), &endp, 10);
        if (errno == ERANGE) is_float = true;  // DataFusion falls back to wider types; Float64 here
        else { e->lit_type = DType::Int64; e->i64 = v; }
      }
      if (is_float) { e->lit_type = DType::Float64; e->f64 = strtod(t.text.c_str(), nullptr); }
      ++p;
      return e;
    }
    if (t.t == Tok::String) {
      auto e = std::make_unique<Expr>();
      e->kind = Expr::Literal; e->lit_type = DType::Utf8; e->str = t.text; ++p;
      return e;
    }
    if (t.t == Tok::Ident) {
      if (t.upper == "NULL") { ++p; auto e = std::make_unique<Expr>(); e->kind = Expr::Literal; e->lit_type = DType::Null; return e; }
      if (t.upper == "TRUE" || t.upper == "FALSE") {
        auto e = std::make_unique<Expr>(); e->kind = Expr::Literal; e->lit_type = DType::Bool; e->b = (t.upper == "TRUE"); ++p; return e;
      }
      if (t.upper == "CASE") unsupported("CASE");
      if (t.upper == "CAST" || t.upper == "TRY_CAST") {
        if (t.upper == "TRY_CAST") unsupported("TRY_CAST");
        ++p;
        expect(Tok::LParen, "(");
        auto inner = parse_expr();
        expect_kw("AS");
        DType ty = parse_type_name();
        expect(Tok::RParen, ")");
        auto e = std::make_unique<Expr>();
        e->kind = Expr::Cast; e->cast_to = ty; e->args.push_back(std::move(inner));
        return e;
      }
      if (peek(1).t == Tok::LParen && !reserved(t.upper)) {  // function call
        auto e = std::make_unique<Expr>();
        e->kind = Expr::Func; e->name = t.text;
        p += 2;
        if (accept_kw("DISTINCT")) e->distinct = true;
        if (accept(Tok::Star)) { e->star_arg = true; }
        else if (cur().t != Tok::RParen) {
          do { e->args.push_back(parse_expr()); } while (accept(Tok::Comma));
        }
        expect(Tok::RParen, ")");
        if (is_kw("OVER")) unsupported("window functions");
        if (is_kw("FILTER")) unsupported("aggregate FILTER");
        return e;
      }
    }
    if (t.t == Tok::Ident || t.t == Tok::QuotedIdent) {
      auto e = std::make_unique<Expr>();
      e->kind = Expr::Column;
      e->name = ident("expression");
      if (cur().t == Tok::Dot && (peek(1).t == Tok::Ident || peek(1).t == Tok::QuotedIdent)) {
        ++p;
        e->qualifier = e->name;
        e->name = ident("column name");
      }
      return e;
    }
    syntax("Expected an expression, found: " + describe());
  }
};

}  // namespace

// SessionContext::parse_sql_expr (plugin/expr/mod.rs:111): one scalar expression, nothing after it.
ExprPtr parse_sql_expr(const std::string& text) {
  Parser ps;
  ps.toks = tokenize(text);
  if (ps.toks.size() == 1) syntax("Expected an expression, found: EOF");
  ExprPtr e = ps.parse_expr();
  if (ps.cur().t != Tok::End) syntax("Expected end of expression, found: " + ps.describe());
  return e;
}

Query parse_sql(const std::string& sql) {
  Parser ps;
  ps.toks = tokenize(sql);
  if (ps.toks.size() == 1) syntax("Expected a statement, found: EOF");
  return ps.parse_statement();
}

}  // namespace ark
