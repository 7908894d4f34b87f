// proto_schema.cc — a small `.proto` parser and type resolver (see proto_schema.h).
//
// Accepts proto2 and proto3 files: syntax / package / import (plain, public, weak) / option statements, nested
// message and enum definitions, fields with optional / required / repeated labels and [default = …] / [packed = …]
// options, oneof, map<K, V>, proto2 groups, reserved, extensions and extend (skipped: extensions are not fields of the
// message), service definitions (skipped), `//` and `/* */` comments.  Type names are resolved by protobuf's scoping
// rules: the first component of a relative name is looked up from the innermost scope outward, the rest inside it.
#include "proto_schema.h"

#include <dirent.h>
#include <sys/stat.h>

#include <algorithm>
#include <cerrno>
#include <climits>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <map>
#include <set>
#include <sstream>

#include "common.h"

namespace ark {

namespace {

[[noreturn]] void parse_fail(const std::string& m) { fail(ARK_ERR_CONFIG, "Failed to parse the proto file: " + m); }

struct Tok {
  enum T { Ident, Int, Float, Str, Sym, End } t = End;
  std::string s;  // identifier / number text / decoded string bytes / the symbol
  int line = 0;
};

std::vector<Tok> tokenize(const std::string& src, const std::string& file) {
  std::vector<Tok> out;
  size_t i = 0;
  int line = 1;
  auto err = [&](const std::string& m) { parse_fail(file + ":" + std::to_string(line) + ": " + m); };
  while (i < src.size()) {
    const char c = src[i];
    if (c == '\n') { ++line; ++i; continue; }
    if (isspace((unsigned char)c)) { ++i; continue; }
    if (c == '/' && i + 1 < src.size() && src[i + 1] == '/') { while (i < src.size() && src[i] != '\n') ++i; continue; }
    if (c == '/' && i + 1 < src.size() && src[i + 1] == '*') {
      const size_t e = src.find("*/", i + 2);
      if (e == std::string::npos) err("unterminated comment");
      line += (int)std::count(src.begin() + i, src.begin() + e, '\n');
      i = e + 2;
      continue;
    }
    Tok t;
    t.line = line;
    if (isalpha((unsigned char)c) || c == '_') {
      size_t j = i;
      while (j < src.size() && (isalnum((unsigned char)src[j]) || src[j] == '_')) ++j;
      t.t = Tok::Ident; t.s = src.substr(i, j - i); i = j;
    } else if (isdigit((unsigned char)c) || (c == '.' && i + 1 < src.size() && isdigit((unsigned char)src[i + 1]))) {
      size_t j = i;
      bool flt = false;
      if (c == '0' && j + 1 < src.size() && (src[j + 1] == 'x' || src[j + 1] == 'X')) {
        j += 2;
        while (j < src.size() && isxdigit((unsigned char)src[j])) ++j;
      } else {
        while (j < src.size() && (isdigit((unsigned char)src[j]) || src[j] == '.')) { flt = flt || src[j] == '.'; ++j; }
        if (j < src.size() && (src[j] == 'e' || src[j] == 'E')) {
          flt = true; ++j;
          if (j < src.size() && (src[j] == '+' || src[j] == '-')) ++j;
          while (j < src.size() && isdigit((unsigned char)src[j])) ++j;
        }
      }
      if (j < src.size() && (isalpha((unsigned char)src[j]) || src[j] == '_')) err("invalid number");
      t.t = flt ? Tok::Float : Tok::Int; t.s = src.substr(i, j - i); i = j;
    } else if (c == '"' || c == '\'') {
      ++i;
      std::string v;
      while (true) {
        if (i >= src.size() || src[i] == '\n') err("unterminated string");
        const char ch = src[i++];
        if (ch == c) break;
        if (ch != '\\') { v += ch; continue; }
        if (i >= src.size()) err("unterminated string");
        const char e = src[i++];
        auto hexv = [](char h) { return isdigit((unsigned char)h) ? h - '0' : (tolower((unsigned char)h) - 'a' + 10); };
        switch (e) {
          case 'n': v += '\n'; break; case 't': v += '\t'; break; case 'r': v += '\r'; break;
          case 'a': v += '\a'; break; case 'b': v += '\b'; break; case 'f': v += '\f'; break; case 'v': v += '\v'; break;
          case 'x': case 'X': {
            int n = 0, val = 0;
            while (n < 2 && i < src.size() && isxdigit((unsigned char)src[i])) { val = val * 16 + hexv(src[i++]); ++n; }
            if (!n) err("bad \\x escape");
            v += (char)val;
            break;
          }
          case 'u': case 'U': {
            const int digits = e == 'u' ? 4 : 8;
            unsigned cp = 0;
            for (int n = 0; n < digits; ++n) {
              if (i >= src.size() || !isxdigit((unsigned char)src[i])) err("bad \\u escape");
              cp = cp * 16 + hexv(src[i++]);
            }
            if (cp < 0x80) v += (char)cp;
            else if (cp < 0x800) { v += (char)(0xC0 | (cp >> 6)); v += (char)(0x80 | (cp & 0x3F)); }
            else if (cp < 0x10000) { v += (char)(0xE0 | (cp >> 12)); v += (char)(0x80 | ((cp >> 6) & 0x3F)); v += (char)(0x80 | (cp & 0x3F)); }
            else { v += (char)(0xF0 | (cp >> 18)); v += (char)(0x80 | ((cp >> 12) & 0x3F)); v += (char)(0x80 | ((cp >> 6) & 0x3F)); v += (char)(0x80 | (cp & 0x3F)); }
            break;
          }
          default:
            if (e >= '0' && e <= '7') {
              int val = e - '0', n = 1;
              while (n < 3 && i < src.size() && src[i] >= '0' && src[i] <= '7') { val = val * 8 + (src[i++] - '0'); ++n; }
              v += (char)val;
            } else v += e;  // \\ \' \" \?
        }
      }
      // adjacent literals concatenate
      if (!out.empty() && out.back().t == Tok::Str) { out.back().s += v; continue; }
      t.t = Tok::Str; t.s = v;
    } else {
      t.t = Tok::Sym; t.s = std::string(1, c); ++i;
    }
    out.push_back(t);
  }
  Tok end;
  end.line = line;
  out.push_back(end);
  return out;
}

enum Label { L_NONE, L_OPTIONAL, L_REQUIRED, L_REPEATED };

struct RawField {
  std::string name, type;  // type: a scalar keyword or a (possibly dotted / leading-dot) type name
  int32_t number = 0;
  Label label = L_NONE;
  bool is_map = false, is_group = false;
  int oneof = -1;
  bool has_default = false;
  Tok dflt;
  bool dflt_neg = false;
};

struct RawMessage {
  std::string full_name, file;
  bool proto3 = false;
  int n_oneofs = 0;
  std::vector<RawField> fields;
};

struct RawEnum {
  std::string full_name;
  std::vector<std::pair<std::string, int32_t>> values;
};

bool is_dir(const std::string& p) { struct stat st; return stat(p.c_str(), &st) == 0 && S_ISDIR(st.st_mode); }
bool is_file(const std::string& p) { struct stat st; return stat(p.c_str(), &st) == 0 && S_ISREG(st.st_mode); }
std::string real_path(const std::string& p) {
  char buf[PATH_MAX];
  return realpath(p.c_str(), buf) ? std::string(buf) : std::string();
}

class Pool {
 public:
  explicit Pool(std::vector<std::string> includes) : includes_(std::move(includes)) {}

  // an input file: it must lie under one of the include directories (its name there is its import path)
  void parse_input(const std::string& path) {
    const std::string rp = real_path(path);
    for (auto& inc : includes_) {
      const std::string ri = real_path(inc);
      if (!ri.empty() && rp.size() > ri.size() && rp.compare(0, ri.size(), ri) == 0 && rp[ri.size()] == '/') { parse_file(rp); return; }
    }
    parse_fail("file " + path + " must reside in an include path");
  }

  void parse_import(const std::string& name, const std::string& from) {
    for (auto& inc : includes_) {
      const std::string p = inc + "/" + name;
      if (is_file(p)) { parse_file(real_path(p)); return; }
    }
    parse_fail(from + ": import \"" + name + "\" was not found in the include paths");
  }

  PbMessage resolve(const std::string& message_type);

 private:
  std::vector<std::string> includes_;
  std::set<std::string> files_;
  std::map<std::string, RawMessage> messages_;
  std::map<std::string, RawEnum> enums_;
  std::set<std::string> packages_;  // every prefix of every package name

  // per-file parse state
  std::vector<Tok> toks_;
  size_t pos_ = 0;
  std::string file_;
  bool proto3_ = false;

  const Tok& peek(size_t k = 0) const { return toks_[std::min(pos_ + k, toks_.size() - 1)]; }
  [[noreturn]] void err(const std::string& m) const { parse_fail(file_ + ":" + std::to_string(peek().line) + ": " + m); }
  bool is_sym(const char* s, size_t k = 0) const { return peek(k).t == Tok::Sym && peek(k).s == s; }
  bool is_word(const char* s, size_t k = 0) const { return peek(k).t == Tok::Ident && peek(k).s == s; }
  bool accept(const char* s) { if (is_sym(s)) { ++pos_; return true; } return false; }
  void expect(const char* s) { if (!accept(s)) err(std::string("expected '") + s + "', found '" + peek().s + "'"); }
  std::string ident() {
    if (peek().t != Tok::Ident) err("expected an identifier, found '" + peek().s + "'");
    return toks_[pos_++].s;
  }
  std::string full_ident() {
    std::string s;
    if (accept(".")) s = ".";
    s += ident();
    while (is_sym(".")) { ++pos_; s += "." + ident(); }
    return s;
  }
  int64_t int_lit(bool neg) {
    if (peek().t != Tok::Int) err("expected an integer, found '" + peek().s + "'");
    const std::string t = toks_[pos_++].s;
    errno = 0;
    const unsigned long long v = strtoull(t.c_str(), nullptr, 0);  // 0x…, 0…, decimal
    if (errno == ERANGE) err("integer out of range: " + t);
    return neg ? -(int64_t)v : (int64_t)v;
  }
  void skip_to_semicolon() {
    while (!is_sym(";")) {
      if (peek().t == Tok::End) err("unexpected end of file");
      if (is_sym("{")) skip_block(); else ++pos_;
    }
    ++pos_;
  }
  void skip_block() {
    expect("{");
    for (int depth = 1; depth > 0; ++pos_) {
      if (peek().t == Tok::End) err("unexpected end of file");
      if (is_sym("{")) ++depth; else if (is_sym("}")) --depth;
    }
  }
  // one constant of an option: returns it (with its sign) for [default = …]
  Tok constant(bool* neg) {
    *neg = false;
    if (is_sym("{")) { skip_block(); return Tok(); }
    if (accept("-")) *neg = true; else accept("+");
    if (peek().t == Tok::End || peek().t == Tok::Sym) err("expected a constant, found '" + peek().s + "'");
    return toks_[pos_++];
  }
  void field_options(RawField& f) {
    if (!accept("[")) return;
    while (true) {
      std::string name;
      if (accept("(")) { name = "(" + full_ident() + ")"; expect(")"); } else name = ident();
      while (accept(".")) name += "." + ident();
      expect("=");
      bool neg;
      Tok v = constant(&neg);
      if (name == "default") { f.has_default = true; f.dflt = v; f.dflt_neg = neg; }
      if (accept(",")) continue;
      expect("]");
      break;
    }
  }

  void parse_file(const std::string& path) {
    if (!files_.insert(path).second) return;
    std::ifstream in(path, std::ios::binary);
    if (!in) parse_fail("cannot read " + path);
    std::stringstream ss;
    ss << in.rdbuf();
    // the parse state of the importing file is kept across the nested parse
    std::vector<Tok> toks = tokenize(ss.str(), path);
    std::swap(toks, toks_);
    const size_t pos = pos_;
    const std::string file = file_;
    const bool p3 = proto3_;
    pos_ = 0; file_ = path; proto3_ = false;
    std::string package;
    bool first = true;
    while (peek().t != Tok::End) {
      if (accept(";")) continue;
      const std::string kw = ident();
      if (kw == "syntax") {
        if (!first) err("syntax must be the first statement");
        expect("=");
        if (peek().t != Tok::Str) err("expected a string");
        const std::string s = toks_[pos_++].s;
        if (s == "proto3") proto3_ = true;
        else if (s != "proto2") err("unknown syntax \"" + s + "\"");
        expect(";");
      } else if (kw == "edition") {
        err("editions are not supported");
      } else if (kw == "package") {
        package = full_ident();
        if (package[0] == '.') err("package names cannot start with '.'");
        for (size_t d = package.find('.'); d != std::string::npos; d = package.find('.', d + 1)) packages_.insert(package.substr(0, d));
        packages_.insert(package);
        expect(";");
      } else if (kw == "import") {
        if (is_word("public") || is_word("weak")) ++pos_;
        if (peek().t != Tok::Str) err("expected the imported file name");
        const std::string name = toks_[pos_++].s;
        expect(";");
        parse_import(name, path);
      } else if (kw == "option") {
        skip_to_semicolon();
      } else if (kw == "message") {
        parse_message(package);
      } else if (kw == "enum") {
        parse_enum(package);
      } else if (kw == "service") {
        ident();
        skip_block();
      } else if (kw == "extend") {
        full_ident();
        skip_block();
      } else {
        err("unexpected '" + kw + "'");
      }
      first = false;
    }
    std::swap(toks, toks_);
    pos_ = pos; file_ = file; proto3_ = p3;
  }

  std::string define(const std::string& scope, const std::string& name) {
    const std::string full = scope.empty() ? name : scope + "." + name;
    if (messages_.count(full) || enums_.count(full)) err("\"" + full + "\" is already defined");
    return full;
  }

  void parse_message(const std::string& scope) {
    RawMessage m;
    m.full_name = define(scope, ident());
    messages_[m.full_name];  // claim the name before nested definitions
    m.file = file_; m.proto3 = proto3_;
    expect("{");
    parse_message_body(m);
    messages_[m.full_name] = std::move(m);
  }

  void parse_message_body(RawMessage& m) {
    while (!accept("}")) {
      if (peek().t == Tok::End) err("unexpected end of file");
      if (accept(";")) continue;
      if (is_word("message") && peek(1).t == Tok::Ident) { ++pos_; parse_message(m.full_name); continue; }
      if (is_word("enum") && peek(1).t == Tok::Ident) { ++pos_; parse_enum(m.full_name); continue; }
      if (is_word("extend")) { ++pos_; full_ident(); skip_block(); continue; }
      if (is_word("option") || is_word("reserved") || is_word("extensions")) { ++pos_; skip_to_semicolon(); continue; }
      if (is_word("oneof") && peek(1).t == Tok::Ident && is_sym("{", 2)) {
        pos_ += 2;
        expect("{");
        const int idx = m.n_oneofs++;
        while (!accept("}")) {
          if (peek().t == Tok::End) err("unexpected end of file");
          if (accept(";")) continue;
          if (is_word("option")) { ++pos_; skip_to_semicolon(); continue; }
          parse_field(m, idx);
        }
        continue;
      }
      parse_field(m, -1);
    }
  }

  void parse_field(RawMessage& m, int oneof) {
    RawField f;
    f.oneof = oneof;
    if (oneof < 0 && (peek(1).t == Tok::Ident || is_sym(".", 1))) {  // a label is followed by the type name
      if (is_word("optional")) { f.label = L_OPTIONAL; ++pos_; }
      else if (is_word("required")) { f.label = L_REQUIRED; ++pos_; }
      else if (is_word("repeated")) { f.label = L_REPEATED; ++pos_; }
    }
    if (is_word("map") && is_sym("<", 1)) {
      pos_ += 2;
      const std::string k = full_ident();
      expect(",");
      const std::string v = full_ident();
      expect(">");
      (void)k; (void)v;
      if (f.label != L_NONE || oneof >= 0) err("map fields cannot have labels or be in a oneof");
      f.is_map = true; f.label = L_REPEATED; f.type = "map";
    } else if (is_word("group") && peek(1).t == Tok::Ident && is_sym("=", 2)) {
      ++pos_;
      f.is_group = true;
    } else {
      f.type = full_ident();
    }
    if (!f.is_map && !f.is_group && m.proto3 == false && f.label == L_NONE && oneof < 0) err("expected \"required\", \"optional\", or \"repeated\"");
    if (m.proto3 && f.label == L_REQUIRED) err("required fields are not allowed in proto3");
    f.name = ident();
    expect("=");
    const int64_t num = int_lit(false);
    if (num < 1 || num > 536870911) err("field number out of range: " + std::to_string(num));
    if (num >= 19000 && num <= 19999) err("field numbers 19000 through 19999 are reserved for the protocol buffer library implementation");
    f.number = (int32_t)num;
    field_options(f);
    if (f.is_group) {
      if (m.proto3) err("groups are not supported in proto3");
      RawMessage g;
      g.full_name = define(m.full_name, f.name);
      messages_[g.full_name];
      g.file = file_; g.proto3 = false;
      expect("{");
      parse_message_body(g);
      f.type = "." + g.full_name;
      messages_[g.full_name] = std::move(g);
      std::string lower = f.name;
      for (auto& ch : lower) ch = (char)tolower((unsigned char)ch);
      f.name = lower;
    } else {
      expect(";");
    }
    for (auto& o : m.fields) {
      if (o.name == f.name) err("\"" + f.name + "\" is already defined in \"" + m.full_name + "\"");
      if (o.number == f.number) err("field number " + std::to_string(f.number) + " has already been used in \"" + m.full_name + "\"");
    }
    m.fields.push_back(std::move(f));
  }

  void parse_enum(const std::string& scope) {
    RawEnum e;
    e.full_name = define(scope, ident());
    expect("{");
    while (!accept("}")) {
      if (peek().t == Tok::End) err("unexpected end of file");
      if (accept(";")) continue;
      if ((is_word("option") || is_word("reserved")) && !is_sym("=", 1)) { ++pos_; skip_to_semicolon(); continue; }
      const std::string name = ident();
      expect("=");
      const bool neg = accept("-");
      const int64_t v = int_lit(neg);
      if (v < INT32_MIN || v > INT32_MAX) err("enum value out of range");
      RawField dummy;
      field_options(dummy);
      expect(";");
      e.values.emplace_back(name, (int32_t)v);
    }
    if (e.values.empty()) err("enum \"" + e.full_name + "\" must contain at least one value");
    enums_[e.full_name] = std::move(e);
  }

  bool is_symbol(const std::string& n) const { return messages_.count(n) || enums_.count(n) || packages_.count(n); }

  // protobuf scoping: the first component from the innermost scope outward, then the whole name inside that scope
  std::string resolve_type(const std::string& name, const std::string& scope, const std::string& where) const {
    if (name[0] == '.') {
      const std::string n = name.substr(1);
      if (messages_.count(n) || enums_.count(n)) return n;
      parse_fail(where + ": \"" + name + "\" is not defined");
    }
    const std::string first = name.substr(0, name.find('.'));
    std::string s = scope;
    while (true) {
      const std::string cand_first = s.empty() ? first : s + "." + first;
      if (is_symbol(cand_first)) {
        const std::string cand = s.empty() ? name : s + "." + name;
        if (messages_.count(cand) || enums_.count(cand)) return cand;
        if (first == name || messages_.count(cand_first) || enums_.count(cand_first))
          parse_fail(where + ": \"" + name + "\" is resolved to \"" + cand + "\", which is not defined");
      }
      if (s.empty()) break;
      const size_t d = s.rfind('.');
      s = d == std::string::npos ? std::string() : s.substr(0, d);
    }
    parse_fail(where + ": \"" + name + "\" is not defined");
  }
};

PbKind scalar_kind(const std::string& t, bool* ok) {
  static const std::map<std::string, PbKind> k = {
      {"double", PbKind::Double}, {"float", PbKind::Float}, {"int64", PbKind::Int64}, {"uint64", PbKind::UInt64},
      {"int32", PbKind::Int32}, {"fixed64", PbKind::Fixed64}, {"fixed32", PbKind::Fixed32}, {"bool", PbKind::Bool},
      {"string", PbKind::String}, {"bytes", PbKind::Bytes}, {"uint32", PbKind::UInt32}, {"sfixed32", PbKind::SFixed32},
      {"sfixed64", PbKind::SFixed64}, {"sint32", PbKind::SInt32}, {"sint64", PbKind::SInt64}};
  auto it = k.find(t);
  *ok = it != k.end();
  return *ok ? it->second : PbKind::Int32;
}

uint64_t double_bits(double d) { uint64_t b; memcpy(&b, &d, 8); return b; }
uint64_t float_bits(float f) { uint32_t b; memcpy(&b, &f, 4); return b; }

PbMessage Pool::resolve(const std::string& message_type) {
  // every field of every message must resolve (protobuf-parse's typecheck), not only those of the requested one
  std::map<std::string, std::vector<PbField>> resolved;
  for (auto& kv : messages_) {
    const RawMessage& m = kv.second;
    std::vector<PbField> out;
    for (const RawField& f : m.fields) {
      const std::string where = m.file + ": " + m.full_name + "." + f.name;
      PbField p;
      p.name = f.name; p.number = f.number; p.oneof = f.oneof;
      p.repeated = f.label == L_REPEATED; p.is_map = f.is_map;
      p.presence = !p.repeated && (f.oneof >= 0 || f.label == L_OPTIONAL || f.label == L_REQUIRED || (!m.proto3 && !f.is_map));
      bool scalar = false;
      if (f.is_map) p.kind = PbKind::Message;
      else if (f.is_group) { p.kind = PbKind::Group; p.type_name = f.type.substr(1); }
      else {
        p.kind = scalar_kind(f.type, &scalar);
        if (!scalar) {
          p.type_name = resolve_type(f.type, m.full_name, where);
          p.kind = enums_.count(p.type_name) ? PbKind::Enum : PbKind::Message;
        }
      }
      if (f.has_default) {
        if (m.proto3) parse_fail(where + ": explicit default values are not allowed in proto3");
        if (p.repeated || p.kind == PbKind::Message || p.kind == PbKind::Group) parse_fail(where + ": this field cannot have a default value");
      }
      if (p.kind == PbKind::Enum) {
        const RawEnum& e = enums_.at(p.type_name);
        p.default_bits = (uint64_t)(int64_t)e.values[0].second;
        if (f.has_default) {
          bool found = false;
          for (auto& v : e.values)
            if (f.dflt.t == Tok::Ident && !f.dflt_neg && v.first == f.dflt.s) { p.default_bits = (uint64_t)(int64_t)v.second; found = true; break; }
          if (!found) parse_fail(where + ": enum type \"" + p.type_name + "\" has no value named \"" + f.dflt.s + "\"");
        }
      } else if (f.has_default) {
        const Tok& t = f.dflt;
        const bool fp = p.kind == PbKind::Double || p.kind == PbKind::Float;
        auto bad = [&]() { parse_fail(where + ": invalid default value"); };
        if (p.kind == PbKind::String || p.kind == PbKind::Bytes) {
          if (t.t != Tok::Str || f.dflt_neg) bad();
          p.default_bytes = t.s;
        } else if (p.kind == PbKind::Bool) {
          if (t.t != Tok::Ident || f.dflt_neg || (t.s != "true" && t.s != "false")) bad();
          p.default_bits = t.s == "true";
        } else if (fp) {
          double d;
          if (t.t == Tok::Int || t.t == Tok::Float) d = strtod(t.s.c_str(), nullptr);
          else if (t.t == Tok::Ident && (t.s == "inf" || t.s == "infinity")) d = INFINITY;
          else if (t.t == Tok::Ident && t.s == "nan") d = NAN;
          else bad();
          if (f.dflt_neg) d = -d;
          p.default_bits = p.kind == PbKind::Double ? double_bits(d) : float_bits((float)d);
        } else {
          if (t.t != Tok::Int) bad();
          errno = 0;
          const unsigned long long mag = strtoull(t.s.c_str(), nullptr, 0);
          if (errno == ERANGE) bad();
          const bool is64 = p.kind == PbKind::Int64 || p.kind == PbKind::SInt64 || p.kind == PbKind::SFixed64 || p.kind == PbKind::UInt64 || p.kind == PbKind::Fixed64;
          const bool uns = p.kind == PbKind::UInt32 || p.kind == PbKind::Fixed32 || p.kind == PbKind::UInt64 || p.kind == PbKind::Fixed64;
          if (uns && f.dflt_neg && mag) bad();
          const unsigned long long lim = uns ? (is64 ? ~0ull : 0xFFFFFFFFull) : (is64 ? (1ull << 63) - (f.dflt_neg ? 0 : 1) : (1ull << 31) - (f.dflt_neg ? 0 : 1));
          if (mag > lim) bad();
          p.default_bits = f.dflt_neg ? (uint64_t)(0 - mag) : (uint64_t)mag;
        }
      }
      out.push_back(std::move(p));
    }
    resolved[m.full_name] = std::move(out);
  }
  auto it = resolved.find(message_type);
  if (it == resolved.end()) fail(ARK_ERR_CONFIG, "The message type could not be found: " + message_type);
  PbMessage msg;
  msg.full_name = message_type;
  msg.fields = std::move(it->second);
  return msg;
}

}  // namespace

PbMessage load_proto_message(const std::vector<std::string>& inputs, const std::vector<std::string>& includes,
                             const std::string& message_type) {
  // list_files_in_dir + the `.proto` extension filter (component/protobuf.rs:42-69): a path that is not a directory adds nothing
  std::vector<std::string> files;
  for (auto& dir : inputs) {
    if (!is_dir(dir)) continue;
    DIR* d = opendir(dir.c_str());
    if (!d) fail(ARK_ERR_CONFIG, "Failed to list proto files: cannot read " + dir);
    std::vector<std::string> here;
    while (dirent* e = readdir(d)) {
      const std::string name = e->d_name;
      const std::string path = dir + "/" + name;
      if (name.size() > 6 && name.compare(name.size() - 6, 6, ".proto") == 0 && is_file(path)) here.push_back(path);
    }
    closedir(d);
    std::sort(here.begin(), here.end());
    files.insert(files.end(), here.begin(), here.end());
  }
  if (files.empty())
    fail(ARK_ERR_CONFIG, "No proto files found in the specified paths. Please ensure the paths contain valid .proto files");
  Pool pool(includes);
  for (auto& f : files) pool.parse_input(f);
  return pool.resolve(message_type);
}

std::string pb_kind_debug(const PbField& f) {
  switch (f.kind) {
    case PbKind::Double: return "Double"; case PbKind::Float: return "Float"; case PbKind::Int64: return "Int64";
    case PbKind::UInt64: return "Uint64"; case PbKind::Int32: return "Int32"; case PbKind::Fixed64: return "Fixed64";
    case PbKind::Fixed32: return "Fixed32"; case PbKind::Bool: return "Bool"; case PbKind::String: return "String";
    case PbKind::Bytes: return "Bytes"; case PbKind::UInt32: return "Uint32"; case PbKind::SFixed32: return "Sfixed32";
    case PbKind::SFixed64: return "Sfixed64"; case PbKind::SInt32: return "Sint32"; case PbKind::SInt64: return "Sint64";
    case PbKind::Enum: return "Enum(" + f.type_name + ")";
    case PbKind::Group: case PbKind::Message: return "Message(" + (f.is_map ? std::string("map entry of ") + f.name : f.type_name) + ")";
  }
  return "?";
}

}  // namespace ark
