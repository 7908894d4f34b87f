// json_mini.h — minimal JSON value parser for processor/buffer configs (the shim serialises the
// component's `serde_json::Value` config back to a string; core/processor/mod.rs:83-90).
#pragma once
#include <cctype>
#include <cerrno>
#include <cstdlib>
#include <map>
#include <memory>
#include <string>
#include <vector>

#include "common.h"

namespace ark {

struct JsonValue {
  enum Kind { Null, Bool, Number, String, Array, Object } kind = Null;
  bool b = false;
  double num = 0;
  bool is_int = false;
  int64_t i64 = 0;
  std::string str;
  std::vector<JsonValue> arr;
  std::vector<std::pair<std::string, JsonValue>> obj;

  const JsonValue* get(const std::string& key) const {
    for (auto& kv : obj) if (kv.first == key) return &kv.second;
    return nullptr;
  }
};

class JsonParser {
 public:
  explicit JsonParser(const std::string& s) : s_(s) {}
  JsonValue parse() {
    JsonValue v = value();
    ws();
    if (p_ != s_.size()) err("trailing characters");
    return v;
  }

 private:
  const std::string& s_;
  size_t p_ = 0;
  [[noreturn]] void err(const std::string& m) {
    fail(ARK_ERR_SERIALIZATION, "invalid JSON config: " + m + " at offset " + std::to_string(p_));
  }
  void ws() { while (p_ < s_.size() && isspace((unsigned char)s_[p_])) ++p_; }
  JsonValue value() {
    ws();
    if (p_ >= s_.size()) err("unexpected end");
    char c = s_[p_];
    JsonValue v;
    if (c == '{') {
      v.kind = JsonValue::Object; ++p_; ws();
      if (p_ < s_.size() && s_[p_] == '}') { ++p_; return v; }
      while (true) {
        ws();
        if (p_ >= s_.size() || s_[p_] != '"') err("expected object key");
        std::string k = string();
        ws();
        if (p_ >= s_.size() || s_[p_] != ':') err("expected ':'");
        ++p_;
        v.obj.emplace_back(k, value());
        ws();
        if (p_ < s_.size() && s_[p_] == ',') { ++p_; continue; }
        if (p_ < s_.size() && s_[p_] == '}') { ++p_; break; }
        err("expected ',' or '}'");
      }
    } else if (c == '[') {
      v.kind = JsonValue::Array; ++p_; ws();
      if (p_ < s_.size() && s_[p_] == ']') { ++p_; return v; }
      while (true) {
        v.arr.push_back(value());
        ws();
        if (p_ < s_.size() && s_[p_] == ',') { ++p_; continue; }
        if (p_ < s_.size() && s_[p_] == ']') { ++p_; break; }
        err("expected ',' or ']'");
      }
    } else if (c == '"') {
      v.kind = JsonValue::String; v.str = string();
    } else if (!s_.compare(p_, 4, "true")) { v.kind = JsonValue::Bool; v.b = true; p_ += 4; }
    else if (!s_.compare(p_, 5, "false")) { v.kind = JsonValue::Bool; v.b = false; p_ += 5; }
    else if (!s_.compare(p_, 4, "null")) { v.kind = JsonValue::Null; p_ += 4; }
    else if (c == '-' || isdigit((unsigned char)c)) {
      size_t q = p_;
      if (s_[q] == '-') ++q;
      while (q < s_.size() && (isdigit((unsigned char)s_[q]) || s_[q] == '.' || s_[q] == 'e' || s_[q] == 'E' || s_[q] == '+' || s_[q] == '-')) ++q;
      std::string t = s_.substr(p_, q - p_);
      v.kind = JsonValue::Number;
      v.num = strtod(t.c_str(), nullptr);
      if (t.find_first_of(".eE") == std::string::npos) {
        errno = 0;
        v.i64 = strtoll(t.c_str(), nullptr, 10);
        v.is_int = errno != ERANGE;  // beyond i64 (e.g. u64::MAX) is a Float64 for arrow-json's inference
      }
      p_ = q;
    } else err(std::string("unexpected character '") + c + "'");
    return v;
  }
  // four hex digits at p_ (serde_json: anything else is an error)
  unsigned hex4() {
    if (p_ + 4 > s_.size()) err("bad \\u escape");
    unsigned v = 0;
    for (int k = 0; k < 4; ++k) {
      const char h = s_[p_++];
      const int d = h >= '0' && h <= '9' ? h - '0' : h >= 'a' && h <= 'f' ? h - 'a' + 10 : h >= 'A' && h <= 'F' ? h - 'A' + 10 : -1;
      if (d < 0) err("bad \\u escape");
      v = v * 16 + (unsigned)d;
    }
    return v;
  }
  // a JSON string → UTF-8.  Only JSON's nine escapes; a surrogate escape must be a high + low pair (combined into one
  // code point, as the device decoder does); raw control characters are errors, as in serde_json.
  std::string string() {
    std::string out;
    ++p_;
    while (true) {
      if (p_ >= s_.size()) err("unterminated string");
      char c = s_[p_++];
      if (c == '"') break;
      if ((unsigned char)c < 0x20) err("control character in string");
      if (c == '\\') {
        if (p_ >= s_.size()) err("bad escape");
        char e = s_[p_++];
        switch (e) {
          case 'n': out += '\n'; break; case 't': out += '\t'; break; case 'r': out += '\r'; break;
          case 'b': out += '\b'; break; case 'f': out += '\f'; break;
          case '"': case '\\': case '/': out += e; break;
          case 'u': {
            unsigned cp = hex4();
            if (cp >= 0xDC00 && cp <= 0xDFFF) err("lone low surrogate in \\u escape");
            if (cp >= 0xD800 && cp <= 0xDBFF) {
              if (p_ + 2 > s_.size() || s_[p_] != '\\' || s_[p_ + 1] != 'u') err("unpaired surrogate in \\u escape");
              p_ += 2;
              const unsigned lo = hex4();
              if (lo < 0xDC00 || lo > 0xDFFF) err("unpaired surrogate in \\u escape");
              cp = 0x10000 + ((cp - 0xD800) << 10) + (lo - 0xDC00);
            }
            if (cp < 0x80) out += (char)cp;
            else if (cp < 0x800) { out += (char)(0xC0 | (cp >> 6)); out += (char)(0x80 | (cp & 0x3F)); }
            else if (cp < 0x10000) { out += (char)(0xE0 | (cp >> 12)); out += (char)(0x80 | ((cp >> 6) & 0x3F)); out += (char)(0x80 | (cp & 0x3F)); }
            else { out += (char)(0xF0 | (cp >> 18)); out += (char)(0x80 | ((cp >> 12) & 0x3F)); out += (char)(0x80 | ((cp >> 6) & 0x3F)); out += (char)(0x80 | (cp & 0x3F)); }
            break;
          }
          default: err(std::string("bad escape '\\") + e + "'");
        }
      } else out += c;
    }
    return out;
  }
};

inline JsonValue parse_json(const std::string& s) { return JsonParser(s).parse(); }

}  // namespace ark
