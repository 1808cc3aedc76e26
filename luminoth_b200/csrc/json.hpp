// Minimal JSON reader for the engine config (input is json.dumps(config) from the wrapper).
#pragma once
#include <cstdlib>
#include <map>
#include <string>
#include <vector>
#include <stdexcept>

namespace lumi {

struct JVal {
  enum Type { Null, Bool, Num, Str, Arr, Obj } t = Null;
  bool b = false;
  double num = 0;
  std::string s;
  std::vector<JVal> arr;
  std::map<std::string, JVal> obj;

  const JVal* find(const std::string& path) const {
    const JVal* cur = this;
    size_t pos = 0;
    while (pos <= path.size()) {
      size_t dot = path.find('.', pos);
      std::string key = path.substr(pos, dot == std::string::npos ? std::string::npos : dot - pos);
      if (cur->t != Obj) return nullptr;
      auto it = cur->obj.find(key);
      if (it == cur->obj.end()) return nullptr;
      cur = &it->second;
      if (dot == std::string::npos) break;
      pos = dot + 1;
    }
    return cur;
  }
  double number(const std::string& path, double def) const {
    const JVal* v = find(path);
    if (!v || v->t == Null) return def;
    if (v->t == Num) return v->num;
    if (v->t == Bool) return v->b ? 1.0 : 0.0;
    throw std::runtime_error("config key '" + path + "' is not a number");
  }
  bool boolean(const std::string& path, bool def) const {
    const JVal* v = find(path);
    if (!v || v->t == Null) return def;
    if (v->t == Bool) return v->b;
    if (v->t == Num) return v->num != 0;
    throw std::runtime_error("config key '" + path + "' is not a boolean");
  }
  std::string str(const std::string& path, const std::string& def) const {
    const JVal* v = find(path);
    if (!v || v->t == Null) return def;
    if (v->t == Str) return v->s;
    throw std::runtime_error("config key '" + path + "' is not a string");
  }
  // as str(), but a null value reads as the empty string: only a missing key takes the default
  std::string str_or_empty(const std::string& path, const std::string& def) const {
    const JVal* v = find(path);
    if (!v) return def;
    if (v->t == Null) return "";
    return str(path, def);
  }
  std::vector<double> numbers(const std::string& path) const {
    std::vector<double> out;
    const JVal* v = find(path);
    if (!v || v->t == Null) return out;
    if (v->t != Arr) throw std::runtime_error("config key '" + path + "' is not a list");
    for (const auto& e : v->arr) {
      if (e.t != Num) throw std::runtime_error("config key '" + path + "' holds a non-number");
      out.push_back(e.num);
    }
    return out;
  }
};

class JParser {
 public:
  explicit JParser(const std::string& s) : s_(s) {}
  JVal parse() {
    JVal v = value();
    ws();
    if (i_ != s_.size()) fail("trailing characters");
    return v;
  }

 private:
  const std::string& s_;
  size_t i_ = 0;
  [[noreturn]] void fail(const std::string& m) { throw std::runtime_error("config JSON: " + m + " at " + std::to_string(i_)); }
  void ws() { while (i_ < s_.size() && (s_[i_] == ' ' || s_[i_] == '\n' || s_[i_] == '\t' || s_[i_] == '\r')) ++i_; }
  bool lit(const char* w) {
    size_t n = std::char_traits<char>::length(w);
    if (s_.compare(i_, n, w) == 0) { i_ += n; return true; }
    return false;
  }
  JVal value() {
    ws();
    if (i_ >= s_.size()) fail("unexpected end");
    char c = s_[i_];
    JVal v;
    if (c == '{') {
      v.t = JVal::Obj; ++i_; ws();
      if (s_[i_] == '}') { ++i_; return v; }
      while (true) {
        ws();
        JVal k = string_();
        ws();
        if (s_[i_] != ':') fail("expected ':'");
        ++i_;
        v.obj[k.s] = value();
        ws();
        if (s_[i_] == ',') { ++i_; continue; }
        if (s_[i_] == '}') { ++i_; break; }
        fail("expected ',' or '}'");
      }
      return v;
    }
    if (c == '[') {
      v.t = JVal::Arr; ++i_; ws();
      if (s_[i_] == ']') { ++i_; return v; }
      while (true) {
        v.arr.push_back(value());
        ws();
        if (s_[i_] == ',') { ++i_; continue; }
        if (s_[i_] == ']') { ++i_; break; }
        fail("expected ',' or ']'");
      }
      return v;
    }
    if (c == '"') return string_();
    if (lit("true")) { v.t = JVal::Bool; v.b = true; return v; }
    if (lit("false")) { v.t = JVal::Bool; v.b = false; return v; }
    if (lit("null")) { v.t = JVal::Null; return v; }
    if (lit("NaN") || lit("Infinity") || lit("-Infinity")) fail("non-finite number");
    char* end = nullptr;
    v.num = std::strtod(s_.c_str() + i_, &end);
    if (end == s_.c_str() + i_) fail("bad value");
    v.t = JVal::Num;
    i_ = end - s_.c_str();
    return v;
  }
  JVal string_() {
    if (s_[i_] != '"') fail("expected string");
    ++i_;
    JVal v; v.t = JVal::Str;
    while (i_ < s_.size() && s_[i_] != '"') {
      if (s_[i_] == '\\') {
        ++i_;
        char e = s_[i_];
        if (e == 'n') v.s += '\n';
        else if (e == 't') v.s += '\t';
        else if (e == 'u') { v.s += '?'; i_ += 4; }
        else v.s += e;
        ++i_;
      } else {
        v.s += s_[i_++];
      }
    }
    if (i_ >= s_.size()) fail("unterminated string");
    ++i_;
    return v;
  }
};

}  // namespace lumi
