// op_params.h -- the string attribute dict of an imperative operator call, parsed the way the
// reference's dmlc::Parameter fields are (scalars: dmlc::stof; tuples: istream >> float), and the
// scalar of the *_scalar operators the way their attribute parser does (std::stod).
#pragma once
#include <cstdlib>
#include <initializer_list>
#include <stdexcept>
#include <string>
#include <type_traits>
#include <utility>
#include <vector>

#include "common.h"
#include "scalar_parse.h"

namespace b200kv {

typedef std::vector<std::pair<std::string, std::string>> Params;

inline const std::string* Find(const Params& p, const std::string& k) {
  for (auto& kv : p) {
    if (kv.first == k) return &kv.second;
  }
  return nullptr;
}

// scalar op parameter: dmlc::Parameter float field (dmlc::stof)
inline float GetF(const Params& p, const std::string& k, float dflt) {
  const std::string* v = Find(p, k);
  return v ? DmlcStof(*v) : dflt;
}

// a parameter without a default value, refused when absent (dmlc::Parameter::Init): float fields
// parsed as GetF does, int fields as GetI, double fields with dmlc::stod, or the string itself
template <typename T = float>
T Required(const Params& p, const char* key, const char* op) {
  const std::string* v = Find(p, key);
  KV_CHECK(v != nullptr) << "Required parameter " << key << " of " << op << " is missing";
  if constexpr (std::is_same<T, std::string>::value) return *v;
  else if constexpr (std::is_same<T, int>::value) return std::atoi(v->c_str());
  else if constexpr (std::is_same<T, double>::value) return DmlcStod(*v);
  else return DmlcStof(*v);
}

// dmlc::Parameter::Init refuses a key its parameter struct does not declare, listing those it does
inline void RejectUnknownKeys(const Params& p, std::initializer_list<const char*> allowed) {
  for (const auto& kv : p) {
    bool known = false;
    std::string list;
    for (const char* k : allowed) {
      known = known || kv.first == k;
      list += (list.empty() ? "" : ", ") + std::string(k);
    }
    KV_CHECK(known) << "Cannot find argument '" << kv.first << "', Possible Arguments: " << list;
  }
}

// the scalar of the reference's *_scalar operators: std::stod (elemwise_binary_scalar_op.h:347-354).
// The kernel then rounds it once to the array's dtype, as BinaryScalarOp's DType(alpha) does.
// Not GetF's dmlc::stof.
inline double StodD(const Params& p, const char* key, const char* op) {
  const std::string v = Required<std::string>(p, key, op);
  try {
    return std::stod(v);
  } catch (const std::exception&) {
    KV_FATAL << op << ": cannot parse " << key << "='" << v << "'";
  }
  return 0.0;
}

// the same for a float32 operand: std::stod, then one rounding to float
inline float StodF(const Params& p, const char* key, const char* op) {
  return static_cast<float>(StodD(p, key, op));
}

inline int GetI(const Params& p, const std::string& k, int dflt) {
  const std::string* v = Find(p, k);
  return v ? std::atoi(v->c_str()) : dflt;
}

inline bool GetB(const Params& p, const std::string& k, bool dflt) {
  const std::string* v = Find(p, k);
  if (!v) return dflt;
  return *v == "True" || *v == "true" || *v == "1";
}

// tuple op parameter "(0.1, 0.2)" / "[0.1, 0.2]": mxnet::Tuple<float> via istream >> float
inline std::vector<float> GetTuple(const Params& p, const std::string& k) {
  const std::string* v = Find(p, k);
  KV_CHECK(v != nullptr) << "Required parameter " << k << " is missing";
  std::vector<float> out;
  const char* s = v->c_str();
  while (*s) {
    if (*s == '(' || *s == ')' || *s == '[' || *s == ']' || *s == ',' || *s == ' ' || *s == 'L') {
      ++s;
      continue;
    }
    char* end = nullptr;
    float f = std::strtof(s, &end);
    KV_CHECK(end != s) << "cannot parse tuple parameter " << k << "='" << *v << "'";
    out.push_back(f);
    s = end;
  }
  return out;
}


// integer tuple "(1, 2, 3)" (mxnet::Tuple<int>)
inline std::vector<int> GetIntTuple(const Params& p, const std::string& k) {
  std::vector<int> out;
  for (float f : GetTuple(p, k)) out.push_back(static_cast<int>(f));
  return out;
}

}  // namespace b200kv
