// scalar_parse.h -- the Python-double -> string -> C++ float hop of the reference, reproduced.
//
// Every optimizer hyper-parameter in the reference is formatted by Python (`str(float)`, i.e.
// repr) and parsed back by the operator's dmlc::Parameter: scalar fields (lr, wd, rescale_grad,
// momentum, clip_gradient, beta1, ...) by dmlc::stof == ParseFloat<float>
// (3rdparty/dmlc-core/include/dmlc/strtonum.h:99-254, via parameter.h:1073-1094), which is NOT a
// correctly rounded conversion (it adds float(int part) + float(frac part) and then scales by
// powers of ten in float); the *_scalar operators by std::stod, then DType(alpha)
// (elemwise_binary_scalar_op.h:347-354, 364-365); tuple fields (lrs, wds of the multi_* ops) by std::istream >> float
// (include/mxnet/tuple.h), which IS correctly rounded. To update weights bit-identically the fused
// path must feed its kernels the same float32 values, so both routes are restated here.
#pragma once
#include <string>

namespace b200kv {

// Python's repr(float) / str(float): shortest round-trip digits, exponent form when the decimal
// exponent is < -4 or >= 16 (Python/pystrtod.c format_float_short, mode 'r').
std::string PyFloatRepr(double v);

// dmlc::stof restated (strtonum.h:99-254). Throws b200kv::Error on malformed input / trailing
// characters like FieldEntry<float>::Set does.
float DmlcStof(const std::string& s);
// dmlc::stod restated (ParseFloat<double, true>): the `double` fields, such as `_full`'s value
double DmlcStod(const std::string& s);

// double -> Python string -> dmlc::stof  (scalar op parameters)
inline float ScalarParam(double v) { return DmlcStof(PyFloatRepr(v)); }
// double -> Python string -> std::stod -> float: the scalar of the *_scalar operators
// (elemwise_binary_scalar_op.h:347-354, 364-365). repr round-trips, so this is the nearest float32.
inline float StodParam(double v) { return static_cast<float>(v); }
// double -> Python string -> istream >> float (tuple op parameters): nearest float32
inline float TupleParam(double v) { return static_cast<float>(v); }

}  // namespace b200kv
