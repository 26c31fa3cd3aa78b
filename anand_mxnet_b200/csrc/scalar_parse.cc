// scalar_parse.cc -- see scalar_parse.h.
#include "scalar_parse.h"

#include <cctype>
#include <charconv>
#include <cmath>
#include <cstdint>
#include <cstdlib>
#include <limits>
#include <type_traits>

#include "common.h"

namespace b200kv {

std::string PyFloatRepr(double v) {
  if (std::isnan(v)) return "nan";
  if (std::isinf(v)) return v > 0 ? "inf" : "-inf";
  std::string out;
  if (std::signbit(v)) {
    out.push_back('-');
    v = -v;
  }
  if (v == 0.0) return out + "0.0";
  char buf[64];
  auto r = std::to_chars(buf, buf + sizeof(buf), v, std::chars_format::scientific);  // shortest
  std::string sci(buf, r.ptr);
  const size_t epos = sci.find('e');
  std::string digits;
  for (size_t i = 0; i < epos; ++i) {
    if (sci[i] != '.') digits.push_back(sci[i]);
  }
  const int exp10 = std::atoi(sci.c_str() + epos + 1);
  const int decpt = exp10 + 1;  // value = 0.d1d2... * 10^decpt
  const int nd = static_cast<int>(digits.size());
  if (decpt <= -4 || decpt > 16) {
    out.push_back(digits[0]);
    if (nd > 1) {
      out.push_back('.');
      out.append(digits, 1, std::string::npos);
    }
    out.push_back('e');
    int e = decpt - 1;
    out.push_back(e < 0 ? '-' : '+');
    e = e < 0 ? -e : e;
    std::string es = std::to_string(e);
    if (es.size() < 2) es = "0" + es;
    return out + es;
  }
  if (decpt <= 0) {
    out += "0.";
    out.append(static_cast<size_t>(-decpt), '0');
    return out + digits;
  }
  if (decpt >= nd) {
    out += digits;
    out.append(static_cast<size_t>(decpt - nd), '0');
    return out + ".0";
  }
  out.append(digits, 0, static_cast<size_t>(decpt));
  out.push_back('.');
  out.append(digits, static_cast<size_t>(decpt), std::string::npos);
  return out;
}

namespace {

// Restatement of ParseFloat<FloatType, true> (3rdparty/dmlc-core/include/dmlc/strtonum.h:99-254):
// every step is taken in FloatType, as there.
template <typename FloatType>
FloatType ParseDmlc(const std::string& s) {
  constexpr bool kDouble = std::is_same<FloatType, double>::value;
  constexpr unsigned kMaxExponent = kDouble ? 308U : 38U;
  constexpr FloatType kMaxSigForMaxExp =
      static_cast<FloatType>(kDouble ? 1.79769313486231570 : 3.402823466);
  constexpr FloatType kMaxSigForNegMaxExp =
      static_cast<FloatType>(kDouble ? 2.22507385850720139 : 1.175494351);
  constexpr int kStrtofMaxDigits = 19;
  const char* p = s.c_str();
  const char* begin = p;
  while (std::isspace(static_cast<unsigned char>(*p))) ++p;
  bool positive = true;
  if (*p == '-') {
    positive = false;
    ++p;
  } else if (*p == '+') {
    ++p;
  }
  auto finish = [&](FloatType value, const char* end) -> FloatType {
    if (end == begin || *end != '\0') {
      KV_FATAL << "Invalid Parameter format: expect " << (kDouble ? "double" : "float")
               << " but value='" << s << "'";
    }
    return value;
  };
  {
    int i = 0;
    while (i < 8 && static_cast<char>((*p) | 32) == "infinity"[i]) { ++i; ++p; }
    if (i == 3 || i == 8) {
      return finish(positive ? std::numeric_limits<FloatType>::infinity()
                             : -std::numeric_limits<FloatType>::infinity(), p);
    }
    p -= i;
    i = 0;
    while (i < 3 && static_cast<char>((*p) | 32) == "nan"[i]) { ++i; ++p; }
    if (i == 3) return finish(std::numeric_limits<FloatType>::quiet_NaN(), p);
    p -= i;
  }
  const char* num_start = p;
  uint64_t predec = 0;
  for (; std::isdigit(static_cast<unsigned char>(*p)); ++p) {
    predec = predec * 10ULL + static_cast<uint64_t>(*p - '0');
  }
  FloatType value = static_cast<FloatType>(predec);
  if (*p == '.') {
    uint64_t pow10 = 1, val2 = 0;
    int digit_cnt = 0;
    ++p;
    while (std::isdigit(static_cast<unsigned char>(*p))) {
      if (digit_cnt < kStrtofMaxDigits) {
        val2 = val2 * 10ULL + static_cast<uint64_t>(*p - '0');
        pow10 *= 10ULL;
      }
      ++p;
      ++digit_cnt;
    }
    value += static_cast<FloatType>(static_cast<double>(val2) / static_cast<double>(pow10));
  }
  if (p == num_start) {
    KV_FATAL << "Invalid Parameter format: expect " << (kDouble ? "double" : "float")
             << " but value='" << s << "'";
  }
  if (*p == 'e' || *p == 'E') {
    ++p;
    bool frac = false;
    FloatType scale = static_cast<FloatType>(1.0f);
    unsigned expon = 0;
    if (*p == '-') {
      frac = true;
      ++p;
    } else if (*p == '+') {
      ++p;
    }
    for (; std::isdigit(static_cast<unsigned char>(*p)); ++p) {
      expon = expon * 10U + static_cast<unsigned>(*p - '0');
    }
    if (expon > kMaxExponent) KV_FATAL << "Out of range value '" << s << "'";
    if (expon == kMaxExponent && ((!frac && value > kMaxSigForMaxExp) ||
                                  (frac && value < kMaxSigForNegMaxExp))) {
      KV_FATAL << "Out of range value '" << s << "'";
    }
    while (expon >= 8U) { scale *= static_cast<FloatType>(1E8f); expon -= 8U; }
    while (expon > 0U) { scale *= static_cast<FloatType>(10.0f); expon -= 1U; }
    value = frac ? (value / scale) : (value * scale);
  }
  if (*p == 'f' || *p == 'F') ++p;
  return finish(positive ? value : -value, p);
}

}  // namespace

float DmlcStof(const std::string& s) { return ParseDmlc<float>(s); }

double DmlcStod(const std::string& s) { return ParseDmlc<double>(s); }

}  // namespace b200kv
