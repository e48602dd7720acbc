// Camera::saveRig (Camera.cpp:158-177, 293-313) for the apps that write rigs: sorted keys, folly's FIXED mode with 10
// digits (RigSimulator's --rig_out) or its default SHORTEST doubles (RigAnalyzer's --output_rig), and an optional
// "comments" array.
#pragma once

#include <algorithm>
#include <charconv>
#include <cmath>
#include <cstdio>
#include <fstream>
#include <string>
#include <utility>
#include <vector>

#include "../../../include/derp_b200.h"
#include "flags.h"

namespace rigjson {

// One camera as the app holds it: rot is its rotation matrix, row-major, rows right, up, backward
struct Camera {
  DerpCameraDesc d{};
  double rot[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  std::string id, group;
};

inline std::string fixed10(double v) {
  char b[512];
  snprintf(b, sizeof b, "%.10f", v);
  return b;
}

// folly's toAppend(double) in SHORTEST mode: double-conversion's ToShortest with flags NO_FLAGS, exponent character
// 'E', decimal notation for decimal exponents in [-6, 21) and exponential notation otherwise ("1E21", "1.5E-7"); no
// trailing ".0", and "-0" for negative zero.  The digits are the shortest that round-trip (std::to_chars).
inline std::string shortest(double v) {
  if (std::isnan(v)) return "NaN";
  if (std::isinf(v)) return v < 0 ? "-Infinity" : "Infinity";
  char b[64];
  const auto r = std::to_chars(b, b + sizeof b, v, std::chars_format::scientific);
  std::string s(b, r.ptr);  // [-]d[.ddd]e[+-]xx
  std::string sign;
  if (s[0] == '-') {
    sign = "-";
    s.erase(0, 1);
  }
  const size_t e = s.find('e');
  const int exp = std::stoi(s.substr(e + 1));
  std::string digits = s.substr(0, e);
  digits.erase(std::remove(digits.begin(), digits.end(), '.'), digits.end());
  if (digits == "0") return sign + "0";
  const int n = (int)digits.size(), point = exp + 1;  // the decimal point sits after `point` digits
  if (exp < -6 || exp >= 21) {
    std::string out = digits.substr(0, 1);
    if (n > 1) out += "." + digits.substr(1);
    return sign + out + "E" + std::to_string(exp);
  }
  if (point <= 0) return sign + "0." + std::string(-point, '0') + digits;
  if (point >= n) return sign + digits + std::string(point - n, '0');
  return sign + digits.substr(0, point) + "." + digits.substr(point);
}

inline std::string quoted(const std::string& s) {  // folly's JSON string escapes
  std::string o = "\"";
  for (unsigned char c : s) {
    if (c == '"' || c == '\\') {
      o += '\\';
      o += (char)c;
    } else if (c < 0x20) {
      char b[8];
      snprintf(b, sizeof b, "\\u%04x", c);
      o += b;
    } else {
      o += (char)c;
    }
  }
  return o + "\"";
}

inline void saveRig(const std::string& path, const std::vector<Camera>& cams, const std::vector<std::string>& comments,
                    bool shortestDoubles) {
  static const char* kTypes[] = {"FTHETA", "RECTILINEAR", "EQUISOLID", "ORTHOGRAPHIC"};
  auto num = [&](double v) { return shortestDoubles ? shortest(v) : fixed10(v); };
  auto vec = [&](const double* v, int n) {
    std::string s = "[";
    for (int i = 0; i < n; ++i) s += std::string(i ? ", " : "") + num(v[i]);
    return s + "]";
  };
  std::string out = "{\n  \"cameras\": [";
  for (size_t i = 0; i < cams.size(); ++i) {
    const Camera& c = cams[i];
    const double right[3] = {c.rot[0], c.rot[1], c.rot[2]}, up[3] = {c.rot[3], c.rot[4], c.rot[5]},
                 fwd[3] = {-c.rot[6], -c.rot[7], -c.rot[8]};
    std::vector<std::pair<std::string, std::string>> kv = {
        {"focal", vec(c.d.focal, 2)},       {"forward", vec(fwd, 3)},  {"id", quoted(c.id)},
        {"origin", vec(c.d.origin, 3)},     {"resolution", vec(c.d.resolution, 2)},
        {"right", vec(right, 3)},           {"type", std::string("\"") + kTypes[c.d.type] + "\""},
        {"up", vec(up, 3)},                 {"version", "1"}};
    if (c.d.has_principal && (c.d.principal[0] != c.d.resolution[0] / 2 || c.d.principal[1] != c.d.resolution[1] / 2))
      kv.push_back({"principal", vec(c.d.principal, 2)});
    if (c.d.distortion[0] != 0 || c.d.distortion[1] != 0 || c.d.distortion[2] != 0)
      kv.push_back({"distortion", vec(c.d.distortion, 3)});
    if (!c.group.empty()) kv.push_back({"group", quoted(c.group)});
    if (c.d.has_fov) {  // isDefaultFov: cosFov == getDefaultCosFov(type)
      const double cosFov = std::cos(c.d.fov);
      const double def = (c.d.type == DERP_CAM_RECTILINEAR || c.d.type == DERP_CAM_ORTHOGRAPHIC) ? 0.0 : -1.0;
      if (cosFov != def) kv.push_back({"fov", num(std::acos(cosFov))});
    }
    std::sort(kv.begin(), kv.end());
    out += std::string(i ? "," : "") + "\n    {";
    for (size_t k = 0; k < kv.size(); ++k)
      out += std::string(k ? "," : "") + "\n      \"" + kv[k].first + "\": " + kv[k].second;
    out += "\n    }";
  }
  out += "\n  ]";
  if (!comments.empty()) {
    out += ",\n  \"comments\": [";
    for (size_t i = 0; i < comments.size(); ++i) out += std::string(i ? ", " : "") + quoted(comments[i]);
    out += "]";
  }
  out += "\n}\n";
  std::ofstream f(path);
  CHECK(f.good()) << "cannot write " << path;
  f << out;
}

}  // namespace rigjson
