// ORACLE — TEST INFRASTRUCTURE ONLY.  gflags for the two reference apps the sweep-view checkers compile
// (GenerateCameraOverlaps.cpp, GenerateEquirect.cpp): DEFINE_* makes a plain global FLAGS_<name> with the default.
#pragma once
#include <cstdint>
#include <string>
#define DEFINE_bool(n, v, h) bool FLAGS_##n = v
#define DEFINE_int32(n, v, h) int32_t FLAGS_##n = v
#define DEFINE_uint64(n, v, h) uint64_t FLAGS_##n = v
#define DEFINE_double(n, v, h) double FLAGS_##n = v
#define DEFINE_string(n, v, h) std::string FLAGS_##n = v
