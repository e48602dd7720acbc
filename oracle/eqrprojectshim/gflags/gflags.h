// ORACLE — TEST INFRASTRUCTURE ONLY.  gflags for the reference's ProjectEquirectsToCameras.cpp (eqrproject.mk): the
// sweep-view checkers' DEFINE_* stand-ins plus the SetUsageMessage its main calls (main is renamed and never run).
#pragma once
#include "../../sweepshim/gflags/gflags.h"
namespace gflags {
inline void SetUsageMessage(const std::string&) {}
}  // namespace gflags
