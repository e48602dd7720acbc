// ORACLE — TEST INFRASTRUCTURE ONLY.  gflags for the reference's RigAnalyzer.cpp (riganalyzer.mk): the sweep-view
// checkers' DEFINE_* stand-ins plus GetArgv, which returns the command line the bridge sets before it runs main.
#pragma once
#include "../../sweepshim/gflags/gflags.h"
namespace gflags {
extern std::string g_refArgv;  // defined in ref_bridge_riganalyzer.cpp
inline std::string GetArgv() { return g_refArgv; }
}  // namespace gflags
