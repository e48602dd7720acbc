// Minimal gflags/glog-compatible front end for the drop-in executables.
//
// The reference's callers (scripts/render/worker.py:66-107, scripts/test/test_master_class.py:161-256)
// run `<App> --flag=value ...` with GLOG_* env vars, and scripts/render/setup.py:52-70 learns each
// binary's flags by scraping `DEFINE_<type>(name, default, "help");` lines from the app's .cpp —
// so the apps here keep exactly that DEFINE_ syntax and the reference's names/defaults/help strings
// (SystemUtil.cpp:99-159 initDep: parse flags, echo them, glog to stderr / --log_dir).
#pragma once

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <ctime>
#include <fstream>
#include <functional>
#include <iostream>
#include <map>
#include <mutex>
#include <sstream>
#include <string>
#include <vector>

namespace flags {

struct FlagInfo {
  std::string name, type, help, def;
  std::function<bool(const std::string&)> set;
  std::function<std::string()> get;
};

inline std::map<std::string, FlagInfo>& registry() {
  static std::map<std::string, FlagInfo> r;
  return r;
}

inline bool parseBool(const std::string& v, bool* out) {
  if (v == "true" || v == "1" || v == "t" || v == "yes" || v == "y") {
    *out = true;
    return true;
  }
  if (v == "false" || v == "0" || v == "f" || v == "no" || v == "n") {
    *out = false;
    return true;
  }
  return false;
}

struct Registrar {
  Registrar(const char* name, const char* type, const char* help, std::string def,
            std::function<bool(const std::string&)> set, std::function<std::string()> get) {
    registry()[name] = FlagInfo{name, type, help, std::move(def), std::move(set), std::move(get)};
  }
};

template <typename T>
inline std::string toStr(const T& v) {
  std::ostringstream s;
  s.precision(17);
  s << v;
  return s.str();
}
inline std::string toStr(const bool& v) { return v ? "true" : "false"; }

#define DERP_DEFINE_FLAG(ctype, tname, name, def, help, parse_expr)                                     \
  ctype FLAGS_##name = def;                                                                             \
  static ::flags::Registrar flag_registrar_##name(                                                      \
      #name, tname, help, ::flags::toStr<ctype>(def),                                                   \
      [](const std::string& v) -> bool { parse_expr },                                                  \
      []() -> std::string { return ::flags::toStr<ctype>(FLAGS_##name); })

#define DEFINE_string(name, def, help) \
  DERP_DEFINE_FLAG(std::string, "string", name, def, help, FLAGS_##name = v; return true;)
#define DEFINE_bool(name, def, help) \
  DERP_DEFINE_FLAG(bool, "bool", name, def, help, return ::flags::parseBool(v, &FLAGS_##name);)
#define DEFINE_int32(name, def, help)                                                                   \
  DERP_DEFINE_FLAG(int, "int32", name, def, help, char* e = nullptr; long x = std::strtol(v.c_str(), &e, 10); \
                   if (v.empty() || *e) return false; FLAGS_##name = (int)x; return true;)
#define DEFINE_uint64(name, def, help)                                                                  \
  DERP_DEFINE_FLAG(uint64_t, "uint64", name, def, help, char* e = nullptr;                                   \
                   unsigned long long x = std::strtoull(v.c_str(), &e, 10);                                   \
                   if (v.empty() || *e || v[0] == '-') return false; FLAGS_##name = (uint64_t)x; return true;)
#define DEFINE_double(name, def, help)                                                                  \
  DERP_DEFINE_FLAG(double, "double", name, def, help, char* e = nullptr; double x = std::strtod(v.c_str(), &e); \
                   if (v.empty() || *e) return false; FLAGS_##name = x; return true;)

// ---- glog-like logging ---------------------------------------------------------------------------
struct LogState {
  std::string program = "derp";
  std::string logDir;
  std::ofstream infoFile, fatalFile;
  std::mutex mu;
  bool toStderr = true;
};
inline LogState& logState() {
  static LogState s;
  return s;
}

inline void logLine(char sev, const char* file, int line, const std::string& msg) {
  LogState& s = logState();
  std::lock_guard<std::mutex> lk(s.mu);
  char ts[64];
  std::time_t t = std::time(nullptr);
  std::tm tmv;
  localtime_r(&t, &tmv);
  std::strftime(ts, sizeof(ts), "%m%d %H:%M:%S", &tmv);
  const char* base = std::strrchr(file, '/');
  std::ostringstream o;
  o << sev << ts << " " << (base ? base + 1 : file) << ":" << line << "] " << msg << "\n";
  const std::string str = o.str();
  if (s.toStderr) std::fputs(str.c_str(), stderr);
  if (s.infoFile.is_open()) {
    s.infoFile << str;
    s.infoFile.flush();
  }
  if (sev == 'F' && s.fatalFile.is_open()) {
    s.fatalFile << str;
    s.fatalFile.flush();
  }
}

struct LogMessage {
  char sev;
  const char* file;
  int line;
  std::ostringstream os;
  LogMessage(char s, const char* f, int l) : sev(s), file(f), line(l) {}
  ~LogMessage() noexcept(false) {
    logLine(sev, file, line, os.str());
    if (sev == 'F') std::abort();  // glog FATAL: message, then abort() (non-zero exit)
  }
};

#define LOG_INFO ::flags::LogMessage('I', __FILE__, __LINE__).os
#define LOG_WARNING ::flags::LogMessage('W', __FILE__, __LINE__).os
#define LOG_ERROR ::flags::LogMessage('E', __FILE__, __LINE__).os
#define LOG_FATAL ::flags::LogMessage('F', __FILE__, __LINE__).os
#define LOG(sev) LOG_##sev
#define CHECK(cond) \
  if (!(cond)) LOG(FATAL) << "Check failed: " #cond " "
#define CHECK_OP(a, b, op) \
  if (!((a)op(b))) LOG(FATAL) << "Check failed: " #a " " #op " " #b " (" << (a) << " vs. " << (b) << ") "
#define CHECK_EQ(a, b) CHECK_OP(a, b, ==)
#define CHECK_NE(a, b) CHECK_OP(a, b, !=)
#define CHECK_LE(a, b) CHECK_OP(a, b, <=)
#define CHECK_LT(a, b) CHECK_OP(a, b, <)
#define CHECK_GE(a, b) CHECK_OP(a, b, >=)
#define CHECK_GT(a, b) CHECK_OP(a, b, >)

inline void printHelp(const std::string& usage) {
  std::cout << usage << "\n  Flags:\n";
  for (auto& kv : registry())
    std::cout << "    -" << kv.second.name << " (" << kv.second.help << ") type: " << kv.second.type
              << " default: " << (kv.second.type == "string" ? "\"" + kv.second.def + "\"" : kv.second.def) << "\n";
}

inline bool setFlag(const std::string& name, const std::string& value, bool fromFile) {
  auto it = registry().find(name);
  if (it == registry().end()) return false;
  if (!it->second.set(value)) {
    std::fprintf(stderr, "ERROR: illegal value '%s' specified for %s flag '%s'\n", value.c_str(),
                 it->second.type.c_str(), name.c_str());
    std::exit(1);
  }
  (void)fromFile;
  return true;
}

inline void parseArgs(std::vector<std::string> args, const std::string& usage, bool fromFile);

inline void parseFlagFile(const std::string& path, const std::string& usage) {
  std::ifstream f(path);
  if (!f.good()) {
    std::fprintf(stderr, "ERROR: cannot read flagfile %s\n", path.c_str());
    std::exit(1);
  }
  std::vector<std::string> args;
  std::string line;
  while (std::getline(f, line)) {
    size_t a = line.find_first_not_of(" \t\r");
    if (a == std::string::npos || line[a] == '#') continue;
    size_t b = line.find_last_not_of(" \t\r");
    args.push_back(line.substr(a, b - a + 1));
  }
  parseArgs(args, usage, true);
}

// built-ins used by the reference's callers: --log_dir, --alsologtostderr, --stderrthreshold, --v, --help, --flagfile
inline void parseArgs(std::vector<std::string> args, const std::string& usage, bool fromFile) {
  LogState& ls = logState();
  for (size_t i = 0; i < args.size(); ++i) {
    std::string a = args[i];
    if (a.size() < 2 || a[0] != '-') {
      std::fprintf(stderr, "ERROR: unexpected argument '%s'\n", a.c_str());
      std::exit(1);
    }
    a = a.substr(a[1] == '-' ? 2 : 1);
    std::string name = a, value;
    bool hasValue = false;
    const size_t eq = a.find('=');
    if (eq != std::string::npos) {
      name = a.substr(0, eq);
      value = a.substr(eq + 1);
      hasValue = true;
    }
    if (name == "help" || name == "helpfull" || name == "helpshort") {
      printHelp(usage);
      std::exit(1);  // gflags exits 1 after --help
    }
    auto takeNext = [&]() {
      if (!hasValue) {
        if (i + 1 >= args.size()) {
          std::fprintf(stderr, "ERROR: flag '%s' is missing its argument\n", name.c_str());
          std::exit(1);
        }
        value = args[++i];
        hasValue = true;
      }
    };
    if (name == "flagfile") {
      takeNext();
      parseFlagFile(value, usage);
      continue;
    }
    if (name == "log_dir") {
      takeNext();
      ls.logDir = value;
      continue;
    }
    if (name == "alsologtostderr" || name == "logtostderr" || name == "stderrthreshold" || name == "v" ||
        name == "minloglevel" || name == "colorlogtostderr") {
      if (!hasValue && i + 1 < args.size() && args[i + 1][0] != '-') ++i;
      continue;  // we always log to stderr (the callers set GLOG_alsologtostderr=1)
    }
    auto it = registry().find(name);
    if (it == registry().end() && name.rfind("no", 0) == 0) {  // --noflag for booleans
      auto nb = registry().find(name.substr(2));
      if (nb != registry().end() && nb->second.type == "bool" && !hasValue) {
        nb->second.set("false");
        continue;
      }
    }
    if (it == registry().end()) {
      std::fprintf(stderr, "ERROR: unknown command line flag '%s'\n", name.c_str());
      if (!fromFile) std::exit(1);  // gflags: unknown flags in a flagfile are ignored, on argv they are fatal
      continue;
    }
    if (it->second.type == "bool" && !hasValue) {
      it->second.set("true");
      continue;
    }
    takeNext();
    setFlag(name, value, fromFile);
  }
}

// system_util::initDep (SystemUtil.cpp:99-159)
inline void initDep(int argc, char** argv, const std::string& usage) {
  LogState& ls = logState();
  const char* base = std::strrchr(argv[0], '/');
  ls.program = base ? base + 1 : argv[0];
  std::vector<std::string> args(argv + 1, argv + argc);
  parseArgs(args, usage, false);
  if (const char* e = std::getenv("GLOG_log_dir"))
    if (ls.logDir.empty()) ls.logDir = e;
  if (!ls.logDir.empty()) {
    ls.infoFile.open(ls.logDir + "/" + ls.program + ".INFO", std::ios::app);
    ls.fatalFile.open(ls.logDir + "/" + ls.program + ".FATAL", std::ios::app);
  }
  // logFlags (SystemUtil.cpp:78-97)
  size_t pad = 0;
  for (auto& kv : registry()) pad = std::max(pad, kv.first.size());
  LOG(INFO) << "Flags:";
  for (auto& kv : registry()) {
    std::string n = kv.first;
    n.resize(pad, ' ');
    LOG(INFO) << "--" << n << " = " << kv.second.get();
  }
}

}  // namespace flags
