// Host-side file formats of the drop-in apps: rig JSON (Camera.cpp:30-75, 244-258), PFM
// (CvUtil.cpp:39-73), PNG via zlib (the reference uses cv::imread / cv::imwrite, CvUtil.cpp:22-37),
// the directory layout (ImageTypes.h:16-47, DerpUtil.cpp:278-330) and the per-camera image loaders
// (ImageUtil.h:42-107, CvUtil.h:227-284 convertImage semantics).
#pragma once

#include <cfloat>
#include <zlib.h>

#include "area_resize.h"
#include "inflate.h"

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <filesystem>
#include <fstream>
#include <iomanip>
#include <map>
#include <memory>
#include <sstream>
#include <string>
#include <vector>

#include "../../../include/derp_b200.h"
#include "flags.h"

namespace fs = std::filesystem;

namespace io {

// ---- JSON (just enough for rig files) ----------------------------------------------------------------
struct Json {
  enum Type { Null, Bool, Num, Str, Arr, Obj } type = Null;
  double num = 0;
  bool b = false;
  std::string str;
  std::vector<Json> arr;
  std::vector<std::pair<std::string, Json>> obj;
  const Json* find(const std::string& k) const {
    for (auto& kv : obj)
      if (kv.first == k) return &kv.second;
    return nullptr;
  }
  const Json& at(const std::string& k) const {
    const Json* j = find(k);
    CHECK(j != nullptr) << "missing JSON key: " << k;
    return *j;
  }
};

class JsonParser {
 public:
  explicit JsonParser(const std::string& s) : s_(s) {}
  Json parse() {
    Json j = value();
    ws();
    CHECK(p_ == s_.size()) << "trailing characters in JSON at offset " << p_;
    return j;
  }

 private:
  const std::string& s_;
  size_t p_ = 0;
  void ws() {
    while (p_ < s_.size() && (s_[p_] == ' ' || s_[p_] == '\n' || s_[p_] == '\t' || s_[p_] == '\r')) ++p_;
  }
  char peek() {
    ws();
    CHECK(p_ < s_.size()) << "unexpected end of JSON";
    return s_[p_];
  }
  void expect(char c) {
    CHECK(peek() == c) << "JSON: expected '" << c << "' at offset " << p_;
    ++p_;
  }
  std::string string() {
    expect('"');
    std::string out;
    while (true) {
      CHECK(p_ < s_.size()) << "unterminated JSON string";
      char c = s_[p_++];
      if (c == '"') break;
      if (c == '\\') {
        CHECK(p_ < s_.size()) << "bad escape";
        char e = s_[p_++];
        switch (e) {
          case 'n': out += '\n'; break;
          case 't': out += '\t'; break;
          case 'r': out += '\r'; break;
          case 'b': out += '\b'; break;
          case 'f': out += '\f'; break;
          case 'u': {
            CHECK(p_ + 4 <= s_.size()) << "bad \\u escape";
            unsigned cp = (unsigned)std::stoul(s_.substr(p_, 4), nullptr, 16);
            p_ += 4;
            if (cp < 0x80) out += (char)cp;
            else if (cp < 0x800) {
              out += (char)(0xC0 | (cp >> 6));
              out += (char)(0x80 | (cp & 0x3F));
            } else {
              out += (char)(0xE0 | (cp >> 12));
              out += (char)(0x80 | ((cp >> 6) & 0x3F));
              out += (char)(0x80 | (cp & 0x3F));
            }
            break;
          }
          default: out += e;
        }
      } else {
        out += c;
      }
    }
    return out;
  }
  Json value() {
    char c = peek();
    Json j;
    if (c == '{') {
      j.type = Json::Obj;
      ++p_;
      if (peek() == '}') {
        ++p_;
        return j;
      }
      while (true) {
        std::string k = string();
        expect(':');
        j.obj.emplace_back(k, value());
        if (peek() == ',') {
          ++p_;
          continue;
        }
        expect('}');
        break;
      }
    } else if (c == '[') {
      j.type = Json::Arr;
      ++p_;
      if (peek() == ']') {
        ++p_;
        return j;
      }
      while (true) {
        j.arr.push_back(value());
        if (peek() == ',') {
          ++p_;
          continue;
        }
        expect(']');
        break;
      }
    } else if (c == '"') {
      j.type = Json::Str;
      j.str = string();
    } else if (s_.compare(p_, 4, "true") == 0) {
      j.type = Json::Bool;
      j.b = true;
      p_ += 4;
    } else if (s_.compare(p_, 5, "false") == 0) {
      j.type = Json::Bool;
      p_ += 5;
    } else if (s_.compare(p_, 4, "null") == 0) {
      p_ += 4;
    } else {
      const char* b = s_.c_str() + p_;
      char* e = nullptr;
      j.type = Json::Num;
      j.num = std::strtod(b, &e);
      CHECK(e != b) << "bad JSON number at offset " << p_;
      p_ += (size_t)(e - b);
    }
    return j;
  }
};

// ---- rig ----------------------------------------------------------------------------------------------
struct Rig {
  std::vector<DerpCameraDesc> cams;
  std::vector<std::string> ids;
  std::vector<std::string> groups;  // "" where the camera has none
};

inline double jnum(const Json& j) {
  if (j.type == Json::Str) return std::stod(j.str);  // folly asDouble accepts numeric strings
  CHECK(j.type == Json::Num) << "expected a number in rig JSON";
  return j.num;
}
template <int N>
inline void jvec(const Json& j, double* out) {
  CHECK_EQ((int)j.arr.size(), N) << "bad vector";
  for (int i = 0; i < N; ++i) out[i] = jnum(j.arr[i]);
}

inline Rig loadRig(const std::string& path) {  // Camera::loadRig (Camera.cpp:244-258)
  std::ifstream f(path);
  std::stringstream ss;
  ss << f.rdbuf();
  const std::string text = ss.str();
  CHECK(!text.empty()) << "could not read JSON file: " << path;
  const Json root = JsonParser(text).parse();
  Rig rig;
  for (const Json& c : root.at("cameras").arr) {
    DerpCameraDesc d;
    std::memset(&d, 0, sizeof(d));
    CHECK_GE(jnum(c.at("version")), 1.0);
    const std::string type = c.at("type").str;
    static const char* names[] = {"FTHETA", "RECTILINEAR", "EQUISOLID", "ORTHOGRAPHIC"};
    d.type = -1;
    for (int i = 0; i < 4; ++i)
      if (type == names[i]) d.type = i;
    CHECK_GE(d.type, 0) << "unknown camera type " << type;
    jvec<3>(c.at("origin"), d.origin);
    jvec<3>(c.at("forward"), d.forward);
    jvec<3>(c.at("up"), d.up);
    jvec<3>(c.at("right"), d.right);
    jvec<2>(c.at("resolution"), d.resolution);
    jvec<2>(c.at("focal"), d.focal);
    if (const Json* p = c.find("principal")) {
      d.has_principal = 1;
      jvec<2>(*p, d.principal);
    }
    if (const Json* p = c.find("distortion")) {
      CHECK_LE((int)p->arr.size(), 3) << "bad distortion";
      for (size_t i = 0; i < p->arr.size(); ++i) d.distortion[i] = jnum(p->arr[i]);
    }
    if (const Json* p = c.find("fov")) {
      d.has_fov = 1;
      d.fov = jnum(*p);
    }
    rig.cams.push_back(d);
    rig.ids.push_back(c.at("id").str);
    const Json* g = c.find("group");
    rig.groups.push_back(g ? g->str : "");
  }
  return rig;
}

// image_util::filterDestinations (ImageUtil.cpp:110-125): indices into rig, in the requested order
inline std::vector<int> filterDestinations(const Rig& rig, const std::string& destinations) {
  std::vector<int> out;
  if (destinations.empty()) {
    for (size_t i = 0; i < rig.ids.size(); ++i) out.push_back((int)i);
    return out;
  }
  std::stringstream ss(destinations);
  std::string dest;
  while (std::getline(ss, dest, ','))
    for (size_t i = 0; i < rig.ids.size(); ++i)
      if (rig.ids[i] == dest) out.push_back((int)i);
  return out;
}

// ---- directory layout (ImageTypes.h:16-47) ------------------------------------------------------------
inline const char* kColorLevels = "video/color_levels";
inline const char* kForegroundMasksLevels = "video/foreground_masks_levels";
inline const char* kBackgroundDispLevels = "background/disparity_levels";
inline const char* kDisparity = "disparity";
inline const char* kDisparityLevels = "disparity_levels";
inline const char* kDisparityTimeFilteredLevels = "disparity_time_filtered_levels";
inline const char* kCost = "cost";
inline const char* kConfidence = "confidence";
inline const char* kMismatches = "mismatches";

inline std::string levelDir(const std::string& dir, int level) { return dir + "/level_" + std::to_string(level); }

inline std::string zeroPad(int x, int padlen = 6) {  // ImageUtil.h:42-46
  std::ostringstream ss;
  ss << std::setw(padlen) << std::setfill('0') << x;
  return ss.str();
}

inline bool isHidden(const fs::path& p) { return p.filename().string()[0] == '.'; }

inline std::vector<fs::path> visibleFilesSorted(const fs::path& dir) {  // FilesystemUtil.h:53-68
  std::vector<fs::path> r;
  for (const auto& e : fs::directory_iterator(dir))
    if (fs::is_regular_file(e) && !isHidden(e.path())) r.push_back(e.path());
  std::sort(r.begin(), r.end());
  return r;
}

inline std::string firstExtension(const fs::path& dir) {  // FilesystemUtil.h:91-95
  const auto files = visibleFilesSorted(dir);
  CHECK_GT(files.size(), 0u) << "no visible files in " << dir.string();
  return files[0].extension().string();
}

inline fs::path imagePath(const fs::path& dir, const std::string& camId, const std::string& frame,
                          const std::string& extension = "") {  // ImageUtil.h:48-56
  const fs::path camDir = dir / camId;
  const std::string ext = extension.empty() ? firstExtension(camDir) : extension;
  return camDir / (frame + ext);
}

// ---- PFM (CvUtil.cpp:39-73): "Pf\n<W> <H>\n-1.0\n" + little-endian rows, top row first -------------
inline void writePfm(const fs::path& path, const float* data, int w, int h) {
  std::ofstream f(path, std::ios::binary);
  CHECK(f.good()) << "cannot write " << path.string();
  f << "Pf\n" << w << " " << h << "\n-1.0\n";
  f.write(reinterpret_cast<const char*>(data), (std::streamsize)w * h * sizeof(float));
}

inline std::vector<float> readPfm(const fs::path& path, int* w, int* h) {
  std::ifstream f(path, std::ios::binary);
  CHECK(f.good()) << "cannot load file: " << path.string();
  std::string format;
  std::getline(f, format);
  CHECK(format == "Pf") << "expected 'Pf' in 1-channel .pfm file header: " << path.string();
  double endian;
  f >> *w >> *h >> endian;
  CHECK_LE(endian, 0.0) << "only little endian .pfm files supported: " << path.string();
  f.ignore();
  std::vector<float> m((size_t)*w * *h);
  f.read(reinterpret_cast<char*>(m.data()), (std::streamsize)m.size() * sizeof(float));
  return m;
}

// ---- PNG (zlib) ---------------------------------------------------------------------------------------
struct Image {
  int w = 0, h = 0, channels = 0, bits = 0;  // bits: 8, 16 (integer) or 32 (float, from .pfm)
  std::vector<uint16_t> u;                   // integer samples (8-bit values stored as-is), interleaved
  std::vector<float> f;                      // float samples (PFM)
};

inline uint32_t be32(const uint8_t* p) { return ((uint32_t)p[0] << 24) | (p[1] << 16) | (p[2] << 8) | p[3]; }

inline Image readPng(const fs::path& path) {
  std::ifstream f(path, std::ios::binary | std::ios::ate);
  CHECK(f.good()) << "failed to load image: " << path.string();
  std::vector<uint8_t> buf((size_t)f.tellg());
  f.seekg(0);
  f.read(reinterpret_cast<char*>(buf.data()), (std::streamsize)buf.size());
  CHECK(f.good()) << "failed to read image: " << path.string();
  static const uint8_t sig[8] = {0x89, 'P', 'N', 'G', 0x0D, 0x0A, 0x1A, 0x0A};
  CHECK(buf.size() > 8 && std::memcmp(buf.data(), sig, 8) == 0) << "not a PNG file: " << path.string();
  size_t p = 8;
  int w = 0, h = 0, depth = 0, ctype = 0, interlace = 0;
  std::vector<uint8_t> idat, palette;
  while (p + 8 <= buf.size()) {
    const uint32_t len = be32(&buf[p]);
    const std::string type(reinterpret_cast<char*>(&buf[p + 4]), 4);
    const uint8_t* data = &buf[p + 8];
    CHECK(p + 12 + len <= buf.size()) << "truncated PNG: " << path.string();
    if (type == "IHDR") {
      w = (int)be32(data);
      h = (int)be32(data + 4);
      depth = data[8];
      ctype = data[9];
      interlace = data[12];
    } else if (type == "PLTE") {
      palette.assign(data, data + len);
    } else if (type == "IDAT") {
      idat.insert(idat.end(), data, data + len);
    } else if (type == "IEND") {
      break;
    }
    p += 12 + len;
  }
  CHECK(w > 0 && h > 0) << "bad PNG header: " << path.string();
  CHECK_EQ(interlace, 0) << "interlaced PNG not supported: " << path.string();
  CHECK(depth == 8 || depth == 16) << "PNG bit depth " << depth << " not supported: " << path.string();
  int ch = 0;
  switch (ctype) {
    case 0: ch = 1; break;
    case 2: ch = 3; break;
    case 3: ch = 1; break;  // palette index, expanded below
    case 4: ch = 2; break;
    case 6: ch = 4; break;
    default: LOG(FATAL) << "bad PNG colour type";
  }
  const int bpp = ch * depth / 8;
  const size_t stride = (size_t)w * bpp;
  std::vector<uint8_t> raw((stride + 1) * h);
  if (!inflate::zlibDecode(idat.data(), idat.size(), raw.data(), raw.size())) {  // declined: let zlib decide
    uLongf outLen = (uLongf)raw.size();
    const int zr = uncompress(raw.data(), &outLen, idat.data(), (uLong)idat.size());
    CHECK(zr == Z_OK && outLen == raw.size()) << "PNG inflate failed: " << path.string();
  }
  // undo the row filters (PNG specification, section 9): one tight loop per filter type; the first bpp bytes of a row have
  // no left neighbour, the first row has no row above
  std::vector<uint8_t> pix(stride * h);
  const std::vector<uint8_t> zeros(stride, 0);
  for (int y = 0; y < h; ++y) {
    const uint8_t ft = raw[y * (stride + 1)];
    const uint8_t* in = &raw[y * (stride + 1) + 1];
    uint8_t* out = &pix[y * stride];
    const uint8_t* up = y ? out - stride : zeros.data();
    const size_t head = std::min<size_t>(bpp, stride);
    switch (ft) {
      case 0: std::memcpy(out, in, stride); break;
      case 1:
        for (size_t i = 0; i < head; ++i) out[i] = in[i];
        for (size_t i = head; i < stride; ++i) out[i] = (uint8_t)(in[i] + out[i - bpp]);
        break;
      case 2:
        for (size_t i = 0; i < stride; ++i) out[i] = (uint8_t)(in[i] + up[i]);
        break;
      case 3:
        for (size_t i = 0; i < head; ++i) out[i] = (uint8_t)(in[i] + (up[i] >> 1));
        for (size_t i = head; i < stride; ++i) out[i] = (uint8_t)(in[i] + ((out[i - bpp] + up[i]) >> 1));
        break;
      case 4:
        for (size_t i = 0; i < head; ++i) out[i] = (uint8_t)(in[i] + up[i]);  // a = c = 0: the predictor is b
        for (size_t i = head; i < stride; ++i) {
          const int a = out[i - bpp], b = up[i], c = up[i - bpp];
          const int pa = std::abs(b - c), pb = std::abs(a - c), pc = std::abs(a + b - 2 * c);
          out[i] = (uint8_t)(in[i] + ((pa <= pb && pa <= pc) ? a : (pb <= pc ? b : c)));
        }
        break;
      default: LOG(FATAL) << "bad PNG filter";
    }
  }
  Image img;
  img.w = w;
  img.h = h;
  img.bits = depth;
  if (ctype == 3) {  // palette -> RGB 8 bit
    CHECK_EQ(depth, 8);
    img.channels = 3;
    img.u.resize((size_t)w * h * 3);
    for (size_t i = 0; i < (size_t)w * h; ++i)
      for (int c = 0; c < 3; ++c) img.u[i * 3 + c] = palette[pix[i] * 3 + c];
  } else {
    // samples are big-endian; PNG stores RGB(A), OpenCV hands out BGR(A) (cv::imread IMREAD_UNCHANGED): one pass does both
    img.channels = ch;
    img.u.resize((size_t)w * h * ch);
    const size_t n = (size_t)w * h;
    uint16_t* dst = img.u.data();
    const uint8_t* src = pix.data();
    auto sample = [&](size_t k) -> uint16_t { return depth == 8 ? src[k] : (uint16_t)((src[2 * k] << 8) | src[2 * k + 1]); };
    if (ch >= 3) {
      for (size_t i = 0; i < n; ++i) {
        const size_t at = i * ch;
        dst[at] = sample(at + 2);
        dst[at + 1] = sample(at + 1);
        dst[at + 2] = sample(at);
        if (ch == 4) dst[at + 3] = sample(at + 3);
      }
    } else {
      for (size_t k = 0; k < n * ch; ++k) dst[k] = sample(k);
    }
    return img;
  }
  // palette: R, G, B entries -> B, G, R
  for (size_t i = 0; i < (size_t)w * h; ++i) std::swap(img.u[i * 3], img.u[i * 3 + 2]);
  return img;
}

inline void pngChunk(std::ofstream& f, const char* type, const std::vector<uint8_t>& data) {
  uint8_t len[4] = {(uint8_t)(data.size() >> 24), (uint8_t)(data.size() >> 16), (uint8_t)(data.size() >> 8),
                    (uint8_t)data.size()};
  f.write(reinterpret_cast<char*>(len), 4);
  f.write(type, 4);
  if (!data.empty()) f.write(reinterpret_cast<const char*>(data.data()), (std::streamsize)data.size());
  uLong crc = crc32(0L, reinterpret_cast<const Bytef*>(type), 4);
  if (!data.empty()) crc = crc32(crc, data.data(), (uInt)data.size());
  uint8_t c[4] = {(uint8_t)(crc >> 24), (uint8_t)(crc >> 16), (uint8_t)(crc >> 8), (uint8_t)crc};
  f.write(reinterpret_cast<char*>(c), 4);
}

// 8-bit PNG, `channels` = 1 (gray), 3 (BGR input, written as RGB) or 4 (BGRA input, written as RGBA) — what cv::imwrite produces for a CV_32F matrix:
// it converts to CV_8U first (convertTo, i.e. saturate_cast<uchar>(cvRound(v)); modules/imgcodecs loadsave.cpp)
inline void writePng8(const fs::path& path, const uint8_t* data, int w, int h, int channels) {
  std::ofstream f(path, std::ios::binary);
  CHECK(f.good()) << "failed to save image: " << path.string();
  static const uint8_t sig[8] = {0x89, 'P', 'N', 'G', 0x0D, 0x0A, 0x1A, 0x0A};
  f.write(reinterpret_cast<const char*>(sig), 8);
  std::vector<uint8_t> ihdr(13);
  ihdr[0] = w >> 24; ihdr[1] = w >> 16; ihdr[2] = w >> 8; ihdr[3] = w;
  ihdr[4] = h >> 24; ihdr[5] = h >> 16; ihdr[6] = h >> 8; ihdr[7] = h;
  ihdr[8] = 8;
  ihdr[9] = channels == 1 ? 0 : channels == 3 ? 2 : 6;
  pngChunk(f, "IHDR", ihdr);
  const size_t stride = (size_t)w * channels;
  std::vector<uint8_t> raw((stride + 1) * h);
  for (int y = 0; y < h; ++y) {
    uint8_t* out = &raw[(size_t)y * (stride + 1)];
    *out++ = 0;
    const uint8_t* in = data + (size_t)y * stride;
    if (channels == 1) {
      std::memcpy(out, in, stride);
    } else if (channels == 3) {
      for (int x = 0; x < w; ++x, in += 3, out += 3) {
        out[0] = in[2];
        out[1] = in[1];
        out[2] = in[0];
      }
    } else {
      for (int x = 0; x < w; ++x, in += 4, out += 4) {
        out[0] = in[2];
        out[1] = in[1];
        out[2] = in[0];
        out[3] = in[3];
      }
    }
  }
  uLongf clen = compressBound((uLong)raw.size());
  std::vector<uint8_t> comp(clen);
  CHECK(compress2(comp.data(), &clen, raw.data(), (uLong)raw.size(), 3) == Z_OK) << "PNG deflate failed";
  comp.resize(clen);
  pngChunk(f, "IDAT", comp);
  pngChunk(f, "IEND", {});
}
inline void writePng8Gray(const fs::path& path, const uint8_t* data, int w, int h) { writePng8(path, data, w, h, 1); }
// saturate_cast<uchar>(float) = saturate_cast<uchar>(cvRound(v)): cvRound is cvtss2si, which answers INT_MIN for NaN and for
// anything outside the int range (e.g. the +inf cost ping-pong leaves on skipped pixels) -> 0 after the clamp
inline uint8_t saturateU8(float v) {
  if (!(v > -2147483648.0f && v < 2147483648.0f)) return 0;
  const long r = std::lrintf(v);
  return (uint8_t)(r < 0 ? 0 : r > 255 ? 255 : r);
}

// 32-bit float OpenEXR file (scan lines, no compression) of 1 channel ("Y", like OpenCV's grayscale EXR output) or 3
// interleaved B, G, R channels (channels "B", "G", "R", as OpenCV names them): the layout of the OpenEXR file-format
// document — magic, version, attribute list, line offset table, scan lines holding each channel's row in chlist order.
inline void writeExrFloatChannels(const fs::path& path, const float* data, int w, int h, int channels) {
  std::ofstream f(path, std::ios::binary);
  CHECK(f.good()) << "failed to save image: " << path.string();
  std::vector<uint8_t> hd;
  auto put32 = [&](std::vector<uint8_t>& v, uint32_t x) {
    for (int i = 0; i < 4; ++i) v.push_back((uint8_t)(x >> (8 * i)));
  };
  auto putF = [&](std::vector<uint8_t>& v, float x) {
    uint32_t u;
    std::memcpy(&u, &x, 4);
    put32(v, u);
  };
  auto putS = [&](std::vector<uint8_t>& v, const char* s) {
    while (*s) v.push_back((uint8_t)*s++);
    v.push_back(0);
  };
  auto attr = [&](const char* name, const char* type, const std::vector<uint8_t>& val) {
    putS(hd, name);
    putS(hd, type);
    put32(hd, (uint32_t)val.size());
    hd.insert(hd.end(), val.begin(), val.end());
  };
  put32(hd, 20000630u);  // magic
  put32(hd, 2u);         // version 2, single-part scan-line file
  CHECK(channels == 1 || channels == 3) << "EXR output of 1 or 3 channels";
  static const char* names3[3] = {"B", "G", "R"};  // chlist order (alphabetical); B is interleaved channel 0
  {
    std::vector<uint8_t> v;
    for (int c = 0; c < channels; ++c) {
      putS(v, channels == 1 ? "Y" : names3[c]);
      put32(v, 2);  // FLOAT
      put32(v, 0);  // pLinear + reserved
      put32(v, 1);  // xSampling
      put32(v, 1);  // ySampling
    }
    v.push_back(0);
    attr("channels", "chlist", v);
  }
  attr("compression", "compression", {0});
  {
    std::vector<uint8_t> v;
    put32(v, 0);
    put32(v, 0);
    put32(v, (uint32_t)(w - 1));
    put32(v, (uint32_t)(h - 1));
    attr("dataWindow", "box2i", v);
    attr("displayWindow", "box2i", v);
  }
  attr("lineOrder", "lineOrder", {0});
  {
    std::vector<uint8_t> v;
    putF(v, 1.0f);
    attr("pixelAspectRatio", "float", v);
  }
  {
    std::vector<uint8_t> v;
    putF(v, 0.0f);
    putF(v, 0.0f);
    attr("screenWindowCenter", "v2f", v);
  }
  {
    std::vector<uint8_t> v;
    putF(v, 1.0f);
    attr("screenWindowWidth", "float", v);
  }
  hd.push_back(0);  // end of header
  f.write(reinterpret_cast<const char*>(hd.data()), (std::streamsize)hd.size());
  const uint64_t lineBytes = 8 + (uint64_t)w * 4 * channels;
  uint64_t ofs = hd.size() + (uint64_t)h * 8;
  for (int y = 0; y < h; ++y, ofs += lineBytes) {
    uint8_t b[8];
    for (int i = 0; i < 8; ++i) b[i] = (uint8_t)(ofs >> (8 * i));
    f.write(reinterpret_cast<const char*>(b), 8);
  }
  std::vector<float> row((size_t)w);
  for (int y = 0; y < h; ++y) {
    std::vector<uint8_t> l;
    put32(l, (uint32_t)y);
    put32(l, (uint32_t)(w * 4 * channels));
    f.write(reinterpret_cast<const char*>(l.data()), 8);
    for (int c = 0; c < channels; ++c) {
      for (int x = 0; x < w; ++x) row[x] = data[((size_t)y * w + x) * channels + c];
      f.write(reinterpret_cast<const char*>(row.data()), (std::streamsize)w * 4);
    }
  }
  CHECK(f.good()) << "failed to save image: " << path.string();
}
inline void writeExrFloat(const fs::path& path, const float* data, int w, int h) { writeExrFloatChannels(path, data, w, h, 1); }

// 16-bit PNG, `channels` = 1 (gray), 3 (BGR input, written as RGB) or 4 (BGRA input, written as RGBA)
inline void writePng16(const fs::path& path, const uint16_t* data, int w, int h, int channels) {
  std::ofstream f(path, std::ios::binary);
  CHECK(f.good()) << "failed to save image: " << path.string();
  static const uint8_t sig[8] = {0x89, 'P', 'N', 'G', 0x0D, 0x0A, 0x1A, 0x0A};
  f.write(reinterpret_cast<const char*>(sig), 8);
  std::vector<uint8_t> ihdr(13);
  ihdr[0] = w >> 24; ihdr[1] = w >> 16; ihdr[2] = w >> 8; ihdr[3] = w;
  ihdr[4] = h >> 24; ihdr[5] = h >> 16; ihdr[6] = h >> 8; ihdr[7] = h;
  ihdr[8] = 16;
  ihdr[9] = channels == 1 ? 0 : channels == 4 ? 6 : 2;  // grey, RGB from BGR, RGBA from BGRA
  pngChunk(f, "IHDR", ihdr);
  const size_t stride = (size_t)w * channels * 2;
  std::vector<uint8_t> raw((stride + 1) * h);
  for (int y = 0; y < h; ++y) {
    uint8_t* out = &raw[y * (stride + 1)];
    *out++ = 0;
    for (int x = 0; x < w; ++x)
      for (int c = 0; c < channels; ++c) {
        const int sc = channels >= 3 && c < 3 ? 2 - c : c;
        const uint16_t v = data[((size_t)y * w + x) * channels + sc];
        *out++ = (uint8_t)(v >> 8);
        *out++ = (uint8_t)v;
      }
  }
  uLongf clen = compressBound((uLong)raw.size());
  std::vector<uint8_t> comp(clen);
  CHECK(compress2(comp.data(), &clen, raw.data(), (uLong)raw.size(), 3) == Z_OK) << "PNG deflate failed";
  comp.resize(clen);
  pngChunk(f, "IDAT", comp);
  pngChunk(f, "IEND", {});
}

// ---- mesh_util::writePfm (MeshUtil.h:24-70): the "pfm" output of ConvertToBinary, the mesh rasterised back onto the depth
// grid.  Faces in order, the last one covering a pixel centre wins; a pixel is covered when its three barycentric
// coordinates are >= 0 ("ignore rasterization rules, just include all edges"); uncovered pixels stay -FLT_MAX.  The 2 x 2
// system of calcBarycentrics is solved by elimination with partial pivoting — the reference calls Eigen's
// colPivHouseholderQr, whose last-bit rounding decides coverage for pixel centres that lie exactly ON an edge or a vertex
// (which they do for an unsimplified mesh: its vertexes ARE the pixel centres); values agree to float rounding either way.
// vtx: x, y, z per vertex as written to .vtx (float32); width / height: the depth grid; resolution: the camera's.
inline std::vector<float> rasterMesh(const float* vtx, const uint32_t* idx, size_t numFaces, int width, int height,
                                     double resolutionX, double resolutionY) {
  std::vector<float> dst((size_t)width * height, -FLT_MAX);
  const double sx = width / resolutionX, sy = height / resolutionY;
  for (size_t f = 0; f < numFaces; ++f) {
    double t[3][3];
    for (int i = 0; i < 3; ++i) {
      const float* v = vtx + 3 * (size_t)idx[3 * f + i];
      t[i][0] = (double)v[0] * sx;
      t[i][1] = (double)v[1] * sy;
      t[i][2] = (double)v[2];
    }
    const double minX = std::min(std::min(t[0][0], t[1][0]), t[2][0]), maxX = std::max(std::max(t[0][0], t[1][0]), t[2][0]);
    const double minY = std::min(std::min(t[0][1], t[1][1]), t[2][1]), maxY = std::max(std::max(t[0][1], t[1][1]), t[2][1]);
    const double bx = t[2][0], by = t[2][1];
    // m^T of calcBarycentrics: columns are (row 0 - base) and (row 1 - base)
    const double a00 = t[0][0] - bx, a01 = t[1][0] - bx, a10 = t[0][1] - by, a11 = t[1][1] - by;
    for (int y = (int)std::floor(minY); y < std::ceil(maxY); ++y)
      for (int x = (int)std::floor(minX); x < std::ceil(maxX); ++x) {
        double A[2][3] = {{a00, a01, (x + 0.5) - bx}, {a10, a11, (y + 0.5) - by}};
        if (std::abs(A[1][0]) > std::abs(A[0][0]))
          for (int j = 0; j < 3; ++j) std::swap(A[0][j], A[1][j]);
        const double fct = A[1][0] / A[0][0];
        const double b1 = (A[1][2] - fct * A[0][2]) / (A[1][1] - fct * A[0][1]);
        const double b0 = (A[0][2] - A[0][1] * b1) / A[0][0];
        const double b2 = 1 - b0 - b1;
        if (b0 >= 0 && b1 >= 0 && b2 >= 0) {
          CHECK(0 <= x && x < width) << x << width;
          CHECK(0 <= y && y < height) << y << height;
          dst[(size_t)y * width + x] = (float)((t[0][2] * b0 + t[1][2] * b1) + t[2][2] * b2);
        }
      }
  }
  return dst;
}

// ---- cv_util::loadImage<T> semantics (CvUtil.h:171-284) -----------------------------------------------
inline Image loadUnchanged(const fs::path& path) {
  const std::string ext = path.extension().string();
  if (ext == ".pfm") {
    Image img;
    img.channels = 1;
    img.bits = 32;
    img.f = readPfm(path, &img.w, &img.h);
    return img;
  }
  CHECK(ext == ".png") << "only .png and .pfm inputs are supported by this build (got " << path.string() << ")";
  return readPng(path);
}

inline int cvRoundD(double v) { return (int)std::lrint(v); }

// cv_util::loadImage<cv::Vec4f>: integer samples * (1 / max), alpha 1 when the file has none
inline std::vector<float> loadColorF32x4(const fs::path& p, int* w, int* h) {
  const Image img = loadUnchanged(p);
  *w = img.w;
  *h = img.h;
  const size_t n = (size_t)img.w * img.h;
  std::vector<float> out(n * 4);
  const float scale = img.bits == 16 ? 1.0f / 65535.0f : 1.0f / 255.0f;
  for (size_t i = 0; i < n; ++i)
    for (int c = 0; c < 4; ++c) {
      float v = 1.0f;
      if (c < 3 || img.channels == 4) {
        const size_t idx = i * img.channels + (img.channels >= 3 ? c : 0);
        v = img.bits == 32 ? img.f[idx] : img.u[idx] * scale;
      }
      out[i * 4 + c] = v;
    }
  return out;
}

// image_util::verifyImagePaths: every camera has every frame of [first, last] (ext "" = the directory's first extension)
inline void verifyImagePaths(const std::string& dir, const Rig& rig, int first, int last, const std::string& ext) {
  for (const std::string& id : rig.ids)
    for (int f = first; f <= last; ++f) {
      const fs::path p = ext.empty() ? imagePath(dir, id, zeroPad(f)) : fs::path(dir) / id / (zeroPad(f) + ext);
      CHECK(fs::exists(p)) << "missing file: " << p.string();
    }
}

// loadImage<cv::Vec3w>: depth -> 16U (8U scaled by 65535/255 = 257, float by 65535 with rounding and
// saturation), then channels -> 3 (gray replicated, alpha dropped)
inline std::vector<uint16_t> loadColor16(const fs::path& path, int* w, int* h) {
  const Image img = loadUnchanged(path);
  *w = img.w;
  *h = img.h;
  const size_t n = (size_t)img.w * img.h;
  std::vector<uint16_t> out(n * 3);
  auto conv = [&](size_t idx) -> uint16_t {
    if (img.bits == 16) return img.u[idx];
    if (img.bits == 8) return (uint16_t)cvRoundD(img.u[idx] * (double)(65535.0f / 255.0f));
    const double v = (double)img.f[idx] * 65535.0;
    const int r = v != v ? 0 : cvRoundD(v);
    return (uint16_t)(r < 0 ? 0 : r > 65535 ? 65535 : r);
  };
  for (size_t i = 0; i < n; ++i)
    for (int c = 0; c < 3; ++c) {
      const int sc = img.channels >= 3 ? c : 0;
      out[i * 3 + c] = conv(i * img.channels + sc);
    }
  return out;
}

// loadImage<cv::Vec4b> followed by cv::cvtColor(BGRA2RGBA) (ConvertToBinary.cpp:138-146, the ".rgba" stream): depth -> 8U
// (16U scaled by the float 255/65535 with rounding and saturation, cv::Mat::convertTo), channels -> 4 (alpha 255 when
// the file has none, gray replicated), then B and R swapped.  Bytes R, G, B, A per pixel.
inline std::vector<uint8_t> loadRgba8(const fs::path& path, int* w, int* h) {
  const Image img = loadUnchanged(path);
  CHECK(img.bits == 8 || img.bits == 16) << "colour image expected: " << path.string();
  *w = img.w;
  *h = img.h;
  const size_t n = (size_t)img.w * img.h;
  const float a = 255.0f / 65535.0f;
  auto conv = [&](size_t idx) -> uint8_t {
    if (img.bits == 8) return (uint8_t)img.u[idx];
    const int r = (int)std::lrintf((float)img.u[idx] * a);  // saturate_cast<uchar>(src * alpha) in float
    return (uint8_t)(r > 255 ? 255 : r);
  };
  std::vector<uint8_t> out(n * 4);
  for (size_t i = 0; i < n; ++i) {
    const size_t at = i * img.channels;
    const uint8_t b = conv(at), g = img.channels >= 3 ? conv(at + 1) : b, r = img.channels >= 3 ? conv(at + 2) : b;
    out[i * 4 + 0] = r;
    out[i * 4 + 1] = g;
    out[i * 4 + 2] = b;
    out[i * 4 + 3] = img.channels == 4 ? conv(at + 3) : (img.channels == 2 ? conv(at + 1) : 255);
  }
  return out;
}

// cv_util::gaussianBlur(image, radius) = cv::GaussianBlur(image, (2 r + 1)^2, sigma 0) (CvUtil.h:302-312) on a 16-bit
// 3-channel image, radius 1..3: OpenCV's fixed-point path with its table kernels for sizes up to 7 — (1 2 1) / 4,
// (1 4 6 4 1) / 16, (2 7 14 18 14 7 2) / 64 — i.e. the integer-weighted sum, + half, shifted; BORDER_REFLECT_101 (pinned to
// cv2 in tests/test_apps.py).  GenerateForegroundMasks blurs with the library at every radius (derp_foreground_mask,
// derp_gaussian_blur); this host restatement stays as IoSelfTest --mode=gauss's reference for the table kernels.
inline std::vector<uint16_t> gaussianBlurU16C3(const std::vector<uint16_t>& src, int w, int h, int radius) {
  CHECK(radius >= 1 && radius <= 3) << "--blur_radius up to 3 (OpenCV's table kernels); got " << radius;
  static const int kernels[3][7] = {{1, 2, 1}, {1, 4, 6, 4, 1}, {2, 7, 14, 18, 14, 7, 2}};
  const int* k = kernels[radius - 1];
  const int n = 2 * radius + 1, shift = radius == 1 ? 2 : (radius == 2 ? 4 : 6);
  auto reflect = [](int i, int size) {
    if (size == 1) return 0;
    while (i < 0 || i >= size) i = i < 0 ? -i : 2 * (size - 1) - i;
    return i;
  };
  std::vector<uint32_t> rows((size_t)w * h * 3);  // horizontal pass, exact: <= 65535 * 64
  for (int y = 0; y < h; ++y)
    for (int x = 0; x < w; ++x)
      for (int c = 0; c < 3; ++c) {
        uint32_t s = 0;
        for (int i = 0; i < n; ++i) s += (uint32_t)k[i] * src[((size_t)y * w + reflect(x + i - radius, w)) * 3 + c];
        rows[((size_t)y * w + x) * 3 + c] = s;
      }
  std::vector<uint16_t> dst((size_t)w * h * 3);
  const uint64_t half = (uint64_t)1 << (2 * shift - 1);
  for (int y = 0; y < h; ++y)
    for (int x = 0; x < w; ++x)
      for (int c = 0; c < 3; ++c) {
        uint64_t s = 0;
        for (int j = 0; j < n; ++j) s += (uint64_t)k[j] * rows[((size_t)reflect(y + j - radius, h) * w + x) * 3 + c];
        dst[((size_t)y * w + x) * 3 + c] = (uint16_t)((s + half) >> (2 * shift));
      }
  return dst;
}

// cv_util::scaleImage's output size (CvUtil.h:150-153): std::round of the scaled extent
inline void scaledSize(int w, int h, double scale, int* dw, int* dh) {
  *dw = (int)std::round(w * scale);
  *dh = (int)std::round(h * scale);
}

// image_util::loadScaledImage<cv::Vec4b>(..., --color_scale, INTER_AREA) for the ".rgba" stream (ConvertToBinary.cpp:140-142):
// the 8-bit 4-channel image shrunk with cv::resize INTER_AREA (the channel order does not matter to a per-channel filter)
inline std::vector<uint8_t> scaleRgba8(const std::vector<uint8_t>& rgba, int* w, int* h, double scale) {
  int dw, dh;
  scaledSize(*w, *h, scale, &dw, &dh);
  CHECK(dw >= 1 && dh >= 1 && dw <= *w && dh <= *h) << "--color_scale must shrink the image";
  if (dw == *w && dh == *h) return rgba;
  std::vector<uint8_t> out((size_t)dw * dh * 4);
  area::resize(rgba.data(), *w, *h, 4, out.data(), dw, dh);
  *w = dw;
  *h = dh;
  return out;
}

// The RGBA8 surface bc7_util::compressBC7 hands to the block encoder when ConvertToBinary runs with --color_scale < 1
// (ConvertToBinary.cpp:127-137, BC7Util.h:45-67): the stored image -> [0, 1] floats (CvUtil.h:196-207; grey replicated, an
// alpha channel would be carried along and dropped later: skipped here) -> cv::resize INTER_AREA to the scaled size ->
// gammaCorrect per channel with the host's powf, exactly the reference's call -> R, G, B, 255.
inline std::vector<uint8_t> bc7SurfaceScaled(const Image& img, double scale, float gamma, int* outW, int* outH) {
  CHECK((img.bits == 8 || img.bits == 16) && (img.channels == 1 || img.channels == 3 || img.channels == 4))
      << "Conversion from " << img.channels << " channels to 4 channels not supported";  // CvUtil.h:261-262
  const size_t n = (size_t)img.w * img.h;
  const float toUnit = 1.0f / (img.bits == 16 ? 65535.0f : 255.0f);
  std::vector<float> bgr(n * 3);
  for (size_t i = 0; i < n; ++i)
    for (int c = 0; c < 3; ++c) bgr[i * 3 + c] = (float)img.u[i * img.channels + (img.channels == 1 ? 0 : c)] * toUnit;
  int dw, dh;
  scaledSize(img.w, img.h, scale, &dw, &dh);
  CHECK(dw >= 1 && dh >= 1 && dw <= img.w && dh <= img.h) << "--color_scale must shrink the image";
  std::vector<float> small;
  const float* px = bgr.data();
  if (dw != img.w || dh != img.h) {  // resizeImage returns the input when the size does not change
    small.resize((size_t)dw * dh * 3);
    area::resize(bgr.data(), img.w, img.h, 3, small.data(), dw, dh, /*simdAsFourChannels=*/true);  // the reference resizes BGRA
    px = small.data();
  }
  std::vector<uint8_t> rgba((size_t)dw * dh * 4);
  for (size_t i = 0; i < (size_t)dw * dh; ++i) {
    for (int c = 0; c < 3; ++c) rgba[i * 4 + c] = (uint8_t)(std::pow(px[i * 3 + 2 - c], gamma) * 255.0f + 0.5f);
    rgba[i * 4 + 3] = 255;
  }
  *outW = dw;
  *outH = dh;
  return rgba;
}

// loadImage<float>: .pfm as-is; integer images scaled by 1/max
inline std::vector<float> loadFloat(const fs::path& path, int* w, int* h) {
  const Image img = loadUnchanged(path);
  *w = img.w;
  *h = img.h;
  const size_t n = (size_t)img.w * img.h;
  if (img.bits == 32) return img.f;
  std::vector<float> out(n);
  const float scale = 1.0f / (img.bits == 16 ? 65535.0f : 255.0f);
  for (size_t i = 0; i < n; ++i) {
    if (img.channels >= 3) {  // BGR2GRAY
      const float b = img.u[i * img.channels] * scale, g = img.u[i * img.channels + 1] * scale,
                  r = img.u[i * img.channels + 2] * scale;
      out[i] = 0.114f * b + 0.587f * g + 0.299f * r;
    } else {
      out[i] = img.u[i * img.channels] * scale;
    }
  }
  return out;
}

// loadImage<bool>: depth -> 8U, threshold > 127 -> 1 (CvUtil.h:236-239), first channel / gray
inline std::vector<uint8_t> loadMask(const fs::path& path, int* w, int* h) {
  const Image img = loadUnchanged(path);
  *w = img.w;
  *h = img.h;
  const size_t n = (size_t)img.w * img.h;
  std::vector<uint8_t> out(n);
  for (size_t i = 0; i < n; ++i) {
    int v8;
    if (img.bits == 32) {
      const double v = (double)img.f[i] * 255.0;
      v8 = std::min(255, std::max(0, v != v ? 0 : cvRoundD(v)));
    } else {
      int v;
      if (img.channels >= 3) {
        const int b = img.u[i * img.channels], g = img.u[i * img.channels + 1], r = img.u[i * img.channels + 2];
        v = (int)std::lrint(0.114 * b + 0.587 * g + 0.299 * r);
      } else {
        v = img.u[i * img.channels];
      }
      v8 = img.bits == 16 ? std::min(255, cvRoundD(v * (double)(255.0f / 65535.0f))) : v;
    }
    out[i] = v8 > 127 ? 1 : 0;
  }
  return out;
}

// cv_util::convertTo<uint16_t>(disparity) for the png outputs: clamp(d,0,1)*65535, NaN -> 0
inline std::vector<uint16_t> disparityTo16(const float* d, size_t n) {
  std::vector<uint16_t> out(n);
  for (size_t i = 0; i < n; ++i) {
    const float v = d[i] * 65535.0f;
    const int r = v != v ? 0 : (v >= 2147483648.0f ? 65535 : (v <= -2147483648.0f ? 0 : (int)std::lrintf(v)));
    out[i] = (uint16_t)(r < 0 ? 0 : r > 65535 ? 65535 : r);
  }
  return out;
}

// output_formats handling shared by the three apps (pfm always for DerpCLI/TemporalBilateralFilter)
inline void saveDisparity(const fs::path& stem, const std::string& ext, const float* d, int w, int h) {
  fs::create_directories(stem.parent_path());
  if (ext == "pfm") {
    writePfm(stem.string() + ".pfm", d, w, h);
  } else if (ext == "png") {
    const auto v = disparityTo16(d, (size_t)w * h);
    writePng16(stem.string() + ".png", v.data(), w, h, 1);
  } else if (ext == "exr") {
    writeExrFloat(stem.string() + ".exr", d, w, h);
  } else {
    LOG(FATAL) << "Invalid type: " << ext;
  }
}

}  // namespace io
