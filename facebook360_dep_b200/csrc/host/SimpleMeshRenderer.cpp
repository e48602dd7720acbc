// SimpleMeshRenderer — drop-in for source/render/SimpleMeshRenderer.cpp's file output without OpenGL.
// Renders the rig's disparity (and colour) canopies from --position in one of nine formats and writes one image per
// frame.  Rendering runs in libderp_b200.so (derp_canopy_render, csrc/derp_rephoto.cuh) under documented
// rasterisation, filtering and resampling rules instead of a GL driver's; the background compositing, layouts and file
// conversion are the reference's host code (smr_host.h).  INTEGRATION.md lists what differs from a GL run; the
// on-screen viewer (an empty --format) and the jpg / tif writers are not available.
#include "../../../include/derp_canopy.h"
#include "io.h"
#include "smr_host.h"

#include <array>
#include <set>

const std::string kUsage = R"(
  - Reads a set of disparity (and optionally color) images for a rig and renders a fused version.
  It outputs images in a specified format (on-screen rendering is not available in this build).

  - Example:
    ./SimpleMeshRenderer \
    --first=000000 \
    --last=000000 \
    --rig=/path/to/rigs/rig.json \
    --color=/path/to/video/color \
    --disparity=/path/to/output/disparity \
    --output=/path/to/output/meshes \
    --format=cubecolor
)";

DEFINE_string(cameras, "", "comma-separated cameras to render (empty for all)");
DEFINE_string(color, "", "path to input color images (required)");
DEFINE_string(disparity, "", "path to disparity images (required)");
DEFINE_string(background, "", "path to optional background image");
DEFINE_string(background_equirect, "", "path to optional background equirect image");
DEFINE_string(file_type, "png", "Supports any image type allowed in OpenCV");
DEFINE_string(first, "000000", "first frame to process (lexical)");
DEFINE_string(forward, "-1.0 0.0 0.0", "forward for rendering");
DEFINE_int32(height, -1, "height of the rendering (pixels), default is width / 2");
DEFINE_double(horizontal_fov, 90, "horizontal field of view for rendering (degrees)");
DEFINE_bool(ignore_alpha_blend, false, "ignore alpha blend (useful if rendering single camera)");
DEFINE_string(last, "000000", "last frame to process (lexical) (ignored if on-screen rendering)");
DEFINE_string(output, "", "path to output directory");
DEFINE_string(position, "0.0 0.0 0.0", "position to render from (m)");
DEFINE_string(rig, "", "path to camera rig .json (required)");
DEFINE_string(up, "0.0 0.0 1.0", "up for rendering");
DEFINE_int32(width, 3072, "width of the rendering (pixels)");
DEFINE_string(format, "", "cubecolor, cubedisp, eqrcolor, eqrdisp, lr180, snapcolor, snapdisp, tb3dof, tbstereo (empty = on-screen rendering)");
DEFINE_int32(gpu, 0, "CUDA device to use");

#define DERP_CALL(expr)                                                    \
  do {                                                                     \
    const int rc_ = (expr);                                                \
    if (rc_ != 0) LOG(FATAL) << #expr << " failed: " << derp_last_error(); \
  } while (0)

namespace {

const std::set<std::string> kFormats = {"cubecolor", "cubedisp", "eqrcolor", "eqrdisp", "lr180",
                                        "snapcolor", "snapdisp", "tb3dof",   "tbstereo"};

void verifyInputs(const io::Rig& rig) {
  CHECK_NE(FLAGS_disparity, "");
  CHECK_NE(FLAGS_first, "");
  if (!FLAGS_format.empty()) CHECK_NE(FLAGS_last, "");
  const int first = std::stoi(FLAGS_first), last = std::stoi(FLAGS_last);
  io::verifyImagePaths(FLAGS_disparity, rig, first, last, ".pfm");
  if (!FLAGS_color.empty()) io::verifyImagePaths(FLAGS_color, rig, first, last, "");
  CHECK_GT(FLAGS_width, 0);
  CHECK_EQ(FLAGS_width % 2, 0) << "width must be a multiple of 2";
  if (FLAGS_height == -1) FLAGS_height = FLAGS_width / 2;
  if (!FLAGS_format.empty()) CHECK(kFormats.count(FLAGS_format)) << "Invalid format: " << FLAGS_format;
  static const std::set<std::string> kAllColor = {"eqrcolor", "cubecolor", "tbstereo", "lr180", "snapcolor"};
  if (kAllColor.count(FLAGS_format)) CHECK_NE(FLAGS_color, "") << FLAGS_format << " needs --color to be set";
}

std::array<float, 3> decodeVector(const std::string& flag) {
  std::array<float, 3> r;
  std::istringstream s(flag);
  s >> r[0] >> r[1] >> r[2];
  CHECK(s) << "Unexpected flag " << flag;
  return r;
}

struct Image {
  std::vector<float> px;  // B, G, R, A
  int w = 0, h = 0;
};

// The rig's canopies, loaded once per frame
struct Frame {
  std::vector<DerpCameraDesc> cams;
  std::vector<std::vector<float>> disps, colors;
  int dw = 0, dh = 0, cw = 0, ch = 0;
};

Image render(const Frame& fr, bool disparity, int projection, int outW, int outH, float ipd, const float* matrix) {
  const std::array<float, 3> position = decodeVector(FLAGS_position);
  std::vector<const float*> dp, cp;
  for (const auto& d : fr.disps) dp.push_back(d.data());
  for (const auto& c : fr.colors) cp.push_back(c.data());
  Image img;
  img.w = projection == DERP_CANOPY_EQUIRECT ? 2 * outH : outW;
  img.h = projection == DERP_CANOPY_CUBEMAP ? 6 * outH : outH;
  img.px.resize((size_t)img.w * img.h * 4);
  DERP_CALL(derp_canopy_render(FLAGS_gpu, fr.cams.data(), (int)fr.cams.size(), dp.data(), fr.dw, fr.dh, cp.data(), fr.cw,
                               fr.ch, projection, position.data(), matrix, outW, outH, ipd, !FLAGS_ignore_alpha_blend,
                               DERP_CANOPY_SVD, disparity ? nullptr : img.px.data(), disparity ? img.px.data() : nullptr,
                               nullptr));
  return img;
}

Image equirect(const Frame& fr, bool disparity, float ipd) {
  return render(fr, disparity, DERP_CANOPY_EQUIRECT, 2 * FLAGS_height, FLAGS_height, ipd, nullptr);
}

Image loadImage(const std::string& path) {
  Image img;
  img.px = io::loadColorF32x4(path, &img.w, &img.h);
  return img;
}

// SimpleMeshWindow::generate: --background by alphaBlend, then --background_equirect
Image generate(Image fore) {
  if (!FLAGS_background.empty()) {
    const Image back = loadImage(FLAGS_background);
    CHECK_EQ(fore.h, back.h);
    CHECK_EQ(fore.w, back.w);
    smr::alphaBlend(fore.px.data(), back.px.data(), (size_t)fore.w * fore.h);
  }
  if (!FLAGS_background_equirect.empty()) {
    const Image equi = loadImage(FLAGS_background_equirect);
    const std::array<float, 3> position = decodeVector(FLAGS_position), forward = decodeVector(FLAGS_forward),
                               up = decodeVector(FLAGS_up);
    float R[9];
    CHECK(smr::forwardUp(forward.data(), up.data(), R)) << FLAGS_forward << "/" << FLAGS_up << " not unitary";
    smr::backgroundEquirect(fore.px.data(), fore.w, fore.h, equi.px.data(), equi.w, equi.h, R, position.data(),
                            FLAGS_horizontal_fov);
  }
  return fore;
}

Image snapshot(const Frame& fr, bool disparity) {
  const std::array<float, 3> position = decodeVector(FLAGS_position), forward = decodeVector(FLAGS_forward),
                             up = decodeVector(FLAGS_up);
  float M[16];
  DERP_CALL(derp_canopy_snapshot_matrix(position.data(), forward.data(), up.data(), FLAGS_horizontal_fov, FLAGS_width,
                                        FLAGS_height, M));
  return render(fr, disparity, DERP_CANOPY_PERSPECTIVE, FLAGS_width, FLAGS_height, 0.0f, M);
}

Image stack(const Image& top, const Image& bottom) {
  Image r;
  r.w = top.w;
  r.h = top.h + bottom.h;
  r.px = smr::stackVertical(top.px, bottom.px);
  return r;
}

void save(const fs::path& path, const Image& img) {
  fs::create_directories(path.parent_path());
  const size_t n = (size_t)img.w * img.h;
  if (FLAGS_file_type == "exr") {  // convertImage<cv::Vec3f>: the B, G, R channels as they are
    std::vector<float> bgr(n * 3);
    for (size_t i = 0; i < n; ++i)
      for (int c = 0; c < 3; ++c) bgr[3 * i + c] = img.px[4 * i + c];
    io::writeExrFloatChannels(path, bgr.data(), img.w, img.h, 3);
  } else {
    const std::vector<uint16_t> v = smr::toPng16(img.px.data(), n);
    io::writePng16(path, v.data(), img.w, img.h, 3);
  }
}

}  // namespace

int main(int argc, char** argv) {
  flags::initDep(argc, argv, kUsage);
  CHECK_NE(FLAGS_rig, "");
  const io::Rig full = io::loadRig(FLAGS_rig);
  io::Rig rig;
  for (int i : io::filterDestinations(full, FLAGS_cameras)) {
    rig.cams.push_back(full.cams[i]);
    rig.ids.push_back(full.ids[i]);
  }
  CHECK_GT(rig.cams.size(), 0u);
  verifyInputs(rig);
  CHECK(!FLAGS_format.empty()) << "on-screen rendering (an empty --format) is not available in this build; choose one of "
                                  "cubecolor, cubedisp, eqrcolor, eqrdisp, lr180, snapcolor, snapdisp, tb3dof, tbstereo";
  CHECK(FLAGS_file_type == "png" || FLAGS_file_type == "exr")
      << "unsupported --file_type " << FLAGS_file_type << ": this build writes png and exr";
  LOG(INFO) << "backend " << derp_backend();

  const int first = std::stoi(FLAGS_first), last = std::stoi(FLAGS_last);
  for (int iFrame = first; iFrame <= last; ++iFrame) {
    const std::string frameName = io::zeroPad(iFrame);
    LOG(INFO) << "Processing frame " << frameName << "...";
    Frame fr;
    fr.cams = rig.cams;
    for (size_t i = 0; i < rig.ids.size(); ++i) {
      int w, h;
      fr.disps.push_back(io::readPfm(fs::path(FLAGS_disparity) / rig.ids[i] / (frameName + ".pfm"), &w, &h));
      if (i == 0) {
        fr.dw = w;
        fr.dh = h;
      }
      CHECK(w == fr.dw && h == fr.dh) << "disparity maps of one frame must share a size";
    }
    for (size_t i = 0; i < rig.ids.size(); ++i) {
      int w = fr.dw, h = fr.dh;
      if (FLAGS_color.empty()) {  // loadColors' dummy images
        fr.colors.emplace_back((size_t)w * h * 4, 0.0f);
      } else {
        fr.colors.push_back(io::loadColorF32x4(io::imagePath(FLAGS_color, rig.ids[i], frameName), &w, &h));
      }
      if (i == 0) {
        fr.cw = w;
        fr.ch = h;
      }
      CHECK(w == fr.cw && h == fr.ch) << "color images of one frame must share a size";
    }
    const std::string& f = FLAGS_format;
    const float halfIpdM = 0.032f;  // left = halfIpdM, right = -halfIpdM
    Image out;
    if (f == "eqrcolor" || f == "eqrdisp") {
      out = generate(equirect(fr, f == "eqrdisp", 0.0f));
    } else if (f == "cubecolor" || f == "cubedisp") {
      out = generate(render(fr, f == "cubedisp", DERP_CANOPY_CUBEMAP, FLAGS_height, FLAGS_height, 0.0f, nullptr));
    } else if (f == "tbstereo" || f == "lr180") {
      const Image left = generate(equirect(fr, false, halfIpdM)), right = generate(equirect(fr, false, -halfIpdM));
      Image st;
      if (f == "tbstereo") {
        st = stack(left, right);
      } else {
        st.w = 2 * (left.w / 2);
        st.h = left.h;
        st.px = smr::lr180(left.px, right.px, left.w, left.h);
      }
      out = generate(st);
    } else if (f == "tb3dof") {
      out = generate(stack(generate(equirect(fr, false, 0.0f)), generate(equirect(fr, true, 0.0f))));
    } else {
      out = generate(snapshot(fr, f == "snapdisp"));
    }
    const fs::path filename = fs::path(FLAGS_output) / (frameName + "." + FLAGS_file_type);
    save(filename, out);
    LOG(INFO) << "File saved in " << filename;
  }
  return EXIT_SUCCESS;
}
