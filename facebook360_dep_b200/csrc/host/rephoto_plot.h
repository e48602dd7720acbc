// Plot of ComputeRephotographyErrors (rephoto_util::stackResults, RephotographyUtil.h:130-181): five panels side by side
// — reference colour, reference disparity, rendered colour and rendered disparity (both black outside the mask), and
// the score as a JET heat map — each the 6 * edge x edge stacked cubemap.  The cv::putText overlay of the averages is
// not drawn: the log line carries the numbers.  Host code shared by the app and the CPU checker (tests/rephoto_oracle.cpp), pinned to cv2 by
// tests/golden/rephoto_vectors.npz.
#pragma once

#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

namespace rephoto_plot {

// cv::applyColorMap(COLORMAP_JET) of the gray levels 0..255, B, G, R (cv2 4.13)
static const uint8_t kJet[256][3] = {
    {128, 0, 0}, {132, 0, 0}, {136, 0, 0}, {140, 0, 0}, {144, 0, 0}, {148, 0, 0}, {152, 0, 0}, {156, 0, 0},
    {160, 0, 0}, {164, 0, 0}, {168, 0, 0}, {172, 0, 0}, {176, 0, 0}, {180, 0, 0}, {184, 0, 0}, {188, 0, 0},
    {192, 0, 0}, {196, 0, 0}, {200, 0, 0}, {204, 0, 0}, {208, 0, 0}, {212, 0, 0}, {216, 0, 0}, {220, 0, 0},
    {224, 0, 0}, {228, 0, 0}, {232, 0, 0}, {236, 0, 0}, {240, 0, 0}, {244, 0, 0}, {248, 0, 0}, {252, 0, 0},
    {255, 0, 0}, {255, 4, 0}, {255, 8, 0}, {255, 12, 0}, {255, 16, 0}, {255, 20, 0}, {255, 24, 0}, {255, 28, 0},
    {255, 32, 0}, {255, 36, 0}, {255, 40, 0}, {255, 44, 0}, {255, 48, 0}, {255, 52, 0}, {255, 56, 0}, {255, 60, 0},
    {255, 64, 0}, {255, 68, 0}, {255, 72, 0}, {255, 76, 0}, {255, 80, 0}, {255, 84, 0}, {255, 88, 0}, {255, 92, 0},
    {255, 96, 0}, {255, 100, 0}, {255, 104, 0}, {255, 108, 0}, {255, 112, 0}, {255, 116, 0}, {255, 120, 0}, {255, 124, 0},
    {255, 128, 0}, {255, 132, 0}, {255, 136, 0}, {255, 140, 0}, {255, 144, 0}, {255, 148, 0}, {255, 152, 0}, {255, 156, 0},
    {255, 160, 0}, {255, 164, 0}, {255, 168, 0}, {255, 172, 0}, {255, 176, 0}, {255, 180, 0}, {255, 184, 0}, {255, 188, 0},
    {255, 192, 0}, {255, 196, 0}, {255, 200, 0}, {255, 204, 0}, {255, 208, 0}, {255, 212, 0}, {255, 216, 0}, {255, 220, 0},
    {255, 224, 0}, {255, 228, 0}, {255, 232, 0}, {255, 236, 0}, {255, 240, 0}, {255, 244, 0}, {255, 248, 0}, {255, 252, 0},
    {254, 255, 2}, {250, 255, 6}, {246, 255, 10}, {242, 255, 14}, {238, 255, 18}, {234, 255, 22}, {230, 255, 26}, {226, 255, 30},
    {222, 255, 34}, {218, 255, 38}, {214, 255, 42}, {210, 255, 46}, {206, 255, 50}, {202, 255, 54}, {198, 255, 58}, {194, 255, 62},
    {190, 255, 66}, {186, 255, 70}, {182, 255, 74}, {178, 255, 78}, {174, 255, 82}, {170, 255, 86}, {166, 255, 90}, {162, 255, 94},
    {158, 255, 98}, {154, 255, 102}, {150, 255, 106}, {146, 255, 110}, {142, 255, 114}, {138, 255, 118}, {134, 255, 122}, {130, 255, 126},
    {126, 255, 130}, {122, 255, 134}, {118, 255, 138}, {114, 255, 142}, {110, 255, 146}, {106, 255, 150}, {102, 255, 154}, {98, 255, 158},
    {94, 255, 162}, {90, 255, 166}, {86, 255, 170}, {82, 255, 174}, {78, 255, 178}, {74, 255, 182}, {70, 255, 186}, {66, 255, 190},
    {62, 255, 194}, {58, 255, 198}, {54, 255, 202}, {50, 255, 206}, {46, 255, 210}, {42, 255, 214}, {38, 255, 218}, {34, 255, 222},
    {30, 255, 226}, {26, 255, 230}, {22, 255, 234}, {18, 255, 238}, {14, 255, 242}, {10, 255, 246}, {6, 255, 250}, {1, 255, 254},
    {0, 252, 255}, {0, 248, 255}, {0, 244, 255}, {0, 240, 255}, {0, 236, 255}, {0, 232, 255}, {0, 228, 255}, {0, 224, 255},
    {0, 220, 255}, {0, 216, 255}, {0, 212, 255}, {0, 208, 255}, {0, 204, 255}, {0, 200, 255}, {0, 196, 255}, {0, 192, 255},
    {0, 188, 255}, {0, 184, 255}, {0, 180, 255}, {0, 176, 255}, {0, 172, 255}, {0, 168, 255}, {0, 164, 255}, {0, 160, 255},
    {0, 156, 255}, {0, 152, 255}, {0, 148, 255}, {0, 144, 255}, {0, 140, 255}, {0, 136, 255}, {0, 132, 255}, {0, 128, 255},
    {0, 124, 255}, {0, 120, 255}, {0, 116, 255}, {0, 112, 255}, {0, 108, 255}, {0, 104, 255}, {0, 100, 255}, {0, 96, 255},
    {0, 92, 255}, {0, 88, 255}, {0, 84, 255}, {0, 80, 255}, {0, 76, 255}, {0, 72, 255}, {0, 68, 255}, {0, 64, 255},
    {0, 60, 255}, {0, 56, 255}, {0, 52, 255}, {0, 48, 255}, {0, 44, 255}, {0, 40, 255}, {0, 36, 255}, {0, 32, 255},
    {0, 28, 255}, {0, 24, 255}, {0, 20, 255}, {0, 16, 255}, {0, 12, 255}, {0, 8, 255}, {0, 4, 255}, {0, 0, 255},
    {0, 0, 252}, {0, 0, 248}, {0, 0, 244}, {0, 0, 240}, {0, 0, 236}, {0, 0, 232}, {0, 0, 228}, {0, 0, 224},
    {0, 0, 220}, {0, 0, 216}, {0, 0, 212}, {0, 0, 208}, {0, 0, 204}, {0, 0, 200}, {0, 0, 196}, {0, 0, 192},
    {0, 0, 188}, {0, 0, 184}, {0, 0, 180}, {0, 0, 176}, {0, 0, 172}, {0, 0, 168}, {0, 0, 164}, {0, 0, 160},
    {0, 0, 156}, {0, 0, 152}, {0, 0, 148}, {0, 0, 144}, {0, 0, 140}, {0, 0, 136}, {0, 0, 132}, {0, 0, 128},
};

// cv::Mat::convertTo(CV_8U, 255): saturate_cast<uchar>(cvRound(v * 255)); NaN and values outside the int range -> 0
inline uint8_t toU8(float v) {
  const float s = v * 255.0f;
  if (!(s > -2147483648.0f && s < 2147483648.0f)) return 0;
  const long r = std::lrintf(s);
  return (uint8_t)(r < 0 ? 0 : r > 255 ? 255 : r);
}

// cv::cvtColor(BGR2GRAY) of 8-bit pixels: the fixed-point weights of OpenCV's integer path
inline uint8_t gray(uint8_t b, uint8_t g, uint8_t r) { return (uint8_t)((b * 3735 + g * 19235 + r * 9798 + 16384) >> 15); }

// 255 - convertImage<Vec3b>(score), applyColorMap(JET) (which takes the gray level of a 3-channel input), zero outside
// the mask.  score: float B, G, R [h][w]; out: B, G, R bytes [h][w]
inline void jetPanel(const float* score, const uint8_t* mask, int w, int h, uint8_t* out) {
  for (size_t i = 0; i < (size_t)w * h; ++i) {
    const uint8_t b = 255 - toU8(score[3 * i]), g = 255 - toU8(score[3 * i + 1]), r = 255 - toU8(score[3 * i + 2]);
    const uint8_t* c = kJet[gray(b, g, r)];
    for (int k = 0; k < 3; ++k) out[3 * i + k] = mask[i] ? c[k] : 0;
  }
}

// The whole plot, B, G, R bytes [h][5 * w].  The cubemaps are float B, G, R, A [h][w]; mask non-zero where scored.
inline std::vector<uint8_t> stackResults(const float* refColor, const float* refDisp, const float* renColor,
                                         const float* renDisp, const float* score, const uint8_t* mask, int w, int h) {
  std::vector<uint8_t> jet((size_t)w * h * 3), plot((size_t)w * h * 15);
  jetPanel(score, mask, w, h, jet.data());
  const float* panels[4] = {refColor, refDisp, renColor, renDisp};
  for (int y = 0; y < h; ++y)
    for (int x = 0; x < w; ++x) {
      const size_t i = (size_t)y * w + x;
      for (int p = 0; p < 5; ++p) {
        uint8_t* o = &plot[((size_t)y * 5 * w + (size_t)p * w + x) * 3];
        for (int k = 0; k < 3; ++k) {
          if (p == 4) o[k] = jet[3 * i + k];
          else o[k] = (p >= 2 && !mask[i]) ? 0 : toU8(panels[p][4 * i + k]);
        }
      }
    }
  return plot;
}

}  // namespace rephoto_plot
