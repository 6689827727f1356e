// rpg_svo_b200/host/host_klt_demo.cpp -- the two-view initialisation's per-frame work through the C++ host mirror:
// svo::initialization::detectFeatures on frame 0, then trackKlt of frames 1..3 against it (KltHomographyInit::addFirstFrame
// / addSecondFrame keep px_ref, px_cur and f_ref across frames).  Prints the tracked count and the median disparity of
// every frame, and every kept point ("pt frame index px_ref px_cur f_cur disparity", index = position in the detection).
// usage: host_klt_demo [pinhole|atan]
// The frames (752 x 480): frame k = a 7 x 7 box blur of an integer hash texture shifted by (3k, 2k) px, contrast stretched
// (tests/klt_host_scene.py builds the same bytes).
#include <cstdio>
#include <cstring>

#include "svo_host.h"

static std::vector<uint8_t> frame_image(int k, int W, int H) {
  auto base = [](int x, int y) { return (((uint32_t)x * 73856093u) ^ ((uint32_t)y * 19349663u)) >> 8 & 255u; };
  std::vector<uint8_t> img((size_t)W * H);
  for (int y = 0; y < H; ++y)
    for (int x = 0; x < W; ++x) {
      uint32_t s = 0;
      for (int j = -3; j <= 3; ++j)
        for (int i = -3; i <= 3; ++i) s += base(x + i + 3 * k, y + j + 2 * k);
      const uint32_t v = std::min(std::max(s / 49, 100u), 155u) - 100u;  // contrast stretched from [100, 155] to [0, 255]
      img[(size_t)y * W + x] = (uint8_t)(v * 255u / 55u);
    }
  return img;
}

int main(int argc, char** argv) {
  const int W = 752, H = 480, n_frames = 4, n_levels = 5;
  const bool atan = argc > 1 && std::strcmp(argv[1], "atan") == 0;
  try {
    svo::Context ctx(0);
    svo::PinholeCamera pinhole(W, H, 315.5, 315.5, 376.0, 240.0);
    svo::ATANCamera atan_cam(W, H, 0.509326, 0.796651, 0.45905, 0.510056, 0.9320);
    svo::AbstractCamera* cam = atan ? static_cast<svo::AbstractCamera*>(&atan_cam) : &pinhole;
    std::vector<uint8_t> img0 = frame_image(0, W, H);
    svo::FramePtr ref(new svo::Frame(ctx, cam, img0.data(), n_levels, 0.0));
    std::vector<svo::Point2f> px_ref, px_cur;
    std::vector<svo::Vector3d> f_ref, f_cur;
    std::vector<double> disparities;
    svo::initialization::detectFeatures(ref, px_ref, f_ref);
    px_cur = px_ref;  // addFirstFrame: the initial flow is the reference position
    std::vector<int> index(px_ref.size());
    for (size_t i = 0; i < index.size(); ++i) index[i] = (int)i;
    std::printf("detected %zu corners\n", px_ref.size());
    for (int k = 1; k < n_frames; ++k) {
      std::vector<uint8_t> img = frame_image(k, W, H);
      svo::FramePtr cur(new svo::Frame(ctx, cam, img.data(), n_levels, 0.0));
      const std::vector<svo::Point2f> before = px_ref;
      svo::initialization::trackKlt(ref, cur, px_ref, px_cur, f_ref, f_cur, disparities);
      // the detection index of every kept point: px_ref keeps its values, so match them in order
      std::vector<int> kept;
      for (size_t i = 0, j = 0; i < before.size() && j < px_ref.size(); ++i)
        if (before[i].x == px_ref[j].x && before[i].y == px_ref[j].y) { kept.push_back(index[i]); ++j; }
      index = kept;
      if (index.size() != px_ref.size() || f_ref.size() != px_ref.size() || f_cur.size() != px_ref.size()) {
        std::fprintf(stderr, "inconsistent sizes after trackKlt\n");
        return 1;
      }
      std::vector<double> d = disparities;
      double median = 0;
      if (!d.empty()) {
        std::nth_element(d.begin(), d.begin() + d.size() / 2, d.end());
        median = d[d.size() / 2];
      }
      std::printf("frame %d tracked %zu median_disparity %.4f\n", k, px_ref.size(), median);
      for (size_t i = 0; i < px_ref.size(); ++i)
        std::printf("pt %d %d %.9g %.9g %.9g %.9g %.17g %.17g %.17g %.17g\n", k, index[i], px_ref[i].x, px_ref[i].y, px_cur[i].x,
                    px_cur[i].y, f_cur[i][0], f_cur[i][1], f_cur[i][2], disparities[i]);
    }
  } catch (const std::exception& e) {
    std::fprintf(stderr, "host_klt_demo: %s\n", e.what());
    return 1;
  }
  return 0;
}
