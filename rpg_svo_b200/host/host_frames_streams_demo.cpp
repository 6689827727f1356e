// rpg_svo_b200/host/host_frames_streams_demo.cpp -- the new frames of several camera streams through svo_host.h, twice:
// once with one `new svo::Frame(ctx, cam, img, n_levels, ts)` per stream, once with one svo::streams::newFrames call (one
// batched upload, one launch per pyramid stage).  The streams mix five image sizes, widths that are and are not multiples of
// 16, and pinhole and ATAN cameras; the batches run with 5 and with 2 levels under both pyramid rules.  Prints a digest of
// every level and every tiled copy of every frame from both paths; the two must be equal.  Then checks that the refusals
// throw before any frame is created.
//   usage: host_frames_streams_demo
#include <cinttypes>
#include <cstdio>
#include <memory>
#include <vector>

#include "svo_host.h"

namespace {

std::vector<uint8_t> image(int s, int W, int H) {
  std::vector<uint8_t> img((size_t)W * H);
  for (int y = 0; y < H; ++y)
    for (int x = 0; x < W; ++x) img[(size_t)y * W + x] = (uint8_t)((((uint32_t)(x + 31 * s) * 73856093u) ^ ((uint32_t)y * 19349663u)) >> 11);
  return img;
}

uint64_t digest(svo::Context& ctx, const svo::FramePtr& f) {
  uint64_t h = 1469598103934665603ULL;
  auto add = [&](const std::vector<uint8_t>& b) {
    for (uint8_t v : b) { h ^= v; h *= 1099511628211ULL; }
  };
  for (const svo::Image& im : f->img_pyr_) {
    std::vector<uint8_t> lv((size_t)im.cols * im.rows), tl((size_t)((im.cols + 3) / 4) * ((im.rows + 3) / 4) * 16);
    ctx.check(svo_b200_frame_download_level(ctx.get(), f->device(), im.level, lv.data()));
    ctx.check(svo_b200_frame_download_level_tiled(ctx.get(), f->device(), im.level, tl.data()));
    add(lv);
    add(tl);
  }
  return h;
}

}  // namespace

int main() {
  try {
    svo::Context ctx(0);
    svo::PinholeCamera pin752{752, 480, 315.5, 315.5, 376.0, 240.0}, pin640{640, 480, 320.0, 320.0, 320.0, 240.0},
        pin644{644, 484, 320.0, 320.0, 322.0, 242.0}, pin96{96, 48, 50.0, 50.0, 48.0, 24.0}, pin17{17, 9, 10.0, 10.0, 8.5, 4.5};
    svo::ATANCamera atan752{752, 480, 0.509326, 0.796651, 0.45905, 0.510056, 0.9320};
    const std::vector<svo::AbstractCamera*> deep = {&pin752, &pin640, &pin644, &atan752, &pin640}, shallow = {&pin96, &pin17, &pin752};
    bool ok = true;
    int n = 0, equal = 0;
    for (int rule : {SVO_B200_PYR_X86, SVO_B200_PYR_SCALAR}) {
      ctx.check(svo_b200_set_pyramid_rule(ctx.get(), rule));
      for (int n_levels : {5, 2}) {
        const std::vector<svo::AbstractCamera*>& cams = n_levels == 5 ? deep : shallow;
        std::vector<std::vector<uint8_t>> imgs;
        std::vector<const uint8_t*> ptrs;
        for (size_t s = 0; s < cams.size(); ++s) imgs.push_back(image((int)s + 7 * n_levels + rule, cams[s]->width(), cams[s]->height()));
        for (const auto& im : imgs) ptrs.push_back(im.data());
        std::vector<svo::FramePtr> batched = svo::streams::newFrames(ctx, cams, ptrs, n_levels, std::vector<double>(cams.size(), 0.5));
        for (size_t s = 0; s < cams.size(); ++s) {
          svo::FramePtr single(new svo::Frame(ctx, cams[s], ptrs[s], n_levels, 0.5));
          const uint64_t a = digest(ctx, single), b = digest(ctx, batched[s]);
          std::printf("rule %d levels %d frame %zu %dx%d constructor %016" PRIx64 " batched %016" PRIx64 "\n", rule, n_levels, s,
                      cams[s]->width(), cams[s]->height(), a, b);
          ++n;
          equal += a == b;
        }
      }
    }
    std::printf("frames %d equal %d\n", n, equal);
    ok = ok && n > 0 && equal == n;

    // refusals: each throws before any frame is created (a created frame would show as a device allocation)
    const std::vector<uint8_t> img = image(0, 752, 480);
    int thrown = 0, tried = 0;
    auto attempt = [&](const char* name, const std::vector<svo::AbstractCamera*>& cams, const std::vector<const uint8_t*>& ptrs,
                       const std::vector<double>& ts, bool runtime) {
      ++tried;
      try {
        svo::streams::newFrames(ctx, cams, ptrs, 5, ts);
      } catch (const std::invalid_argument&) {
        thrown += !runtime;
        return;
      } catch (const std::runtime_error&) {
        thrown += runtime;
        return;
      }
      std::printf("refusal %s: not thrown\n", name);
    };
    attempt("null-image", {&pin752, &pin752}, {img.data(), nullptr}, {0.0, 0.0}, true);
    attempt("null-camera", {&pin752, nullptr}, {img.data(), img.data()}, {0.0, 0.0}, false);
    attempt("lengths", {&pin752, &pin752}, {img.data()}, {0.0, 0.0}, false);
    attempt("timestamps", {&pin752}, {img.data()}, {}, false);
    std::printf("refusals thrown %d of %d\n", thrown, tried);
    ok = ok && thrown == tried;
    std::printf("empty batch %zu frames\n", svo::streams::newFrames(ctx, {}, {}, 5, {}).size());
    return ok ? 0 : 1;
  } catch (const std::exception& e) {
    std::fprintf(stderr, "host_frames_streams_demo: %s\n", e.what());
    return 2;
  }
}
