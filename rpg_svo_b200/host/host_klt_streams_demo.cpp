// rpg_svo_b200/host/host_klt_streams_demo.cpp -- the two-view initialisation of several camera streams through svo_host.h,
// twice on identically built streams: once with one initialization::trackKlt call per stream and frame, once with one
// svo::streams::trackKlt call per frame (one batched pyramid build, one tracking launch).  The streams mix pinhole and
// ATAN cameras and two image sizes, and two of them share one first keyframe.  Prints a digest of every stream's px_ref,
// px_cur, f_ref, f_cur and disparities after every frame; the two digests must be equal.  Then checks that every refusal of
// streams::trackKlt throws std::invalid_argument and leaves every vector as it was.
//   usage: host_klt_streams_demo
#include <cinttypes>
#include <cstdio>
#include <cstring>
#include <memory>
#include <vector>

#include "svo_host.h"

namespace {

constexpr int kStreams = 6, kFrames = 4, kLevels = 5;

// frame k of stream s: host_klt_demo's blurred hash texture, shifted by (3k, 2k) px from a per-stream origin
std::vector<uint8_t> frame_image(int s, int k, int W, int H) {
  auto base = [](int x, int y) { return (((uint32_t)x * 73856093u) ^ ((uint32_t)y * 19349663u)) >> 8 & 255u; };
  const int ox = 37 * s, oy = 23 * s;
  std::vector<uint8_t> img((size_t)W * H);
  for (int y = 0; y < H; ++y)
    for (int x = 0; x < W; ++x) {
      uint32_t sum = 0;
      for (int j = -3; j <= 3; ++j)
        for (int i = -3; i <= 3; ++i) sum += base(x + i + 3 * k + ox, y + j + 2 * k + oy);
      const uint32_t v = std::min(std::max(sum / 49, 100u), 155u) - 100u;
      img[(size_t)y * W + x] = (uint8_t)(v * 255u / 55u);
    }
  return img;
}

struct Digest {
  uint64_t h = 1469598103934665603ULL;
  void add(const void* p, size_t n) {
    const uint8_t* b = static_cast<const uint8_t*>(p);
    for (size_t i = 0; i < n; ++i) { h ^= b[i]; h *= 1099511628211ULL; }
  }
  template <class T> void vec(const std::vector<T>& v) { size_t n = v.size(); add(&n, sizeof(n)); add(v.data(), n * sizeof(T)); }
};

// the cameras: stream s % 4 = 0 752 x 480 pinhole, 1 640 x 480 ATAN, 2 752 x 480 ATAN, 3 640 x 480 pinhole
struct Cameras {
  svo::PinholeCamera pin752{752, 480, 315.5, 315.5, 376.0, 240.0}, pin640{640, 480, 320.0, 320.0, 320.0, 240.0};
  svo::ATANCamera atan752{752, 480, 0.509326, 0.796651, 0.45905, 0.510056, 0.9320}, atan640{640, 480, 0.52, 0.69, 0.5, 0.5, 0.85};
  svo::AbstractCamera* of(int s) {
    switch (s % 4) {
      case 0: return &pin752;
      case 1: return &atan640;
      case 2: return &atan752;
      default: return &pin640;
    }
  }
};

struct Streams {
  std::vector<svo::FramePtr> refs;
  std::vector<std::vector<svo::Point2f>> px_ref, px_cur;
  std::vector<std::vector<svo::Vector3d>> f_ref, f_cur;
  std::vector<std::vector<double>> disp;
  uint64_t digest() const {
    Digest g;
    for (size_t s = 0; s < refs.size(); ++s) { g.vec(px_ref[s]); g.vec(px_cur[s]); g.vec(f_ref[s]); g.vec(f_cur[s]); g.vec(disp[s]); }
    return g.h;
  }
};

// first keyframes and their detections (addFirstFrame): stream 4 shares stream 0's keyframe
Streams first_frames(svo::Context& ctx, Cameras& cams) {
  Streams st;
  st.px_ref.resize(kStreams); st.px_cur.resize(kStreams); st.f_ref.resize(kStreams); st.f_cur.resize(kStreams); st.disp.resize(kStreams);
  for (int s = 0; s < kStreams; ++s) {
    if (s == 4) {
      st.refs.push_back(st.refs[0]);
    } else {
      svo::AbstractCamera* cam = cams.of(s);
      const std::vector<uint8_t> img = frame_image(s, 0, cam->width(), cam->height());
      st.refs.emplace_back(new svo::Frame(ctx, cam, img.data(), kLevels, 0.0));
    }
    svo::initialization::detectFeatures(st.refs[s], st.px_ref[s], st.f_ref[s]);
    st.px_cur[s] = st.px_ref[s];  // the initial flow is the reference position
  }
  return st;
}

std::vector<svo::FramePtr> next_frames(svo::Context& ctx, Cameras& cams, int k) {
  std::vector<svo::FramePtr> cur;
  for (int s = 0; s < kStreams; ++s) {
    svo::AbstractCamera* cam = cams.of(s == 4 ? 0 : s);
    const std::vector<uint8_t> img = frame_image(s == 4 ? 0 : s, k + (s == 4 ? 1 : 0), cam->width(), cam->height());
    cur.emplace_back(new svo::Frame(ctx, cam, img.data(), kLevels, 0.0));
  }
  return cur;
}

}  // namespace

int main() {
  try {
    svo::Context ctx(0);
    Cameras cams;
    bool ok = true;
    uint64_t dg[2] = {0, 0};
    size_t pts[2] = {0, 0};
    for (int run = 0; run < 2; ++run) {
      Streams st = first_frames(ctx, cams);
      Digest g;
      for (int k = 1; k < kFrames; ++k) {
        std::vector<svo::FramePtr> cur = next_frames(ctx, cams, k);
        if (run == 0) {
          for (int s = 0; s < kStreams; ++s)
            svo::initialization::trackKlt(st.refs[s], cur[s], st.px_ref[s], st.px_cur[s], st.f_ref[s], st.f_cur[s], st.disp[s]);
        } else {
          svo::streams::trackKlt(st.refs, cur, st.px_ref, st.px_cur, st.f_ref, st.f_cur, st.disp);
        }
        const uint64_t d = st.digest();
        g.add(&d, sizeof(d));
        for (int s = 0; s < kStreams; ++s) {
          pts[run] += st.px_ref[s].size();
          if (run == 1) std::printf("frame %d stream %d tracked %zu\n", k, s, st.px_ref[s].size());
        }
      }
      dg[run] = g.h;
    }
    std::printf("sequential %016" PRIx64 " points %zu\n", dg[0], pts[0]);
    std::printf("batched    %016" PRIx64 " points %zu\n", dg[1], pts[1]);
    ok = ok && dg[0] == dg[1] && pts[0] > 0;

    // refusals: each throws std::invalid_argument with every vector as it was
    {
      Streams st = first_frames(ctx, cams);
      std::vector<svo::FramePtr> cur = next_frames(ctx, cams, 1);
      const uint64_t before = st.digest();
      int thrown = 0, n = 0;
      auto attempt = [&](const char* name, const std::vector<svo::FramePtr>& refs, const std::vector<svo::FramePtr>& curs, Streams& x) {
        ++n;
        try {
          svo::streams::trackKlt(refs, curs, x.px_ref, x.px_cur, x.f_ref, x.f_cur, x.disp);
        } catch (const std::invalid_argument&) {
          ++thrown;
          return;
        }
        std::printf("refusal %s: not thrown\n", name);
      };
      {  // one vector shorter than the frame lists
        std::vector<std::vector<svo::Point2f>> saved = st.px_cur;
        st.px_cur.pop_back();
        attempt("lengths", st.refs, cur, st);
        st.px_cur.push_back(saved.back());
      }
      {
        std::vector<svo::FramePtr> refs = st.refs;
        refs.pop_back();
        attempt("frame-lists", refs, cur, st);
      }
      {
        std::vector<svo::FramePtr> c2 = cur;
        c2[3] = nullptr;
        attempt("null-cur", st.refs, c2, st);
        std::vector<svo::FramePtr> r2 = st.refs;
        r2[5] = nullptr;
        attempt("null-ref", r2, cur, st);
      }
      const uint64_t after = st.digest();
      std::printf("refusals thrown %d of %d vectors %s\n", thrown, n, after == before ? "unchanged" : "changed");
      ok = ok && thrown == n && after == before;
      // a frame on another device: needs a second GPU
      std::unique_ptr<svo::Context> other;
      try { other.reset(new svo::Context(1)); } catch (const std::exception&) {}
      if (other) {
        std::vector<svo::FramePtr> c2 = cur;
        const std::vector<uint8_t> img = frame_image(2, 1, 752, 480);
        c2[2].reset(new svo::Frame(*other, cams.of(2), img.data(), kLevels, 0.0));
        const uint64_t b2 = st.digest();
        bool threw = false;
        try { svo::streams::trackKlt(st.refs, c2, st.px_ref, st.px_cur, st.f_ref, st.f_cur, st.disp, &ctx); }
        catch (const std::invalid_argument&) { threw = true; }
        std::printf("device refusal %s vectors %s\n", threw ? "thrown" : "not-thrown", st.digest() == b2 ? "unchanged" : "changed");
        ok = ok && threw && st.digest() == b2;
        c2[2].reset();
      } else {
        std::printf("device refusal skipped (one device)\n");
      }
    }
    return ok ? 0 : 1;
  } catch (const std::exception& e) {
    std::fprintf(stderr, "host_klt_streams_demo: %s\n", e.what());
    return 2;
  }
}
