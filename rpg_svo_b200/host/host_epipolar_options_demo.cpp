// rpg_svo_b200/host/host_epipolar_options_demo.cpp -- Matcher::Options of the epipolar search through svo_host.h:
//   1. a DepthFilter subclass that sets matcher_.options_ (align_1d, no sub-pixel refinement) gets a different result
//      from the default filter on the same seeds, equal to the C ABI's depth filter under the same setting;
//   2. a Matcher with align_1d sets h_inv_ where align1D runs (also on a failed alignment, NaN on a zero-length line) and
//      keeps it where it does not;
//   3. streams::updateSeeds refuses filters whose matcher_.options_ differ, before any launch.
// Prints one line per check and "epipolar options demo: ok"; exits 1 at the first failed check.
//   usage: host_epipolar_options_demo
#include <cmath>
#include <cstdio>
#include <cstring>
#include <stdexcept>
#include <vector>

#include "svo_host.h"

namespace {

int g_failed = 0;
void check(bool ok, const char* what) {
  std::printf("%s: %s\n", ok ? "ok  " : "FAIL", what);
  if (!ok) g_failed = 1;
}

// a textured plane z = 2 m; camera at world position c with identity rotation: T_f_w = [I | -c]
svo::FramePtr render(svo::Context& ctx, svo::PinholeCamera* cam, const svo::Vector3d& c) {
  const int w = cam->width(), h = cam->height();
  std::vector<uint8_t> img((size_t)w * h);
  for (int v = 0; v < h; ++v)
    for (int u = 0; u < w; ++u) {
      const double z = 2.0 - c[2], X = (u - cam->cx_) / cam->fx_ * z + c[0], Y = (v - cam->cy_) / cam->fy_ * z + c[1];
      const double t = std::sin(X * 173.0) * std::cos(Y * 131.0) + 0.5 * std::sin((X + 2 * Y) * 411.0);
      img[(size_t)v * w + u] = (uint8_t)std::lround(128.0 + 80.0 * t);
    }
  svo::FramePtr f(new svo::Frame(ctx, cam, img.data(), 3, 0.0));
  const double T[12] = {1, 0, 0, -c[0], 0, 1, 0, -c[1], 0, 0, 1, -c[2]};
  std::memcpy(f->T_f_w_.m, T, sizeof(T));
  return f;
}

// The reference's pattern (INTEGRATION.md section 7): a subclass reaches the protected matcher_.
struct EdgeFilter : svo::DepthFilter {
  explicit EdgeFilter(callback_t cb) : svo::DepthFilter(cb) {
    matcher_.options_.align_1d = true;
    matcher_.options_.subpix_refinement = false;
  }
};

struct Seeds {
  std::vector<float> a, b, mu, s2;
  size_t n = 0;
};
Seeds snapshot(svo::DepthFilter& df) {
  Seeds s;
  for (const svo::Seed& sd : df.getSeeds()) { s.a.push_back(sd.a); s.b.push_back(sd.b); s.mu.push_back(sd.mu); s.s2.push_back(sd.sigma2); }
  s.n = s.a.size();
  return s;
}
bool same(const Seeds& x, const Seeds& y) {
  return x.n == y.n && std::memcmp(x.a.data(), y.a.data(), 4 * x.n) == 0 && std::memcmp(x.b.data(), y.b.data(), 4 * x.n) == 0 &&
         std::memcmp(x.mu.data(), y.mu.data(), 4 * x.n) == 0 && std::memcmp(x.s2.data(), y.s2.data(), 4 * x.n) == 0;
}

}  // namespace

int main() {
  svo::Context ctx(0);
  svo::PinholeCamera cam(752, 480, 315.5, 315.5, 376.0, 240.0);
  svo::FramePtr kf = render(ctx, &cam, {0, 0, 0});
  svo::FramePtr cur = render(ctx, &cam, {0.12, 0.03, 0.02});
  std::vector<svo::Feature*> ftrs;
  for (int v = 40, i = 0; v < 440; v += 37)
    for (int u = 40; u < 712; u += 41, ++i) {
      const int L = i % 3;
      ftrs.push_back(new svo::Feature(kf.get(), {(double)((u >> L) << L), (double)((v >> L) << L)}, L));
    }
  auto noop = [](svo::Point* p, double) { delete p; };

  // 1. matcher_.options_ of a subclass reach the launch
  svo::DepthFilter plain(noop);
  EdgeFilter edge(noop);
  plain.addKeyframe(kf, ftrs, 2.0, 0.5);
  edge.addKeyframe(kf, ftrs, 2.0, 0.5);
  const Seeds before = snapshot(edge);
  plain.updateSeeds(cur);
  edge.updateSeeds(cur);
  const Seeds p = snapshot(plain), e = snapshot(edge);
  check(edge.n_updates_ > 20 && plain.n_updates_ > 20, "both filters update seeds");
  check(!same(p, e), "align_1d without refinement changes the filter's result");
  svo_b200_epipolar_options set{};
  ctx.check(svo_b200_get_epipolar_options(ctx.get(), &set));
  check(set.align_1d == 1 && set.subpix_refinement == 0 && set.epi_search_edgelet_filtering == 1 &&
            set.epi_search_edgelet_max_angle == 0.7,
        "the filter's launch set the context's options from matcher_.options_");
  {  // the same seeds through the C ABI under the same setting
    const size_t M = before.n;
    std::vector<const svo_b200_frame*> refs{kf->device()};
    std::vector<int> ri(M, 0), lv, ty(M, 0), bi(M, svo::Seed::batch_counter());
    std::vector<double> px, f, gr(2 * M, 0.0), pc(2 * M), z(M);
    for (svo::Feature* ft : ftrs) { lv.push_back(ft->level); px.push_back(ft->px[0]); px.push_back(ft->px[1]);
                                    f.push_back(ft->f[0]); f.push_back(ft->f[1]); f.push_back(ft->f[2]); }
    Seeds s = before;
    std::vector<float> zr(M, 2.0f);
    std::vector<uint8_t> st(M);
    const svo_b200_camera c = cam.c_abi();
    const svo_b200_depth_options opt = {3, 200.0, 2, 10, 1000};
    ctx.check(svo_b200_depth_filter_update(ctx.get(), refs.data(), kf->T_f_w_.m, 1, cur->device(), cur->T_f_w_.m, &c, &opt, (int)M,
                                           ri.data(), px.data(), f.data(), lv.data(), ty.data(), gr.data(), bi.data(),
                                           svo::Seed::batch_counter(), s.a.data(), s.b.data(), s.mu.data(), zr.data(),
                                           s.s2.data(), st.data(), pc.data(), z.data(), nullptr));
    size_t n_kept = 0, n_same = 0;
    std::list<svo::Seed>::const_iterator it = edge.getSeeds().begin();
    for (size_t m = 0; m < M; ++m) {
      if (st[m] == SVO_B200_SEED_CONVERGED || st[m] == SVO_B200_SEED_NAN || st[m] == SVO_B200_SEED_TOO_OLD) continue;
      ++n_kept;
      n_same += it->a == s.a[m] && it->b == s.b[m] && it->mu == s.mu[m] && it->sigma2 == s.s2[m];
      ++it;
    }
    check(n_kept == e.n && n_same == n_kept, "the subclass's seeds equal the C ABI's under the same setting");
  }

  // 2. Matcher::h_inv_
  svo::Matcher m1, m2;
  m1.options_.align_1d = true;
  m2.h_inv_ = m1.h_inv_ = -1.0;
  svo::Feature* ft = ftrs[40];
  const double d = 2.0 / ft->f[2];
  double depth = 0.0;
  const bool ok1 = m1.findEpipolarMatchDirect(*kf, *cur, *ft, d, d / 1.001, d / 0.999, depth);
  check(m1.h_inv_ != -1.0 && std::isfinite(m1.h_inv_) && m1.h_inv_ > 0.0, "align_1d sets h_inv_ (short line)");
  std::printf("      h_inv_ %.9g, success %d, depth %.6f (true %.6f)\n", m1.h_inv_, (int)ok1, depth, d);
  m2.findEpipolarMatchDirect(*kf, *cur, *ft, d, d / 1.3, d / 0.7, depth);
  check(m2.h_inv_ == -1.0, "align2D leaves h_inv_ as it was");
  const bool ok0 = m1.findEpipolarMatchDirect(*kf, *cur, *ft, d, d, d, depth);
  check(!ok0 && std::isnan(m1.h_inv_), "a zero-length line runs align1D along a NaN direction: h_inv_ NaN, no match");

  // 3. mixed settings in one streams call
  EdgeFilter e2(noop);
  svo::DepthFilter p2(noop);
  e2.addKeyframe(kf, ftrs, 2.0, 0.5);
  p2.addKeyframe(kf, ftrs, 2.0, 0.5);
  const Seeds e2_before = snapshot(e2), p2_before = snapshot(p2);
  const uint64_t launches = svo_b200_launch_count(ctx.get());
  bool refused = false;
  try {
    svo::streams::updateSeeds({&e2, &p2}, {cur, cur});
  } catch (const std::invalid_argument& ex) {
    refused = true;
    std::printf("      refused: %s\n", ex.what());
  }
  check(refused && svo_b200_launch_count(ctx.get()) == launches && same(snapshot(e2), e2_before) && same(snapshot(p2), p2_before),
        "streams::updateSeeds refuses mixed matcher_.options_ before any launch");
  svo::streams::updateSeeds({&e2}, {cur});
  check(same(snapshot(e2), e), "one stream of the subclass equals its own updateSeeds");

  for (svo::Feature* f : ftrs) delete f;
  if (g_failed) return 1;
  std::printf("epipolar options demo: ok\n");
  return 0;
}
