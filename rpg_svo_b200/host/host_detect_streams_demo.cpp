// rpg_svo_b200/host/host_detect_streams_demo.cpp -- keyframe seeding of several camera streams through svo_host.h, each
// stage twice on identically built streams: once per object (DepthFilter::addKeyframe, FastDetector::detect,
// initialization::detectFeatures) and once batched (svo::streams::addKeyframes / detect / detectFeatures, one detection
// launch per stage).  Prints a digest of every object's state after each run; the two digests of a stage must be equal.
// Then checks that every refusal of streams::addKeyframes and streams::detect throws std::invalid_argument and leaves the
// objects as they were.
//   usage: host_detect_streams_demo
// Scenes are rendered here: a textured plane z = 2 m seen by cameras with identity rotation at different positions.
#include <cinttypes>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <random>
#include <vector>

#include "svo_host.h"

namespace {

constexpr double kPlaneZ = 2.0;
constexpr int kLevels = 5, kStreams = 6, kRounds = 2, kExistingFeatures = 120;

// value noise on the plane, two octaves, bilinear: texture a few pixels wide at 2 m
double lattice(int64_t i, int64_t j, uint32_t salt) {
  uint64_t h = (uint64_t)i * 0x9E3779B97F4A7C15ULL ^ ((uint64_t)j + 0x632BE59BD9B4E019ULL) * 0xC2B2AE3D27D4EB4FULL ^ salt;
  h ^= h >> 29; h *= 0xBF58476D1CE4E5B9ULL; h ^= h >> 32;
  return (double)(h & 0xFFFF) / 65535.0;
}
double noise(double x, double y, uint32_t salt) {
  const double fx = std::floor(x), fy = std::floor(y), tx = x - fx, ty = y - fy;
  const int64_t i = (int64_t)fx, j = (int64_t)fy;
  const double a = lattice(i, j, salt), b = lattice(i + 1, j, salt), c = lattice(i, j + 1, salt), d = lattice(i + 1, j + 1, salt);
  return (a * (1 - tx) + b * tx) * (1 - ty) + (c * (1 - tx) + d * tx) * ty;
}
uint8_t texture(double X, double Y) {
  const double v = 0.65 * noise(X / 0.02, Y / 0.02, 1) + 0.35 * noise(X / 0.007, Y / 0.007, 2);
  return (uint8_t)std::lround(20.0 + 215.0 * v);
}

// camera at world position c, identity rotation: T_f_w = [I | -c]
svo::FramePtr render(svo::Context& ctx, svo::PinholeCamera* cam, const svo::Vector3d& c, double ts) {
  const int w = cam->width(), h = cam->height();
  std::vector<uint8_t> img((size_t)w * h);
  for (int v = 0; v < h; ++v)
    for (int u = 0; u < w; ++u) {
      const double z = kPlaneZ - c[2];
      img[(size_t)v * w + u] = texture((u - cam->cx_) / cam->fx_ * z + c[0], (v - cam->cy_) / cam->fy_ * z + c[1]);
    }
  svo::FramePtr f(new svo::Frame(ctx, cam, img.data(), kLevels, ts));
  const double T[12] = {1, 0, 0, -c[0], 0, 1, 0, -c[1], 0, 0, 1, -c[2]};
  std::memcpy(f->T_f_w_.m, T, sizeof(T));
  return f;
}

// a keyframe that already carries features (those the tracker matched): its cells are occupied for the detector
svo::FramePtr keyframe(svo::Context& ctx, svo::PinholeCamera* cam, int s, int round) {
  svo::FramePtr f = render(ctx, cam, {0.05 * s + 0.07 * round, -0.03 * s + 0.02 * round, 0.01 * round}, round);
  std::mt19937 rng(1000 * round + s);
  std::uniform_real_distribution<double> U(0.0, 1.0);
  for (int i = 0; i < kExistingFeatures; ++i) {
    const int L = i % 3;
    const double u = std::floor(8 + (cam->width() - 16) * U(rng)), v = std::floor(8 + (cam->height() - 16) * U(rng));
    f->addFeature(new svo::Feature(f.get(), {(double)(((int)u >> L) << L), (double)(((int)v >> L) << L)}, L));
  }
  f->setKeyframe();
  return f;
}

struct Digest {
  uint64_t h = 1469598103934665603ULL;
  void add(const void* p, size_t n) {
    const uint8_t* b = static_cast<const uint8_t*>(p);
    for (size_t i = 0; i < n; ++i) { h ^= b[i]; h *= 1099511628211ULL; }
  }
  template <class T> void add(const T& v) { add(&v, sizeof(T)); }
};

// ---- depth filters: S streams, kRounds keyframes each -----------------------------------------------------------------
struct Stream {
  svo::PinholeCamera* cam;
  svo::feature_detection::DetectorPtr detector;
  std::unique_ptr<svo::DepthFilter> filter;
  std::vector<svo::FramePtr> kfs;
  double depth_mean, depth_min;
};

void build(svo::Context& ctx, std::vector<svo::PinholeCamera*>& cams, std::vector<std::unique_ptr<Stream>>& out) {
  for (int s = 0; s < kStreams; ++s) {
    out.emplace_back(new Stream);
    Stream& d = *out.back();
    d.cam = cams[s % cams.size()];
    const int cell = s % 3 == 0 ? 25 : 30, levels = s % 4 == 3 ? 2 : 3;  // detectors differ in cell size and levels
    d.detector.reset(new svo::feature_detection::FastDetector(d.cam->width(), d.cam->height(), cell, levels));
    d.filter.reset(new svo::DepthFilter(d.detector, [](svo::Point*, double) {}));
    d.filter->triang_min_corner_score_ = 20.0 + 15.0 * (s % 3);
    for (int r = 0; r < kRounds; ++r) d.kfs.push_back(keyframe(ctx, d.cam, s, r));
    d.depth_mean = 2.0 + 0.1 * s;
    d.depth_min = 0.5 + 0.05 * s;
  }
}

// every filter's seeds (ids, batch ids, a, b, mu, z_range, sigma2, feature px / level / bearing, the keyframe it lies in)
// and the process-wide counters
uint64_t digest(const std::vector<std::unique_ptr<Stream>>& st, size_t* n_seeds) {
  Digest g;
  *n_seeds = 0;
  for (const auto& d : st) {
    for (const svo::Seed& sd : d->filter->getSeeds()) {
      g.add(sd.id); g.add(sd.batch_id);
      g.add(sd.a); g.add(sd.b); g.add(sd.mu); g.add(sd.z_range); g.add(sd.sigma2);
      g.add(sd.ftr->px); g.add(sd.ftr->level); g.add(sd.ftr->f);
      int k = -1;
      for (size_t i = 0; i < d->kfs.size(); ++i) if (d->kfs[i].get() == sd.ftr->frame) k = (int)i;
      g.add(k);
      ++*n_seeds;
    }
    for (const auto& kf : d->kfs) g.add(kf->fts_.size());
  }
  g.add(svo::Seed::batch_counter());
  g.add(svo::Seed::seed_counter());
  return g.h;
}

void add_keyframes_per_object(std::vector<std::unique_ptr<Stream>>& st) {
  for (int r = 0; r < kRounds; ++r)
    for (auto& d : st) d->filter->addKeyframe(d->kfs[r], d->depth_mean, d->depth_min);
}

void add_keyframes_batched(std::vector<std::unique_ptr<Stream>>& st) {
  for (int r = 0; r < kRounds; ++r) {
    std::vector<svo::DepthFilter*> filters;
    std::vector<svo::FramePtr> frames;
    std::vector<double> mean, min;
    for (auto& d : st) { filters.push_back(d->filter.get()); frames.push_back(d->kfs[r]); mean.push_back(d->depth_mean); min.push_back(d->depth_min); }
    svo::streams::addKeyframes(filters, frames, mean, min);
  }
}

void reset_counters() { svo::Seed::batch_counter() = 0; svo::Seed::seed_counter() = 0; }

// ---- FastDetector::detect: each detector twice (grid filled from the keyframe's features, then from nothing: that
// second call sees the grid the first one left) -------------------------------------------------------------------------
uint64_t detect_run(std::vector<std::unique_ptr<Stream>>& st, bool batched, size_t* n_ftrs) {
  Digest g;
  *n_ftrs = 0;
  for (int r = 0; r < kRounds; ++r) {
    std::vector<svo::feature_detection::FastDetector*> dets;
    std::vector<svo::FramePtr> frames;
    std::vector<double> thr;
    std::vector<svo::Features> fts(st.size());
    for (auto& d : st) {
      dets.push_back(static_cast<svo::feature_detection::FastDetector*>(d->detector.get()));
      frames.push_back(d->kfs[r]);
      thr.push_back(d->filter->triang_min_corner_score_);
      if (r == 0) d->detector->setExistingFeatures(d->kfs[r]->fts_);
    }
    if (batched) {
      svo::streams::detect(dets, frames, thr, fts);
    } else {
      for (size_t s = 0; s < st.size(); ++s) dets[s]->detect(frames[s].get(), thr[s], fts[s]);
    }
    for (auto& f : fts) {
      g.add(f.size());
      for (svo::Feature* x : f) { g.add(x->px); g.add(x->level); g.add(x->f); ++*n_ftrs; delete x; }
    }
  }
  return g.h;
}

// ---- initialization::detectFeatures ------------------------------------------------------------------------------------
uint64_t init_run(std::vector<std::unique_ptr<Stream>>& st, bool batched, size_t* n_ftrs) {
  std::vector<svo::FramePtr> frames;
  for (auto& d : st) frames.push_back(d->kfs[0]);
  std::vector<std::vector<svo::Point2f>> px(frames.size());
  std::vector<std::vector<svo::Vector3d>> f(frames.size());
  if (batched) {
    svo::streams::detectFeatures(frames, px, f);
  } else {
    for (size_t s = 0; s < frames.size(); ++s) svo::initialization::detectFeatures(frames[s], px[s], f[s]);
  }
  Digest g;
  *n_ftrs = 0;
  for (size_t s = 0; s < frames.size(); ++s) {
    g.add(px[s].size());
    for (size_t i = 0; i < px[s].size(); ++i) { g.add(px[s][i].x); g.add(px[s][i].y); g.add(f[s][i]); ++*n_ftrs; }
  }
  return g.h;
}

}  // namespace

int main() {
  try {
    svo::Context ctx(0);
    svo::PinholeCamera cam752(752, 480, 315.5, 315.5, 376.0, 240.0), cam640(640, 480, 320.0, 320.0, 320.0, 240.0);
    std::vector<svo::PinholeCamera*> cams{&cam752, &cam640};
    bool ok = true;

    // DepthFilter::addKeyframe: per object, then batched, on identically built streams
    uint64_t kd[2];
    size_t seeds[2];
    for (int run = 0; run < 2; ++run) {
      std::vector<std::unique_ptr<Stream>> st;
      build(ctx, cams, st);
      reset_counters();
      if (run == 0) add_keyframes_per_object(st); else add_keyframes_batched(st);
      kd[run] = digest(st, &seeds[run]);
    }
    printf("keyframes per-object %016" PRIx64 " seeds %zu\n", kd[0], seeds[0]);
    printf("keyframes batched    %016" PRIx64 " seeds %zu\n", kd[1], seeds[1]);
    ok = ok && kd[0] == kd[1];

    uint64_t dd[2], id[2];
    size_t nd[2], ni[2];
    for (int run = 0; run < 2; ++run) {
      std::vector<std::unique_ptr<Stream>> st;
      build(ctx, cams, st);
      dd[run] = detect_run(st, run == 1, &nd[run]);
      id[run] = init_run(st, run == 1, &ni[run]);
    }
    printf("detect per-object %016" PRIx64 " features %zu\n", dd[0], nd[0]);
    printf("detect batched    %016" PRIx64 " features %zu\n", dd[1], nd[1]);
    printf("init per-object %016" PRIx64 " features %zu\n", id[0], ni[0]);
    printf("init batched    %016" PRIx64 " features %zu\n", id[1], ni[1]);
    ok = ok && dd[0] == dd[1] && id[0] == id[1];

    // refusals: each throws std::invalid_argument before any object changes.  The streams that took part then run their
    // per-object addKeyframe; the digest must equal the per-object run's above (grids, seeds, counters untouched).
    {
      std::vector<std::unique_ptr<Stream>> st;
      build(ctx, cams, st);
      reset_counters();
      std::vector<svo::DepthFilter*> all;
      std::vector<svo::FramePtr> frames;
      std::vector<double> mean, min;
      for (auto& d : st) { all.push_back(d->filter.get()); frames.push_back(d->kfs[0]); mean.push_back(d->depth_mean); min.push_back(d->depth_min); }
      svo::DepthFilter threaded(svo::feature_detection::DetectorPtr(new svo::feature_detection::FastDetector(752, 480, 30, 3)),
                                [](svo::Point*, double) {});
      threaded.startThread();
      svo::DepthFilter no_detector([](svo::Point*, double) {});
      svo::DepthFilter shares(st[1]->detector, [](svo::Point*, double) {});
      struct Case { const char* name; svo::DepthFilter* extra; };
      const Case cases[] = {{"listed-twice", st[2]->filter.get()}, {"thread", &threaded}, {"no-detector", &no_detector},
                            {"shared-detector", &shares}};
      int thrown = 0, n = 0;
      for (const Case& c : cases) {
        std::vector<svo::DepthFilter*> f = all;
        std::vector<svo::FramePtr> fr = frames;
        std::vector<double> me = mean, mi = min;
        f.push_back(c.extra); fr.push_back(frames[0]); me.push_back(2.0); mi.push_back(0.5);
        ++n;
        try { svo::streams::addKeyframes(f, fr, me, mi); } catch (const std::invalid_argument&) { ++thrown; continue; }
        printf("refusal %s: not thrown\n", c.name);
      }
      {  // streams::detect with a detector listed twice
        std::vector<svo::feature_detection::FastDetector*> dets;
        for (auto& d : st) dets.push_back(static_cast<svo::feature_detection::FastDetector*>(d->detector.get()));
        dets.push_back(dets[0]);
        std::vector<svo::FramePtr> fr = frames;
        fr.push_back(frames[0]);
        std::vector<svo::Features> fts(dets.size());
        ++n;
        try { svo::streams::detect(dets, fr, std::vector<double>(dets.size(), 20.0), fts); } catch (const std::invalid_argument&) { ++thrown; }
      }
      threaded.stopThread();
      size_t ns = 0;
      const uint64_t before = digest(st, &ns);
      add_keyframes_per_object(st);  // the counters are still those reset_counters left
      size_t n_after;
      const uint64_t after = digest(st, &n_after);
      const bool unchanged = ns == 0 && after == kd[0];
      printf("refusals thrown %d of %d objects %s seeds-before %zu %016" PRIx64 "\n", thrown, n, unchanged ? "unchanged" : "changed", ns, before);
      ok = ok && thrown == n && unchanged;
    }
    return ok ? 0 : 1;
  } catch (const std::exception& e) {
    fprintf(stderr, "host_detect_streams_demo: %s\n", e.what());
    return 2;
  }
}
