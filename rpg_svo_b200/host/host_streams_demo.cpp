// rpg_svo_b200/host/host_streams_demo.cpp -- several camera streams through the depth filter and the reprojector of
// svo_host.h, each stage twice on identically built streams: once per object (DepthFilter::updateSeeds,
// Reprojector::reprojectMap) and once batched (svo::streams::updateSeeds / reprojectMap, one launch per stage).  Prints a
// digest of every object's state after each run; the two digests of a stage must be equal.
//   usage: host_streams_demo
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
constexpr int kLevels = 5;

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

struct Digest {
  uint64_t h = 1469598103934665603ULL;
  void add(const void* p, size_t n) {
    const uint8_t* b = static_cast<const uint8_t*>(p);
    for (size_t i = 0; i < n; ++i) { h ^= b[i]; h *= 1099511628211ULL; }
  }
  template <class T> void add(const T& v) { add(&v, sizeof(T)); }
};

// ---- depth filter ----------------------------------------------------------------------------------------------------
constexpr int kDepthStreams = 6, kDepthFrames = 5;  // 10 cm more baseline per frame, so that seeds converge within the run

struct DepthStream {
  svo::MapPointCandidates candidates;
  std::unique_ptr<svo::DepthFilter> filter;
  svo::FramePtr kf;
  std::vector<svo::FramePtr> frames;
};

void build_depth(svo::Context& ctx, std::vector<svo::PinholeCamera*>& cams, std::vector<std::unique_ptr<DepthStream>>& out) {
  for (int s = 0; s < kDepthStreams; ++s) {
    out.emplace_back(new DepthStream);
    DepthStream& d = *out.back();
    svo::PinholeCamera* cam = cams[s % cams.size()];
    d.filter.reset(new svo::DepthFilter(std::bind(&svo::MapPointCandidates::newCandidatePoint, &d.candidates,
                                                  std::placeholders::_1, std::placeholders::_2)));
    const svo::Vector3d c0{0.03 * s, -0.02 * s, 0.0};
    d.kf = render(ctx, cam, c0, 0.0);
    d.kf->setKeyframe();
    std::vector<svo::Feature*> ftrs;
    int i = 0;
    for (int v = 24; v < cam->height() - 24; v += 22 + s)
      for (int u = 24; u < cam->width() - 24; u += 22 + s, ++i) {
        const int L = i % 3;
        ftrs.push_back(new svo::Feature(d.kf.get(), {(double)((u >> L) << L), (double)((v >> L) << L)}, L));
      }
    d.filter->addKeyframe(d.kf, ftrs, 2.6 + 0.1 * s, 0.5);
    for (int k = 1; k <= kDepthFrames; ++k)
      d.frames.push_back(render(ctx, cam, {c0[0] + 0.1 * k, c0[1] + 0.02 * k, 0.01 * k}, k));
  }
}

uint64_t digest_depth(const std::vector<std::unique_ptr<DepthStream>>& st, size_t* n_seeds, size_t* n_cand) {
  Digest g;
  *n_seeds = *n_cand = 0;
  for (const auto& d : st) {
    g.add(d->filter->n_updates_);
    g.add(d->filter->n_failed_matches_);
    for (const svo::Seed& sd : d->filter->getSeeds()) {
      g.add(sd.a); g.add(sd.b); g.add(sd.mu); g.add(sd.z_range); g.add(sd.sigma2);
      g.add(sd.ftr->px);
      ++*n_seeds;
    }
    for (auto& c : d->candidates.candidates_) { g.add(c.first->pos_); g.add(c.second->px); ++*n_cand; }
  }
  return g.h;
}

// ---- reprojector -----------------------------------------------------------------------------------------------------
constexpr int kReprojStreams = 4, kMapKfs = 3, kMapPoints = 500, kMapCandidates = 60;

struct ReprojStream {
  svo::Map map;
  std::vector<svo::Point*> pts;
  std::unique_ptr<svo::Reprojector> reprojector;
  svo::FramePtr cur;
  std::vector<std::pair<svo::FramePtr, size_t>> overlap;
};

void build_reproject(svo::Context& ctx, std::vector<svo::PinholeCamera*>& cams, std::vector<std::unique_ptr<ReprojStream>>& out) {
  for (int s = 0; s < kReprojStreams; ++s) {
    out.emplace_back(new ReprojStream);
    ReprojStream& r = *out.back();
    svo::PinholeCamera* cam = cams[s % cams.size()];
    std::mt19937 rng(100 + s);
    std::uniform_real_distribution<double> U(0.0, 1.0);
    std::vector<svo::FramePtr> kfs;
    for (int k = 0; k < kMapKfs; ++k) kfs.push_back(render(ctx, cam, {0.08 * k - 0.04 * s, 0.03 * k, 0.02 * k}, k));
    const double half_w = 0.9 * kPlaneZ * cam->cx_ / cam->fx_, half_h = 0.9 * kPlaneZ * cam->cy_ / cam->fy_;
    for (int p = 0; p < kMapPoints + kMapCandidates; ++p) {
      const svo::Vector3d pos{-half_w + 2 * half_w * U(rng), -half_h + 2 * half_h * U(rng), kPlaneZ};
      svo::Point* pt = new svo::Point(pos);
      const bool cand = p >= kMapPoints;
      pt->type_ = cand ? svo::Point::TYPE_CANDIDATE : (U(rng) < 0.6 ? svo::Point::TYPE_UNKNOWN : svo::Point::TYPE_GOOD);
      pt->n_failed_reproj_ = (int)(U(rng) * (cand ? 32 : 17));
      pt->n_succeeded_reproj_ = (int)(U(rng) * 12);
      r.pts.push_back(pt);
      svo::Feature* first = nullptr;
      for (int k = 0; k < kMapKfs; ++k) {
        if (!cand && U(rng) > 0.7) continue;
        const svo::Vector2d px = kfs[k]->w2c(pos);
        const int L = (int)(U(rng) * 3);
        const svo::Vector2d pl{std::round(px[0] / (1 << L)) * (1 << L), std::round(px[1] / (1 << L)) * (1 << L)};
        if (pl[0] < 12 || pl[1] < 12 || pl[0] >= cam->width() - 12 || pl[1] >= cam->height() - 12) continue;
        svo::Feature* f = new svo::Feature(kfs[k].get(), pt, pl, cam->cam2world(pl), L);
        if (U(rng) < 0.12) { f->type = svo::Feature::EDGELET; const double a = 6.283 * U(rng); f->grad = {std::cos(a), std::sin(a)}; }
        pt->addFrameRef(f);
        first = f;
        if (cand) break;  // a converged seed: one observation, not in its keyframe's fts_
        kfs[k]->addFeature(f);
      }
      if (cand && first) r.map.point_candidates_.candidates_.push_back(svo::MapPointCandidates::PointCandidate(pt, first));
      if (U(rng) < 0.25) for (double& x : pt->pos_) x += 0.1 * (U(rng) - 0.5);  // map error: these matches fail
      if (!cand && U(rng) < 0.02) pt->type_ = svo::Point::TYPE_DELETED;
    }
    for (auto& k : kfs) { k->setKeyframe(); r.map.addKeyframe(k); }
    r.cur = render(ctx, cam, {0.08 * (kMapKfs - 1) - 0.04 * s + 0.03, 0.03 * (kMapKfs - 1) + 0.02, 0.03}, 10.0);
    svo::Reprojector::Options opt;
    opt.max_fts = 80 + 40 * s;
    opt.grid_size = s % 2 ? 40 : 30;
    r.reprojector.reset(new svo::Reprojector(cam, r.map, opt, 7 + s));
  }
}

uint64_t digest_reproject(const std::vector<std::unique_ptr<ReprojStream>>& st, size_t* n_matches, size_t* n_new) {
  Digest g;
  *n_matches = *n_new = 0;
  for (const auto& r : st) {
    g.add(r->reprojector->n_matches_);
    g.add(r->reprojector->n_trials_);
    *n_matches += r->reprojector->n_matches_;
    std::vector<svo::FramePtr> kfs(r->map.keyframes_.begin(), r->map.keyframes_.end());
    for (auto& o : r->overlap) {
      int k = -1;
      for (size_t i = 0; i < kfs.size(); ++i) if (kfs[i] == o.first) k = (int)i;
      g.add(k); g.add(o.second);
    }
    for (svo::Feature* f : r->cur->fts_) {
      int p = -1;
      for (size_t i = 0; i < r->pts.size(); ++i) if (r->pts[i] == f->point) p = (int)i;
      g.add(p); g.add(f->px); g.add(f->level); g.add(f->type); g.add(f->grad);
      ++*n_new;
    }
    for (svo::Point* p : r->pts) { g.add(p->type_); g.add(p->n_failed_reproj_); g.add(p->n_succeeded_reproj_); }
    g.add(r->map.trash_points_.size());
    g.add(r->map.point_candidates_.trash_points_.size());
    g.add(r->map.point_candidates_.candidates_.size());
  }
  return g.h;
}

void release(std::vector<std::unique_ptr<ReprojStream>>& st) {  // the map owns its trash and remaining candidates
  for (auto& r : st) {
    std::set<svo::Point*> map_owned(r->map.trash_points_.begin(), r->map.trash_points_.end());
    map_owned.insert(r->map.point_candidates_.trash_points_.begin(), r->map.point_candidates_.trash_points_.end());
    for (auto& c : r->map.point_candidates_.candidates_) map_owned.insert(c.first);
    r->map.emptyTrash();
    for (svo::Point* p : r->pts) if (!map_owned.count(p)) delete p;
  }
}

}  // namespace

int main() {
  try {
    svo::Context ctx(0);
    svo::PinholeCamera cam752(752, 480, 315.5, 315.5, 376.0, 240.0), cam640(640, 480, 320.0, 320.0, 320.0, 240.0);
    std::vector<svo::PinholeCamera*> cams{&cam752, &cam640};

    // depth filter: per object, then batched, on identically built streams
    uint64_t dd[2];
    size_t seeds[2], cands[2];
    for (int run = 0; run < 2; ++run) {
      std::vector<std::unique_ptr<DepthStream>> st;
      build_depth(ctx, cams, st);
      for (int k = 0; k < kDepthFrames; ++k) {
        if (run == 0) {
          for (auto& d : st) d->filter->addFrame(d->frames[k]);  // no mapper thread: addFrame -> updateSeeds
        } else {
          std::vector<svo::DepthFilter*> filters;
          std::vector<svo::FramePtr> frames;
          for (auto& d : st) { filters.push_back(d->filter.get()); frames.push_back(d->frames[k]); }
          svo::streams::updateSeeds(filters, frames);
        }
      }
      dd[run] = digest_depth(st, &seeds[run], &cands[run]);
    }
    printf("depth per-object %016" PRIx64 " seeds %zu candidates %zu\n", dd[0], seeds[0], cands[0]);
    printf("depth batched    %016" PRIx64 " seeds %zu candidates %zu\n", dd[1], seeds[1], cands[1]);

    // reprojector
    uint64_t rd[2];
    size_t matches[2], added[2];
    for (int run = 0; run < 2; ++run) {
      std::vector<std::unique_ptr<ReprojStream>> st;
      build_reproject(ctx, cams, st);
      if (run == 0) {
        for (auto& r : st) r->reprojector->reprojectMap(r->cur, r->overlap);
      } else {
        std::vector<svo::Reprojector*> rp;
        std::vector<svo::FramePtr> frames;
        std::vector<std::vector<std::pair<svo::FramePtr, size_t>>> overlap(st.size());
        for (auto& r : st) { rp.push_back(r->reprojector.get()); frames.push_back(r->cur); }
        svo::streams::reprojectMap(rp, frames, overlap);
        for (size_t s = 0; s < st.size(); ++s) st[s]->overlap = overlap[s];
      }
      rd[run] = digest_reproject(st, &matches[run], &added[run]);
      release(st);
    }
    printf("reproject per-object %016" PRIx64 " matches %zu new features %zu\n", rd[0], matches[0], added[0]);
    printf("reproject batched    %016" PRIx64 " matches %zu new features %zu\n", rd[1], matches[1], added[1]);
    return dd[0] == dd[1] && rd[0] == rd[1] ? 0 : 1;
  } catch (const std::exception& e) {
    fprintf(stderr, "host_streams_demo: %s\n", e.what());
    return 2;
  }
}
