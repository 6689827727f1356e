// oracle/svo_oracle_klt.cpp -- CPU restatement of the two-view initialisation's KLT tracking (TEST INFRASTRUCTURE ONLY,
// built by oracle/klt.mk).  The reference's trackKlt (svo/src/initialization.cpp:127-169) calls
//   cv::calcOpticalFlowPyrLK(ref_img, cur_img, px_ref, px_cur, status, err, Size(30, 30), 4,
//                            TermCriteria(COUNT + EPS, 30, 0.001), OPTFLOW_USE_INITIAL_FLOW)
// on two plain 8-bit images.
//
// [EXT] OpenCV's pyramidal Lucas-Kanade (modules/video/src/lkpyramid.cpp: buildOpticalFlowPyramid, calcScharrDeriv,
// LKTrackerInvoker; J.-Y. Bouguet, "Pyramidal implementation of the Lucas Kanade feature tracker", 2000), restated from
// its published algorithm:
//   pyramid      level 0 = the image; level l+1 = pyrDown(level l): a separable [1 4 6 4 1] filter with reflect-101
//                borders, even rows and columns kept, (sum + 128) >> 8; size ((w+1)/2, (h+1)/2).  Levels stop once the
//                next one would be no larger than the window in either dimension.  Every level is read through a
//                window-wide reflect-101 border.
//   derivatives  Scharr on every level of the previous image: dx = [-1 0 1] across of [3 10 3] down, dy = [3 10 3] across
//                of [-1 0 1] down, reflect-101 borders, int16 pairs; zero outside the level.
//   tracker      coarse to fine; half-window (win-1)/2; window corner floor(pt - halfWin); bilinear weights with 14 bits
//                (cvRound); the reference window sampled once per level (intensity << 5 and derivatives, descaled);
//                A summed in float and scaled by 2^-20; lost when min eigenvalue / win^2 < 1e-4 or det < FLT_EPSILON;
//                per iteration b, delta = A^-1 b, stop when delta.delta <= eps^2 or the iteration limit is reached, and
//                step back half a step when two consecutive steps nearly cancel (both |components| of their sum < 0.01).
//                Out-of-bounds and eigenvalue failures clear the status only at level 0.
// [EXT] summation order: OpenCV's own float sums run in the order of its SIMD lanes, which the tests do not rely on.  The
// sums here are 32 strided partial sums (pixel p of the window into partial p mod 32, in increasing p) combined by
// pairwise halving (partial[i] + partial[i ^ 16], then ^ 8, ^ 4, ^ 2, ^ 1): one order fixed for the oracle and the kernel
// alike, so that the two agree bit for bit.
#include <float.h>
#include <math.h>
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <vector>

namespace {

constexpr int kMaxLevels = 8;  // SVO_B200_MAX_LEVELS
constexpr float kMinEig = 1e-4f;

int reflect101(int p, int len) {  // cv::borderInterpolate(p, len, BORDER_REFLECT_101)
  if (len == 1) return 0;
  while (p < 0 || p >= len) p = p < 0 ? -p : 2 * len - p - 2;
  return p;
}

// A level with a `B`-pixel border on every side (reflect-101 for images, zero for derivatives).
struct Padded {
  int w = 0, h = 0, B = 0;
  std::vector<uint8_t> img;   // (w+2B) x (h+2B)
  std::vector<int16_t> der;   // (w+2B) x (h+2B) x 2, or empty
  int stride() const { return w + 2 * B; }
  const uint8_t* I(int x, int y) const { return img.data() + (size_t)(y + B) * stride() + (x + B); }
  const int16_t* D(int x, int y) const { return der.data() + ((size_t)(y + B) * stride() + (x + B)) * 2; }
};

int level_sizes(int w, int h, int max_level, int win, int* ws, int* hs) {
  int n = 0;
  for (int level = 0; level <= max_level && level < kMaxLevels; ++level) {
    ws[level] = w; hs[level] = h;
    n = level + 1;
    w = (w + 1) / 2; h = (h + 1) / 2;
    if (w <= win || h <= win) break;
  }
  return n;
}

std::vector<uint8_t> pyr_down(const std::vector<uint8_t>& src, int w, int h, int dw, int dh) {
  static const int k[5] = {1, 4, 6, 4, 1};
  std::vector<int> rows((size_t)h * dw);
  for (int y = 0; y < h; ++y)
    for (int x = 0; x < dw; ++x) {
      int s = 0;
      for (int j = 0; j < 5; ++j) s += k[j] * src[(size_t)y * w + reflect101(2 * x + j - 2, w)];
      rows[(size_t)y * dw + x] = s;
    }
  std::vector<uint8_t> dst((size_t)dw * dh);
  for (int y = 0; y < dh; ++y)
    for (int x = 0; x < dw; ++x) {
      int s = 0;
      for (int i = 0; i < 5; ++i) s += k[i] * rows[(size_t)reflect101(2 * y + i - 2, h) * dw + x];
      dst[(size_t)y * dw + x] = (uint8_t)((s + 128) >> 8);
    }
  return dst;
}

void scharr(const std::vector<uint8_t>& s, int w, int h, std::vector<int16_t>& d) {
  d.assign((size_t)w * h * 2, 0);
  auto at = [&](int x, int y) { return (int)s[(size_t)reflect101(y, h) * w + reflect101(x, w)]; };
  for (int y = 0; y < h; ++y)
    for (int x = 0; x < w; ++x) {
      auto sm = [&](int xx) { return (at(xx, y - 1) + at(xx, y + 1)) * 3 + at(xx, y) * 10; };
      auto df = [&](int xx) { return at(xx, y + 1) - at(xx, y - 1); };
      d[((size_t)y * w + x) * 2] = (int16_t)(sm(x + 1) - sm(x - 1));
      d[((size_t)y * w + x) * 2 + 1] = (int16_t)((df(x + 1) + df(x - 1)) * 3 + df(x) * 10);
    }
}

int build(const uint8_t* img, int w, int h, int max_level, int win, bool deriv, std::vector<Padded>& pyr,
          std::vector<std::vector<uint8_t>>* plain = nullptr, std::vector<std::vector<int16_t>>* plain_der = nullptr) {
  int ws[kMaxLevels], hs[kMaxLevels];
  const int n = level_sizes(w, h, max_level, win, ws, hs);
  pyr.assign(n, Padded());
  std::vector<uint8_t> cur(img, img + (size_t)w * h);
  for (int l = 0; l < n; ++l) {
    if (l > 0) cur = pyr_down(cur, ws[l - 1], hs[l - 1], ws[l], hs[l]);
    Padded& P = pyr[l];
    P.w = ws[l]; P.h = hs[l]; P.B = win;
    const int S = P.stride(), R = P.h + 2 * win;
    P.img.resize((size_t)S * R);
    for (int y = 0; y < R; ++y)
      for (int x = 0; x < S; ++x) P.img[(size_t)y * S + x] = cur[(size_t)reflect101(y - win, P.h) * P.w + reflect101(x - win, P.w)];
    std::vector<int16_t> d;
    if (deriv) {
      scharr(cur, P.w, P.h, d);
      P.der.assign((size_t)S * R * 2, 0);
      for (int y = 0; y < P.h; ++y) memcpy(&P.der[((size_t)(y + win) * S + win) * 2], &d[(size_t)y * P.w * 2], (size_t)P.w * 4);
    }
    if (plain) plain->push_back(cur);
    if (plain_der) plain_der->push_back(d);
  }
  return n;
}

inline int descale(int x, int n) { return (x + (1 << (n - 1))) >> n; }

// 32 strided partial sums combined pairwise (see the file header).
struct LaneSum {
  float v[32];
  LaneSum() { for (float& x : v) x = 0.f; }
  float total() const {
    float a[32];
    memcpy(a, v, sizeof a);
    for (int off = 16; off >= 1; off >>= 1) {
      float b[32];
      for (int i = 0; i < 32; ++i) b[i] = a[i] + a[i ^ off];
      memcpy(a, b, sizeof a);
    }
    return a[0];
  }
};

inline double bounds_margin(float x, float y, int w, int h, int win) {
  return std::min(std::min((double)x + win, (double)w - x), std::min((double)y + win, (double)h - y));
}

}  // namespace

extern "C" {

/* Exit reasons, as SVO_B200_KLT_* of include/svo_b200.h. */
enum { KLT_CONVERGED = 0, KLT_HALF_STEP = 1, KLT_MAX_ITER = 2, KLT_OUT_OF_BOUNDS = 3, KLT_SMALL_EIG = 4, KLT_NOT_RUN = -1 };

/* Level count and sizes of the LK pyramid (ws, hs: kMaxLevels ints). */
int orc_klt_levels(int w, int h, int max_level, int win, int* ws, int* hs) { return level_sizes(w, h, max_level, win, ws, hs); }

/* The levels (interior, concatenated) and, if der_out, the Scharr derivatives of each level (interleaved dx, dy). */
int orc_klt_pyramid(const uint8_t* img, int w, int h, int max_level, int win, uint8_t* img_out, int16_t* der_out) {
  std::vector<Padded> pyr;
  std::vector<std::vector<uint8_t>> plain;
  std::vector<std::vector<int16_t>> plain_der;
  const int n = build(img, w, h, max_level, win, der_out != nullptr, pyr, &plain, &plain_der);
  for (int l = 0; l < n; ++l) {
    memcpy(img_out, plain[l].data(), plain[l].size());
    img_out += plain[l].size();
    if (der_out) { memcpy(der_out, plain_der[l].data(), plain_der[l].size() * 2); der_out += plain_der[l].size(); }
  }
  return n;
}

/* calcOpticalFlowPyrLK(prev, next, prev_pts, next_pts, ..., Size(win, win), max_level, (COUNT + EPS, max_iter, eps),
 * OPTFLOW_USE_INITIAL_FLOW) for n points.  next_pts: in = initial flow, out = tracked.  Per point: status, reason (how
 * level 0 ended); per point and level (kMaxLevels each, KLT_NOT_RUN / 0 / NaN where not built): level_reason, iters (steps
 * taken), and 5 margins -- min |eps^2 - delta.delta| and min |max(|sum_x|, |sum_y|) - 0.01| over the level's steps (the
 * convergence and half-step tests), minEig - 1e-4 and det - FLT_EPSILON, and the smallest distance of a tested window
 * corner to the bounds it is tested against (+inf where a test did not run).  Returns the number of levels. */
int orc_klt_track(const uint8_t* prev, const uint8_t* next, int w, int h, int max_level, int win, int max_iter, double eps,
                  int n, const float* prev_pts, float* next_pts, uint8_t* status, int* reason, int* level_reason, int* iters,
                  double* margins) {
  std::vector<Padded> P, N;
  const int nl = std::min(build(prev, w, h, max_level, win, true, P), build(next, w, h, max_level, win, false, N));
  const int maxL = nl - 1;
  max_iter = std::min(std::max(max_iter, 0), 100);
  eps = std::min(std::max(eps, 0.), 10.);
  const double eps2 = eps * eps;
  const float hw = (win - 1) * 0.5f;
  const int W_BITS = 14, W_BITS1 = 14;
  const float FLT_SCALE = 1.f / (1 << 20);
  const double inf = INFINITY;
  std::vector<int16_t> Iw((size_t)win * win), dIw((size_t)win * win * 2);
  for (int i = 0; i < n; ++i) {
    status[i] = 1;
    reason[i] = KLT_NOT_RUN;
    for (int l = 0; l < kMaxLevels; ++l) {
      level_reason[i * kMaxLevels + l] = KLT_NOT_RUN;
      iters[i * kMaxLevels + l] = 0;
      for (int m = 0; m < 5; ++m) margins[(i * kMaxLevels + l) * 5 + m] = l < nl ? inf : NAN;
    }
    for (int level = maxL; level >= 0; --level) {
      const Padded &I = P[level], &J = N[level];
      double* mg = margins + (i * kMaxLevels + level) * 5;
      int& why = level_reason[i * kMaxLevels + level];
      int& it = iters[i * kMaxLevels + level];
      const float sc = (float)(1. / (1 << level));
      float px = prev_pts[2 * i] * sc, py = prev_pts[2 * i + 1] * sc;
      float nx, ny;
      if (level == maxL) { nx = next_pts[2 * i] * sc; ny = next_pts[2 * i + 1] * sc; }
      else { nx = next_pts[2 * i] * 2.f; ny = next_pts[2 * i + 1] * 2.f; }
      next_pts[2 * i] = nx; next_pts[2 * i + 1] = ny;
      px -= hw; py -= hw;
      int ipx = (int)floorf(px), ipy = (int)floorf(py);
      mg[4] = std::min(mg[4], fabs(bounds_margin(px, py, I.w, I.h, win)));
      if (ipx < -win || ipx >= I.w || ipy < -win || ipy >= I.h) {
        why = KLT_OUT_OF_BOUNDS;
        if (level == 0) status[i] = 0;
        continue;
      }
      float a = px - ipx, b = py - ipy;
      int iw00 = (int)lrintf((1.f - a) * (1.f - b) * (1 << W_BITS));
      int iw01 = (int)lrintf(a * (1.f - b) * (1 << W_BITS));
      int iw10 = (int)lrintf((1.f - a) * b * (1 << W_BITS));
      int iw11 = (1 << W_BITS) - iw00 - iw01 - iw10;
      LaneSum sA11, sA12, sA22;
      for (int p = 0; p < win * win; ++p) {
        const int x = p % win, y = p / win;
        const uint8_t* s = I.I(ipx + x, ipy + y);
        const int16_t* d = I.D(ipx + x, ipy + y);
        const int st = I.stride(), ds = st * 2;
        const int ival = descale(s[0] * iw00 + s[1] * iw01 + s[st] * iw10 + s[st + 1] * iw11, W_BITS1 - 5);
        const int ixval = descale(d[0] * iw00 + d[2] * iw01 + d[ds] * iw10 + d[ds + 2] * iw11, W_BITS1);
        const int iyval = descale(d[1] * iw00 + d[3] * iw01 + d[ds + 1] * iw10 + d[ds + 3] * iw11, W_BITS1);
        Iw[p] = (int16_t)ival; dIw[2 * p] = (int16_t)ixval; dIw[2 * p + 1] = (int16_t)iyval;
        sA11.v[p & 31] += (float)(ixval * ixval);
        sA12.v[p & 31] += (float)(ixval * iyval);
        sA22.v[p & 31] += (float)(iyval * iyval);
      }
      const float A11 = sA11.total() * FLT_SCALE, A12 = sA12.total() * FLT_SCALE, A22 = sA22.total() * FLT_SCALE;
      float D = A11 * A22 - A12 * A12;
      const float minEig = (A22 + A11 - sqrtf((A11 - A22) * (A11 - A22) + 4.f * A12 * A12)) / (float)(2 * win * win);
      mg[2] = (double)minEig - (double)kMinEig;
      mg[3] = (double)D - (double)FLT_EPSILON;
      if (minEig < kMinEig || D < FLT_EPSILON) {
        why = KLT_SMALL_EIG;
        if (level == 0) status[i] = 0;
        continue;
      }
      D = 1.f / D;
      nx -= hw; ny -= hw;
      float pdx = 0.f, pdy = 0.f;
      why = KLT_MAX_ITER;
      for (int j = 0; j < max_iter; ++j) {
        const int inx = (int)floorf(nx), iny = (int)floorf(ny);
        mg[4] = std::min(mg[4], fabs(bounds_margin(nx, ny, J.w, J.h, win)));
        if (inx < -win || inx >= J.w || iny < -win || iny >= J.h) {
          why = KLT_OUT_OF_BOUNDS;
          if (level == 0) status[i] = 0;
          break;
        }
        a = nx - inx; b = ny - iny;
        iw00 = (int)lrintf((1.f - a) * (1.f - b) * (1 << W_BITS));
        iw01 = (int)lrintf(a * (1.f - b) * (1 << W_BITS));
        iw10 = (int)lrintf((1.f - a) * b * (1 << W_BITS));
        iw11 = (1 << W_BITS) - iw00 - iw01 - iw10;
        LaneSum sb1, sb2;
        for (int p = 0; p < win * win; ++p) {
          const int x = p % win, y = p / win, st = J.stride();
          const uint8_t* s = J.I(inx + x, iny + y);
          const int diff = descale(s[0] * iw00 + s[1] * iw01 + s[st] * iw10 + s[st + 1] * iw11, W_BITS1 - 5) - Iw[p];
          sb1.v[p & 31] += (float)(diff * dIw[2 * p]);
          sb2.v[p & 31] += (float)(diff * dIw[2 * p + 1]);
        }
        const float b1 = sb1.total() * FLT_SCALE, b2 = sb2.total() * FLT_SCALE;
        const float dx = (A12 * b2 - A22 * b1) * D, dy = (A12 * b1 - A11 * b2) * D;
        nx += dx; ny += dy;
        next_pts[2 * i] = nx + hw; next_pts[2 * i + 1] = ny + hw;
        it = j + 1;
        const double dd = (double)dx * dx + (double)dy * dy;
        mg[0] = std::min(mg[0], fabs(eps2 - dd));
        if (dd <= eps2) { why = KLT_CONVERGED; break; }
        if (j > 0) {
          const float sx = dx + pdx, sy = dy + pdy;
          mg[1] = std::min(mg[1], fabs(std::max((double)fabsf(sx), (double)fabsf(sy)) - 0.01));
          if ((double)fabsf(sx) < 0.01 && (double)fabsf(sy) < 0.01) {
            next_pts[2 * i] -= dx * 0.5f; next_pts[2 * i + 1] -= dy * 0.5f;
            why = KLT_HALF_STEP;
            break;
          }
        }
        pdx = dx; pdy = dy;
      }
    }
    reason[i] = level_reason[i * kMaxLevels];
  }
  return nl;
}

}  // extern "C"
