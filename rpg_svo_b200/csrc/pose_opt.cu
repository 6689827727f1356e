// rpg_svo_b200/csrc/pose_opt.cu -- pose_optimizer::optimizeGaussNewton on sm_90a.
//
// Replaces svo/src/pose_optimizer.cpp:28-161: robust (Tukey weights, MAD scale) Gauss-Newton on the
// unit-plane reprojection error of one frame, outlier culling, covariance and the median error
// statistics.  One CTA per frame runs the whole optimisation on the device (<= n_iter iterations without a
// host round trip); a batch of frames is one launch (grid = #frames).
//   * the per-observation constants -- point position, project2d(f), 1/(1<<level) -- are computed once and
//     kept in shared memory (SoA, conflict free): an iteration re-reads 48 B per observation from shared
//     memory instead of 52 B from global memory and performs no division but the two of project2d(xyz),
//     which are a Newton reciprocal + one correction step (correctly rounded, like the reference's `/`);
//   * every iteration ends in a 28-value block reduction (21 unique A entries, 6 b entries, chi2: transposed
//     warp shuffles, one shared-memory hop, ONE barrier), after which warp 0 alone -- all lanes redundantly, in
//     registers -- factorises the 6x6 system, applies T <- exp(dT) * T and the accept / rollback rule and
//     publishes the pose (second barrier);
//   * the three medians ([EXT] vk::getMedian = nth_element at floor(n/2)) are exact order statistics by an
//     MSB-first radix select on order-preserving keys that stops as soon as one candidate is left (3-4 passes of
//     8 bits instead of 8); error_init and error_final are selected in the same passes.
// All arithmetic is f64 except the f32 error vector / Tukey weight, as in the reference.
#include <cstdio>
#include <cstring>
#include <vector>

#include "ctx.h"
#include "svo_math.cuh"

namespace svo {

#ifndef SVO_SIA_DEBUG
#define SVO_SIA_DEBUG 0  // instrumented build (SVO_B200_EXTRA_NVCC_FLAGS=-DSVO_SIA_DEBUG=1): thread 0 of frame 0 prints clock64 section timings
#endif
#if SVO_SIA_DEBUG
#define PO_DBG(...) __VA_ARGS__
#else
#define PO_DBG(...)
#endif

constexpr int kPoThreads = 512;
constexpr int kPoWarps = kPoThreads / 32;
constexpr int kPoK = 28;

struct PoseOptParams {
  const double* f;      // all frames' observations, concatenated
  const double* pos;
  const int* level;
  uint8_t* has_point;   // in/out
  const int* obs_offset;  // B+1
  const double* fx;       // B: cam->errorMultiplier2()
  int n_iter;
  double reproj_thresh;
  double* T_io;  // B*12
  svo_b200_pose_opt_result* out;  // B
};

struct PoseOptShared {
  double part[kPoWarps * kPoK];
  double sums[kPoK];
  double R[9], t[3];
  double A[36];
  double cov[36];
  double med[2];
  Pose T, T_old;   // frame->T_f_w_ and the roll-back copy (warp 0)
  double chi2;
  Solver6 sol;
  double x[8];
  int done, iters, n_pivoted, cov_pivoted;  // n_pivoted / cov_pivoted: which solves took the fallback (reported)
  unsigned hist[2][256];
  int sel_bin[2], sel_k[2], sel_cnt[2];
};

// [EXT] vk::robust_cost::TukeyWeightFunction::value, b = 4.6851f
__device__ __forceinline__ float tukey_weight(float x) {
  const float b_square = __fmul_rn(4.6851f, 4.6851f);
  const float x_square = __fmul_rn(x, x);
  if (x_square <= b_square) {
    const float tmp = __fsub_rn(1.0f, __fdiv_rn(x_square, b_square));
    return __fmul_rn(tmp, tmp);
  }
  return 0.0f;
}

// Per-warp partial sums of K values into s.part, then ONE barrier.  Afterwards po_total(k) (any thread) adds the
// per-warp partials of value k in warp order.
template <int K>
__device__ __forceinline__ void po_partials(double (&v)[K], PoseOptShared& s) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (K == kPoK) {  // 28 = 16 + 8 (transposed reductions) + 4 (tree)
    double a16[16], a8[8], a4[4];
#pragma unroll
    for (int k = 0; k < 16; ++k) a16[k] = v[k];
#pragma unroll
    for (int k = 0; k < 8; ++k) a8[k] = v[16 + k];
#pragma unroll
    for (int k = 0; k < 4; ++k) a4[k] = v[24 + k];
    warp_reduce_t<16>(a16);
    warp_reduce_t<8>(a8);
    warp_sum<4>(a4);
    if ((lane & 1) == 0) s.part[warp * kPoK + (lane >> 1)] = a16[0];
    if ((lane & 3) == 0) s.part[warp * kPoK + 16 + (lane >> 2)] = a8[0];
    if (lane == 0) {
#pragma unroll
      for (int k = 0; k < 4; ++k) s.part[warp * kPoK + 24 + k] = a4[k];
    }
  } else {
    warp_sum<K>(v);
    if (lane == 0) {
#pragma unroll
      for (int k = 0; k < K; ++k) s.part[warp * kPoK + k] = v[k];
    }
  }
  __syncthreads();
}
__device__ __forceinline__ double po_total(const PoseOptShared& s, int k) {
  double acc = 0.0;
#pragma unroll
  for (int w = 0; w < kPoWarps; ++w) acc += s.part[w * kPoK + k];
  return acc;
}

// k-th smallest (0-based) of the valid entries of NA arrays at once (same validity flags, same k): exact order
// statistics by MSB-first radix select on order-preserving 64-bit keys, 8 bits per pass, shared-memory histograms,
// warp-parallel bin scan.  An array drops out as soon as its selected bin holds a single candidate (that element is
// then found in the next sweep).  Results in s.med[a] (NaN if there are no more than k valid entries).
__device__ __forceinline__ unsigned long long order_key(double d) {
  const unsigned long long u = (unsigned long long)__double_as_longlong(d);
  return (u >> 63) ? ~u : (u | 0x8000000000000000ULL);
}
template <int NA>
__device__ void block_kth(const double* const (&v)[NA], const uint8_t* valid, int N, int k, PoseOptShared& s) {
  unsigned long long prefix[NA], mask[NA];
  int kk[NA], state[NA];  // state: 0 = selecting, 1 = one candidate left (pick it up in the next sweep), 2 = done
#pragma unroll
  for (int a = 0; a < NA; ++a) { prefix[a] = 0; mask[a] = 0; kk[a] = k; state[a] = 0; }
  for (int pass = 7; pass >= -1; --pass) {
    bool any = false;
#pragma unroll
    for (int a = 0; a < NA; ++a) any = any || state[a] != 2;
    if (!any) break;
    const int shift = pass * 8;
    for (int b = threadIdx.x; b < 256 * NA; b += blockDim.x) (&s.hist[0][0])[b] = 0;
    __syncthreads();
    for (int i = threadIdx.x; i < N; i += blockDim.x) {
      if (!valid[i]) continue;
#pragma unroll
      for (int a = 0; a < NA; ++a) {
        if (state[a] == 2) continue;
        const unsigned long long key = order_key(v[a][i]);
        if ((key & mask[a]) != prefix[a]) continue;
        if (state[a] == 1 || pass < 0) s.med[a] = v[a][i];  // the single remaining candidate (ties: identical values)
        else atomicAdd(&s.hist[a][(unsigned)(key >> shift) & 255u], 1u);
      }
    }
    __syncthreads();
    if (threadIdx.x < 32 * NA) {  // warp a scans array a: lane l owns bins [8l, 8l+8)
      const int a = threadIdx.x >> 5, lane = threadIdx.x & 31;
      const int st_a = (NA == 1 || a == 0) ? state[0] : state[NA - 1];
      const int kk_a = (NA == 1 || a == 0) ? kk[0] : kk[NA - 1];
      if (st_a == 0 && pass >= 0) {
        unsigned loc[8], sum = 0;
#pragma unroll
        for (int j = 0; j < 8; ++j) { loc[j] = s.hist[a][8 * lane + j]; sum += loc[j]; }
        unsigned inc = sum;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const unsigned t = __shfl_up_sync(0xffffffffu, inc, o);
          if (lane >= o) inc += t;
        }
        const unsigned exc = inc - sum;
        const int target = kk_a;
        const unsigned hit = __ballot_sync(0xffffffffu, inc > (unsigned)target);
        if (hit == 0) {
          if (lane == 0) s.sel_bin[a] = -1;
        } else if (lane == __ffs(hit) - 1) {
          unsigned cum = exc;
          int bin = 8 * lane;
          unsigned cnt = 0;
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            if (cum + loc[j] > (unsigned)target) { bin = 8 * lane + j; cnt = loc[j]; break; }
            cum += loc[j];
          }
          s.sel_bin[a] = bin;
          s.sel_k[a] = target - (int)cum;
          s.sel_cnt[a] = (int)cnt;
        }
      }
    }
    __syncthreads();
#pragma unroll
    for (int a = 0; a < NA; ++a) {
      if (state[a] == 1 || (state[a] == 0 && pass < 0)) { state[a] = 2; continue; }
      if (state[a] != 0) continue;
      if (s.sel_bin[a] < 0) {  // fewer than k+1 valid entries
        if (threadIdx.x == 0) s.med[a] = __longlong_as_double(0x7ff8000000000000LL);
        state[a] = 2;
        continue;
      }
      prefix[a] |= (unsigned long long)s.sel_bin[a] << shift;
      mask[a] |= 0xffULL << shift;
      kk[a] = s.sel_k[a];
      if (s.sel_cnt[a] == 1 || pass == 0) state[a] = 1;  // unique candidate, or all 64 bits fixed: equal values
    }
  }
  __syncthreads();
}

// SoA view of one frame's observations in shared memory
struct PoObs {
  double *px, *py, *pz, *fxn, *fyn, *sic, *work, *init;
  uint8_t* valid;
};

// rcp_rn seeds its Newton steps with the f32 reciprocal: inside (1e-30, 1e30) that seed is finite and nonzero and the
// result is the correctly rounded 1/d; outside it (or for 0, inf, NaN) the seed is 0 or inf and only IEEE division is 1/d.
__device__ __forceinline__ bool rcp_in_range(double d) {
  const double a = fabs(d);
  return a > 1e-30 && a < 1e30;
}

// e = (project2d(f) - project2d(T_f_w * pos)) / (1 << level)  (:52-54, :82-85, :135-137); xyz_f out
__device__ __forceinline__ void reproj_error(const PoObs& o, int i, const double (&R)[9], const double (&t)[3], double& ex,
                                             double& ey, double (&p)[3], double& z_inv) {
  const double X = o.px[i], Y = o.py[i], Z = o.pz[i];
  p[0] = R[0] * X + R[1] * Y + R[2] * Z + t[0];
  p[1] = R[3] * X + R[4] * Y + R[5] * Z + t[1];
  p[2] = R[6] * X + R[7] * Y + R[8] * Z + t[2];
  const double sic = o.sic[i];
  double qx, qy;
  if (rcp_in_range(p[2])) {
    z_inv = rcp_rn(p[2]);
    qx = div_rn(p[0], p[2], z_inv);
    qy = div_rn(p[1], p[2], z_inv);
  } else {  // a point on, behind-and-near or far beyond the camera plane: the reference's IEEE division
    z_inv = 1.0 / p[2];
    qx = p[0] / p[2];
    qy = p[1] / p[2];
  }
  ex = (o.fxn[i] - qx) * sic;
  ey = (o.fyn[i] - qy) * sic;
}

__global__ void __launch_bounds__(kPoThreads) pose_opt_kernel(PoseOptParams P) {
  extern __shared__ __align__(16) unsigned char po_smem[];
  PoseOptShared& s = *reinterpret_cast<PoseOptShared*>(po_smem);
  const int fr = blockIdx.x;
  const int o0 = P.obs_offset[fr], N = P.obs_offset[fr + 1] - o0;
  const int Np = (N + 1) & ~1;
  PoObs o;
  o.px = reinterpret_cast<double*>(po_smem + ((sizeof(PoseOptShared) + 15) & ~size_t(15)));
  o.py = o.px + Np; o.pz = o.py + Np; o.fxn = o.pz + Np; o.fyn = o.fxn + Np; o.sic = o.fyn + Np;
  o.work = o.sic + Np; o.init = o.work + Np;
  o.valid = reinterpret_cast<uint8_t*>(o.init + Np);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const double fx = P.fx[fr];
  uint8_t* has_point = P.has_point + o0;
  PO_DBG(long long tc[8]; tc[0] = clock64();)

  // ---- per-observation constants, once ------------------------------------------------------------
  // (the loads of an observation do not wait for its has_point flag, and two observations per thread are in flight
  // together: the phase is a chain of first-touch global loads, not arithmetic)
  double cnt[1] = {0.0};
  for (int i0 = tid; i0 < N; i0 += 2 * kPoThreads) {
    const int i1 = i0 + kPoThreads;
    const bool in1 = i1 < N;
    const size_t g0 = (size_t)(o0 + i0), g1 = (size_t)(o0 + (in1 ? i1 : i0));
    const uint8_t hp0 = has_point[i0], hp1 = in1 ? has_point[i1] : (uint8_t)0;
    const double a0 = P.pos[3 * g0], a1 = P.pos[3 * g0 + 1], a2 = P.pos[3 * g0 + 2];
    const double f00 = P.f[3 * g0], f01 = P.f[3 * g0 + 1], f02 = P.f[3 * g0 + 2];
    const int l0 = P.level[g0];
    const double b0 = P.pos[3 * g1], b1 = P.pos[3 * g1 + 1], b2 = P.pos[3 * g1 + 2];
    const double f10 = P.f[3 * g1], f11 = P.f[3 * g1 + 1], f12 = P.f[3 * g1 + 2];
    const int l1 = P.level[g1];
    o.valid[i0] = hp0;
    if (hp0) {
      o.px[i0] = a0; o.py[i0] = a1; o.pz[i0] = a2;
      o.fxn[i0] = f00 / f02;  // vk::project2d(f)
      o.fyn[i0] = f01 / f02;
      o.sic[i0] = 1.0 / (double)(1 << l0);
      cnt[0] += 1.0;
    }
    if (in1) {
      o.valid[i1] = hp1;
      if (hp1) {
        o.px[i1] = b0; o.py[i1] = b1; o.pz[i1] = b2;
        o.fxn[i1] = f10 / f12;
        o.fyn[i1] = f11 / f12;
        o.sic[i1] = 1.0 / (double)(1 << l1);
        cnt[0] += 1.0;
      }
    }
  }
  // pose: every thread derives R, t from the input itself (same arithmetic everywhere)
  double R[9], t[3];
  {
    const Pose T0 = pose_from_rt12(P.T_io + 12 * (size_t)fr);
    qmatrix(T0.q, R);
    t[0] = T0.t[0]; t[1] = T0.t[1]; t[2] = T0.t[2];
    if (tid == 0) { s.T = T0; s.T_old = T0; s.chi2 = 0.0; }
  }
  if (tid == 0) {
    s.done = 0; s.iters = 0; s.n_pivoted = 0;
    for (int k = 0; k < 36; ++k) s.A[k] = 0.0;
  }
  po_partials<1>(cnt, s);
  const int num_obs = (int)po_total(s, 0);
  if (num_obs == 0) {  // errors.empty() -> return (:57-58)
    if (tid == 0) {
      svo_b200_pose_opt_result r;
      memset(&r, 0, sizeof(r));
      P.out[fr] = r;
    }
    return;
  }
  PO_DBG(tc[1] = clock64();)
  // ---- scale of the error for robust estimation (:47-60) ------------------------------------
  for (int i = tid; i < N; i += kPoThreads) {
    if (!o.valid[i]) continue;
    double ex, ey, p[3], zi;
    reproj_error(o, i, R, t, ex, ey, p, zi);
    o.work[i] = (double)(float)sqrt(ex * ex + ey * ey);  // errors.push_back(e.norm()) -> float
  }
  __syncthreads();
  {
    const double* const arr[1] = {o.work};
    block_kth<1>(arr, o.valid, N, num_obs / 2, s);
  }
  // [EXT] MADScaleEstimator: 1.48f * median (float arithmetic)
  const double estimated_scale = (double)__fmul_rn(1.48f, (float)s.med[0]);
  double scale = estimated_scale;

  PO_DBG(tc[2] = clock64();)
  // ---- Gauss-Newton (:63-121) -------------------------------------------------------------------
  for (int iter = 0; iter < P.n_iter; ++iter) {
    if (iter == 5) scale = 0.85 / fx;  // (:69-70)
    const bool scale_fast = rcp_in_range(scale);  // a float-subnormal or zero MAD scale divides by IEEE rules
    const double scale_rcp = scale_fast ? rcp_rn(scale) : 0.0;
    double acc[kPoK];
#pragma unroll
    for (int k = 0; k < kPoK; ++k) acc[k] = 0.0;
    for (int i = tid; i < N; i += kPoThreads) {
      if (!o.valid[i]) continue;
      double ex, ey, p[3], z_inv;
      reproj_error(o, i, R, t, ex, ey, p, z_inv);
      const double sic = o.sic[i];
      // Frame::jacobian_xyz2uv (frame.h:116-138), then J *= sqrt_inv_cov
      const double x = p[0], y = p[1], z_inv_2 = z_inv * z_inv;
      double J0[6], J1[6];
      J0[0] = -z_inv; J0[1] = 0.0; J0[2] = x * z_inv_2; J0[3] = y * J0[2]; J0[4] = -(1.0 + x * J0[2]); J0[5] = y * z_inv;
      J1[0] = 0.0; J1[1] = -z_inv; J1[2] = y * z_inv_2; J1[3] = 1.0 + y * J1[2]; J1[4] = -J0[3]; J1[5] = -x * z_inv;
#pragma unroll
      for (int k = 0; k < 6; ++k) { J0[k] *= sic; J1[k] *= sic; }
      const double e_sq = ex * ex + ey * ey;
      if (iter == 0) o.init[i] = e_sq;  // chi2_vec_init (:87-88)
      const double en = sqrt(e_sq);
      const double w = (double)tukey_weight((float)(scale_fast ? div_rn(en, scale, scale_rcp) : en / scale));  // e.norm() / scale, correctly rounded
      int idx = 0;
#pragma unroll
      for (int r = 0; r < 6; ++r)
#pragma unroll
        for (int c = r; c < 6; ++c, ++idx) acc[idx] += (J0[r] * J0[c] + J1[r] * J1[c]) * w;
#pragma unroll
      for (int r = 0; r < 6; ++r) acc[21 + r] -= (J0[r] * ex + J1[r] * ey) * w;
      acc[27] += e_sq * w;
    }
    po_partials<kPoK>(acc, s);  // barrier A
    if (warp == 0) {
      // warp 0: totals (lane k adds value k over the warps), then every lane runs the 6x6 solve and the update
      // redundantly in registers; lane 0 publishes
      if (lane < kPoK) s.sums[lane] = po_total(s, lane);
      __syncwarp();
      double h[21], b[6];
#pragma unroll
      for (int k = 0; k < 21; ++k) h[k] = s.sums[k];
#pragma unroll
      for (int k = 0; k < 6; ++k) b[k] = s.sums[21 + k];
      const double new_chi2 = s.sums[27];
      if (lane == 0) {
#pragma unroll
        for (int r = 0; r < 6; ++r)
#pragma unroll
          for (int c = r; c < 6; ++c) { s.A[r * 6 + c] = h[upper_idx(r, c)]; s.A[c * 6 + r] = h[upper_idx(r, c)]; }
      }
      double dT[6];
      Fact6 F;
      if (fact6_compute_upper(h, F)) {
        fact6_solve(F, b, dT);
      } else {  // degenerate A: the pivoted Eigen-like LDL^T, through shared memory
        __syncwarp();
        if (lane == 0) {
          for (int k = 0; k < 36; ++k) s.sol.ldl[k] = s.A[k];
          ldlt6_factor(s.sol.ldl, s.sol.tr);
          for (int k = 0; k < 6; ++k) s.x[k] = b[k];
          ldlt6_solve(s.sol.ldl, s.sol.tr, s.x);
          s.n_pivoted++;
        }
        __syncwarp();
#pragma unroll
        for (int k = 0; k < 6; ++k) dT[k] = s.x[k];
      }
      int done = 0;
      Pose T = s.T;
      __syncwarp();
      if ((iter > 0 && new_chi2 > s.chi2) || isnan(dT[0])) {
        T = s.T_old;  // roll-back (:100-107)
        done = 1;
        __syncwarp();
        if (lane == 0) s.T = T;
      } else {
        const Pose Tn = pose_mul_fast(se3_exp_fast(dT), T);  // exp(dT) * T  (:110)
        double m = 0;
#pragma unroll
        for (int k = 0; k < 6; ++k) m = fmax(m, fabs(dT[k]));
        if (m <= 0.0000000001) done = 1;  // EPS (global.h:77)
        __syncwarp();
        if (lane == 0) { s.T_old = T; s.T = Tn; s.chi2 = new_chi2; }
        T = Tn;
      }
      if (lane == 0) {
        qmatrix(T.q, s.R);
        s.t[0] = T.t[0]; s.t[1] = T.t[1]; s.t[2] = T.t[2];
        s.done = done;
        s.iters++;
      }
    }
    __syncthreads();  // barrier B
#pragma unroll
    for (int k = 0; k < 9; ++k) R[k] = s.R[k];
    t[0] = s.t[0]; t[1] = s.t[1]; t[2] = s.t[2];
    if (s.done) break;
  }

  PO_DBG(tc[3] = clock64();)
  // ---- remove measurements with too large reprojection error (:129-145) ------------------------
  const double thresh = P.reproj_thresh / fx;
  double del[1] = {0.0};
  for (int i = tid; i < N; i += kPoThreads) {
    if (!o.valid[i]) continue;
    double ex, ey, p[3], zi;
    reproj_error(o, i, R, t, ex, ey, p, zi);
    const double e_sq = ex * ex + ey * ey;
    o.work[i] = e_sq;  // chi2_vec_final
    if (sqrt(e_sq) > thresh) del[0] += 1.0;
  }
  po_partials<1>(del, s);
  const int n_deleted = (int)po_total(s, 0);
  // medians use the pre-culling validity flags: both vectors hold one entry per original observation
  {
    const double* const arr[2] = {o.init, o.work};
    block_kth<2>(arr, o.valid, N, num_obs / 2, s);
  }
  PO_DBG(tc[4] = clock64();)
  const double med_init = (P.n_iter > 0) ? s.med[0] : 0.0;
  const double med_final = s.med[1];
  for (int i = tid; i < N; i += kPoThreads)
    if (o.valid[i] && sqrt(o.work[i]) > thresh) has_point[i] = 0;  // point = NULL

  // Cov_ = (A * fx^2)^-1  (:125-126).  Warp 0: every lane factorises A fx^2 (register LDL^T, redundantly), lane j < 6
  // solves for the unit vector e_j = column j of the inverse -- ~0.8 K cycles instead of a one-thread elimination
  // with 36 dependent divisions (9.5 K).  A degenerate A falls back to Gauss-Jordan with partial pivoting.
  if (warp == 0) {
    const double f2 = fx * fx;
    double h[21];
    {
      int idx = 0;
#pragma unroll
      for (int r = 0; r < 6; ++r)
#pragma unroll
        for (int c = r; c < 6; ++c, ++idx) h[idx] = s.A[r * 6 + c] * f2;
    }
    Fact6 F;
    const bool ok = fact6_compute_upper(h, F);
    if (lane == 0) s.cov_pivoted = ok ? 0 : 1;
    if (ok) {
      double e[6], x[6];
#pragma unroll
      for (int k = 0; k < 6; ++k) e[k] = (k == lane) ? 1.0 : 0.0;
      fact6_solve(F, e, x);
      if (lane < 6) {
#pragma unroll
        for (int k = 0; k < 6; ++k) s.cov[k * 6 + lane] = x[k];
      }
    } else if (lane == 0) {
      double M[6][12];
      for (int a = 0; a < 6; ++a)
        for (int b = 0; b < 6; ++b) { M[a][b] = s.A[a * 6 + b] * f2; M[a][6 + b] = (a == b) ? 1.0 : 0.0; }
      for (int c = 0; c < 6; ++c) {
        int p = c;
        for (int rr = c + 1; rr < 6; ++rr)
          if (fabs(M[rr][c]) > fabs(M[p][c])) p = rr;
        if (p != c)
          for (int j = 0; j < 12; ++j) { const double tmp = M[c][j]; M[c][j] = M[p][j]; M[p][j] = tmp; }
        const double d = 1.0 / M[c][c];
        for (int j = 0; j < 12; ++j) M[c][j] *= d;
        for (int rr = 0; rr < 6; ++rr)
          if (rr != c) {
            const double fct = M[rr][c];
            for (int j = 0; j < 12; ++j) M[rr][j] -= fct * M[c][j];
          }
      }
      for (int a = 0; a < 6; ++a)
        for (int b = 0; b < 6; ++b) s.cov[a * 6 + b] = M[a][6 + b];
    }
    __syncwarp();
  }
  if (tid == 0) {
    svo_b200_pose_opt_result r;
    memset(&r, 0, sizeof(r));
    for (int k = 0; k < 36; ++k) r.cov[k] = s.cov[k];
    r.estimated_scale = estimated_scale * fx;
    r.error_init = sqrt(med_init) * fx;
    r.error_final = sqrt(med_final) * fx;
    r.num_obs = (long long)num_obs - (long long)n_deleted;
    r.n_iter_done = s.iters;
    r.n_pivoted_solves = (int16_t)s.n_pivoted;
    r.cov_pivoted = (int16_t)s.cov_pivoted;
    P.out[fr] = r;
    pose_to_rt12(s.T, P.T_io + 12 * (size_t)fr);
    PO_DBG(if (fr == 0) printf("[po dbg] N %d iters %d cycles: constants %lld scale-median %lld gauss-newton %lld cull+medians %lld cov+out %lld\n",
                              N, s.iters, tc[1] - tc[0], tc[2] - tc[1], tc[3] - tc[2], tc[4] - tc[3], (long long)clock64() - tc[4]);)
  }
}

}  // namespace svo

using namespace svo;

extern "C" int svo_b200_pose_optimize_batch(svo_b200_ctx* ctx, int B, double reproj_thresh, int n_iter, const double* fx,
                                            double* T_f_w_io, const int* obs_offset, const double* f,
                                            const double* point_pos, const int* level, uint8_t* has_point_io,
                                            svo_b200_pose_opt_result* out) {
  if (!ctx || B < 0 || n_iter < 0 || (B > 0 && (!fx || !T_f_w_io || !obs_offset || !out)))
    return set_err(ctx, SVO_B200_EINVAL, "pose_optimize_batch: bad arguments");
  if (B == 0) return 0;
  // every check comes before anything is written: a refused call leaves out, T_f_w_io and has_point_io as they were
  const int base = obs_offset[0], total = obs_offset[B] - base;
  if (base < 0) return set_err(ctx, SVO_B200_EINVAL, "pose_optimize_batch: obs_offset[0] is negative");
  int max_n = 0;
  for (int b = 0; b < B; ++b) {
    const int n = obs_offset[b + 1] - obs_offset[b];
    if (n < 0) return set_err(ctx, SVO_B200_EINVAL, "pose_optimize_batch: obs_offset not monotone");
    if (n > max_n) max_n = n;
  }
  if (total > 0 && (!f || !point_pos || !level || !has_point_io))
    return set_err(ctx, SVO_B200_EINVAL, "pose_optimize_batch: NULL observation arrays");
  // sqrt_inv_cov = 1.0 / (1 << level) is defined for levels 0..30 only
  for (int i = base; i < base + total; ++i)
    if (has_point_io[i] && (level[i] < 0 || level[i] > 30))
      return set_err(ctx, SVO_B200_EINVAL, "pose_optimize_batch: observation %d has level %d outside [0, 30]", i - base, level[i]);
  const size_t smem = ((sizeof(PoseOptShared) + 15) & ~size_t(15)) + (sizeof(double) * 8 + 1) * (size_t)((max_n + 1) & ~1) + 16;
  if (smem > (size_t)ctx->max_smem_optin)
    return set_err(ctx, SVO_B200_ELIMIT, "pose_optimize: %d observations in one frame need %zu B of shared memory", max_n, smem);
  memset(out, 0, sizeof(*out) * (size_t)B);
  if (total == 0) return 0;  // errors.empty() -> return, for every frame
  cudaSetDevice(ctx->device);
  std::vector<int> off((size_t)B + 1);
  for (int b = 0; b <= B; ++b) off[b] = obs_offset[b] - base;
  Staging st(ctx);
  PoseOptParams P;
  st.in(f + 3 * (size_t)base, 3 * (size_t)total, &P.f);
  st.in(point_pos + 3 * (size_t)base, 3 * (size_t)total, &P.pos);
  st.in(level + base, total, &P.level);
  st.in(off.data(), B + 1, &P.obs_offset);
  st.in(fx, B, &P.fx);
  st.inout(T_f_w_io, 12 * (size_t)B, &P.T_io);
  st.inout(has_point_io + base, total, &P.has_point);
  st.inout(out, B, &P.out);  // zeroed above
  int rc;
  if ((rc = st.open()) || (rc = st.send())) return rc;
  P.n_iter = n_iter;
  P.reproj_thresh = reproj_thresh;
  SVO_CUDA_CHECK(ctx, cudaFuncSetAttribute(pose_opt_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  if ((rc = launch_kernels(ctx, 1, [&] { pose_opt_kernel<<<B, kPoThreads, smem, ctx->stream>>>(P); }))) return rc;
  return st.receive();
}

extern "C" int svo_b200_pose_optimize(svo_b200_ctx* ctx, double reproj_thresh, int n_iter, double fx,
                                      double* T_f_w_io, const double* f, const double* point_pos, const int* level,
                                      uint8_t* has_point_io, int N, svo_b200_pose_opt_result* out) {
  if (!ctx || !T_f_w_io || !out || N < 0 || n_iter < 0 || (N > 0 && (!f || !point_pos || !level || !has_point_io)))
    return set_err(ctx, SVO_B200_EINVAL, "pose_optimize: bad arguments");
  const int off[2] = {0, N};
  return svo_b200_pose_optimize_batch(ctx, 1, reproj_thresh, n_iter, &fx, T_f_w_io, off, f, point_pos, level, has_point_io, out);
}

// ================================================================================================
// Point::optimize (svo/src/point.cpp:119-177): 3-DoF Gauss-Newton on a point's world position over
// the frames observing it.  Points are independent: one thread per point, observations streamed from
// global memory; the 3x3 system is solved with the same pivoted LDL^T as Eigen's (tiny, in registers).
// ================================================================================================
namespace svo {

__device__ inline void ldlt3_solve(double (&A)[3][3], const double (&b)[3], double (&x)[3]) {
  int tr[3];
  for (int k = 0; k < 3; ++k) {
    int big = k;
    double bigv = fabs(A[k][k]);
    for (int i = k + 1; i < 3; ++i)
      if (fabs(A[i][i]) > bigv) { bigv = fabs(A[i][i]); big = i; }
    tr[k] = big;
    if (big != k) {
      for (int j = 0; j < k; ++j) { const double s = A[k][j]; A[k][j] = A[big][j]; A[big][j] = s; }
      for (int i = big + 1; i < 3; ++i) { const double s = A[i][k]; A[i][k] = A[i][big]; A[i][big] = s; }
      { const double s = A[k][k]; A[k][k] = A[big][big]; A[big][big] = s; }
      for (int i = k + 1; i < big; ++i) { const double s = A[i][k]; A[i][k] = A[big][i]; A[big][i] = s; }
    }
    if (k > 0) {
      double temp[3], acc = 0;
      for (int j = 0; j < k; ++j) { temp[j] = A[j][j] * A[k][j]; acc += A[k][j] * temp[j]; }
      A[k][k] -= acc;
      for (int i = k + 1; i < 3; ++i) {
        double a2 = 0;
        for (int j = 0; j < k; ++j) a2 += A[i][j] * temp[j];
        A[i][k] -= a2;
      }
    }
    const double akk = A[k][k];
    const bool ok = fabs(akk) > 0.0;
    if (k == 0 && !ok) { tr[0] = 0; tr[1] = 1; tr[2] = 2; break; }
    if (ok)
      for (int i = k + 1; i < 3; ++i) A[i][k] /= akk;
  }
  for (int i = 0; i < 3; ++i) x[i] = b[i];
  for (int i = 0; i < 3; ++i) { const int j = tr[i]; const double s = x[i]; x[i] = x[j]; x[j] = s; }
  for (int i = 1; i < 3; ++i)
    for (int j = 0; j < i; ++j) x[i] -= A[i][j] * x[j];
  for (int i = 0; i < 3; ++i) x[i] = (fabs(A[i][i]) > 5.562684646268003e-309) ? x[i] / A[i][i] : 0.0;
  for (int i = 1; i >= 0; --i)
    for (int j = i + 1; j < 3; ++j) x[i] -= A[j][i] * x[j];
  for (int i = 2; i >= 0; --i) { const int j = tr[i]; const double s = x[i]; x[i] = x[j]; x[j] = s; }
}

__global__ void point_optimize_kernel(int P, int n_iter, const int* __restrict__ obs_offset,
                                      const int* __restrict__ obs_frame, const double* __restrict__ obs_f,
                                      const double* __restrict__ frame_T, double* __restrict__ pos_io) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  double pos[3] = {pos_io[3 * p], pos_io[3 * p + 1], pos_io[3 * p + 2]};
  double old_point[3] = {pos[0], pos[1], pos[2]};
  double chi2 = 0.0;
  const int o0 = obs_offset[p], o1 = obs_offset[p + 1];
  for (int it = 0; it < n_iter; ++it) {
    double A[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}}, b[3] = {0, 0, 0}, new_chi2 = 0.0;
    for (int o = o0; o < o1; ++o) {
      const double* T = frame_T + 12 * (size_t)obs_frame[o];
      const double px = T[0] * pos[0] + T[1] * pos[1] + T[2] * pos[2] + T[3];
      const double py = T[4] * pos[0] + T[5] * pos[1] + T[6] * pos[2] + T[7];
      const double pz = T[8] * pos[0] + T[9] * pos[1] + T[10] * pos[2] + T[11];
      const double z_inv = 1.0 / pz, z_inv_sq = z_inv * z_inv;
      const double pj[2][3] = {{z_inv, 0.0, -px * z_inv_sq}, {0.0, z_inv, -py * z_inv_sq}};
      double J[2][3];
#pragma unroll
      for (int r = 0; r < 2; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) J[r][c] = -(pj[r][0] * T[c] + pj[r][1] * T[4 + c] + pj[r][2] * T[8 + c]);
      const double ex = obs_f[3 * o] / obs_f[3 * o + 2] - px / pz, ey = obs_f[3 * o + 1] / obs_f[3 * o + 2] - py / pz;
      new_chi2 += ex * ex + ey * ey;
#pragma unroll
      for (int r = 0; r < 3; ++r) {
#pragma unroll
        for (int c = 0; c < 3; ++c) A[r][c] += J[0][r] * J[0][c] + J[1][r] * J[1][c];
        b[r] -= J[0][r] * ex + J[1][r] * ey;
      }
    }
    double dp[3];
    ldlt3_solve(A, b, dp);
    if ((it > 0 && new_chi2 > chi2) || isnan(dp[0])) {
      pos[0] = old_point[0]; pos[1] = old_point[1]; pos[2] = old_point[2];  // roll-back
      break;
    }
    for (int k = 0; k < 3; ++k) { old_point[k] = pos[k]; pos[k] += dp[k]; }
    chi2 = new_chi2;
    if (fmax(fabs(dp[0]), fmax(fabs(dp[1]), fabs(dp[2]))) <= 0.0000000001) break;
  }
  pos_io[3 * p] = pos[0]; pos_io[3 * p + 1] = pos[1]; pos_io[3 * p + 2] = pos[2];
}

}  // namespace svo

extern "C" int svo_b200_point_optimize_batch(svo_b200_ctx* ctx, int P, int n_iter, const int* obs_offset,
                                             const int* obs_frame, const double* obs_f, const double* frame_T_f_w,
                                             int n_frames, double* pos_io) {
  if (!ctx || P < 0 || n_iter < 0 || n_frames <= 0 || (P > 0 && (!obs_offset || !obs_frame || !obs_f || !frame_T_f_w || !pos_io)))
    return set_err(ctx, SVO_B200_EINVAL, "point_optimize_batch: bad arguments");
  if (P == 0) return 0;
  // the kernel walks [off[p], off[p+1]) of the staged observations: every such range must lie inside the staged ones
  for (int p = 0; p <= P; ++p)
    if (obs_offset[p] < (p ? obs_offset[p - 1] : 0))
      return set_err(ctx, SVO_B200_EINVAL, "point_optimize_batch: obs_offset[%d] is negative or decreasing", p);
  const int n_obs = obs_offset[P] - obs_offset[0];
  for (int o = 0; o < n_obs; ++o)
    if (obs_frame[obs_offset[0] + o] < 0 || obs_frame[obs_offset[0] + o] >= n_frames)
      return set_err(ctx, SVO_B200_EINVAL, "point_optimize_batch: obs_frame[%d] out of range", o);
  cudaSetDevice(ctx->device);
  std::vector<int> off((size_t)P + 1);
  for (int p = 0; p <= P; ++p) off[p] = obs_offset[p] - obs_offset[0];
  Staging st(ctx);
  const int *d_off, *d_frame;
  const double *d_f, *d_T;
  double* d_pos;
  st.in(off.data(), P + 1, &d_off);
  st.in(obs_frame + obs_offset[0], n_obs, &d_frame);
  st.in(obs_f + 3 * (size_t)obs_offset[0], 3 * (size_t)n_obs, &d_f);
  st.in(frame_T_f_w, 12 * (size_t)n_frames, &d_T);
  st.inout(pos_io, 3 * (size_t)P, &d_pos);
  int rc;
  if ((rc = st.open()) || (rc = st.send())) return rc;
  const int threads = 128, blocks = (P + threads - 1) / threads;
  if ((rc = launch_kernels(ctx, 1, [&] {
         point_optimize_kernel<<<blocks, threads, 0, ctx->stream>>>(P, n_iter, d_off, d_frame, d_f, d_T, d_pos);
       })))
    return rc;
  return st.receive();
}
