// rpg_svo_b200/host/host_robust_demo.cpp -- svo::SparseImgAlign with a robust cost through the C++ host classes
// (svo_host.h): two Frames with Features/Points, then
//   SparseImgAlign img_align(max, min, 30, GaussNewton, false, false);
//   img_align.setRobustCostFunction(MADScale, weight);   // [EXT] vk::NLLSSolver
//   img_align.run(ref, cur);  img_align.getFisherInformation();
// and, on the same context, an object without a robust cost (its run() must not inherit the other's mode).
// Inputs come from a binary dump written by tests/test_sia_robust_gpu.py, results go to a second file that the test
// compares with the CPU oracle.   usage: host_robust_demo in.bin out.bin
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "svo_host.h"

template <class T>
static void rd(FILE* f, T* p, size_t n) {
  if (fread(p, sizeof(T), n, f) != n) { fprintf(stderr, "host_robust_demo: short read\n"); exit(2); }
}

int main(int argc, char** argv) {
  if (argc != 3) { fprintf(stderr, "usage: %s in.bin out.bin\n", argv[0]); return 2; }
  FILE* fi = fopen(argv[1], "rb");
  if (!fi) { perror("open input"); return 2; }
  int hdr[7];
  rd(fi, hdr, 7);
  const int w = hdr[0], h = hdr[1], n_levels = hdr[2], N = hdr[3], max_level = hdr[4], min_level = hdr[5], weight = hdr[6];
  double camv[4];
  rd(fi, camv, 4);
  std::vector<uint8_t> ref_img((size_t)w * h), cur_img((size_t)w * h), has_point(N);
  rd(fi, ref_img.data(), ref_img.size());
  rd(fi, cur_img.data(), cur_img.size());
  svo::SE3 T_ref_w;
  rd(fi, T_ref_w.m, 12);
  std::vector<double> px(2 * N), f(3 * N), pos(3 * N);
  rd(fi, px.data(), px.size());
  rd(fi, f.data(), f.size());
  rd(fi, pos.data(), pos.size());
  rd(fi, has_point.data(), has_point.size());
  fclose(fi);

  try {
    svo::Context ctx(0);
    svo::PinholeCamera cam(w, h, camv[0], camv[1], camv[2], camv[3]);
    svo::FramePtr frame_ref(new svo::Frame(ctx, &cam, ref_img.data(), n_levels, 0.0));
    std::vector<svo::Point*> points;
    for (int i = 0; i < N; ++i) {
      svo::Point* pt = has_point[i] ? new svo::Point({pos[3 * i], pos[3 * i + 1], pos[3 * i + 2]}) : nullptr;
      if (pt) points.push_back(pt);
      frame_ref->addFeature(new svo::Feature(frame_ref.get(), pt, {px[2 * i], px[2 * i + 1]}, {f[3 * i], f[3 * i + 1], f[3 * i + 2]}, 0));
    }
    frame_ref->T_f_w_ = T_ref_w;
    FILE* fo = fopen(argv[2], "wb");
    if (!fo) { perror("open output"); return 2; }
    svo::SparseImgAlign robust(max_level, min_level, 30, svo::SparseImgAlign::GaussNewton, false, false);
    robust.setRobustCostFunction(svo::SparseImgAlign::MADScale, svo::SparseImgAlign::WeightFunctionType(weight));
    svo::SparseImgAlign plain(max_level, min_level, 30, svo::SparseImgAlign::GaussNewton, false, false);
    for (svo::SparseImgAlign* a : {&robust, &plain}) {  // robust first: plain must run without weights afterwards
      svo::FramePtr frame_cur(new svo::Frame(ctx, &cam, cur_img.data(), n_levels, 1.0));
      frame_cur->T_f_w_ = T_ref_w;  // the current frame starts at the reference pose
      const long long n_tracked = (long long)a->run(frame_ref, frame_cur);
      const svo::Matrix6d fisher = a->getFisherInformation();
      fwrite(frame_cur->T_f_w_.m, sizeof(double), 12, fo);
      fwrite(&n_tracked, sizeof(n_tracked), 1, fo);
      fwrite(fisher.data(), sizeof(double), 36, fo);
      printf("host_robust_demo: %s: tracked %lld patches, t = (%.6f %.6f %.6f), I(0,0) = %.6g\n", a == &robust ? "robust" : "plain",
             n_tracked, frame_cur->T_f_w_.m[3], frame_cur->T_f_w_.m[7], frame_cur->T_f_w_.m[11], fisher[0]);
    }
    fclose(fo);
    bool threw = false;
    try {
      robust.setRobustCostFunction(svo::SparseImgAlign::TDistScale, svo::SparseImgAlign::TDistWeight);
    } catch (const std::invalid_argument&) {
      threw = true;
    }
    if (!threw) { fprintf(stderr, "host_robust_demo: TDistScale accepted\n"); return 1; }
    for (svo::Point* p : points) delete p;
  } catch (const std::exception& e) {
    fprintf(stderr, "host_robust_demo: %s\n", e.what());
    return 1;
  }
  return 0;
}
