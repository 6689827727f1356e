// tests/camera_probe.cu -- runs the device camera functions every projecting kernel inlines (svo_math.cuh
// cam_world2cam / cam_cam2world) over arrays, with the CamDev the library's own svo::cam_to_dev derives, for
// tests/test_camera_edges_gpu.py.  Built by that test with the library's nvcc flags (-fmad=false) and linked against
// libsvo_b200.so; nothing here restates camera code.
//
//   camera_probe IN OUT
//   IN:  svo_b200_camera, int64 n_w, int64 n_c, n_w x 3 doubles (xyz), n_c x 2 doubles (pixels)
//   OUT: n_w x 2 doubles (world2cam(xyz / z)), n_c x 3 doubles (cam2world)
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "../rpg_svo_b200/csrc/ctx.h"
#include "../rpg_svo_b200/csrc/svo_math.cuh"

__global__ void world2cam_kernel(svo::CamDev c, const double* xyz, long long n, double* uv) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= n) return;
  double u, v;
  svo::cam_world2cam(c, xyz[3 * i] / xyz[3 * i + 2], xyz[3 * i + 1] / xyz[3 * i + 2], u, v);  // project2d, then world2cam
  uv[2 * i] = u;
  uv[2 * i + 1] = v;
}

__global__ void cam2world_kernel(svo::CamDev c, const double* px, long long n, double* f) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= n) return;
  double b[3];
  svo::cam_cam2world(c, px[2 * i], px[2 * i + 1], b);
  f[3 * i] = b[0];
  f[3 * i + 1] = b[1];
  f[3 * i + 2] = b[2];
}

#define CHECK(call)                                                                         \
  do {                                                                                      \
    cudaError_t e_ = (call);                                                                \
    if (e_ != cudaSuccess) {                                                                \
      fprintf(stderr, "camera_probe: %s: %s\n", #call, cudaGetErrorString(e_));             \
      return 1;                                                                             \
    }                                                                                       \
  } while (0)

int main(int argc, char** argv) {
  if (argc != 3) {
    fprintf(stderr, "usage: camera_probe IN OUT\n");
    return 2;
  }
  FILE* in = fopen(argv[1], "rb");
  if (!in) return 2;
  svo_b200_camera cam;
  long long n[2];
  if (fread(&cam, sizeof(cam), 1, in) != 1 || fread(n, sizeof(n), 1, in) != 1 || n[0] < 0 || n[1] < 0) return 2;
  std::vector<double> xyz(3 * n[0] + 1), px(2 * n[1] + 1), uv(2 * n[0] + 1), f(3 * n[1] + 1);
  if (fread(xyz.data(), sizeof(double), 3 * n[0], in) != (size_t)(3 * n[0]) ||
      fread(px.data(), sizeof(double), 2 * n[1], in) != (size_t)(2 * n[1]))
    return 2;
  fclose(in);
  svo::CamDev c;
  if (svo::cam_to_dev(nullptr, &cam, c) != 0) {
    fprintf(stderr, "camera_probe: cam_to_dev refused the camera\n");
    return 3;
  }
  double *d_xyz, *d_px, *d_uv, *d_f;
  CHECK(cudaMalloc(&d_xyz, xyz.size() * sizeof(double)));
  CHECK(cudaMalloc(&d_px, px.size() * sizeof(double)));
  CHECK(cudaMalloc(&d_uv, uv.size() * sizeof(double)));
  CHECK(cudaMalloc(&d_f, f.size() * sizeof(double)));
  CHECK(cudaMemcpy(d_xyz, xyz.data(), xyz.size() * sizeof(double), cudaMemcpyHostToDevice));
  CHECK(cudaMemcpy(d_px, px.data(), px.size() * sizeof(double), cudaMemcpyHostToDevice));
  if (n[0]) world2cam_kernel<<<(unsigned)((n[0] + 127) / 128), 128>>>(c, d_xyz, n[0], d_uv);
  if (n[1]) cam2world_kernel<<<(unsigned)((n[1] + 127) / 128), 128>>>(c, d_px, n[1], d_f);
  CHECK(cudaGetLastError());
  CHECK(cudaMemcpy(uv.data(), d_uv, uv.size() * sizeof(double), cudaMemcpyDeviceToHost));
  CHECK(cudaMemcpy(f.data(), d_f, f.size() * sizeof(double), cudaMemcpyDeviceToHost));
  cudaFree(d_xyz); cudaFree(d_px); cudaFree(d_uv); cudaFree(d_f);
  FILE* out = fopen(argv[2], "wb");
  if (!out) return 2;
  fwrite(uv.data(), sizeof(double), 2 * n[0], out);
  fwrite(f.data(), sizeof(double), 3 * n[1], out);
  fclose(out);
  return 0;
}
