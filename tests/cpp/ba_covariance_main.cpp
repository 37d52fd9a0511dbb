// svs::StereoGraph::computeMarginals on a window written by tests/test_ba_covariance_gpu.py:
//   int32 P, L, E, C, npairs, iters, robust; float64 cam[4], lambda;
//   float64 T_qt[P][7]; int32 fixed[P]; float64 xyz_anchor[L][3];
//   int32 e_point[E], e_pose[E], e_anchor[E]; float64 e_obs[E][3], e_info[E][3];
//   int32 c_i[C], c_j[C]; float64 c_T[C][7], c_Lambda[C][36]; int32 pair_i[npairs], pair_j[npairs]   (pose indices)
// Frames get the ids 5000 - 3 i and points 11 l + 2 (the caller's ids, not indices).  optimize(iters, robust), then
// computeMarginals(lambda) with the pairs named by frame id; writes pose_cov [P][36], pair_cov [npairs][36],
// point_cov [L][9].  Exit 0 on success, 1 if the factor failed, 2 on bad input, 3 without a GPU.
#include <cstdio>
#include <utility>
#include <vector>

#include "svs_b200.hpp"

template <typename T>
static bool rd(FILE* f, std::vector<T>& v, size_t n) {
  v.resize(n);
  return fread(v.data(), sizeof(T), n, f) == n;
}

int main(int argc, char** argv) {
  if (argc < 3) { printf("usage: ba_covariance_main in.bin out.bin\n"); return 2; }
  FILE* f = fopen(argv[1], "rb");
  if (!f) return 2;
  std::vector<int> hdr, fixed, ep, es, ea, ci, cj, pi, pj;
  std::vector<double> cam, T, xyz, obs, info, cT, cL;
  bool ok = rd(f, hdr, 7) && rd(f, cam, 5);
  const int P = ok ? hdr[0] : 0, L = ok ? hdr[1] : 0, E = ok ? hdr[2] : 0, C = ok ? hdr[3] : 0, n = ok ? hdr[4] : 0;
  ok = ok && P > 0 && L >= 0 && E >= 0 && C >= 0 && n >= 0 && rd(f, T, 7 * (size_t)P) && rd(f, fixed, P) &&
       rd(f, xyz, 3 * (size_t)L) && rd(f, ep, E) && rd(f, es, E) && rd(f, ea, E) && rd(f, obs, 3 * (size_t)E) &&
       rd(f, info, 3 * (size_t)E) && rd(f, ci, C) && rd(f, cj, C) && rd(f, cT, 7 * (size_t)C) && rd(f, cL, 36 * (size_t)C) &&
       rd(f, pi, n) && rd(f, pj, n);
  fclose(f);
  if (!ok) { printf("BAD_INPUT\n"); return 2; }
  auto frame = [](int i) { return 5000 - 3 * i; };
  auto point = [](int l) { return 11 * l + 2; };

  svs::StereoGraph g;
  if (!g.valid()) { printf("NO_GPU %s\n", g.last_error()); return 3; }
  g.setCamera(cam[0], cam[1], cam[2], cam[3]);
  for (int i = 0; i < P; ++i) {
    svs::SE3d X;
    for (int k = 0; k < 4; ++k) X.q[k] = T[7 * i + k];
    for (int k = 0; k < 3; ++k) X.t[k] = T[7 * i + 4 + k];
    g.addPose(frame(i), X, fixed[i] != 0);
  }
  for (int l = 0; l < L; ++l) g.addPoint(point(l), &xyz[3 * (size_t)l]);
  for (int e = 0; e < E; ++e) g.addObs(&obs[3 * (size_t)e], &info[3 * (size_t)e], point(ep[e]), frame(es[e]), frame(ea[e]));
  for (int c = 0; c < C; ++c) {
    svs::SE3d X;
    for (int k = 0; k < 4; ++k) X.q[k] = cT[7 * c + k];
    for (int k = 0; k < 3; ++k) X.t[k] = cT[7 * c + 4 + k];
    g.addConstraint(X, &cL[36 * (size_t)c], frame(ci[c]), frame(cj[c]));
  }
  const int it = g.optimize(svs::OptParams(hdr[5], hdr[6] != 0));
  if (it < 0) { printf("OPTIMIZE_FAILED %d %s\n", it, g.last_error()); return 2; }
  std::vector<std::pair<int, int>> pairs(n);
  for (int k = 0; k < n; ++k) pairs[k] = {frame(pi[k]), frame(pj[k])};
  std::vector<double> pose_cov, point_cov, pair_cov;
  const bool done = g.computeMarginals(cam[4], &pose_cov, &point_cov, pairs, &pair_cov);
  FILE* o = fopen(argv[2], "wb");
  if (!o) return 2;
  fwrite(pose_cov.data(), 8, pose_cov.size(), o);
  fwrite(pair_cov.data(), 8, pair_cov.size(), o);
  fwrite(point_cov.data(), 8, point_cov.size(), o);
  fclose(o);
  printf("%s iterations=%d\n", done ? "OK" : "FACTOR_FAILED", it);
  return done ? 0 : 1;
}
