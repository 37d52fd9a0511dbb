// Drives svs::DeviceMap::prepareForOptimization (include/svs_b200.hpp): setPoseGraph, one prepare, windowState, then a
// refused prepare (inner_window_size >= double_window_size) that must throw std::runtime_error.
// Input: float64 little-endian: V, Np, nnz, nnzN, root, loop, inner, dbl, then the map (poses, anchor, xyz, vis_ptr,
// vis_pose, center, level) and the pose graph (nbr_ptr, nbr_id, nbr_strength, nbr_T, nbr_Lambda).
// Output: float64: do_optimization, P, window_vertex, inner, L, active_point, C, c_i, c_j, c_T, c_Lambda, window_type[V],
// marginalized[nnzN], poses[V][7].  Exit 3 with NO_GPU, 4 when the refusal does not throw.
#include <cstdio>
#include <stdexcept>
#include <vector>

#include "svs_b200.hpp"

static std::vector<double> in;
static size_t at = 0;
template <typename T>
static std::vector<T> take(size_t n) {
  std::vector<T> v(n);
  for (size_t i = 0; i < n; ++i) v[i] = (T)in[at++];
  return v;
}

int main(int argc, char** argv) {
  if (argc < 3) return 2;
  FILE* f = fopen(argv[1], "rb");
  if (!f) return 2;
  double x;
  while (fread(&x, sizeof(double), 1, f) == 1) in.push_back(x);
  fclose(f);
  const std::vector<int> hd = take<int>(8);
  const int V = hd[0], Np = hd[1], nnz = hd[2], nn = hd[3], root = hd[4], loop = hd[5], inner = hd[6], dbl = hd[7];
  auto poses = take<double>(7 * (size_t)V);
  auto anchor = take<int>(Np);
  auto xyz = take<double>(3 * (size_t)Np);
  auto vptr = take<int>((size_t)Np + 1);
  auto vpose = take<int>(nnz);
  auto cen = take<double>(3 * (size_t)nnz);
  auto lvl = take<int>(nnz);
  svs::DeviceMap::PoseGraph g;
  g.nbr_ptr = take<int>((size_t)V + 1); g.nbr_id = take<int>(nn); g.nbr_strength = take<int>(nn);
  g.nbr_T = take<double>(7 * (size_t)nn); g.nbr_Lambda = take<double>(36 * (size_t)nn);
  svs::DeviceMap dm;
  if (!dm.valid()) {
    printf("NO_GPU %s\n", dm.last_error());
    return 3;
  }
  if (!dm.set(poses, anchor, xyz, vptr, vpose, cen, lvl) || !dm.setPoseGraph(g)) {
    printf("set: %s\n", dm.last_error());
    return 1;
  }
  svs::DeviceMap::DoubleWindow w;
  const bool do_opt = dm.prepareForOptimization(root, loop, inner, dbl, &w);
  std::vector<unsigned char> wt, mg;
  dm.windowState(&wt, &mg);
  bool threw = false;
  try {
    svs::DeviceMap::DoubleWindow w2;
    dm.prepareForOptimization(root, loop, dbl, dbl, &w2);
  } catch (const std::runtime_error&) {
    threw = true;
  }
  if (!threw) return 4;
  std::vector<double> got;
  if (!dm.poseGraph(&g)) return 1;
  std::vector<double> P(7 * (size_t)V);
  if (svs_map_get(dm.handle(), P.data(), nullptr) != SVS_OK) return 1;
  auto put = [&](auto const& v) { for (auto e : v) got.push_back((double)e); };
  got.push_back(do_opt); got.push_back((double)w.window_vertex.size()); put(w.window_vertex); put(w.inner);
  got.push_back((double)w.active_point.size()); put(w.active_point);
  got.push_back((double)w.c_i.size()); put(w.c_i); put(w.c_j); put(w.c_T); put(w.c_Lambda);
  put(wt); put(mg); put(P);
  FILE* o = fopen(argv[2], "wb");
  if (!o) return 2;
  fwrite(got.data(), sizeof(double), got.size(), o);
  fclose(o);
  return 0;
}
