// Drives svs::DeviceMap's pose-graph growth (include/svs_b200.hpp): setPoseGraph with an empty graph, one addKeyframe
// with its strength table and edges, then addEdges; the same calls go through the C ABI on a second handle and both
// graphs must be equal bit for bit.
// Input: float64 little-endian: V, Np, nnz, oldkey, n_new, n_track, covis_thr, width, height, n_edges, moved, then the
// map (poses, anchor, xyz, vis_ptr, vis_pose, center, level), T_newkey_from_oldkey, the keyframe's arrays, the edges
// (v1, v2, strength) and T_moved_from_w[7].
// Output: float64: n_table, the table rows, then nbr_ptr, nbr_id, nbr_strength, nbr_T, nbr_Lambda.  Exit 3 with NO_GPU.
#include <cstdio>
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
  const std::vector<int> hd = take<int>(11);
  const int V = hd[0], Np = hd[1], nnz = hd[2], oldkey = hd[3], nn = hd[4], nt = hd[5], thr = hd[6], w = hd[7], h = hd[8];
  const int ne = hd[9], moved = hd[10];
  auto poses = take<double>(7 * (size_t)V);
  auto anchor = take<int>(Np);
  auto xyz = take<double>(3 * (size_t)Np);
  auto vptr = take<int>((size_t)Np + 1);
  auto vpose = take<int>(nnz);
  auto cen = take<double>(3 * (size_t)nnz);
  auto lvl = take<int>(nnz);
  auto T = take<double>(7);
  auto na = take<int>(nn);
  auto nx = take<double>(3 * (size_t)nn), nac = take<double>(3 * (size_t)nn);
  auto nal = take<int>(nn);
  auto nc = take<double>(3 * (size_t)nn);
  auto nl = take<int>(nn);
  auto tp = take<int>(nt);
  auto tc = take<double>(3 * (size_t)nt);
  auto tl = take<int>(nt);
  auto v1 = take<int>(ne), v2 = take<int>(ne), es = take<int>(ne);
  auto Tm = take<double>(7);

  svs::DeviceMap dm;
  svs_map* c = nullptr;
  if (!dm.valid() || svs_map_create(-1, &c) != SVS_OK) {
    printf("NO_GPU %s\n", dm.last_error());
    return 3;
  }
  svs::DeviceMap::PoseGraph g0;
  g0.nbr_ptr.assign((size_t)V + 1, 0);
  std::vector<int> table;
  int n_edges = 0;
  if (!dm.set(poses, anchor, xyz, vptr, vpose, cen, lvl) || !dm.setPoseGraph(g0) ||
      dm.addKeyframe(oldkey, T.data(), na, nx, nac, nal, nc, nl, tp, tc, tl, thr, w, h, &table, &n_edges) != V ||
      !dm.addEdges(v1, v2, es, moved, Tm.data())) {
    printf("FAIL wrapper: %s\n", dm.last_error());
    return 1;
  }
  // the C ABI on a second handle
  std::vector<int> rows(2 * (size_t)V);
  int v = 0, q = 0, nrow = 0, ne2 = 0;
  if (svs_map_set(c, V, poses.data(), Np, anchor.data(), xyz.data(), vptr.data(), vpose.data(), cen.data(), lvl.data()) != SVS_OK ||
      svs_map_set_pose_graph(c, g0.nbr_ptr.data(), nullptr, nullptr, nullptr, nullptr) != SVS_OK ||
      svs_map_add_keyframe_graph(c, oldkey, T.data(), nn, na.data(), nx.data(), nac.data(), nal.data(), nc.data(), nl.data(), nt,
                                 tp.data(), tc.data(), tl.data(), thr, w, h, &v, &q, &nrow, rows.data(), &ne2) != SVS_OK ||
      svs_map_add_edges(c, ne, v1.data(), v2.data(), es.data(), moved, Tm.data()) != SVS_OK) {
    printf("FAIL C ABI: %s\n", svs_map_last_error(c));
    return 1;
  }
  svs::DeviceMap::PoseGraph g;
  if (!dm.poseGraph(&g)) return 1;
  int nnzN = 0;
  svs_map_get_graph(c, 0, &nnzN, nullptr, nullptr, nullptr, nullptr, nullptr);
  std::vector<int> p2((size_t)V + 2), i2(nnzN + 1), s2(nnzN + 1);
  std::vector<double> T2(7 * (size_t)nnzN + 7), L2(36 * (size_t)nnzN + 36);
  svs_map_get_graph(c, nnzN, &nnzN, p2.data(), i2.data(), s2.data(), T2.data(), L2.data());
  svs_map_destroy(c);
  rows.resize(2 * (size_t)nrow); i2.resize(nnzN); s2.resize(nnzN); T2.resize(7 * (size_t)nnzN); L2.resize(36 * (size_t)nnzN);
  if (rows != table || ne2 != n_edges || p2 != g.nbr_ptr || i2 != g.nbr_id || s2 != g.nbr_strength || T2 != g.nbr_T ||
      L2 != g.nbr_Lambda) {
    printf("FAIL wrapper and C ABI differ\n");
    return 1;
  }
  FILE* o = fopen(argv[2], "wb");
  if (!o) return 2;
  auto put = [&](const auto& vec) { for (auto e : vec) { const double d = (double)e; fwrite(&d, sizeof(double), 1, o); } };
  put(std::vector<int>{(int)table.size() / 2});
  put(table); put(g.nbr_ptr); put(g.nbr_id); put(g.nbr_strength); put(g.nbr_T); put(g.nbr_Lambda);
  fclose(o);
  printf("OK edges %d\n", n_edges);
  return 0;
}
