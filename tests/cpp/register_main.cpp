// Drives svs::DeviceMap::localRegisterFrame (include/svs_b200.hpp) on one map and svs_localRegisterFrame on a second
// copy with their own matcher and pose handles, and checks that both give the same bits.  Input (little-endian):
//   int V, Np, nnz, nlv; double poses[V][7]; int anchor[Np]; double xyz[Np][3]; int vis_ptr[Np+1], vis_pose[nnz];
//   double center[nnz][3]; int level[nnz]; int nbr_ptr[V+1], nbr_id[nbr_ptr[V]]; per level int w, h, double f, px, py;
//   double cam[4]; int covis, root, P, window[P], slot[V], nslot; per slot per level uint8 [h][w]; the root frame per
//   level uint8 [h][w], float disp[h0][w0]; per level int nkp, xy[nkp][2], content[nkp].
// Output: int counts[11] (svs_register_result order), double T_align1[7], T_newroot_from_oldroot[7],
// T_newroot_from_w[7], int ns, stats[ns][7], int nt, point[nt], level[nt], committed[nt], double uvu[nt][3].
// Exit 3 with NO_GPU without a device.
#include <algorithm>
#include <cstdio>
#include <cstring>
#include <vector>

#include "svs_b200.hpp"

template <class T>
static bool rd(FILE* f, T* p, size_t n) { return fread(p, sizeof(T), n, f) == n; }

struct Handles {
  svs::DeviceMap map;
  svs::GuidedMatcher* m = nullptr;
  svs::BA_SE3_XYZ_STEREO ba{8192};
};

int main(int argc, char** argv) {
  if (argc < 3) return 2;
  FILE* f = fopen(argv[1], "rb");
  if (!f) return 2;
  int V, Np, nnz, nlv;
  if (!rd(f, &V, 1) || !rd(f, &Np, 1) || !rd(f, &nnz, 1) || !rd(f, &nlv, 1)) return 2;
  if (V <= 0 || V > (1 << 20) || Np < 0 || Np > (1 << 24) || nnz < 0 || nnz > (1 << 26) || nlv <= 0 || nlv > SVS_MATCH_MAX_LEVELS)
    return 2;
  std::vector<double> poses(7 * (size_t)V), xyz(3 * (size_t)Np), center(3 * (size_t)nnz);
  std::vector<int> anchor(Np), vis_ptr(Np + 1), vis_pose(nnz), level(nnz), nbr_ptr(V + 1);
  if (!rd(f, poses.data(), poses.size()) || !rd(f, anchor.data(), anchor.size()) || !rd(f, xyz.data(), xyz.size()) ||
      !rd(f, vis_ptr.data(), vis_ptr.size()) || !rd(f, vis_pose.data(), vis_pose.size()) ||
      !rd(f, center.data(), center.size()) || !rd(f, level.data(), level.size()) || !rd(f, nbr_ptr.data(), nbr_ptr.size()))
    return 2;
  std::vector<int> nbr_id(nbr_ptr[V]);
  if (!rd(f, nbr_id.data(), nbr_id.size())) return 2;
  std::vector<svs_match_level> lv(nlv);
  for (auto& L : lv)
    if (!rd(f, &L.w, 1) || !rd(f, &L.h, 1) || !rd(f, &L.f, 1) || !rd(f, &L.px, 1) || !rd(f, &L.py, 1)) return 2;
  svs_cam cam;
  int covis, root, P, nslot;
  if (!rd(f, &cam.f, 1) || !rd(f, &cam.px, 1) || !rd(f, &cam.py, 1) || !rd(f, &cam.b, 1) || !rd(f, &covis, 1) ||
      !rd(f, &root, 1) || !rd(f, &P, 1))
    return 2;
  std::vector<int> window(P), slot(V);
  if (!rd(f, window.data(), P) || !rd(f, slot.data(), V) || !rd(f, &nslot, 1)) return 2;
  auto read_pyr = [&](std::vector<std::vector<unsigned char>>* pyr) {
    pyr->resize(nlv);
    for (int l = 0; l < nlv; ++l) {
      (*pyr)[l].resize((size_t)lv[l].w * lv[l].h);
      if (!rd(f, (*pyr)[l].data(), (*pyr)[l].size())) return false;
    }
    return true;
  };
  std::vector<std::vector<std::vector<unsigned char>>> slots(nslot);
  for (auto& p : slots)
    if (!read_pyr(&p)) return 2;
  std::vector<std::vector<unsigned char>> cur;
  std::vector<float> disp((size_t)lv[0].w * lv[0].h);
  if (!read_pyr(&cur) || !rd(f, disp.data(), disp.size())) return 2;
  std::vector<std::vector<int>> kxy(nlv), kc(nlv);
  for (int l = 0; l < nlv; ++l) {
    int n;
    if (!rd(f, &n, 1)) return 2;
    kxy[l].resize(2 * (size_t)n); kc[l].resize(n);
    if (!rd(f, kxy[l].data(), kxy[l].size()) || !rd(f, kc[l].data(), kc[l].size())) return 2;
  }
  fclose(f);

  Handles a, b;
  svs::GuidedMatcher ma(lv, nslot, 8192), mb(lv, nslot, 8192);
  a.m = &ma; b.m = &mb;
  if (!a.map.valid() || !ma.valid() || !a.ba.valid()) {
    printf("NO_GPU %s\n", a.map.valid() ? "matcher or pose handle" : "map handle");
    return 3;
  }
  for (Handles* h : {&a, &b}) {
    if (!h->map.set(poses, anchor, xyz, vis_ptr, vis_pose, center, level)) { printf("FAIL set: %s\n", h->map.last_error()); return 1; }
    if (!h->map.setGraph(nbr_ptr, nbr_id)) { printf("FAIL setGraph: %s\n", h->map.last_error()); return 1; }
    svs_matcher* mh = h->m->handle();
    std::vector<int> pitch(nlv);
    for (int l = 0; l < nlv; ++l) pitch[l] = lv[l].w;
    for (int s = 0; s < nslot; ++s) {
      std::vector<const unsigned char*> ptr(nlv);
      for (int l = 0; l < nlv; ++l) ptr[l] = slots[s][l].data();
      const double I7[7] = {0, 0, 0, 1, 0, 0, 0};
      if (svs_matcher_set_keyframe(mh, s, I7, ptr.data(), pitch.data()) != SVS_OK) { printf("FAIL slot\n"); return 1; }
    }
    std::vector<const unsigned char*> ptr(nlv);
    for (int l = 0; l < nlv; ++l) ptr[l] = cur[l].data();
    if (svs_matcher_set_current(mh, ptr.data(), pitch.data(), disp.data(), lv[0].w) != SVS_OK) { printf("FAIL current\n"); return 1; }
    for (int l = 0; l < nlv; ++l)
      if (svs_matcher_set_features(mh, l, kxy[l].data(), kc[l].data(), (int)kc[l].size()) != SVS_OK) { printf("FAIL features\n"); return 1; }
  }
  svs_register_result ra{}, rb{};
  std::vector<svs_register_stats> sa;
  svs::DeviceMap::RegisterTracks tr;
  bool registered;
  try {
    registered = a.map.localRegisterFrame(ma, a.ba, cam, covis, root, window, slot, &ra, &sa, &tr);
  } catch (const std::exception& e) {
    printf("FAIL localRegisterFrame: %s\n", e.what());
    return 1;
  }
  const int ct = Np > 0 ? Np : 1;
  std::vector<svs_register_stats> sb(V);
  std::vector<int> tp(ct), tl(ct), tc(ct);
  std::vector<double> tu(3 * (size_t)ct);
  if (svs_localRegisterFrame(b.map.handle(), mb.handle(), b.ba.handle(), &cam, covis, root, P, window.data(), slot.data(), &rb, V,
                             sb.data(), ct, tp.data(), tu.data(), tl.data(), tc.data()) != SVS_OK) {
    printf("FAIL C ABI: %s\n", b.map.last_error());
    return 1;
  }
  const int nt = (int)tr.point.size(), ns = (int)sa.size();
  if (std::memcmp(&ra, &rb, offsetof(svs_register_result, lm)) != 0 || registered != (rb.registered != 0) ||
      std::memcmp(sa.data(), sb.data(), sizeof(svs_register_stats) * (size_t)ns) != 0 ||
      !std::equal(tr.point.begin(), tr.point.end(), tp.begin()) || !std::equal(tr.level.begin(), tr.level.end(), tl.begin()) ||
      !std::equal(tr.committed.begin(), tr.committed.end(), tc.begin()) ||
      std::memcmp(tr.uvu.data(), tu.data(), sizeof(double) * 3 * (size_t)nt) != 0) {
    printf("FAIL the C++ layer and the C ABI differ\n");
    return 1;
  }
  FILE* o = fopen(argv[2], "wb");
  const int counts[11] = {ra.registered, ra.stage, ra.n_direct, ra.n_neighborhood, ra.n_candidates, ra.n_matched1,
                          ra.n_matched2, ra.n_tracks, ra.n_stats, ra.n_neighbors, ra.n_committed};
  fwrite(counts, sizeof(int), 11, o);
  fwrite(ra.T_align1, sizeof(double), 7, o);
  fwrite(ra.T_newroot_from_oldroot, sizeof(double), 7, o);
  fwrite(ra.T_newroot_from_w, sizeof(double), 7, o);
  fwrite(&ns, sizeof(int), 1, o);
  fwrite(sa.data(), sizeof(svs_register_stats), ns, o);
  fwrite(&nt, sizeof(int), 1, o);
  fwrite(tr.point.data(), sizeof(int), nt, o);
  fwrite(tr.level.data(), sizeof(int), nt, o);
  fwrite(tr.committed.data(), sizeof(int), nt, o);
  fwrite(tr.uvu.data(), sizeof(double), 3 * (size_t)nt, o);
  fclose(o);
  printf("OK registered=%d tracks=%d\n", ra.registered, nt);
  return 0;
}
