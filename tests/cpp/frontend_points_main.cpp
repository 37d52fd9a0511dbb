// Drives svs::GuidedMatcher::{matchAndTrack, processMatchedPoints, addNewPoints, addMorePoints} and
// svs::shallWeDropNewKeyframe (include/svs_b200.hpp) on one matcher and the C ABI on a second one, and checks that both
// give the same bits.  Input (little-endian): int nlv; per level int w, h, double f, px, py; double cam[4]; the keyframe
// per level uint8 [h][w]; the current frame per level uint8 [h][w]; float disp[h0][w0]; per level int nkp, xy[nkp][2],
// content[nkp]; double T_cur[7], T_key_w[7]; int n_groups, sizes[n_groups]; svs_match_point pts[sum]; int nmax.
// Output: int num_obs, num_new, drop, ng; svs_tracked_point[ng]; svs_point_stats; int nfresh; svs_new_point[nfresh];
// int nmore; svs_new_point[nmore].  Exit 3 with NO_GPU without a device, 4 when the two paths differ.
#include <cstdio>
#include <cstring>
#include <vector>

#include "svs_b200.hpp"

template <class T>
static bool rd(FILE* f, T* p, size_t n) { return fread(p, sizeof(T), n, f) == n; }
template <class T>
static void wr(FILE* f, const T* p, size_t n) { fwrite(p, sizeof(T), n, f); }
template <class T>
static bool same(const std::vector<T>& a, const std::vector<T>& b) {
  return a.size() == b.size() && (a.empty() || memcmp(a.data(), b.data(), sizeof(T) * a.size()) == 0);
}

int main(int argc, char** argv) {
  if (argc < 3) return 2;
  FILE* f = fopen(argv[1], "rb");
  if (!f) return 2;
  int nlv;
  if (!rd(f, &nlv, 1) || nlv <= 0 || nlv > SVS_MATCH_MAX_LEVELS) return 2;
  std::vector<svs_match_level> lv(nlv);
  for (auto& L : lv)
    if (!rd(f, &L.w, 1) || !rd(f, &L.h, 1) || !rd(f, &L.f, 1) || !rd(f, &L.px, 1) || !rd(f, &L.py, 1)) return 2;
  svs_cam cam;
  if (!rd(f, &cam.f, 1) || !rd(f, &cam.px, 1) || !rd(f, &cam.py, 1) || !rd(f, &cam.b, 1)) return 2;
  std::vector<std::vector<unsigned char>> kf(nlv), cur(nlv);
  for (auto* pyr : {&kf, &cur})
    for (int l = 0; l < nlv; ++l) {
      (*pyr)[l].resize((size_t)lv[l].w * lv[l].h);
      if (!rd(f, (*pyr)[l].data(), (*pyr)[l].size())) return 2;
    }
  std::vector<float> disp((size_t)lv[0].w * lv[0].h);
  if (!rd(f, disp.data(), disp.size())) return 2;
  std::vector<std::vector<int>> xy(nlv), content(nlv);
  for (int l = 0; l < nlv; ++l) {
    int n;
    if (!rd(f, &n, 1) || n < 0) return 2;
    xy[l].resize(2 * (size_t)n); content[l].resize(n);
    if (!rd(f, xy[l].data(), xy[l].size()) || !rd(f, content[l].data(), content[l].size())) return 2;
  }
  double T_cur[7], T_key_w[7];
  int ng;
  if (!rd(f, T_cur, 7) || !rd(f, T_key_w, 7) || !rd(f, &ng, 1) || ng < 2) return 2;
  std::vector<int> sizes(ng);
  if (!rd(f, sizes.data(), ng)) return 2;
  std::vector<std::vector<svs_match_point>> groups(ng);
  for (int g = 0; g < ng; ++g) {
    groups[g].resize(sizes[g]);
    if (!rd(f, groups[g].data(), groups[g].size())) return 2;
  }
  int nmax;
  if (!rd(f, &nmax, 1)) return 2;
  fclose(f);

  svs::GuidedMatcher a(lv), b(lv);
  if (!a.valid() || !b.valid()) { fprintf(stderr, "NO_GPU: svs::GuidedMatcher needs a CUDA device\n"); return 3; }
  std::vector<const unsigned char*> kp(nlv), cp(nlv);
  std::vector<int> pitch(nlv);
  for (int l = 0; l < nlv; ++l) { kp[l] = kf[l].data(); cp[l] = cur[l].data(); pitch[l] = lv[l].w; }
  for (svs_matcher* h : {a.handle(), b.handle()}) {
    if (svs_matcher_set_keyframe(h, 0, T_key_w, kp.data(), pitch.data()) != SVS_OK ||
        svs_matcher_set_current(h, cp.data(), pitch.data(), disp.data(), lv[0].w) != SVS_OK)
      return 5;
    for (int l = 0; l < nlv; ++l)
      if (svs_matcher_set_features(h, l, xy[l].data(), content[l].data(), (int)content[l].size()) != SVS_OK) return 5;
  }
  // the wrapper
  std::vector<svs_new_point> fresh_a, more_a;
  std::vector<svs_match_point> rows;
  if (a.addNewPoints(cam, 1, &fresh_a, &rows) < 0) return 5;
  std::vector<svs_match_result> td_a;
  int num_new_a = 0;
  const int num_obs_a = a.matchAndTrack(T_cur, T_key_w, groups, nmax, &td_a, &num_new_a);
  int boundary = 0;
  for (int g = 0; g + 1 < ng; ++g) boundary += sizes[g];
  std::vector<svs_tracked_point> tr_a;
  svs::PointStatistics st_a;
  int flags_a[9];
  bool drop_a = false;
  if (num_obs_a < 0 || a.processMatchedPoints(T_cur, cam, boundary, &tr_a, &st_a, flags_a, &drop_a) < 0) return 5;
  if (drop_a != svs::shallWeDropNewKeyframe(st_a, T_cur)) return 4;
  if (a.addMorePoints(cam, 2, &more_a, &rows) < 0) return 5;
  // the C ABI
  const svs_frontend_params p = SVS_FRONTEND_PARAMS_DEFAULT;
  const double I[7] = {0, 0, 0, 1, 0, 0, 0};
  int cap = 0;
  for (int l = 0; l < nlv; ++l) cap += (p.num_max_points >> l) + 1;
  std::vector<svs_new_point> fresh_b(cap), more_b(cap);
  std::vector<svs_match_point> rows_b(cap);
  const int nf = svs_addMorePoints(b.handle(), 1, I, &cam, 1, &p, fresh_b.data(), rows_b.data(), cap, nullptr);
  std::vector<svs_match_point> pts;
  std::vector<int> ends;
  for (const auto& g : groups) { pts.insert(pts.end(), g.begin(), g.end()); ends.push_back((int)pts.size()); }
  std::vector<svs_match_result> td_b(pts.size());
  int num_new_b = 0, num_obs_b = 0;
  if (nf < 0 || svs_match_track(b.handle(), T_cur, T_key_w, pts.data(), (int)pts.size(), ng, ends.data(), nmax, 4, 22, 10,
                                td_b.data(), &num_new_b, &num_obs_b) != SVS_OK)
    return 5;
  std::vector<svs_tracked_point> tr_b(pts.size());
  svs_point_stats st_b;
  int flags_b[9], drop_b = 0;
  const int ngb = svs_processMatchedPoints(b.handle(), T_cur, &cam, boundary, &p, tr_b.data(), &st_b, flags_b, &drop_b);
  if (ngb < 0) return 5;
  tr_b.resize(ngb);
  const int nm = svs_addMorePoints(b.handle(), 0, I, &cam, 2, &p, more_b.data(), rows_b.data(), cap, nullptr);
  if (nm < 0) return 5;
  fresh_b.resize(nf); more_b.resize(nm);
  if (!same(td_a, td_b) || num_new_a != num_new_b || num_obs_a != num_obs_b || !same(tr_a, tr_b) ||
      memcmp(&st_a, &st_b, sizeof st_a) || memcmp(flags_a, flags_b, sizeof flags_a) || (int)drop_a != drop_b ||
      !same(fresh_a, fresh_b) || !same(more_a, more_b)) {
    fprintf(stderr, "the wrapper and the C ABI differ\n");
    return 4;
  }
  FILE* o = fopen(argv[2], "wb");
  if (!o) return 2;
  const int head[4] = {num_obs_a, num_new_a, (int)drop_a, (int)tr_a.size()};
  wr(o, head, 4);
  wr(o, tr_a.data(), tr_a.size());
  wr(o, &st_a, 1);
  const int nfa = (int)fresh_a.size(), nma = (int)more_a.size();
  wr(o, &nfa, 1); wr(o, fresh_a.data(), fresh_a.size());
  wr(o, &nma, 1); wr(o, more_a.data(), more_a.size());
  fclose(o);
  return 0;
}
