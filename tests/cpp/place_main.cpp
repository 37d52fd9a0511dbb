// Drives svs::PlaceRecognizer (include/svs_b200.hpp) over a keyframe sequence and checks every call against the
// C ABI on a second handle.  Input (little-endian): int W, double cam[4], float words[W][64], int K, then per keyframe
// int id, n, do_loop, n_excl, int excl[n_excl], float desc[n][64], double uvu[n][3].
// Output: per keyframe int best_id, num_inliers, loop_found, then double T[7].  Exit 3 with NO_GPU without a device.
#include <cstdio>
#include <cstring>
#include <vector>

#include "svs_b200.hpp"

template <class T>
static bool rd(FILE* f, T* p, size_t n) { return fread(p, sizeof(T), n, f) == n; }

int main(int argc, char** argv) {
  if (argc < 3) return 2;
  FILE* f = fopen(argv[1], "rb");
  if (!f) return 2;
  int W = 0, K = 0;
  svs_cam cam;
  if (!rd(f, &W, 1) || !rd(f, &cam.f, 1) || !rd(f, &cam.px, 1) || !rd(f, &cam.py, 1) || !rd(f, &cam.b, 1)) return 2;
  std::vector<float> words(64 * (size_t)W);
  if (!rd(f, words.data(), words.size()) || !rd(f, &K, 1)) return 2;
  svs::PlaceRecognizer pr(words, cam);
  svs_place* c = nullptr;
  if (!pr.valid() || svs_place_create(-1, W, words.data(), &cam, &c) != SVS_OK) {
    printf("NO_GPU %s\n", pr.last_error());
    return 3;
  }
  FILE* out = fopen(argv[2], "wb");
  int loops = 0;
  for (int k = 0; k < K; ++k) {
    int hd[4];
    if (!rd(f, hd, 4)) return 2;
    const int id = hd[0], n = hd[1], do_loop = hd[2], ne = hd[3];
    std::vector<int> excl(ne);
    std::vector<float> desc(64 * (size_t)n);
    std::vector<double> uvu(3 * (size_t)n);
    if (!rd(f, excl.data(), ne) || !rd(f, desc.data(), desc.size()) || !rd(f, uvu.data(), uvu.size())) return 2;
    svs::DetectedLoop loop;
    std::vector<int> iq, it;
    if (!pr.addLocation(id, desc, uvu, excl, do_loop != 0, &loop, &iq, &it)) {
      printf("FAIL addLocation %d: %s\n", id, pr.last_error());
      return 1;
    }
    svs_place_result r;
    std::vector<int> cq((size_t)n + 1), ct((size_t)n + 1);
    svs_place_params p = SVS_PLACE_PARAMS_DEFAULT;
    if (svs_place_add_location(c, id, n, desc.data(), uvu.data(), do_loop, ne, excl.data(), &p, &r, cq.data(),
                               ct.data()) != SVS_OK) {
      printf("FAIL C ABI %d: %s\n", id, svs_place_last_error(c));
      return 1;
    }
    const svs_place_result& a = pr.last_result();
    const bool same = a.best_keyframe_id == r.best_keyframe_id && a.num_inliers == r.num_inliers &&
                      a.num_matches == r.num_matches && a.loop_found == r.loop_found &&
                      std::memcmp(a.T_query_from_loop, r.T_query_from_loop, sizeof r.T_query_from_loop) == 0 &&
                      std::equal(iq.begin(), iq.end(), cq.begin()) && std::equal(it.begin(), it.end(), ct.begin());
    if (!same) {
      printf("FAIL keyframe %d: the C++ layer and the C ABI differ\n", id);
      return 1;
    }
    if (r.loop_found) {
      if (loop.query_keyframe_id != id || loop.loop_keyframe_id != r.best_keyframe_id ||
          std::memcmp(loop.T_query_from_loop.q, r.T_query_from_loop, 4 * sizeof(double)) != 0) {
        printf("FAIL keyframe %d: DetectedLoop\n", id);
        return 1;
      }
      ++loops;
    }
    const int o3[3] = {r.best_keyframe_id, r.num_inliers, r.loop_found};
    fwrite(o3, sizeof(int), 3, out);
    fwrite(r.T_query_from_loop, sizeof(double), 7, out);
  }
  fclose(out);
  fclose(f);
  svs_place_destroy(c);
  printf("OK keyframes=%d loops=%d\n", K, loops);
  return 0;
}
