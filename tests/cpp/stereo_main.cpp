// Drives svs::StereoBM (include/svs_b200.hpp) on one stereo pair and checks it against the C ABI on a second handle.
// Input (little-endian): int w, h, num_disparities, then the left and the right image, w*h bytes each.
// Output: the w*h float disparity map.  Exit 3 with NO_GPU without a device.
#include <cstdio>
#include <cstring>
#include <vector>

#include "svs_b200.hpp"

int main(int argc, char** argv) {
  if (argc < 3) return 2;
  FILE* f = fopen(argv[1], "rb");
  if (!f) return 2;
  int hd[3];
  if (fread(hd, sizeof(int), 3, f) != 3) return 2;
  const int w = hd[0], h = hd[1], nd = hd[2];
  std::vector<unsigned char> left((size_t)w * h), right((size_t)w * h);
  if (fread(left.data(), 1, left.size(), f) != left.size() || fread(right.data(), 1, right.size(), f) != right.size()) return 2;
  fclose(f);
  svs::StereoBM bm(w, h, nd);
  svs_stereo* c = nullptr;
  if (!bm.valid() || svs_stereo_create(-1, w, h, nd, &c) != SVS_OK) {
    printf("NO_GPU %s\n", bm.last_error());
    return 3;
  }
  std::vector<float> a((size_t)w * h), b((size_t)w * h);
  if (!bm.calcDisparity(left.data(), w, right.data(), w) || !bm.disparity(a.data())) {
    printf("FAIL calcDisparity: %s\n", bm.last_error());
    return 1;
  }
  const float* d = nullptr;
  int stride = 0;
  if (!bm.disparityDevice(&d, &stride) || !d || stride < w) {
    printf("FAIL disparityDevice\n");
    return 1;
  }
  if (svs_stereo_compute(c, left.data(), w, 0, right.data(), w, 0) != SVS_OK || svs_stereo_get(c, b.data()) != SVS_OK) {
    printf("FAIL C ABI: %s\n", svs_stereo_last_error(c));
    return 1;
  }
  if (std::memcmp(a.data(), b.data(), a.size() * sizeof(float)) != 0) {
    printf("FAIL the C++ layer and the C ABI differ\n");
    return 1;
  }
  svs_stereo_destroy(c);
  FILE* out = fopen(argv[2], "wb");
  fwrite(a.data(), sizeof(float), a.size(), out);
  fclose(out);
  int valid = 0;
  for (float v : a) valid += v > 0;
  printf("OK %dx%d valid=%d\n", w, h, valid);
  return 0;
}
