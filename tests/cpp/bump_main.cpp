// svs::Bump (scavislam_b200/csrc/handle.cuh), the layout every module's device buffers are carved with: the sizing
// pass and the carve pass agree, every array is 256-byte aligned, the arrays are disjoint and in take order, n = 0 still
// gets a slot, and a nullptr base hands out nullptr.  Prints one line per failed check and exits 1 on any.
#include <cstdio>
#include <cstdlib>
#include <cstdint>
#include <vector>

#include "handle.cuh"

namespace {

struct Rec { double a[3]; };   // 24 bytes: a size that does not divide 256

struct Taken { size_t off, bytes; const char* p; };

int failures = 0;
void check(bool ok, const char* what, size_t i) {
  if (!ok) { std::printf("FAIL %s (array %zu)\n", what, i); ++failures; }
}

// the same takes on any base: the offset each array starts at, its bytes, and the pointer handed out
template <typename T>
void take(svs::Bump& m, size_t n, std::vector<Taken>& out) {
  const size_t off = m.off;
  const T* p = m.take<T>(n);
  out.push_back({off, n * sizeof(T), reinterpret_cast<const char*>(p)});
}
size_t carve(svs::Bump& m, std::vector<Taken>& out) {
  take<char>(m, 3, out);
  take<double>(m, 0, out);
  take<int>(m, 1000, out);
  take<Rec>(m, 7, out);
  take<unsigned long long>(m, 33, out);
  take<unsigned char>(m, 256, out);
  take<int>(m, 0, out);
  return m.off;
}

}  // namespace

int main() {
  std::vector<Taken> sz, cv;
  svs::Bump s{nullptr};
  const size_t total = carve(s, sz);
  for (size_t i = 0; i < sz.size(); ++i) check(sz[i].p == nullptr, "a nullptr base hands out nullptr", i);

  char* base = static_cast<char*>(std::aligned_alloc(256, total));
  if (!base) { std::printf("FAIL aligned_alloc\n"); return 1; }
  svs::Bump m{base};
  check(carve(m, cv) == total, "the carve pass ends where the sizing pass did", 0);
  check(sz.size() == cv.size(), "both passes take the same arrays", 0);
  for (size_t i = 0; i < cv.size() && i < sz.size(); ++i) {
    check(cv[i].off == sz[i].off, "both passes give the same offset", i);
    check(cv[i].p == base + cv[i].off, "the pointer lies at its offset", i);
    check(reinterpret_cast<uintptr_t>(cv[i].p) % 256 == 0, "256-byte aligned", i);
    const size_t end = i + 1 < cv.size() ? cv[i + 1].off : total;
    check(end > cv[i].off, "every array, n = 0 included, gets a slot", i);
    check(cv[i].off + cv[i].bytes <= end, "disjoint from the next array", i);
    check(end - cv[i].off == (cv[i].bytes + 255) / 256 * 256 + (cv[i].bytes == 0 ? 256 : 0), "the smallest 256-byte slot", i);
  }
  check(cv.empty() || cv[0].off == 0, "the first array starts the buffer", 0);
  std::free(base);
  if (failures) return 1;
  std::printf("OK %zu arrays in %zu bytes\n", cv.size(), total);
  return 0;
}
