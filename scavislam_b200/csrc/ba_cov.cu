// ba_cov.cu -- k_ba_point_cov: the landmark blocks of (H + lambda I)^-1 (svs_ba_covariance).
//
// With H = [[A, B], [B^T, C]] over (poses, landmarks), S = A - B C^-1 B^T the reduced system and Z = S^-1, the block of
// landmark l is
//     Sigma_ll = D + D M D,    M = sum_{a,b} Hpl_a^T Z_ab Hpl_b,    D = (Hll + lambda I)^-1,
// over the slots a, b of l (anchor, then observers; Hpl_a = BaDev::W of the slot, Hll = BaDev::Dbl, both as the build
// left them).  Every pose pair of a track lies in the factor's pattern, so Z_ab comes from the selected inversion.
// Zero-weight padding slots and fixed poses have Hpl = 0 and add exactly nothing.  Z_ba = Z_ab^T, so M is summed over
// the pairs a <= b, a pair a < b adding C + C^T with C = Hpl_a^T Z_ab Hpl_b.
#include "ba_dev.cuh"
#include "ba_kernels.cuh"

namespace svs {

namespace {

constexpr int kCovThreads = 256;
constexpr int kShortTrack = 8;   // slots of a track a group of kShortLanes lanes takes; longer tracks get a warp
constexpr int kShortLanes = 8;

// One group of LANES lanes per landmark of `list` (nullptr: landmark idx) whose slot count falls on this instance's
// side of kShortTrack.  Lane `sub` takes the pairs sub, sub + LANES, ... of the a-major list of pairs a <= b; the nine
// partial sums are reduced over the group by a butterfly, which leaves the same bits on every lane.  The output is in
// the caller's landmark order, row-major, its lower triangle the mirror of the upper.
template <int LANES>
__global__ void __launch_bounds__(kCovThreads)
k_ba_point_cov(BaDev d, const double* __restrict__ Z, const int* __restrict__ list, int n, double lambda,
               double* __restrict__ out) {
  const int lane = threadIdx.x & 31, sub = lane & (LANES - 1);
  const int idx = (int)((blockIdx.x * (unsigned)kCovThreads + threadIdx.x) / LANES);
  if (idx >= n) return;   // whole groups leave together
  const int li = list ? __ldg(list + idx) : idx;
  const int s0 = __ldg(d.lm_sptr + li), K = __ldg(d.lm_sptr + li + 1) - s0;
  if ((K > kShortTrack) != (LANES == 32)) return;   // the other instance's landmark
  const unsigned gmask = LANES == 32 ? 0xffffffffu : ((1u << LANES) - 1u) << (lane & ~(LANES - 1));
  const int e0 = __ldg(d.lm_eptr + li), k = __ldg(d.lm_eptr + li + 1) - e0;
  double* o = out + 9 * (size_t)__ldg(d.lm_user + li);
  if (k == 0 || d.ctl->chol_fail) {
    for (int q = sub; q < 9; q += LANES) o[q] = 0.;
    return;
  }
  const int off = __ldg(d.lm_self + li) ? 0 : 1, ia = __ldg(d.lm_anchor + li), P = d.P;
  const size_t ns = (size_t)d.nslots;
  const double* __restrict__ W = d.W + s0;
  double M[9];
#pragma unroll
  for (int q = 0; q < 9; ++q) M[q] = 0.;
  int a = 0, rem = sub;   // pair (a, a + rem)
  while (a < K && rem >= K - a) { rem -= K - a; ++a; }
  while (a < K) {
    const int b = a + rem;
    const int pa = a == 0 ? ia : __ldg(d.e_pose + e0 + a - off);
    const int pb = b == 0 ? ia : __ldg(d.e_pose + e0 + b - off);
    const int t = __ldg(d.tbl + (size_t)pa * P + pb);
    const double* Zab = Z + 36 * (size_t)(t >> 1);
    const int zr = (t & 1) ? 1 : 6, zc = (t & 1) ? 6 : 1;   // element (r, q) of Z_ab is Zab[r zr + q zc]
    double Hb[18];
#pragma unroll
    for (int q = 0; q < 18; ++q) Hb[q] = __ldg(W + q * ns + b);
    double Cab[9];
#pragma unroll
    for (int q = 0; q < 9; ++q) Cab[q] = 0.;
#pragma unroll
    for (int r = 0; r < 6; ++r) {
      double u0 = 0., u1 = 0., u2 = 0.;   // row r of Z_ab Hpl_b
#pragma unroll
      for (int q = 0; q < 6; ++q) {
        const double z = __ldg(Zab + r * zr + q * zc);
        u0 = fma(z, Hb[3 * q], u0);
        u1 = fma(z, Hb[3 * q + 1], u1);
        u2 = fma(z, Hb[3 * q + 2], u2);
      }
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        const double h = __ldg(W + (3 * r + i) * ns + a);   // Hpl_a (r, i)
        Cab[3 * i] = fma(h, u0, Cab[3 * i]);
        Cab[3 * i + 1] = fma(h, u1, Cab[3 * i + 1]);
        Cab[3 * i + 2] = fma(h, u2, Cab[3 * i + 2]);
      }
    }
    if (a == b) {
#pragma unroll
      for (int q = 0; q < 9; ++q) M[q] += Cab[q];
    } else {
#pragma unroll
      for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) M[3 * i + j] += Cab[3 * i + j] + Cab[3 * j + i];
    }
    rem += LANES;
    while (a < K && rem >= K - a) { rem -= K - a; ++a; }
  }
#pragma unroll
  for (int q = 0; q < 9; ++q)
#pragma unroll
    for (int s = LANES / 2; s > 0; s >>= 1) M[q] += __shfl_xor_sync(gmask, M[q], s);
  double D[9];
  inv3_sym_lambda(d.Dbl + 12 * (size_t)li, lambda, D);
#pragma unroll
  for (int q = 0; q < 9; ++q) {
    const int i = min(q / 3, q % 3), j = max(q / 3, q % 3);   // (i, j) and (j, i) get the same bits
    double s = D[3 * i + j];
#pragma unroll
    for (int p = 0; p < 3; ++p) {
      const double dm = D[3 * i] * M[p] + D[3 * i + 1] * M[3 + p] + D[3 * i + 2] * M[6 + p];   // (D M)(i, p)
      s = fma(dm, D[3 * p + j], s);
    }
    if (q % LANES == sub) o[q] = s;
  }
}

template <int LANES>
void launch_one(const BaDev& d, const double* Z, const int* list, int n, double lambda, double* out, cudaStream_t st) {
  if (n <= 0) return;
  const long long threads = (long long)n * LANES;
  k_ba_point_cov<LANES><<<(unsigned)((threads + kCovThreads - 1) / kCovThreads), kCovThreads, 0, st>>>(d, Z, list, n, lambda,
                                                                                                       out);
}

}  // namespace

// Tracks of up to kShortTrack slots (most of them): kShortLanes lanes each, over all landmarks; the longer tracks, which
// the build also lists apart (gen_lm: 9..32 slots or no observations, long_lm: more than 32), one warp each.
void launch_point_cov(const BaDev& d, const double* Z, double lambda, double* out, cudaStream_t st) {
  launch_one<kShortLanes>(d, Z, nullptr, d.L, lambda, out, st);
  launch_one<32>(d, Z, d.gen_lm, d.ngen, lambda, out, st);
  launch_one<32>(d, Z, d.long_lm, d.nlong, lambda, out, st);
}

}  // namespace svs
