// place.cu -- PlaceRecognizer::addLocation (scavislam/placerecognizer.cpp:206-324) on the device: vocabulary words,
// TF-IDF scores over the stored places (calcLoopStatistics, :131-172), the brute-force match against the best
// candidate and the 3-point absolute-orientation RANSAC of geometricCheck (:175-202, ransac.cpp:29-137,
// ransac_models.cpp:27-181).  Semantics and deviations: include/svs_b200.h (svs_place).
//
// One call is one stream of kernels with no host round trip: the inputs go in, one result record comes back.
//   k_place_nn (words)  -> k_place_assign -> k_place_score -> k_place_select -> k_place_nn (match, reads the winner
//   from device memory) -> k_place_match_fin -> k_place_ransac -> k_place_finish -> k_place_insert
// Built with -fmad=false: the descriptor distance is an explicit __fmaf_rn chain, everything else is restated
// operation by operation as oracle/place_oracle.c writes it.
#include <algorithm>
#include <climits>
#include <cmath>
#include <cstring>
#include <string>
#include <unordered_map>
#include <vector>

#include <cuda_runtime.h>

#include "../../include/svs_b200.h"
#include "handle.cuh"

// named (not anonymous) so the kernels keep stable symbol names in traces: place::k_place_nn, ...
namespace place {

constexpr int kDim = 64;
constexpr int kTile = 64;           // query rows per CTA and train rows per shared-memory tile
constexpr int kNNThreads = 256;     // 16 x 16 threads, each a 4 x 4 tile of (query, train) pairs
constexpr int kMaxDraws = 64;
constexpr int kJacobiSweeps = 32;
constexpr int kRansacWarps = 4;
constexpr float kWordRadius = 0.1f;

struct PlaceRes {           // the record one call reads back
  int best_place;           // index into the database, -1 = none
  int best_kf;
  float best_score;
  int num_matches;
  int num_inliers;
  int nwords;
  int ndistinct;
  int best_h;
  int num_hyp;
  int pad;
  double T[7];
};

struct Cam { double f, px, py, b; };

// ---------------------------------------------------------------- nearest neighbour
// Train rows [t0, t1) of tile size kTile; CTA (bx, by) takes query block bx and the by-th slice of the train tiles.
// With sel != nullptr the train set is the stored place *sel (nothing to do when it is -1).
__global__ void __launch_bounds__(kNNThreads) k_place_nn(const float* __restrict__ Q, int n, const float* __restrict__ T,
                                                         int m, const int* sel, const int* __restrict__ row_off,
                                                         const int* __restrict__ nrows,
                                                         unsigned long long* __restrict__ best) {
  if (sel) {
    const int k = *sel;
    if (k < 0) return;
    T += (size_t)row_off[k] * kDim;
    m = nrows[k];
  }
  const int tiles = (m + kTile - 1) / kTile;
  const int per = (tiles + gridDim.y - 1) / gridDim.y;
  const int tb = blockIdx.y * per, te = min(tiles, tb + per);
  if (tb >= te) return;
  __shared__ __align__(16) float sQ[kDim][kTile];
  __shared__ __align__(16) float sT[kDim][kTile];
  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
  const int q0 = blockIdx.x * kTile;
  for (int it = tid; it < kTile * kDim / 4; it += kNNThreads) {
    const int qi = it % kTile, k4 = (it / kTile) * 4;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (q0 + qi < n) v = *reinterpret_cast<const float4*>(Q + (size_t)(q0 + qi) * kDim + k4);
    sQ[k4][qi] = v.x; sQ[k4 + 1][qi] = v.y; sQ[k4 + 2][qi] = v.z; sQ[k4 + 3][qi] = v.w;
  }
  unsigned long long run[4] = {~0ull, ~0ull, ~0ull, ~0ull};
  for (int tile = tb; tile < te; ++tile) {
    const int j0 = tile * kTile;
    __syncthreads();
    for (int it = tid; it < kTile * kDim / 4; it += kNNThreads) {
      const int ti = it % kTile, k4 = (it / kTile) * 4;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (j0 + ti < m) v = *reinterpret_cast<const float4*>(T + (size_t)(j0 + ti) * kDim + k4);
      sT[k4][ti] = v.x; sT[k4 + 1][ti] = v.y; sT[k4 + 2][ti] = v.z; sT[k4 + 3][ti] = v.w;
    }
    __syncthreads();
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
#pragma unroll 8
    for (int k = 0; k < kDim; ++k) {
      const float4 q = *reinterpret_cast<const float4*>(&sQ[k][ty * 4]);
      const float4 t = *reinterpret_cast<const float4*>(&sT[k][tx * 4]);
      const float qv[4] = {q.x, q.y, q.z, q.w}, tv[4] = {t.x, t.y, t.z, t.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float d = __fsub_rn(qv[i], tv[j]);
          acc[i][j] = __fmaf_rn(d, d, acc[i][j]);
        }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int idx = j0 + tx * 4 + j;
      if (idx >= m) continue;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        // non-negative float bits order like the floats: the packed minimum is (distance, lowest index)
        const unsigned long long key = ((unsigned long long)__float_as_uint(acc[i][j]) << 32) | (unsigned)idx;
        run[i] = min(run[i], key);
      }
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
#pragma unroll
    for (int o = 8; o >= 1; o >>= 1) run[i] = min(run[i], __shfl_xor_sync(0xffffffffu, run[i], o));
    const int q = q0 + ty * 4 + i;
    if (tx == 0 && q < n) atomicMin(best + q, run[i]);
  }
}

// word[r] = nearest word when its distance is below the radius; per-word first row and count of this keyframe
__global__ void k_place_assign(const unsigned long long* __restrict__ best, int n, int* __restrict__ word,
                               int* __restrict__ first_row, int* __restrict__ kf_count, PlaceRes* res) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  const unsigned long long b = best[r];
  const float d = __uint_as_float((unsigned)(b >> 32));
  const int w = d < kWordRadius ? (int)(unsigned)(b & 0xffffffffu) : -1;
  word[r] = w;
  if (w < 0) return;
  atomicMin(first_row + w, r);
  atomicAdd(kf_count + w, 1);
  atomicAdd(&res->nwords, 1);
}

// ---------------------------------------------------------------- TF-IDF
// One warp per stored place k: 32 rows at a time, each lane binary-searches its row's word in k's sorted
// (word, count) list; lane 0 adds the 32 products in row order.  c_w(r) = places holding w before this call, plus
// the current keyframe once an earlier row of it took w (the reference inserts into inverted_index_ per descriptor).
__global__ void k_place_score(int L, int n, const int* __restrict__ word, const int* __restrict__ first_row,
                              const int* __restrict__ cw, const int* __restrict__ wl_off, const int* __restrict__ wl_n,
                              const int* __restrict__ wl_word, const int* __restrict__ wl_count,
                              const int* __restrict__ nwords, const unsigned char* __restrict__ excluded,
                              float* __restrict__ score) {
  const int k = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (k >= L) return;
  float s = 0.f;
  if (!excluded[k]) {
    const int* lw = wl_word + wl_off[k];
    const int* lc = wl_count + wl_off[k];
    const int len = wl_n[k];
    const float fL = (float)L, fnw = (float)nwords[k];
    for (int r0 = 0; r0 < n; r0 += 32) {
      const int r = r0 + lane;
      float val = 0.f;
      const int w = r < n ? word[r] : -1;
      if (w >= 0) {
        int lo = 0, hi = len;
        while (lo < hi) {
          const int mid = (lo + hi) >> 1;
          if (lw[mid] < w) lo = mid + 1; else hi = mid;
        }
        if (lo < len && lw[lo] == w) {
          const int c = cw[w] + (first_row[w] < r ? 1 : 0);
          val = __fmul_rn(__fdiv_rn((float)lc[lo], fnw), __fdiv_rn(fL, (float)c));
        }
      }
      const int last = min(32, n - r0);
      for (int j = 0; j < last; ++j) s = __fadd_rn(s, __shfl_sync(0xffffffffu, val, j));   // +0 leaves s >= 0 alone
    }
  }
  if (lane == 0) score[k] = s;
}

struct Cand { float s; int id, k; };

__device__ __forceinline__ Cand better(Cand a, Cand b) {
  if (b.k < 0) return a;
  if (a.k < 0) return b;
  if (b.s > a.s || (b.s == a.s && b.id < a.id)) return b;
  return a;
}

// the largest score > 2, ties to the smallest keyframe id
__global__ void __launch_bounds__(1024) k_place_select(int L, const float* __restrict__ score,
                                                       const int* __restrict__ place_id, PlaceRes* res) {
  __shared__ Cand sc[32];
  Cand c{0.f, 0, -1};
  for (int k = threadIdx.x; k < L; k += blockDim.x)
    if (score[k] > 2.f) c = better(c, Cand{score[k], place_id[k], k});
  for (int o = 16; o >= 1; o >>= 1) {
    Cand d{__shfl_xor_sync(0xffffffffu, c.s, o), __shfl_xor_sync(0xffffffffu, c.id, o),
           __shfl_xor_sync(0xffffffffu, c.k, o)};
    c = better(c, d);
  }
  if ((threadIdx.x & 31) == 0) sc[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    Cand b{0.f, 0, -1};
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) b = better(b, sc[w]);
    res->best_place = b.k;
    res->best_kf = b.k >= 0 ? b.id : -1;
    res->best_score = b.k >= 0 ? b.s : 0.f;
  }
}

__global__ void k_place_match_fin(const unsigned long long* __restrict__ best, int n, const int* __restrict__ nrows,
                                  PlaceRes* res, int* __restrict__ train_idx, float* __restrict__ dist) {
  const int k = res->best_place;
  if (k < 0 || nrows[k] == 0) return;
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r == 0) res->num_matches = n;
  if (r >= n) return;
  const unsigned long long b = best[r];
  train_idx[r] = (int)(unsigned)(b & 0xffffffffu);
  dist[r] = __fsqrt_rn(__uint_as_float((unsigned)(b >> 32)));
}

// ---------------------------------------------------------------- geometry (double)
__device__ __forceinline__ void unmap_uvu(const Cam& c, const double* uvu, double* xyz) {
  const double sd = __ddiv_rn(__dsub_rn(uvu[0], uvu[2]), c.b);
  const double z = __ddiv_rn(c.f, sd);
  xyz[0] = __dmul_rn(__ddiv_rn(__dsub_rn(uvu[0], c.px), c.f), z);
  xyz[1] = __dmul_rn(__ddiv_rn(__dsub_rn(uvu[1], c.py), c.f), z);
  xyz[2] = z;
}

__device__ __forceinline__ bool below_threshold(const Cam& c, const double* R, const double* t, const double* X,
                                                const double* obs, double thr2) {
  double p[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) p[i] = ((R[3 * i] * X[0] + R[3 * i + 1] * X[1]) + R[3 * i + 2] * X[2]) + t[i];
  const double u = c.f * (p[0] / p[2]) + c.px;
  const double v = c.f * (p[1] / p[2]) + c.py;
  const double ur = (p[0] - c.b) / p[2] * c.f + c.px;
  const double du = obs[0] - u, dv = obs[1] - v, dr = obs[2] - ur;
  return du * du < thr2 && dv * dv < thr2 && dr * dr < thr2;
}

// Kabsch with H = sum p1 p0^T on the centred triple, one-sided Jacobi SVD, u3 = u1 x u2, determinant fix
__device__ void kabsch(const double* p0_in, const double* p1_in, double* R, double* t) {
  double p0[9], p1[9], c0[3], c1[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    c0[i] = ((p0_in[i] + p0_in[3 + i]) + p0_in[6 + i]) * (1.0 / 3.0);
    c1[i] = ((p1_in[i] + p1_in[3 + i]) + p1_in[6 + i]) * (1.0 / 3.0);
  }
#pragma unroll
  for (int a = 0; a < 3; ++a)
#pragma unroll
    for (int i = 0; i < 3; ++i) { p0[3 * a + i] = p0_in[3 * a + i] - c0[i]; p1[3 * a + i] = p1_in[3 * a + i] - c1[i]; }
  double A[9], V[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) A[3 * i + j] = (p1[i] * p0[j] + p1[3 + i] * p0[3 + j]) + p1[6 + i] * p0[6 + j];
  for (int sweep = 0; sweep < kJacobiSweeps; ++sweep) {
    bool rotated = false;
#pragma unroll
    for (int pq = 0; pq < 3; ++pq) {
      const int p = pq == 2 ? 1 : 0, q = pq == 0 ? 1 : 2;
      const double al = (A[p] * A[p] + A[3 + p] * A[3 + p]) + A[6 + p] * A[6 + p];
      const double be = (A[q] * A[q] + A[3 + q] * A[3 + q]) + A[6 + q] * A[6 + q];
      const double ga = (A[p] * A[q] + A[3 + p] * A[3 + q]) + A[6 + p] * A[6 + q];
      if (!(fabs(ga) > 1e-15 * sqrt(al * be))) continue;
      const double ze = (be - al) / (2.0 * ga);
      const double tt = (ze >= 0.0 ? 1.0 : -1.0) / (fabs(ze) + sqrt(1.0 + ze * ze));
      const double cs = 1.0 / sqrt(1.0 + tt * tt), sn = cs * tt;
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        const double ap = A[3 * i + p], aq = A[3 * i + q];
        A[3 * i + p] = cs * ap - sn * aq;
        A[3 * i + q] = sn * ap + cs * aq;
        const double vp = V[3 * i + p], vq = V[3 * i + q];
        V[3 * i + p] = cs * vp - sn * vq;
        V[3 * i + q] = sn * vp + cs * vq;
      }
      rotated = true;
    }
    if (!rotated) break;
  }
  double sg[3];
#pragma unroll
  for (int j = 0; j < 3; ++j) sg[j] = sqrt((A[j] * A[j] + A[3 + j] * A[3 + j]) + A[6 + j] * A[6 + j]);
  int o[3] = {0, 1, 2};
  for (int a = 0; a < 2; ++a)
    for (int b = 0; b < 2 - a; ++b)
      if (sg[o[b + 1]] > sg[o[b]]) { const int tmp = o[b]; o[b] = o[b + 1]; o[b + 1] = tmp; }
  double u1[3], u2[3], u3[3], v1[3], v2[3], v3[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    u1[i] = A[3 * i + o[0]] / sg[o[0]];
    u2[i] = A[3 * i + o[1]] / sg[o[1]];
    v1[i] = V[3 * i + o[0]]; v2[i] = V[3 * i + o[1]]; v3[i] = V[3 * i + o[2]];
  }
  u3[0] = u1[1] * u2[2] - u1[2] * u2[1];
  u3[1] = u1[2] * u2[0] - u1[0] * u2[2];
  u3[2] = u1[0] * u2[1] - u1[1] * u2[0];
  for (int pass = 0; pass < 2; ++pass) {
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int j = 0; j < 3; ++j) R[3 * i + j] = (v1[i] * u1[j] + v2[i] * u2[j]) + v3[i] * u3[j];
    const double det = R[0] * (R[4] * R[8] - R[5] * R[7]) - R[1] * (R[3] * R[8] - R[5] * R[6]) +
                       R[2] * (R[3] * R[7] - R[4] * R[6]);
    if (!(det < 0.0)) break;
#pragma unroll
    for (int i = 0; i < 3; ++i) v3[i] = -v3[i];
  }
#pragma unroll
  for (int i = 0; i < 3; ++i) t[i] = c0[i] - ((R[3 * i] * c1[0] + R[3 * i + 1] * c1[1]) + R[3 * i + 2] * c1[2]);
}

__device__ __forceinline__ unsigned long long splitmix_next(unsigned long long& st) {
  unsigned long long z = (st += 0x9E3779B97F4A7C15ull);
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

// the sampling loop of RanSaC::compute with hypothesis h's own stream; false = void after kMaxDraws draws
__device__ bool draw_triple(unsigned long long seed, int h, int nmatch, const int* train_idx, int* tri) {
  unsigned long long st = seed ^ (0xD1B54A32D192ED03ull * (unsigned long long)(h + 1));
  int draws = 0;
  for (;;) {
    for (int i = 0; i < 3; ++i) {
      bool dup;
      do {
        if (draws == kMaxDraws) return false;
        tri[i] = (int)(((splitmix_next(st) >> 32) * (unsigned long long)nmatch) >> 32);
        ++draws;
        dup = false;
        for (int j = 0; j < i; ++j) dup |= tri[j] == tri[i];
      } while (dup);
    }
    bool clash = false;
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < i; ++j) clash |= tri[i] == tri[j] || train_idx[tri[i]] == train_idx[tri[j]];
    if (!clash) return true;
  }
}

struct RansacArgs {
  const PlaceRes* res;
  int n, num_ransac;
  unsigned long long seed;
  double thr2;
  Cam cam;
  const double* uvu;
  const double* xyz;      // the database's points
  const int* row_off;
  const int* train_idx;
  int* hyp_triple;        // [H][3]
  int* hyp_inl;           // [H], -1 = void
  double* hyp_RT;         // [H][12]
};

// one warp per hypothesis: lane 0 draws, every lane solves the same triple, the warp counts the inliers
__global__ void __launch_bounds__(kRansacWarps * 32) k_place_ransac(RansacArgs a) {
  const int k = a.res->best_place;
  if (k < 0 || a.n < 3) return;
  const int h = blockIdx.x * kRansacWarps + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (h >= a.num_ransac) return;
  int tri[3] = {-1, -1, -1};
  int ok = 0;
  if (lane == 0) ok = draw_triple(a.seed, h, a.n, a.train_idx, tri);
  ok = __shfl_sync(0xffffffffu, ok, 0);
#pragma unroll
  for (int i = 0; i < 3; ++i) tri[i] = __shfl_sync(0xffffffffu, tri[i], 0);
  if (lane < 3) a.hyp_triple[3 * h + lane] = ok ? tri[lane] : -1;
  if (!ok) {
    if (lane == 0) a.hyp_inl[h] = -1;
    return;
  }
  const double* xyz = a.xyz + 3 * (size_t)a.row_off[k];
  double p0[9], p1[9], R[9], t[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    unmap_uvu(a.cam, a.uvu + 3 * (size_t)tri[i], p0 + 3 * i);
    const double* X = xyz + 3 * (size_t)a.train_idx[tri[i]];
    p1[3 * i] = X[0]; p1[3 * i + 1] = X[1]; p1[3 * i + 2] = X[2];
  }
  kabsch(p0, p1, R, t);
  int inl = 0;
  for (int r = lane; r < a.n; r += 32)
    inl += below_threshold(a.cam, R, t, xyz + 3 * (size_t)a.train_idx[r], a.uvu + 3 * (size_t)r, a.thr2);
  inl = __reduce_add_sync(0xffffffffu, inl);
  if (lane == 0) a.hyp_inl[h] = inl;
  if (lane < 9) a.hyp_RT[12 * (size_t)h + lane] = R[lane];
  else if (lane < 12) a.hyp_RT[12 * (size_t)h + lane] = t[lane - 9];
}

// exclusive block scan of one int per thread (blockDim.x = 1024); *total receives the sum
__device__ int block_excl_scan(int v, int* total) {
  __shared__ int ws[32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) ws[wid] = x;
  __syncthreads();
  if (wid == 0) {
    int s = lane < (int)(blockDim.x >> 5) ? ws[lane] : 0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, s, o);
      if (lane >= o) s += y;
    }
    ws[lane] = s;
  }
  __syncthreads();
  const int incl = x + (wid > 0 ? ws[wid - 1] : 0);
  *total = ws[(blockDim.x >> 5) - 1];
  __syncthreads();
  return incl - v;
}

// Eigen's Quaternion-from-rotation-matrix
__device__ void quat_from_R(const double* R, double* q) {
  const double tr = (R[0] + R[4]) + R[8];
  if (tr > 0.0) {
    double s = sqrt(tr + 1.0);
    q[3] = 0.5 * s;
    s = 0.5 / s;
    q[0] = (R[7] - R[5]) * s;
    q[1] = (R[2] - R[6]) * s;
    q[2] = (R[3] - R[1]) * s;
  } else {
    int i = 0;
    if (R[4] > R[0]) i = 1;
    if (R[8] > R[3 * i + i]) i = 2;
    const int j = (i + 1) % 3, k = (j + 1) % 3;
    double s = sqrt(R[3 * i + i] - R[3 * j + j] - R[3 * k + k] + 1.0);
    q[i] = 0.5 * s;
    s = 0.5 / s;
    q[3] = (R[3 * k + j] - R[3 * j + k]) * s;
    q[j] = (R[3 * j + i] + R[3 * i + j]) * s;
    q[k] = (R[3 * k + i] + R[3 * i + k]) * s;
  }
}

// best hypothesis (most inliers, lowest h), its inliers in match order, the result record
__global__ void __launch_bounds__(1024) k_place_finish(RansacArgs a, int* __restrict__ inl_q, int* __restrict__ inl_t) {
  PlaceRes* res = const_cast<PlaceRes*>(a.res);
  const int k = res->best_place;
  if (k < 0 || a.n < 3) return;
  __shared__ int sBest;
  __shared__ double sRT[12];
  if (threadIdx.x == 0) {
    int bh = -1, bi = 0;
    for (int h = 0; h < a.num_ransac; ++h)
      if (a.hyp_inl[h] > bi) { bi = a.hyp_inl[h]; bh = h; }
    sBest = bh;
    for (int i = 0; i < 12; ++i) sRT[i] = bh >= 0 ? a.hyp_RT[12 * (size_t)bh + i] : (i == 0 || i == 4 || i == 8 ? 1.0 : 0.0);
  }
  __syncthreads();
  double R[9], t[3];
#pragma unroll
  for (int i = 0; i < 9; ++i) R[i] = sRT[i];
#pragma unroll
  for (int i = 0; i < 3; ++i) t[i] = sRT[9 + i];
  const double* xyz = a.xyz + 3 * (size_t)a.row_off[k];
  int base = 0;
  for (int r0 = 0; r0 < a.n; r0 += blockDim.x) {
    const int r = r0 + threadIdx.x;
    const int f = r < a.n && below_threshold(a.cam, R, t, xyz + 3 * (size_t)a.train_idx[r], a.uvu + 3 * (size_t)r, a.thr2);
    int total;
    const int pos = base + block_excl_scan(f, &total);
    if (f) { inl_q[pos] = r; inl_t[pos] = a.train_idx[r]; }
    base += total;
  }
  if (threadIdx.x == 0) {
    res->num_inliers = base;
    res->best_h = sBest;
    res->num_hyp = a.num_ransac;
    quat_from_R(R, res->T);
    for (int i = 0; i < 3; ++i) res->T[4 + i] = t[i];
  }
}

// Insert the new place: sorted (word, count) list by a scan over the vocabulary, c_w += 1 for its words, the
// per-keyframe scratch reset, xyz = unmap_uvu(uvu) of its rows, and its entry in the per-place arrays.
struct InsertArgs {
  int W, n, L, row_off, wl_off, id;
  Cam cam;
  const double* uvu;
  int* first_row;
  int* kf_count;
  int* cw;
  int* wl_word;
  int* wl_count;
  double* xyz;
  int* p_row_off;
  int* p_nrows;
  int* p_wl_off;
  int* p_wl_n;
  int* p_nwords;
  int* p_id;
  PlaceRes* res;
};

__global__ void __launch_bounds__(1024) k_place_insert(InsertArgs a) {
  int base = 0;
  for (int w0 = 0; w0 < a.W; w0 += blockDim.x) {
    const int w = w0 + threadIdx.x;
    const int c = w < a.W ? a.kf_count[w] : 0;
    int total;
    const int pos = base + block_excl_scan(c > 0, &total);
    if (c > 0) {
      a.wl_word[a.wl_off + pos] = w;
      a.wl_count[a.wl_off + pos] = c;
      a.cw[w] += 1;
      a.kf_count[w] = 0;
      a.first_row[w] = INT_MAX;
    }
    base += total;
  }
  for (int r = threadIdx.x; r < a.n; r += blockDim.x) unmap_uvu(a.cam, a.uvu + 3 * (size_t)r, a.xyz + 3 * ((size_t)a.row_off + r));
  if (threadIdx.x == 0) {
    a.p_row_off[a.L] = a.row_off; a.p_nrows[a.L] = a.n; a.p_wl_off[a.L] = a.wl_off; a.p_wl_n[a.L] = base;
    a.p_nwords[a.L] = a.res->nwords; a.p_id[a.L] = a.id;
    a.res->ndistinct = base;
  }
}

__global__ void k_fill_int(int* p, int n, int v) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}

}  // namespace place

using namespace place;

// ---------------------------------------------------------------- handle
template <class T>
struct DevArr {             // device array that grows geometrically and keeps its contents
  T* p = nullptr;
  size_t cap = 0;
  cudaError_t reserve(size_t need, cudaStream_t s) {
    if (need <= cap) return cudaSuccess;
    const size_t nc = std::max(need, 2 * cap);
    T* q = nullptr;
    cudaError_t e = cudaMalloc(&q, nc * sizeof(T));
    if (e != cudaSuccess) return e;
    if (cap) {
      e = cudaMemcpyAsync(q, p, cap * sizeof(T), cudaMemcpyDeviceToDevice, s);
      if (e == cudaSuccess) e = cudaStreamSynchronize(s);
      if (e != cudaSuccess) { cudaFree(q); return e; }
    }
    cudaFree(p);
    p = q;
    cap = nc;
    return cudaSuccess;
  }
  void release() { cudaFree(p); p = nullptr; cap = 0; }
};

struct svs_place : svs::Handle {
  int W = 0, sms = 132;
  Cam cam{};
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  // vocabulary and per-word state
  float* d_words = nullptr;
  int* d_cw = nullptr;          // places holding each word
  int* d_first_row = nullptr;   // scratch of the current keyframe (INT_MAX between calls)
  int* d_kf_count = nullptr;    // scratch of the current keyframe (0 between calls)
  // database
  int L = 0, rows = 0, wl = 0, max_rows = 0;
  std::unordered_map<int, int> index_of;
  std::vector<int> ids;
  DevArr<float> desc;           // [rows][64]
  DevArr<double> xyz;           // [rows][3]
  DevArr<int> wl_word, wl_count;
  DevArr<int> p_row_off, p_nrows, p_wl_off, p_wl_n, p_nwords, p_id;
  // per call
  DevArr<double> uvu;
  DevArr<unsigned long long> best_word, best_match;
  DevArr<int> word, train_idx, inl_q, inl_t, hyp_triple, hyp_inl;
  DevArr<float> dist, score;
  DevArr<double> hyp_RT;
  DevArr<unsigned char> excluded;
  PlaceRes* d_res = nullptr;
  PlaceRes last{};
  int last_n = 0, last_L = 0, last_scored = 0;
};

// the split of the nearest-neighbour kernel: query blocks of kTile rows; the train tiles are divided over enough
// CTAs that the grid covers about two waves of the device, never more slices than tiles
static dim3 nn_grid(int n, int m, int sms) {
  const int qb = (n + kTile - 1) / kTile, tiles = (m + kTile - 1) / kTile;
  const int want = (2 * sms + qb - 1) / qb;
  return dim3(qb, std::max(1, std::min(tiles, want)));
}

extern "C" {

int svs_place_create(int device, int num_words, const float* words, const svs_cam* cam, svs_place** out) {
  if (!out) return SVS_ERR_INVALID;
  *out = nullptr;
  if (num_words <= 0 || !words || !cam) return SVS_ERR_INVALID;
  svs_place* h = new svs_place();
  if (int rc = svs::open_handle(h, device)) {
    delete h;
    return rc;
  }
  h->W = num_words;
  h->cam = Cam{cam->f, cam->px, cam->py, cam->b};
  auto fail = [&]() { svs_place_destroy(h); return SVS_ERR_CUDA; };
  cudaDeviceGetAttribute(&h->sms, cudaDevAttrMultiProcessorCount, device);
  if (cudaEventCreate(&h->ev0) != cudaSuccess || cudaEventCreate(&h->ev1) != cudaSuccess ||
      cudaMalloc(&h->d_words, sizeof(float) * kDim * (size_t)num_words) != cudaSuccess ||
      cudaMalloc(&h->d_cw, sizeof(int) * (size_t)num_words) != cudaSuccess ||
      cudaMalloc(&h->d_first_row, sizeof(int) * (size_t)num_words) != cudaSuccess ||
      cudaMalloc(&h->d_kf_count, sizeof(int) * (size_t)num_words) != cudaSuccess ||
      cudaMalloc(&h->d_res, sizeof(PlaceRes)) != cudaSuccess)
    return fail();
  if (cudaMemcpyAsync(h->d_words, words, sizeof(float) * kDim * (size_t)num_words, cudaMemcpyHostToDevice, h->stream) !=
          cudaSuccess ||
      cudaMemsetAsync(h->d_cw, 0, sizeof(int) * (size_t)num_words, h->stream) != cudaSuccess ||
      cudaMemsetAsync(h->d_kf_count, 0, sizeof(int) * (size_t)num_words, h->stream) != cudaSuccess)
    return fail();
  k_fill_int<<<(num_words + 255) / 256, 256, 0, h->stream>>>(h->d_first_row, num_words, INT_MAX);
  if (cudaGetLastError() != cudaSuccess || cudaStreamSynchronize(h->stream) != cudaSuccess) return fail();
  *out = h;
  return SVS_OK;
}

void svs_place_destroy(svs_place* h) {
  if (!h) return;
  svs::begin_close(h);
  for (auto* a : {&h->desc, &h->score, &h->dist}) a->release();
  for (auto* a : {&h->xyz, &h->uvu, &h->hyp_RT}) a->release();
  for (auto* a : {&h->wl_word, &h->wl_count, &h->p_row_off, &h->p_nrows, &h->p_wl_off, &h->p_wl_n, &h->p_nwords,
                  &h->p_id, &h->word, &h->train_idx, &h->inl_q, &h->inl_t, &h->hyp_triple, &h->hyp_inl})
    a->release();
  h->best_word.release(); h->best_match.release(); h->excluded.release();
  cudaFree(h->d_words); cudaFree(h->d_cw); cudaFree(h->d_first_row); cudaFree(h->d_kf_count); cudaFree(h->d_res);
  if (h->ev0) cudaEventDestroy(h->ev0);
  if (h->ev1) cudaEventDestroy(h->ev1);
  delete h;
}

const char* svs_place_last_error(const svs_place* h) { return svs::last_error(h); }

int svs_place_add_location(svs_place* h, int keyframe_id, int n, const float* desc, const double* uvu,
                           int do_loop_detection, int n_exclude, const int* exclude_ids, const svs_place_params* p,
                           svs_place_result* res, int* inlier_query, int* inlier_train) {
  if (!h) return SVS_ERR_INVALID;
  const svs_place_params prm = p ? *p : svs_place_params SVS_PLACE_PARAMS_DEFAULT;
  if (!res) { h->err = "res is NULL"; return SVS_ERR_INVALID; }
  if (n < 0 || (n > 0 && (!desc || !uvu))) { h->err = "n < 0 or a NULL array with n > 0"; return SVS_ERR_INVALID; }
  if (n_exclude < 0 || (n_exclude > 0 && !exclude_ids)) { h->err = "bad exclude set"; return SVS_ERR_INVALID; }
  if (prm.num_ransac < 0) { h->err = "num_ransac < 0"; return SVS_ERR_INVALID; }
  if (!(prm.pixel_thr > 0.0) || !std::isfinite(prm.pixel_thr)) { h->err = "pixel_thr not > 0 and finite"; return SVS_ERR_INVALID; }
  if (h->index_of.count(keyframe_id)) { h->err = "keyframe id already in the database"; return SVS_ERR_INVALID; }
  SVS_CK(h, cudaSetDevice(h->device));
  cudaStream_t s = h->stream;
  const int L = h->L, H = prm.num_ransac;
  const size_t n1 = (size_t)std::max(n, 1);
  // storage: the database grows geometrically; the per-call buffers keep their largest size
  SVS_CK(h, h->desc.reserve(((size_t)h->rows + n1) * kDim, s));
  SVS_CK(h, h->xyz.reserve(((size_t)h->rows + n1) * 3, s));
  SVS_CK(h, h->wl_word.reserve((size_t)h->wl + n1, s));
  SVS_CK(h, h->wl_count.reserve((size_t)h->wl + n1, s));
  for (auto* a : {&h->p_row_off, &h->p_nrows, &h->p_wl_off, &h->p_wl_n, &h->p_nwords, &h->p_id})
    SVS_CK(h, a->reserve((size_t)L + 1, s));
  SVS_CK(h, h->score.reserve((size_t)L + 1, s));
  SVS_CK(h, h->excluded.reserve((size_t)L + 1, s));
  SVS_CK(h, h->uvu.reserve(3 * n1, s));
  SVS_CK(h, h->best_word.reserve(n1, s));
  SVS_CK(h, h->best_match.reserve(n1, s));
  for (auto* a : {&h->word, &h->train_idx, &h->inl_q, &h->inl_t}) SVS_CK(h, a->reserve(n1, s));
  SVS_CK(h, h->dist.reserve(n1, s));
  SVS_CK(h, h->hyp_triple.reserve(3 * (size_t)std::max(H, 1), s));
  SVS_CK(h, h->hyp_inl.reserve((size_t)std::max(H, 1), s));
  SVS_CK(h, h->hyp_RT.reserve(12 * (size_t)std::max(H, 1), s));

  std::vector<unsigned char> excl((size_t)L + 1, 0);
  for (int e = 0; e < n_exclude; ++e) {
    auto it = h->index_of.find(exclude_ids[e]);
    if (it != h->index_of.end()) excl[it->second] = 1;
  }
  PlaceRes init{};
  init.best_place = -1; init.best_kf = -1; init.best_h = -1;
  init.T[3] = 1.0;
  float* q = h->desc.p + (size_t)h->rows * kDim;   // the new rows go straight into the database
  SVS_CK(h, cudaEventRecord(h->ev0, s));
  SVS_CK(h, cudaMemcpyAsync(h->d_res, &init, sizeof init, cudaMemcpyHostToDevice, s));
  if (n > 0) {
    SVS_CK(h, cudaMemcpyAsync(q, desc, sizeof(float) * kDim * (size_t)n, cudaMemcpyHostToDevice, s));
    SVS_CK(h, cudaMemcpyAsync(h->uvu.p, uvu, sizeof(double) * 3 * (size_t)n, cudaMemcpyHostToDevice, s));
    SVS_CK(h, cudaMemsetAsync(h->best_word.p, 0xff, sizeof(unsigned long long) * (size_t)n, s));
    k_place_nn<<<nn_grid(n, h->W, h->sms), kNNThreads, 0, s>>>(q, n, h->d_words, h->W, nullptr, nullptr, nullptr,
                                                                 h->best_word.p);
    k_place_assign<<<(n + 255) / 256, 256, 0, s>>>(h->best_word.p, n, h->word.p, h->d_first_row, h->d_kf_count, h->d_res);
  }
  const bool scored = do_loop_detection && L > 0 && n > 0;
  if (scored) {
    SVS_CK(h, cudaMemcpyAsync(h->excluded.p, excl.data(), (size_t)L, cudaMemcpyHostToDevice, s));
    k_place_score<<<(L + 7) / 8, 256, 0, s>>>(L, n, h->word.p, h->d_first_row, h->d_cw, h->p_wl_off.p, h->p_wl_n.p,
                                              h->wl_word.p, h->wl_count.p, h->p_nwords.p, h->excluded.p, h->score.p);
    k_place_select<<<1, 1024, 0, s>>>(L, h->score.p, h->p_id.p, h->d_res);
    // the match and the geometric check read the candidate from device memory and return at once without one
    SVS_CK(h, cudaMemsetAsync(h->best_match.p, 0xff, sizeof(unsigned long long) * (size_t)n, s));
    k_place_nn<<<nn_grid(n, h->max_rows, h->sms), kNNThreads, 0, s>>>(q, n, h->desc.p, 0, &h->d_res->best_place,
                                                                       h->p_row_off.p, h->p_nrows.p, h->best_match.p);
    k_place_match_fin<<<(n + 255) / 256, 256, 0, s>>>(h->best_match.p, n, h->p_nrows.p, h->d_res, h->train_idx.p,
                                                      h->dist.p);
    RansacArgs ra;
    ra.res = h->d_res; ra.n = n; ra.num_ransac = H; ra.seed = prm.seed; ra.thr2 = prm.pixel_thr * prm.pixel_thr;
    ra.cam = h->cam; ra.uvu = h->uvu.p; ra.xyz = h->xyz.p; ra.row_off = h->p_row_off.p; ra.train_idx = h->train_idx.p;
    ra.hyp_triple = h->hyp_triple.p; ra.hyp_inl = h->hyp_inl.p; ra.hyp_RT = h->hyp_RT.p;
    if (H > 0) k_place_ransac<<<(H + kRansacWarps - 1) / kRansacWarps, kRansacWarps * 32, 0, s>>>(ra);
    k_place_finish<<<1, 1024, 0, s>>>(ra, h->inl_q.p, h->inl_t.p);
  }
  InsertArgs ia;
  ia.W = h->W; ia.n = n; ia.L = L; ia.row_off = h->rows; ia.wl_off = h->wl; ia.id = keyframe_id; ia.cam = h->cam;
  ia.uvu = h->uvu.p; ia.first_row = h->d_first_row; ia.kf_count = h->d_kf_count; ia.cw = h->d_cw;
  ia.wl_word = h->wl_word.p; ia.wl_count = h->wl_count.p; ia.xyz = h->xyz.p;
  ia.p_row_off = h->p_row_off.p; ia.p_nrows = h->p_nrows.p; ia.p_wl_off = h->p_wl_off.p; ia.p_wl_n = h->p_wl_n.p;
  ia.p_nwords = h->p_nwords.p; ia.p_id = h->p_id.p; ia.res = h->d_res;
  k_place_insert<<<1, 1024, 0, s>>>(ia);
  SVS_CK(h, cudaGetLastError());
  SVS_CK(h, cudaEventRecord(h->ev1, s));
  PlaceRes r{};
  SVS_CK(h, cudaMemcpyAsync(&r, h->d_res, sizeof r, cudaMemcpyDeviceToHost, s));
  SVS_CK(h, cudaStreamSynchronize(s));
  if (r.num_inliers > 0 && inlier_query)
    SVS_CK(h, cudaMemcpy(inlier_query, h->inl_q.p, sizeof(int) * (size_t)r.num_inliers, cudaMemcpyDeviceToHost));
  if (r.num_inliers > 0 && inlier_train)
    SVS_CK(h, cudaMemcpy(inlier_train, h->inl_t.p, sizeof(int) * (size_t)r.num_inliers, cudaMemcpyDeviceToHost));
  // the place is in the database: update the host's view of it
  h->index_of[keyframe_id] = L;
  h->ids.push_back(keyframe_id);
  h->L = L + 1;
  h->rows += n;
  h->wl += r.ndistinct;
  h->max_rows = std::max(h->max_rows, n);
  h->last = r;
  h->last_n = n;
  h->last_L = L;
  h->last_scored = scored;
  res->best_keyframe_id = r.best_kf;
  res->best_score = r.best_score;
  res->num_matches = r.num_matches;
  res->num_inliers = r.num_inliers;
  res->loop_found = r.num_inliers > 30;
  for (int i = 0; i < 7; ++i) res->T_query_from_loop[i] = r.T[i];
  float ms = 0.f;
  cudaEventElapsedTime(&ms, h->ev0, h->ev1);
  res->ms = ms;
  return SVS_OK;
}

int svs_place_num_places(const svs_place* h) { return h ? h->L : SVS_ERR_INVALID; }

int svs_place_last_words(const svs_place* h, int* word) {
  if (!h || (h->last_n > 0 && !word)) return SVS_ERR_INVALID;
  if (h->last_n > 0 && cudaMemcpy(word, h->word.p, sizeof(int) * (size_t)h->last_n, cudaMemcpyDeviceToHost) != cudaSuccess)
    return SVS_ERR_CUDA;
  return h->last_n;
}

int svs_place_last_scores(const svs_place* h, int cap, int* keyframe_id, float* score) {
  if (!h || cap < 0 || (cap > 0 && (!keyframe_id || !score))) return SVS_ERR_INVALID;
  if (!h->last_scored) return 0;
  std::vector<float> s((size_t)h->last_L);
  if (cudaMemcpy(s.data(), h->score.p, sizeof(float) * s.size(), cudaMemcpyDeviceToHost) != cudaSuccess)
    return SVS_ERR_CUDA;
  int count = 0;
  for (int k = 0; k < h->last_L; ++k) {
    if (!(s[k] > 0.f)) continue;   // every contribution is positive: score > 0 iff the place received one
    if (count < cap) { keyframe_id[count] = h->ids[k]; score[count] = s[k]; }
    ++count;
  }
  return count;
}

int svs_place_last_matches(const svs_place* h, int* train_idx, float* dist) {
  if (!h) return SVS_ERR_INVALID;
  const int m = h->last.num_matches;
  if (m > 0 && (!train_idx || !dist)) return SVS_ERR_INVALID;
  if (m > 0 && (cudaMemcpy(train_idx, h->train_idx.p, sizeof(int) * (size_t)m, cudaMemcpyDeviceToHost) != cudaSuccess ||
                cudaMemcpy(dist, h->dist.p, sizeof(float) * (size_t)m, cudaMemcpyDeviceToHost) != cudaSuccess))
    return SVS_ERR_CUDA;
  return m;
}

int svs_place_last_hypotheses(const svs_place* h, int cap, int* triple, int* inliers, int* best) {
  if (!h || cap < 0 || (cap > 0 && (!triple || !inliers))) return SVS_ERR_INVALID;
  const int H = h->last.num_hyp, c = std::min(cap, H);
  if (best) *best = h->last.best_h;
  if (c > 0 && (cudaMemcpy(triple, h->hyp_triple.p, sizeof(int) * 3 * (size_t)c, cudaMemcpyDeviceToHost) != cudaSuccess ||
                cudaMemcpy(inliers, h->hyp_inl.p, sizeof(int) * (size_t)c, cudaMemcpyDeviceToHost) != cudaSuccess))
    return SVS_ERR_CUDA;
  return H;
}

}  // extern "C"
