// stereo.cu -- the front end's level-0 disparity on sm_90a: calcDisparityCpu (stereo_frontend.cpp:620-653) and
// method 1 of calcDisparityGpu (:539-565), i.e. cv::StereoBM with preFilterCap 31, SADWindowSize 7, minDisparity 0,
// textureThreshold 10, uniquenessRatio 15, speckleWindowSize 100, speckleRange 32, disp12MaxDiff 1 and
// numberOfDisparities = ndisp.  Every stage is integer until the final /16, and each follows OpenCV 4.x's StereoBM
// rule for rule (checked bit for bit against cv2.StereoBM), so the output is the library's, not an approximation:
//   k_stereo_prefilter  x-Sobel (rows reflect-101) clipped to [0, 62]; columns 0 and w-1 are 31, and so is the last
//                       row of an odd-height image (OpenCV filters rows in pairs)
//   k_stereo_cost       per row Y in [3, h-3) and column X in [ndisp, w): the 7x7 SADs of all ndisp disparities in
//                       shared memory, the texture sum, winner-take-all (ties go to the larger disparity), the
//                       uniqueness test and the 1/16-px parabola
//   k_stereo_lr         per row: the left-right check against the best left pixel of every right pixel (least cost,
//                       then least x), then the invalid border (x < ndisp + 2, x >= w - 3, 3 rows top and bottom)
//   k_stereo_unite / k_stereo_count / k_stereo_final
//                       filterSpeckles: 4-connected components of pixels whose 1/16-px values differ by <= 32,
//                       by union-find over the runs k_stereo_lr leaves in each row; components of <= 100 pixels
//                       become invalid; then float, /16, -1 = invalid
// The window columns follow OpenCV's clamping: a window column xc reads the left image at min(xc, w-1) and the right
// image at min(max(xc, ndisp-1), w-1) - d, which differs from a plain shift only near the image's left and right
// edges, in pixels the border stage later invalidates but which still take part in the left-right check.
#include <cuda_runtime.h>

#include <climits>
#include <cstdint>

#include "../../include/svs_b200.h"
#include "handle.cuh"

namespace {

constexpr int kCap = 31;            // preFilterCap
constexpr int kR = 3;               // SADWindowSize / 2
constexpr int kTexture = 10;        // textureThreshold
constexpr int kUniqueness = 15;     // uniquenessRatio
constexpr int kSpeckleSize = 100;   // speckleWindowSize
constexpr int kSpeckleRange = 32;   // speckleRange, in 1/16 px as OpenCV applies it to the fixed-point map
constexpr int kMaxDiff12 = 16;      // disp12MaxDiff = 1 px, in 1/16 px
constexpr short kFiltered = -16;    // (minDisparity - 1) << 4
constexpr int kTile = 64;           // output columns per k_stereo_cost block
constexpr int kCostThreads = 256;
constexpr int kWinCols = kTile + 2 * kR;

__global__ void k_stereo_prefilter(const unsigned char* __restrict__ left, int lpitch, const unsigned char* __restrict__ right,
                                   int rpitch, unsigned char* __restrict__ pl, unsigned char* __restrict__ pr, int pitch,
                                   int w, int h) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= w || y >= h) return;
  const unsigned char* src = blockIdx.z ? right : left;
  const int sp = blockIdx.z ? rpitch : lpitch;
  int v = kCap;
  if (x > 0 && x < w - 1 && !((h & 1) && y == h - 1)) {
    const int yu = y > 0 ? y - 1 : 1, yd = y < h - 1 ? y + 1 : y - 1;
    const unsigned char *ru = src + (size_t)yu * sp, *rc = src + (size_t)y * sp, *rd = src + (size_t)yd * sp;
    const int s = (ru[x + 1] - ru[x - 1]) + 2 * (rc[x + 1] - rc[x - 1]) + (rd[x + 1] - rd[x - 1]);
    v = min(max(s, -kCap), kCap) + kCap;
  }
  (blockIdx.z ? pr : pl)[(size_t)y * pitch + x] = (unsigned char)v;
}

// One block per (row Y, 64 columns from Xs).  Shared memory: the 7 pre-filtered rows of both images around the tile,
// the 7-row column sums of every (window column, disparity), then the 7x7 costs of every (pixel, disparity).
__global__ void __launch_bounds__(kCostThreads) k_stereo_cost(const unsigned char* __restrict__ pl,
                                                              const unsigned char* __restrict__ pr, int pitch, int w,
                                                              int ndisp, short* __restrict__ d16,
                                                              unsigned short* __restrict__ c16, int dpitch) {
  extern __shared__ __align__(16) unsigned char smem[];
  const int Y = blockIdx.y + kR, Xs = ndisp + blockIdx.x * kTile, nx = min(kTile, w - Xs), lofs = ndisp - 1;
  const int rw = kWinCols + ndisp - 1;            // right-image columns [Xs - 2 - ndisp, Xs + kTile + 3)
  const int r0 = Xs - 2 - ndisp;
  unsigned short* colsum = reinterpret_cast<unsigned short*>(smem);       // [kWinCols][ndisp]
  unsigned short* cost = colsum + kWinCols * ndisp;                        // [kTile][ndisp]
  int* tcol = reinterpret_cast<int*>(cost + kTile * ndisp);                // [kWinCols]
  unsigned char* sl = reinterpret_cast<unsigned char*>(tcol + kWinCols);   // [7][kWinCols]
  unsigned char* sr = sl + (2 * kR + 1) * kWinCols;                        // [7][rw]
  const int tid = threadIdx.x;

  for (int i = tid; i < (2 * kR + 1) * kWinCols; i += kCostThreads) {
    const int r = i / kWinCols, c = i - r * kWinCols;
    sl[i] = pl[(size_t)(Y - kR + r) * pitch + min(Xs - kR + c, w - 1)];
  }
  for (int i = tid; i < (2 * kR + 1) * rw; i += kCostThreads) {
    const int r = i / rw, c = i - r * rw;
    sr[i] = pr[(size_t)(Y - kR + r) * pitch + min(max(r0 + c, 0), w - 1)];
  }
  __syncthreads();

  for (int i = tid; i < kWinCols * ndisp; i += kCostThreads) {
    const int xi = i / ndisp, d = i - xi * ndisp;
    const int xc = Xs - kR + xi;
    const int jr = min(max(xc, lofs), w - 1) - d - r0;
    int s = 0;
#pragma unroll
    for (int r = 0; r < 2 * kR + 1; ++r) s += abs((int)sl[r * kWinCols + xi] - (int)sr[r * rw + jr]);
    colsum[i] = (unsigned short)s;
  }
  for (int i = tid; i < kWinCols; i += kCostThreads) {
    int s = 0;
#pragma unroll
    for (int r = 0; r < 2 * kR + 1; ++r) s += abs((int)sl[r * kWinCols + i] - kCap);
    tcol[i] = s;
  }
  __syncthreads();

  for (int i = tid; i < nx * ndisp; i += kCostThreads) {
    const int x = i / ndisp, d = i - x * ndisp;
    int s = 0;
#pragma unroll
    for (int k = 0; k <= 2 * kR; ++k) s += colsum[(x + k) * ndisp + d];
    cost[i] = (unsigned short)s;
  }
  __syncthreads();

  // one warp per pixel, lanes over disparities.  OpenCV scans the index ndisp-1-d and keeps the first minimum, so
  // among equal costs the larger disparity wins: the key (cost, ndisp-1-d) makes that the unsigned minimum.
  const int lane = tid & 31, warp = tid >> 5;
  for (int x = warp; x < nx; x += kCostThreads / 32) {
    const unsigned short* cx = cost + x * ndisp;
    unsigned key = 0xffffffffu;
    for (int d = lane; d < ndisp; d += 32) key = min(key, ((unsigned)cx[d] << 8) | (unsigned)(ndisp - 1 - d));
    key = __reduce_min_sync(0xffffffffu, key);
    const int minsad = (int)(key >> 8), best = ndisp - 1 - (int)(key & 0xff);
    int tsum = 0;
#pragma unroll
    for (int k = 0; k <= 2 * kR; ++k) tsum += tcol[x + k];
    const int thresh = minsad + minsad * kUniqueness / 100;
    bool rival = false;
    for (int d = lane; d < ndisp; d += 32) rival |= abs(d - best) > 1 && (int)cx[d] <= thresh;
    rival = __any_sync(0xffffffffu, rival);
    if (lane == 0) {
      const size_t o = (size_t)Y * dpitch + Xs + x;
      int v = kFiltered;
      if (tsum >= kTexture && !rival) {
        int frac = 0;
        if (best > 0 && best < ndisp - 1) {
          const int p = cx[best - 1], n = cx[best + 1];
          const int den = p + n - 2 * minsad + abs(p - n);
          frac = den != 0 ? (p - n) * 256 / den : 0;
        }
        v = (best * 256 + frac + 15) >> 4;
        c16[o] = (unsigned short)minsad;
      }
      d16[o] = (short)v;
    }
  }
}

// One block per row.  OpenCV's validateDisparity: every valid x >= ndisp claims the right pixel x - round(d); a right
// pixel keeps the claim of least cost, the first (least x) among equal costs.  A pixel is invalid when both right
// pixels around x - d hold a claim that differs from d by more than 1 px.  keys: one row of scratch per row.
// 4-neighbours in one speckle component: both valid and within speckleRange of each other
__device__ __forceinline__ bool speckle_linked(int a, int b) {
  return a != kFiltered && b != kFiltered && abs(a - b) <= kSpeckleRange;
}

__global__ void k_stereo_lr(short* __restrict__ d16, const unsigned short* __restrict__ c16, int dpitch, int w, int h,
                            int ndisp, bool any_valid, unsigned* __restrict__ keys, int* __restrict__ parent,
                            int* __restrict__ size) {
  const int Y = blockIdx.x;
  short* drow = d16 + (size_t)Y * dpitch;
  unsigned* krow = keys + (size_t)Y * w;
  const bool row_ok = any_valid && Y >= kR && Y < h - kR;
  if (row_ok) {
    for (int x = threadIdx.x; x < w; x += blockDim.x) krow[x] = 0xffffffffu;
    __syncthreads();
    for (int x = ndisp + threadIdx.x; x < w; x += blockDim.x) {
      const int d = drow[x];
      if (d != kFiltered) atomicMin(&krow[x - ((d + 8) >> 4)], ((unsigned)c16[(size_t)Y * dpitch + x] << 16) | (unsigned)x);
    }
    __syncthreads();
    for (int x = threadIdx.x; x < w; x += blockDim.x) {   // claim -> the claiming pixel's disparity
      const unsigned k = krow[x];
      krow[x] = k == 0xffffffffu ? (unsigned)(int)kFiltered : (unsigned)(int)drow[k & 0xffffu];
    }
    __syncthreads();
  }
  for (int x = threadIdx.x; x < w; x += blockDim.x) {
    int d = kFiltered;
    if (row_ok && x >= ndisp + kR - 1 && x < w - kR) {
      d = drow[x];
      if (d != kFiltered) {
        const int x0 = x - (d >> 4), x1 = x - ((d + 15) >> 4);
        const int b0 = x0 >= 0 && x0 < w ? (int)krow[x0] : kFiltered, b1 = x1 >= 0 && x1 < w ? (int)krow[x1] : kFiltered;
        if (b0 != kFiltered && abs(b0 - d) > kMaxDiff12 && b1 != kFiltered && abs(b1 - d) > kMaxDiff12) d = kFiltered;
      }
    }
    drow[x] = (short)d;
  }
  __syncthreads();
  // The row's runs of speckle-connected pixels: every pixel's parent is the first pixel of its run (a block-wide
  // running max of the run starts, 256 columns at a time), and that first pixel holds the run's length.  The union
  // pass then only links runs of neighbouring rows.
  __shared__ int wmax[32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  int carry = -1;
  for (int base = 0; base < w; base += blockDim.x) {
    const int x = base + threadIdx.x;
    const int d = x < w ? drow[x] : kFiltered;
    const bool lk = x > 0 && x < w && speckle_linked(d, drow[x - 1]);
    int v = x < w && !lk ? x : -1;
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, v, o);
      if (lane >= o) v = max(v, t);
    }
    if (lane == 31) wmax[wid] = v;
    __syncthreads();
    int pre = carry, last = carry;
    for (int k = 0; k < nw; ++k) {
      if (k < wid) pre = max(pre, wmax[k]);
      last = max(last, wmax[k]);
    }
    if (x < w) {
      const int start = max(v, pre);
      parent[Y * w + x] = Y * w + start;
      if (d != kFiltered && (x + 1 == w || !speckle_linked(drow[x + 1], d))) size[Y * w + start] = x - start + 1;
    }
    __syncthreads();
    carry = last;
  }
}

__device__ __forceinline__ int uf_find(const int* parent, int i) {
  int p;
  while ((p = __ldcg(parent + i)) != i) i = p;
  return i;
}

// Links the sets of a and b, always pointing the larger index at the smaller one.  A failed atomicMin means the node
// gained a parent meanwhile; the loop then carries on from that parent, so no link is lost.
__device__ void uf_unite(int* parent, int a, int b) {
  while (true) {
    a = uf_find(parent, a);
    b = uf_find(parent, b);
    if (a == b) return;
    if (a > b) { const int t = a; a = b; b = t; }
    const int old = atomicMin(parent + b, a);
    if (old == b) return;
    b = old;
  }
}

// Links each run with the runs below it that touch it.  A pixel skips the link when its left neighbours above and below
// are in the same two runs and linked to each other, so every stretch where two runs touch links them once.
__global__ void k_stereo_unite(const short* __restrict__ d16, int dpitch, int w, int h, int* parent) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= w || y + 1 >= h) return;
  const short* row = d16 + (size_t)y * dpitch;
  const int d = row[x], dn = row[x + dpitch];
  if (!speckle_linked(d, dn)) return;
  if (x > 0 && speckle_linked(row[x - 1], row[x - 1 + dpitch]) && speckle_linked(d, row[x - 1]) &&
      speckle_linked(dn, row[x - 1 + dpitch]))
    return;
  uf_unite(parent, y * w + x, (y + 1) * w + x);
}

// Once per run that is not its component's root: its length goes to the root, and the run points at the root directly
// (the sets are final here, so every such write is a true root and concurrent finds stay right).  A root's own
// length is already in place; nothing adds to a run that is not a root.
__global__ void k_stereo_count(const short* __restrict__ d16, int dpitch, int w, int h, int* parent, int* size) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= w || y >= h) return;
  const short* row = d16 + (size_t)y * dpitch;
  if (row[x] == kFiltered || (x > 0 && speckle_linked(row[x], row[x - 1]))) return;   // not the first pixel of a run
  const int s = y * w + x, root = uf_find(parent, s);
  if (root == s) return;
  parent[s] = root;
  atomicAdd(size + root, size[s]);
}

__global__ void k_stereo_final(const short* __restrict__ d16, int dpitch, int w, int h, const int* parent,
                               const int* __restrict__ size, float* __restrict__ out, int ostride) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= w || y >= h) return;
  const int d = d16[(size_t)y * dpitch + x];
  const bool keep = d != kFiltered && __ldcg(size + uf_find(parent, y * w + x)) > kSpeckleSize;
  out[(size_t)y * ostride + x] = (float)(keep ? d : kFiltered) * (1.f / 16.f);
}

constexpr size_t cost_smem(int ndisp) {
  return sizeof(unsigned short) * (size_t)(kWinCols + kTile) * ndisp + sizeof(int) * kWinCols +
         (size_t)(2 * kR + 1) * (kWinCols + kWinCols + ndisp - 1);
}

static_assert(cost_smem(160) <= 48 * 1024, "k_stereo_cost must fit the default shared-memory limit at ndisp 160");

}  // namespace

struct svs_stereo : svs::Handle {
  int w = 0, h = 0, ndisp = 0;
  int pitch8 = 0, dpitch = 0, ostride = 0;
  unsigned char *in[2] = {}, *pf[2] = {};   // host inputs land in `in`; pre-filtered left / right
  short* d16 = nullptr;
  unsigned short* c16 = nullptr;
  unsigned* keys = nullptr;
  int *parent = nullptr, *size = nullptr;
  float* out = nullptr;
};

extern "C" {

int svs_stereo_create(int device, int w, int hgt, int num_disparities, svs_stereo** out) {
  if (!out) return SVS_ERR_INVALID;
  *out = nullptr;
  if (w <= 0 || hgt <= 0 || w > 65535 || hgt > 65535 || (long long)w * hgt > INT_MAX || num_disparities < 16 ||
      num_disparities > 160 || num_disparities % 16)
    return SVS_ERR_INVALID;
  svs_stereo* h = new svs_stereo();
  if (int rc = svs::open_handle(h, device)) {
    delete h;
    return rc;
  }
  h->w = w; h->h = hgt; h->ndisp = num_disparities;
  h->pitch8 = ((w + 255) / 256) * 256;
  h->dpitch = ((w + 63) / 64) * 64;
  h->ostride = h->dpitch;
  const size_t n = (size_t)w * hgt;
  bool ok = true;
  for (int k = 0; k < 2 && ok; ++k)
    ok = cudaMalloc(&h->in[k], (size_t)h->pitch8 * hgt) == cudaSuccess && cudaMalloc(&h->pf[k], (size_t)h->pitch8 * hgt) == cudaSuccess;
  ok = ok && cudaMalloc(&h->d16, sizeof(short) * h->dpitch * hgt) == cudaSuccess;
  ok = ok && cudaMalloc(&h->c16, sizeof(unsigned short) * h->dpitch * hgt) == cudaSuccess;
  ok = ok && cudaMalloc(&h->keys, sizeof(unsigned) * n) == cudaSuccess;
  ok = ok && cudaMalloc(&h->parent, sizeof(int) * n) == cudaSuccess;
  ok = ok && cudaMalloc(&h->size, sizeof(int) * n) == cudaSuccess;
  ok = ok && cudaMalloc(&h->out, sizeof(float) * h->ostride * hgt) == cudaSuccess;
  // until the first compute the map is all zero (no depth)
  ok = ok && cudaMemset2D(h->out, sizeof(float) * h->ostride, 0, sizeof(float) * w, hgt) == cudaSuccess;
  if (!ok) { svs_stereo_destroy(h); return SVS_ERR_CUDA; }
  *out = h;
  return SVS_OK;
}

void svs_stereo_destroy(svs_stereo* h) {
  if (!h) return;
  svs::begin_close(h);
  for (int k = 0; k < 2; ++k) { cudaFree(h->in[k]); cudaFree(h->pf[k]); }
  cudaFree(h->d16); cudaFree(h->c16); cudaFree(h->keys); cudaFree(h->parent); cudaFree(h->size); cudaFree(h->out);
  delete h;
}

const char* svs_stereo_last_error(const svs_stereo* h) { return svs::last_error(h); }

int svs_stereo_compute(svs_stereo* h, const unsigned char* left, int left_pitch, int left_on_device,
                       const unsigned char* right, int right_pitch, int right_on_device) {
  if (!h) return SVS_ERR_INVALID;
  if (!left || !right || left_pitch < h->w || right_pitch < h->w)
    return svs::fail(h, SVS_ERR_INVALID, "svs_stereo_compute: null image or pitch < width");
  if ((left_on_device && !svs::on_device(h->device, left)) || (right_on_device && !svs::on_device(h->device, right)))
    return svs::fail(h, SVS_ERR_INVALID, "svs_stereo_compute: an image flagged as device memory is not on the handle's device");
  cudaSetDevice(h->device);
  const unsigned char* src[2] = {left, right};
  int pitch[2] = {left_pitch, right_pitch};
  const int on_dev[2] = {left_on_device, right_on_device};
  for (int k = 0; k < 2; ++k)
    if (!on_dev[k]) {   // pageable source: the copy has read it when the call returns
      SVS_CK(h, cudaMemcpy2DAsync(h->in[k], h->pitch8, src[k], pitch[k], h->w, h->h, cudaMemcpyHostToDevice, h->stream));
      src[k] = h->in[k];
      pitch[k] = h->pitch8;
    }
  const int w = h->w, hh = h->h, nd = h->ndisp;
  const dim3 blk(32, 8), grid((w + 31) / 32, (hh + 7) / 8);
  k_stereo_prefilter<<<dim3(grid.x, grid.y, 2), blk, 0, h->stream>>>(src[0], pitch[0], src[1], pitch[1], h->pf[0], h->pf[1],
                                                                      h->pitch8, w, hh);
  // OpenCV's valid rectangle is x in [ndisp + 2, w - 3), y in [3, h - 3); without it every pixel is invalid
  const bool any_valid = w > nd + 5 && hh > 2 * kR;
  if (any_valid)
    k_stereo_cost<<<dim3((w - nd + kTile - 1) / kTile, hh - 2 * kR), kCostThreads, cost_smem(nd), h->stream>>>(
        h->pf[0], h->pf[1], h->pitch8, w, nd, h->d16, h->c16, h->dpitch);
  k_stereo_lr<<<hh, 256, 0, h->stream>>>(h->d16, h->c16, h->dpitch, w, hh, nd, any_valid, h->keys, h->parent, h->size);
  k_stereo_unite<<<grid, blk, 0, h->stream>>>(h->d16, h->dpitch, w, hh, h->parent);
  k_stereo_count<<<grid, blk, 0, h->stream>>>(h->d16, h->dpitch, w, hh, h->parent, h->size);
  k_stereo_final<<<grid, blk, 0, h->stream>>>(h->d16, h->dpitch, w, hh, h->parent, h->size, h->out, h->ostride);
  SVS_CK(h, cudaGetLastError());
  SVS_CK(h, cudaStreamSynchronize(h->stream));   // consumers run on their own streams
  return SVS_OK;
}

int svs_stereo_disparity(svs_stereo* h, const float** d_disp, int* stride_floats) {
  if (!h || !d_disp || !stride_floats) return SVS_ERR_INVALID;
  *d_disp = h->out;
  *stride_floats = h->ostride;
  return SVS_OK;
}

int svs_stereo_get(svs_stereo* h, float* out) {
  if (!h || !out) return SVS_ERR_INVALID;
  cudaSetDevice(h->device);
  SVS_CK(h, cudaMemcpy2D(out, sizeof(float) * h->w, h->out, sizeof(float) * h->ostride, sizeof(float) * h->w, h->h,
                         cudaMemcpyDeviceToHost));
  return SVS_OK;
}

}  // extern "C"
