// fast.cu -- grid FAST-9/16 detector on sm_90a, bit-exact with cv::FastFeatureDetector(thr, false)
// run per grid cell as ScaViSLAM does (scavislam/fast_grid.cpp:60-83 FastGrid::detect,
// :86-152 FastGrid::detectAdaptively).
//
// Integer/byte work, HBM-bound at one pass over the uint8 image: instead of re-running the
// detector up to `trials` times per cell like the reference, ONE kernel computes for every
// pixel the largest threshold at which it is still a corner (the segment test is monotone in
// the threshold) and a per-cell histogram of those scores; the adaptive threshold walk then
// becomes a scalar loop over histogram suffix sums, and the keypoints of the final threshold
// are emitted by an order-preserving (raster, per cell) compaction so that the per-cell
// ordinal the reference stores in its quadtree (fast_grid.cpp:75-80) is reproduced exactly.
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

#include <cuda_runtime.h>

#include "../../include/svs_b200.h"
#include "handle.cuh"
#include "internal.cuh"
#include "svs_nvtx.hpp"

namespace {

constexpr int kMaxCells = 64;
constexpr int kTileW = 32, kTileH = 8;

struct CellDev {
  int u0, u1, v0, v1, thr;
};

__constant__ int c_dx[16] = {0, 1, 2, 3, 3, 3, 2, 1, 0, -1, -2, -3, -3, -3, -2, -1};
__constant__ int c_dy[16] = {3, 3, 2, 1, 0, -1, -2, -3, -3, -3, -2, -1, 0, 1, 2, 3};

__device__ __forceinline__ bool has_run9(unsigned m16) {
  const unsigned x = m16 | (m16 << 16);
  const unsigned a = x & (x >> 1);
  const unsigned b = a & (a >> 2);
  const unsigned c = b & (b >> 4);
  return (c & (x >> 8)) != 0u;   // 9 consecutive set bits somewhere on the circle
}

// score+1 of every pixel of every cell's inner region (3 px inside the cell ROI, like cv::FAST
// on img(vrange, urange)), 0 where the pixel is not a corner at threshold t0 of its cell.
__global__ void __launch_bounds__(kTileW * kTileH)
k_fast_score(const uint8_t* __restrict__ img, int pitch, const CellDev* __restrict__ cells, int use_cell_thr, int t0_all,
             uint8_t* __restrict__ score, int* __restrict__ hist) {
  __shared__ uint8_t tile[kTileH + 6][kTileW + 6 + 2];
  __shared__ int shist[256];
  const CellDev cell = cells[blockIdx.z];
  const int iw = cell.u1 - cell.u0 - 6, ih = cell.v1 - cell.v0 - 6;
  const int bx = blockIdx.x * kTileW, by = blockIdx.y * kTileH;
  if (bx >= iw || by >= ih) return;
  const int tid = threadIdx.y * kTileW + threadIdx.x;
  if (hist) shist[tid] = 0;
  // stage the (tile + 3 px apron): always inside the cell ROI
  const int x0 = cell.u0 + bx, y0 = cell.v0 + by;   // top-left of the apron
  for (int i = tid; i < (kTileH + 6) * (kTileW + 6); i += kTileW * kTileH) {
    const int ty = i / (kTileW + 6), tx = i - ty * (kTileW + 6);
    const int x = min(x0 + tx, cell.u1 - 1), y = min(y0 + ty, cell.v1 - 1);
    tile[ty][tx] = img[(size_t)y * pitch + x];
  }
  __syncthreads();
  const int px = bx + threadIdx.x, py = by + threadIdx.y;
  const bool inside = px < iw && py < ih;
  int sc1 = 0;
  if (inside) {
    const int t0 = use_cell_thr ? cell.thr : t0_all;
    const int cx = threadIdx.x + 3, cy = threadIdx.y + 3;
    const int v = tile[cy][cx];
    int d[16];
    unsigned br = 0, dk = 0;
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      d[k] = (int)tile[cy + c_dy[k]][cx + c_dx[k]] - v;
      br |= (d[k] > t0) ? (1u << k) : 0u;
      dk |= (d[k] < -t0) ? (1u << k) : 0u;
    }
    const bool cb = has_run9(br), cd = has_run9(dk);
    if (cb || cd) {
      // exact score: max over the 16 arcs of min over 9 consecutive (|d| - 1), per polarity
      int best = -1;
#pragma unroll
      for (int pol = 0; pol < 2; ++pol) {
        if (pol == 0 ? !cb : !cd) continue;
        int e[16], m2[16], m4[16], m8[16];
#pragma unroll
        for (int k = 0; k < 16; ++k) e[k] = (pol == 0 ? d[k] : -d[k]) - 1;
#pragma unroll
        for (int k = 0; k < 16; ++k) m2[k] = min(e[k], e[(k + 1) & 15]);
#pragma unroll
        for (int k = 0; k < 16; ++k) m4[k] = min(m2[k], m2[(k + 2) & 15]);
#pragma unroll
        for (int k = 0; k < 16; ++k) m8[k] = min(m4[k], m4[(k + 4) & 15]);
#pragma unroll
        for (int k = 0; k < 16; ++k) best = max(best, min(m8[k], e[(k + 8) & 15]));
      }
      sc1 = min(best, 254) + 1;
      if (hist) atomicAdd(&shist[sc1 - 1], 1);
    }
    score[(size_t)(cell.v0 + 3 + py) * pitch + cell.u0 + 3 + px] = (uint8_t)sc1;
  }
  if (hist) {
    __syncthreads();
    const int c = shist[tid];
    if (c) atomicAdd(&hist[blockIdx.z * 256 + tid], c);
  }
}

struct GridParams {
  int grid_w, grid_h, fast_min, fast_max, min_inner, min_outer, max_inner, max_outer;
};

// The threshold walk of FastGrid::detectAdaptively (fast_grid.cpp:86-152) on histogram suffix sums.
// One warp per cell first turns the cell's 256-bin score histogram into suffix sums in shared memory
// (count of corners at threshold >= s), so that every trial of the walk is one lookup; then one thread per
// grid row walks its cells (prev_thr / prev_prev_thr are shared by the cells of a row).
constexpr int kSelCells = 32;   // cells per launch block (kMaxCells is 64: two rounds at most)
__global__ void __launch_bounds__(kSelCells * 32)
k_fast_select(CellDev* cells, const int* __restrict__ hist, GridParams g, int trials, int* thr_detect) {
  __shared__ int ssuf[kSelCells][257];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int ncells = g.grid_w * g.grid_h;
  const int per_round = (kSelCells / g.grid_w) * g.grid_w;   // whole grid rows per round (grid_w <= kSelCells, checked by the launcher)
  for (int c0 = 0; c0 < ncells; c0 += per_round) {
    const int ci = c0 + warp;
    if (warp < per_round && ci < ncells) {
      // lane owns bins [8 lane, 8 lane + 8): local suffix sums, then a warp scan over the lane totals
      int v[8], tot = 0;
#pragma unroll
      for (int q = 7; q >= 0; --q) { tot += hist[ci * 256 + 8 * lane + q]; v[q] = tot; }
      int above = tot;   // inclusive suffix scan over lanes (higher lanes = higher bins)
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int up = __shfl_down_sync(0xffffffffu, above, o);
        if (lane + o < 32) above += up;
      }
      above -= tot;      // corners in the bins of all higher lanes
#pragma unroll
      for (int q = 0; q < 8; ++q) ssuf[warp][8 * lane + q] = v[q] + above;
      if (lane == 0) ssuf[warp][256] = 0;
    }
    __syncthreads();
    const int rows_here = min(per_round, ncells - c0) / g.grid_w;
    const int j = threadIdx.x;   // grid row within this round
    if (j < rows_here) {
      int prev_thr = -1, prev_prev_thr = -2;
      for (int i = 0; i < g.grid_w; ++i) {
        const int cl = j * g.grid_w + i, ci2 = c0 + cl;
        int thr = cells[ci2].thr;
        int tdet = -1;   // threshold of the last detect() call; -1 = none (trials <= 0)
        for (int trial = 0; trial < trials; ++trial) {
          tdet = thr;
          const int nd = ssuf[cl][min(max(thr, 0), 256)];
          if (prev_prev_thr == thr) { thr = (thr + prev_prev_thr) / 2; break; }
          prev_prev_thr = prev_thr;
          prev_thr = thr;
          if (nd < g.min_inner) {
            if (thr <= g.fast_min) break;
            --thr;
            if (nd < g.min_outer) {
              if (thr <= g.fast_min) break;
              --thr;
              continue;
            }
          } else if (nd > g.max_inner) {
            if (thr >= g.fast_max) break;
            ++thr;
            if (nd > g.max_outer) {
              if (thr >= g.fast_max) break;
              ++thr;
              continue;
            }
          }
          break;
        }
        cells[ci2].thr = thr;
        thr_detect[ci2] = tdet;
      }
    }
    __syncthreads();
  }
}

// keypoints per (cell, row): one warp per row of a cell's inner region
__global__ void k_fast_count(const uint8_t* __restrict__ score, int pitch, const CellDev* __restrict__ cells,
                             const int* __restrict__ thr_detect, int max_rows, int* __restrict__ row_count) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  const int ci = blockIdx.y;
  const CellDev cell = cells[ci];
  const int ih = cell.v1 - cell.v0 - 6, iw = cell.u1 - cell.u0 - 6;
  if (warp >= ih) return;
  const int thr = thr_detect ? thr_detect[ci] : cell.thr;
  int n = 0;
  if (thr >= 0) {
    const uint8_t* row = score + (size_t)(cell.v0 + 3 + warp) * pitch + cell.u0 + 3;
    for (int x = lane; x < iw; x += 32) n += (row[x] > thr) ? 1 : 0;   // score+1 > thr  <=>  score >= thr
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) n += __shfl_xor_sync(0xffffffffu, n, o);
  if (lane == 0) row_count[ci * max_rows + warp] = n;
}

// exclusive scan of the row counts inside each cell (warp per cell), then over cells
__global__ void k_fast_scan(const CellDev* __restrict__ cells, int ncells, int max_rows, int* __restrict__ row_count,
                            int* __restrict__ cell_off) {
  __shared__ int tot[kMaxCells];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int ci = warp; ci < ncells; ci += blockDim.x >> 5) {
    const int ih = max(cells[ci].v1 - cells[ci].v0 - 6, 0);
    int carry = 0;
    for (int r0 = 0; r0 < ih; r0 += 32) {
      const int r = r0 + lane;
      const int v = r < ih ? row_count[ci * max_rows + r] : 0;
      int inc = v;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += t;
      }
      if (r < ih) row_count[ci * max_rows + r] = carry + inc - v;
      carry += __shfl_sync(0xffffffffu, inc, 31);
    }
    if (lane == 0) tot[ci] = carry;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int s = 0;
    for (int ci = 0; ci < ncells; ++ci) { cell_off[ci] = s; s += tot[ci]; }
    cell_off[ncells] = s;
  }
}

__global__ void k_fast_emit(const uint8_t* __restrict__ score, int pitch, const CellDev* __restrict__ cells,
                            const int* __restrict__ thr_detect, int max_rows, const int* __restrict__ row_off,
                            const int* __restrict__ cell_off, int max_out, int* __restrict__ out_xy) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  const int ci = blockIdx.y;
  const CellDev cell = cells[ci];
  const int ih = cell.v1 - cell.v0 - 6, iw = cell.u1 - cell.u0 - 6;
  if (warp >= ih) return;
  const int thr = thr_detect ? thr_detect[ci] : cell.thr;
  if (thr < 0) return;
  const int y = cell.v0 + 3 + warp;
  const uint8_t* row = score + (size_t)y * pitch + cell.u0 + 3;
  int base = cell_off[ci] + row_off[ci * max_rows + warp];
  for (int x0 = 0; x0 < iw; x0 += 32) {
    const int x = x0 + lane;
    const bool hit = x < iw && row[x] > thr;
    const unsigned m = __ballot_sync(0xffffffffu, hit);
    if (hit) {
      const int o = base + __popc(m & ((1u << lane) - 1u));
      if (o < max_out) { out_xy[2 * o] = cell.u0 + 3 + x; out_xy[2 * o + 1] = y; }
    }
    base += __popc(m);
  }
}

}  // namespace

struct svs_fast : svs::Handle {
  int cap_w = 0, cap_h = 0, pitch = 0, w = 0, h = 0;
  uint8_t* d_img = nullptr;
  uint8_t* d_score = nullptr;
  CellDev* d_cells = nullptr;
  int* d_hist = nullptr;
  int* d_thr_detect = nullptr;
  int* d_row = nullptr;
  int* d_cell_off = nullptr;
  int* d_xy = nullptr;
  int cap_xy = 0;
  int* h_pinned = nullptr;   // cell_off + cells + xy staging
  int h_pinned_ints = 0;
  bool has_image = false;
  int last_total = 0, last_ncells = 0;   // result of the last detect call, still on the device (d_xy, d_cell_off)
};

namespace svs {
// keypoints of the last detect call where they lie on the device: xy [n][2], cell_off [ncells + 1] (internal.cuh)
void fast_device_results(svs_fast* f, const int** d_xy, const int** d_cell_off, int* ncells, int* n, int* device) {
  *d_xy = f->d_xy; *d_cell_off = f->d_cell_off; *ncells = f->last_ncells; *n = f->last_total; *device = f->device;
}
}  // namespace svs

extern "C" {

int svs_fast_create(int device, int max_w, int max_h, int max_keypoints, svs_fast** out) {
  if (!out || max_w <= 0 || max_h <= 0 || max_keypoints <= 0) return SVS_ERR_INVALID;
  *out = nullptr;
  svs_fast* h = new svs_fast();
  if (int rc = svs::open_handle(h, device)) {
    delete h;
    return rc;
  }
  h->cap_w = max_w; h->cap_h = max_h;
  h->pitch = ((max_w + 255) / 256) * 256;
  h->cap_xy = max_keypoints;
  bool ok = cudaMalloc(&h->d_img, (size_t)h->pitch * max_h) == cudaSuccess &&
            cudaMalloc(&h->d_score, (size_t)h->pitch * max_h) == cudaSuccess &&
            cudaMalloc(&h->d_cells, sizeof(CellDev) * kMaxCells) == cudaSuccess &&
            cudaMalloc(&h->d_hist, sizeof(int) * 256 * kMaxCells) == cudaSuccess &&
            cudaMalloc(&h->d_thr_detect, sizeof(int) * kMaxCells) == cudaSuccess &&
            cudaMalloc(&h->d_row, sizeof(int) * kMaxCells * (size_t)max_h) == cudaSuccess &&
            cudaMalloc(&h->d_cell_off, sizeof(int) * (kMaxCells + 1)) == cudaSuccess &&
            cudaMalloc(&h->d_xy, sizeof(int) * 2 * (size_t)max_keypoints) == cudaSuccess;
  h->h_pinned_ints = (kMaxCells + 1) + kMaxCells * 5 + 2 * max_keypoints;
  ok = ok && cudaMallocHost(&h->h_pinned, sizeof(int) * (size_t)h->h_pinned_ints) == cudaSuccess;
  if (!ok) {
    svs_fast_destroy(h);
    return SVS_ERR_CUDA;
  }
  *out = h;
  return SVS_OK;
}

void svs_fast_destroy(svs_fast* h) {
  if (!h) return;
  svs::begin_close(h);
  cudaFree(h->d_img); cudaFree(h->d_score); cudaFree(h->d_cells); cudaFree(h->d_hist);
  cudaFree(h->d_thr_detect); cudaFree(h->d_row); cudaFree(h->d_cell_off); cudaFree(h->d_xy);
  if (h->h_pinned) cudaFreeHost(h->h_pinned);
  delete h;
}

const char* svs_fast_last_error(const svs_fast* h) { return svs::last_error(h); }

int svs_fast_set_image(svs_fast* h, const unsigned char* img, int pitch, int w, int hgt) {
  if (!h || !img || w <= 0 || hgt <= 0 || pitch < w) return SVS_ERR_INVALID;
  if (w > h->cap_w || hgt > h->cap_h) { h->err = "image larger than the handle's capacity"; return SVS_ERR_INVALID; }
  cudaSetDevice(h->device);
  SVS_CK(h, cudaMemcpy2DAsync(h->d_img, h->pitch, img, pitch, w, hgt, cudaMemcpyHostToDevice, h->stream));
  h->w = w; h->h = hgt; h->has_image = true;
  return SVS_OK;
}

int svs_fast_set_image_device(svs_fast* h, const unsigned char* d_img, int pitch, int w, int hgt) {
  if (!h || !d_img || w <= 0 || hgt <= 0 || pitch < w) return SVS_ERR_INVALID;
  if (w > h->cap_w || hgt > h->cap_h) { h->err = "image larger than the handle's capacity"; return SVS_ERR_INVALID; }
  cudaSetDevice(h->device);
  SVS_CK(h, cudaMemcpy2DAsync(h->d_img, h->pitch, d_img, pitch, w, hgt, cudaMemcpyDeviceToDevice, h->stream));
  h->w = w; h->h = hgt; h->has_image = true;
  return SVS_OK;
}

static int run_detect(svs_fast* h, svs_fast_cell* cells, int ncells, const svs_fast_grid_params* gp, int trials,
                      int* out_xy, int max_out, int* cell_off, int write_back_thr) {
  if (!h) return SVS_ERR_INVALID;
  if (!h->has_image) { h->err = "no image set"; return SVS_ERR_STATE; }
  if (!cells || ncells <= 0 || ncells > kMaxCells || !cell_off || (max_out > 0 && !out_xy) || max_out < 0) {
    h->err = "bad cell list / output buffers"; return SVS_ERR_INVALID;
  }
  int max_iw = 0, max_ih = 0, t0 = 255;
  for (int c = 0; c < ncells; ++c) {
    const svs_fast_cell& q = cells[c];
    if (q.u0 < 0 || q.v0 < 0 || q.u1 > h->w || q.v1 > h->h || q.u1 < q.u0 || q.v1 < q.v0) {
      h->err = "cell outside the image"; return SVS_ERR_INVALID;
    }
    max_iw = std::max(max_iw, q.u1 - q.u0 - 6);
    max_ih = std::max(max_ih, q.v1 - q.v0 - 6);
    t0 = std::min(t0, q.thr);
  }
  if (gp) {
    if (gp->grid_w * gp->grid_h != ncells) { h->err = "grid size does not match the cell count"; return SVS_ERR_INVALID; }
    if (gp->grid_w < 1 || gp->grid_w > kSelCells) { h->err = "grid wider than 32 cells"; return SVS_ERR_UNSUPPORTED; }
    t0 = std::min(t0, gp->fast_min);
  }
  t0 = std::max(t0, 0);
  cudaSetDevice(h->device);
  const int lim = std::min(max_out, h->cap_xy);
  CellDev* hc = reinterpret_cast<CellDev*>(h->h_pinned + (kMaxCells + 1));
  for (int c = 0; c < ncells; ++c) hc[c] = CellDev{cells[c].u0, cells[c].u1, cells[c].v0, cells[c].v1, cells[c].thr};
  SVS_CK(h, cudaMemcpyAsync(h->d_cells, hc, sizeof(CellDev) * ncells, cudaMemcpyHostToDevice, h->stream));
  if (max_iw > 0 && max_ih > 0) {
    const dim3 blk(kTileW, kTileH), grd((max_iw + kTileW - 1) / kTileW, (max_ih + kTileH - 1) / kTileH, ncells);
    if (gp) SVS_CK(h, cudaMemsetAsync(h->d_hist, 0, sizeof(int) * 256 * ncells, h->stream));
    k_fast_score<<<grd, blk, 0, h->stream>>>(h->d_img, h->pitch, h->d_cells, gp ? 0 : 1, t0, h->d_score,
                                             gp ? h->d_hist : nullptr);
  } else if (gp) {
    SVS_CK(h, cudaMemsetAsync(h->d_hist, 0, sizeof(int) * 256 * ncells, h->stream));
  }
  if (gp) {
    GridParams g{gp->grid_w, gp->grid_h, gp->fast_min, gp->fast_max, gp->min_inner, gp->min_outer, gp->max_inner, gp->max_outer};
    k_fast_select<<<1, kSelCells * 32, 0, h->stream>>>(h->d_cells, h->d_hist, g, trials, h->d_thr_detect);
  }
  const int rows = std::max(max_ih, 1);
  const dim3 wgrid((rows * 32 + 255) / 256, ncells);
  const int* thr_det = gp ? h->d_thr_detect : nullptr;
  k_fast_count<<<wgrid, 256, 0, h->stream>>>(h->d_score, h->pitch, h->d_cells, thr_det, h->cap_h, h->d_row);
  k_fast_scan<<<1, 1024, 0, h->stream>>>(h->d_cells, ncells, h->cap_h, h->d_row, h->d_cell_off);
  k_fast_emit<<<wgrid, 256, 0, h->stream>>>(h->d_score, h->pitch, h->d_cells, thr_det, h->cap_h, h->d_row, h->d_cell_off,
                                            lim, h->d_xy);
  SVS_CK(h, cudaGetLastError());
  SVS_CK(h, cudaMemcpyAsync(h->h_pinned, h->d_cell_off, sizeof(int) * (ncells + 1), cudaMemcpyDeviceToHost, h->stream));
  if (write_back_thr) SVS_CK(h, cudaMemcpyAsync(hc, h->d_cells, sizeof(CellDev) * ncells, cudaMemcpyDeviceToHost, h->stream));
  SVS_CK(h, cudaStreamSynchronize(h->stream));
  const int total = h->h_pinned[ncells];
  h->last_total = std::min(total, lim); h->last_ncells = ncells;
  memcpy(cell_off, h->h_pinned, sizeof(int) * (ncells + 1));
  if (write_back_thr)
    for (int c = 0; c < ncells; ++c) cells[c].thr = hc[c].thr;
  const int ncopy = std::min(total, lim);
  if (ncopy > 0) {
    int* stage = h->h_pinned + (kMaxCells + 1) + kMaxCells * 5;
    SVS_CK(h, cudaMemcpyAsync(stage, h->d_xy, sizeof(int) * 2 * (size_t)ncopy, cudaMemcpyDeviceToHost, h->stream));
    SVS_CK(h, cudaStreamSynchronize(h->stream));
    memcpy(out_xy, stage, sizeof(int) * 2 * (size_t)ncopy);
  }
  return total;
}

int svs_fast_detect(svs_fast* h, const svs_fast_cell* cells, int ncells, int* out_xy, int max_out, int* cell_off) {
  svs::NvtxRange nvtx_("fast");
  if (!cells || ncells <= 0 || ncells > kMaxCells) return SVS_ERR_INVALID;
  std::vector<svs_fast_cell> tmp(cells, cells + ncells);
  return run_detect(h, tmp.data(), ncells, nullptr, 0, out_xy, max_out, cell_off, 0);
}

int svs_fast_detect_adaptively(svs_fast* h, const svs_fast_grid_params* grid, svs_fast_cell* cells, int trials,
                               int* out_xy, int max_out, int* cell_off) {
  svs::NvtxRange nvtx_("fast");
  if (!grid) return SVS_ERR_INVALID;
  return run_detect(h, cells, grid->grid_w * grid->grid_h, grid, trials, out_xy, max_out, cell_off, 1);
}

// FastGrid::FastGrid (fast_grid.cpp:23-58): cell ranges and the inner/outer count bands
int svs_fast_grid_init(int img_w, int img_h, int num_features_per_cell, int boundary_per_cell, int fast_thr,
                       int grid_w, int grid_h, int fast_min, int fast_max, svs_fast_grid_params* grid,
                       svs_fast_cell* cells) {
  if (!grid || !cells || grid_w <= 0 || grid_h <= 0 || grid_w * grid_h > kMaxCells) return SVS_ERR_INVALID;
  grid->grid_w = grid_w; grid->grid_h = grid_h; grid->fast_min = fast_min; grid->fast_max = fast_max;
  grid->min_inner = (int)(num_features_per_cell - boundary_per_cell * 0.33);
  grid->min_outer = num_features_per_cell - boundary_per_cell;
  grid->max_inner = (int)(num_features_per_cell + boundary_per_cell * 0.33);
  grid->max_outer = num_features_per_cell + boundary_per_cell;
  const int cw = img_w / grid_w, ch = img_h / grid_h;
  for (int j = 0; j < grid_h; ++j)
    for (int i = 0; i < grid_w; ++i) {
      svs_fast_cell& c = cells[j * grid_w + i];
      c.u0 = i * cw; c.u1 = i * cw + cw; c.v0 = j * ch; c.v1 = j * ch + ch; c.thr = fast_thr;
    }
  return SVS_OK;
}

}  // extern "C"
