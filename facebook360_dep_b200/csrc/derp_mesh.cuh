// Camera mesh of a disparity map (SURVEY §8(f) rank 4, the geometry half of ConvertToBinary's convertDepth,
// source/mesh_stream/ConvertToBinary.cpp:150-183, before mesh simplification):
//   depth = 1 / disparity [INTER_NEAREST shrink]  ->  mesh_util::getVertexesEquiError (MeshUtil.h:313-338)
//   -> mesh_util::getFaces(wrapHorizontally = false, isRigCoordinates = false, tearRatio) (MeshUtil.h:162-298)
//   -> vertex mask = !isnan(depth) [& foreground mask]  ->  mesh_util::applyMaskToVertexesAndFaces (MeshUtil.h:342-403)
//   -> the float32 / uint32 buffers mesh_util::writeDepth stores as .vtx / .idx (MeshUtil.h:74-93).
// All of it is index work over the depth grid: one pass that decides the (at most two) triangles of every quad, two
// exclusive scans (kept faces per quad, used vertexes) and two emit passes — HBM-bound, no atomics on the data path,
// output order identical to the reference's row-major loops.
#pragma once

#include <cstdint>

namespace derp {

struct MeshGrid {
  int W, H;            // mesh grid (depth map after the optional shrink)
  int srcW;            // width of the disparity map
  const float* disp;   // [srcH][srcW]
  const int* xofs;     // [W]  nearest-neighbour source column (identity without shrink)
  const int* yofs;     // [H]
  const uint8_t* fg;   // nullable foreground mask [fgH][fgW]
  int fgW;
  const int* fgx;      // [W]  nearest-neighbour mask column
  const int* fgy;      // [H]
  double stepX, stepY; // camera.resolution / grid size (MeshUtil.h:324-325)
  double scale;        // camera.getScalarFocal() * kRadius (MeshUtil.h:317)
  float tearRatio;
  int floorZ;          // write z < 0 as FLT_MIN (ConvertToBinary.cpp:199-203, whenever --triangles > 0)
  static constexpr bool kMasked = true;  // vertexes outside the mask are dropped and the rest re-indexed
  __device__ __forceinline__ double corner(int x, int y, bool* valid) const;
};

// depth(y, x) = 1.0f / disparity (cv::divide on floats, IEEE), ConvertToBinary.cpp:152-156
__device__ __forceinline__ float meshDepth(const MeshGrid& g, int x, int y) {
  return 1.0f / __ldg(g.disp + (size_t)__ldg(g.yofs + y) * g.srcW + __ldg(g.xofs + x));
}
// z of the equi-error vertex (MeshUtil.h:326) and the vertex mask (ConvertToBinary.cpp:163-176)
__device__ __forceinline__ double meshZ(const MeshGrid& g, int x, int y, bool* valid) {
  const float depth = meshDepth(g, x, y);
  bool ok = !(depth != depth);
  if (g.fg) ok = ok && (__ldg(g.fg + (size_t)__ldg(g.fgy + y) * g.fgW + __ldg(g.fgx + x)) & 1u);  // Mat_<bool> & Mat_<bool>
  *valid = ok;
  return g.scale / (double)depth;
}
__device__ __forceinline__ double MeshGrid::corner(int x, int y, bool* valid) const { return meshZ(*this, x, y, valid); }

// Equirect mesh of a disparity equirect (CreateObjFromDisparityEquirect.cpp:64-71): mesh_util::getVertexesEquirect
// (MeshUtil.h:298-313) and getFaces(wrapHorizontally = true, isRigCoordinates = true, tearRatio).  Every vertex is kept;
// the distance of a corner is the fp64 norm of its vertex (Eigen's 3-term sum, left to right).
struct EqrGrid {
  int W, H;
  const double* vtx;  // [H][W][3], eqrVertexKernel's output
  float tearRatio;
  static constexpr bool kMasked = false;
  __device__ __forceinline__ double corner(int x, int y, bool* valid) const {
    const double* p = vtx + ((size_t)y * W + x) * 3;
    *valid = true;
    return sqrt((p[0] * p[0] + p[1] * p[1]) + p[2] * p[2]);
  }
};

// getVertexesEquirect, one thread per vertex: depth = fminf(maxDepth, 1.0f / disparity) (fmin's NaN rule: a NaN
// quotient gives maxDepth), vertex = double(depth) * (double(sin(phi) * cos(theta)), double(cos(phi)),
// double(sin(phi) * sin(theta))) with the fp32 products.  sin / cos of theta (per column) and phi (per row) come from
// tables the host built with its C library (derp_equirect_mesh), so no device transcendental enters the vertexes.
__global__ void eqrVertexKernel(int W, int H, const float* __restrict__ disp, float maxDepth,
                                const float* __restrict__ sinTheta, const float* __restrict__ cosTheta,
                                const float* __restrict__ sinPhi, const float* __restrict__ cosPhi,
                                double* __restrict__ vtx) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= W || y >= H) return;
  const size_t i = (size_t)y * W + x;
  const double depth = (double)fminf(maxDepth, 1.0f / __ldg(disp + i));
  const float sp = __ldg(sinPhi + y);
  vtx[i * 3 + 0] = depth * (double)(sp * __ldg(cosTheta + x));
  vtx[i * 3 + 1] = depth * (double)__ldg(cosPhi + y);
  vtx[i * 3 + 2] = depth * (double)(sp * __ldg(sinTheta + x));
}

// cv::resize(src, dst, Size(), f, f) with the default INTER_LINEAR on floats (CreateObjFromDisparityEquirect.cpp:61),
// per output pixel: one horizontal pass per source row of the pair, then the vertical blend, each two fp32 products and
// a sum, unfused (-fmad=false).  Taps are built on the host (derp_equirect_mesh): column x reads source columns
// xofs[x] and xofs[x] + 1 with weights (xw[2x], xw[2x + 1]), or copies column xofs[x] where xcopy[x] (the right border);
// row y blends source rows yofs[2y], yofs[2y + 1] with (yw[2y], yw[2y + 1]).  The host instantiation is pinned to cv2.
struct LinearTaps {
  const int* xofs;
  const uint8_t* xcopy;
  const float* xw;
  const int* yofs;
  const float* yw;
};
__host__ __device__ __forceinline__ float linearRow(const float* row, const LinearTaps& t, int x) {
  const int s = t.xofs[x];
  if (t.xcopy[x]) return row[s];
  const float p0 = row[s] * t.xw[2 * x], p1 = row[s + 1] * t.xw[2 * x + 1];
  return p0 + p1;
}
__host__ __device__ __forceinline__ float linearPixel(const float* src, int sw, const LinearTaps& t, int x, int y) {
  const float r0 = linearRow(src + (size_t)t.yofs[2 * y] * sw, t, x);
  const float r1 = linearRow(src + (size_t)t.yofs[2 * y + 1] * sw, t, x);
  const float p0 = r0 * t.yw[2 * y], p1 = r1 * t.yw[2 * y + 1];
  return p0 + p1;
}
__global__ void resizeLinearKernel(const float* __restrict__ src, int sw, const LinearTaps t, int dw, int dh,
                                   float* __restrict__ dst) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= dw || y >= dh) return;
  dst[(size_t)y * dw + x] = linearPixel(src, sw, t, x, y);
}

struct DepthTag {
  double v;
  int i;
};
// std::tuple<double, int>::operator<
__device__ __forceinline__ bool tagLess(const DepthTag& a, const DepthTag& b) {
  return a.v < b.v || (!(b.v < a.v) && a.i < b.i);
}

// getTriangleMask (MeshUtil.h:162-221); the corner distances come from the grid's policy.  std::sort of four elements is libstdc++'s
// __insertion_sort (stl_algo.h: below the introsort threshold of 16); restated literally so that NaN depths, for which
// operator< is not a strict weak order, give the permutation the reference gets.
__device__ __forceinline__ unsigned triangleMask(double tl, double tr, double bl, double br, float tearRatio) {
  DepthTag v[4] = {{tl, 0}, {tr, 1}, {bl, 2}, {br, 3}};
#pragma unroll
  for (int i = 1; i < 4; ++i) {
    const DepthTag val = v[i];
    if (tagLess(val, v[0])) {
#pragma unroll
      for (int k = i; k > 0; --k) v[k] = v[k - 1];
      v[0] = val;
    } else {
      int last = i;
#pragma unroll
      for (int next = i - 1; next >= 0; --next) {  // unguarded in the original: v[0] stops it (val is not < v[0])
        if (last == next + 1 && tagLess(val, v[next])) {
          v[last] = v[next];
          last = next;
        }
      }
      v[last] = val;
    }
  }
  const double tear = (double)tearRatio;
  if (v[0].v / v[3].v > tear) {
    if (fabs(tl - br) < fabs(tr - bl)) return 1u << 1 | 1u << 2;
    return 1u << 0 | 1u << 3;
  }
  const double lo = v[0].v / v[2].v;
  const double hi = v[1].v / v[3].v;
  if (lo >= tear && lo > hi) return 1u << (v[3].i ^ 0x3);
  if (hi >= tear) return 1u << (v[0].i ^ 0x3);
  return 0u;
}

// corner c (0 tl, 1 tr, 2 bl, 3 br) of the three vertexes of triangle `which`, in addTriangle's order (MeshUtil.h:224-251)
__device__ __forceinline__ int triangleCorner(int which, int k) {
  // which 0: bl tr tl | 1: tl br tr | 2: br tl bl | 3: tr bl br   (2 bits per corner, k = 0 lowest)
  const unsigned code = which == 0 ? (2u | 1u << 2 | 0u << 4)
                      : which == 1 ? (0u | 3u << 2 | 1u << 4)
                      : which == 2 ? (3u | 0u << 2 | 2u << 4)
                                   : (1u | 2u << 2 | 3u << 4);
  return (int)((code >> (2 * k)) & 3u);
}

// pass 1: kept triangles of every quad (bits 0..3 of quadBits) and, for a masked grid, the vertexes they use
template <typename Grid>
__global__ void meshQuadKernel(const Grid g, uint8_t* __restrict__ quadBits, uint8_t* used) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= g.W || y >= g.H) return;
  const size_t base = (size_t)y * g.W + x;
  unsigned kept = 0;
  if (x < g.W - 1 && y < g.H - 1) {
    bool ok[4];
    const double tl = g.corner(x, y, ok + 0), tr = g.corner(x + 1, y, ok + 1), bl = g.corner(x, y + 1, ok + 2),
                 br = g.corner(x + 1, y + 1, ok + 3);
    const unsigned m = triangleMask(tl, tr, bl, br, g.tearRatio);
    const size_t at[4] = {base, base + 1, base + g.W, base + g.W + 1};
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      if (!((m >> t) & 1u)) continue;
      if constexpr (!Grid::kMasked) {
        kept |= 1u << t;
        continue;
      }
      // every triangle of a quad uses all corners but the opposite one
      const bool all = ok[triangleCorner(t, 0)] && ok[triangleCorner(t, 1)] && ok[triangleCorner(t, 2)];
      if (!all) continue;
      kept |= 1u << t;
#pragma unroll
      for (int k = 0; k < 3; ++k) used[at[triangleCorner(t, k)]] = 1;  // same value from every writer
    }
  }
  quadBits[base] = (uint8_t)kept;
}

constexpr int kScanThreads = 256;
constexpr int kScanItems = 8;  // grid cells per thread and tile
constexpr int kScanTile = kScanThreads * kScanItems;

// exclusive scan of one value per thread over a 256-thread CTA; *total = CTA sum
__device__ __forceinline__ unsigned blockExclusive(unsigned v, unsigned* total) {
  __shared__ unsigned warpSum[kScanThreads / 32];
  __shared__ unsigned ctaSum;
  const unsigned lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  unsigned inc = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const unsigned o = __shfl_up_sync(0xffffffffu, inc, d);
    if (lane >= (unsigned)d) inc += o;
  }
  __syncthreads();  // protects warpSum / ctaSum across successive calls
  if (lane == 31) warpSum[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    unsigned w = lane < kScanThreads / 32 ? warpSum[lane] : 0u;
    unsigned winc = w;
#pragma unroll
    for (int d = 1; d < kScanThreads / 32; d <<= 1) {
      const unsigned o = __shfl_up_sync(0xffffffffu, winc, d);
      if (lane >= (unsigned)d) winc += o;
    }
    if (lane < kScanThreads / 32) warpSum[lane] = winc - w;
    if (lane == kScanThreads / 32 - 1) ctaSum = winc;
  }
  __syncthreads();
  *total = ctaSum;
  return warpSum[warp] + inc - v;
}

// pass 2a: per-tile totals of kept faces and used vertexes (kMasked = false: every vertex counts)
template <bool kMasked>
__global__ void __launch_bounds__(kScanThreads) meshTileCountKernel(size_t n, const uint8_t* __restrict__ quadBits,
                                                                    const uint8_t* __restrict__ used,
                                                                    unsigned* __restrict__ tileFaces,
                                                                    unsigned* __restrict__ tileVerts) {
  const size_t i0 = (size_t)blockIdx.x * kScanTile + (size_t)threadIdx.x * kScanItems;
  unsigned f = 0, v = 0;
#pragma unroll
  for (int k = 0; k < kScanItems; ++k)
    if (i0 + k < n) {
      f += __popc((unsigned)quadBits[i0 + k]);
      if constexpr (kMasked) v += used[i0 + k] ? 1u : 0u;
      else v += 1u;
    }
  unsigned tf, tv;
  blockExclusive(f, &tf);
  blockExclusive(v, &tv);
  if (threadIdx.x == 0) {
    tileFaces[blockIdx.x] = tf;
    tileVerts[blockIdx.x] = tv;
  }
}

// pass 2b: exclusive scan of the tile totals (one CTA; a 4096^2 grid has 8192 tiles); totals[0] = faces, [1] = vertexes
__global__ void __launch_bounds__(kScanThreads) meshTileScanKernel(int tiles, unsigned* tileFaces, unsigned* tileVerts,
                                                                   unsigned long long* totals) {
  unsigned carryF = 0, carryV = 0;
  for (int t0 = 0; t0 < tiles; t0 += kScanThreads) {
    const int t = t0 + threadIdx.x;
    const unsigned f = t < tiles ? tileFaces[t] : 0u, v = t < tiles ? tileVerts[t] : 0u;
    unsigned tf, tv;
    const unsigned ef = blockExclusive(f, &tf), ev = blockExclusive(v, &tv);
    if (t < tiles) {
      tileFaces[t] = carryF + ef;
      tileVerts[t] = carryV + ev;
    }
    carryF += tf;
    carryV += tv;
  }
  if (threadIdx.x == 0) {
    totals[0] = carryF;
    totals[1] = carryV;
  }
}

// The emit passes walk a tile in kScanItems rounds of kScanThreads CONSECUTIVE cells (thread t takes cell round * 256 + t),
// carrying the running offset from round to round, so that a warp's outputs are contiguous in memory.

// pass 3: vertexes in grid order (MeshUtil.h:373-388), new index of every used vertex, float32 xyz (writeDepth's cast)
// T = float: writeDepth's cast; T = double: the values the mesh simplifier starts from (ConvertToBinary.cpp:190)
template <typename T>
__global__ void __launch_bounds__(kScanThreads) meshEmitVertexesKernel(const MeshGrid g, const uint8_t* __restrict__ used,
                                                                       const unsigned* __restrict__ tileVerts,
                                                                       unsigned* __restrict__ newIndex,
                                                                       T* __restrict__ vertexes) {
  const size_t n = (size_t)g.W * g.H;
  unsigned running = tileVerts[blockIdx.x];
#pragma unroll 1
  for (int round = 0; round < kScanItems; ++round) {
    const size_t i = (size_t)blockIdx.x * kScanTile + (size_t)round * kScanThreads + threadIdx.x;
    const bool take = i < n && used[i];
    unsigned total;
    const unsigned at = running + blockExclusive(take ? 1u : 0u, &total);
    running += total;
    if (!take) continue;
    const int y = (int)(i / (size_t)g.W), x = (int)(i - (size_t)y * g.W);
    bool ok;
    const double z = meshZ(g, x, y, &ok);
    newIndex[i] = at;
    vertexes[(size_t)at * 3 + 0] = (T)(g.stepX * (x + 0.5));
    vertexes[(size_t)at * 3 + 1] = (T)(g.stepY * (y + 0.5));
    vertexes[(size_t)at * 3 + 2] = (g.floorZ && z < 0) ? (T)1.17549435e-38f : (T)z;
  }
}

// pass 4: faces in quad order, triangles of a quad in ascending `which` (MeshUtil.h:277-283), re-indexed (MeshUtil.h:393-402)
// when the grid is masked, grid indexes otherwise
template <bool kMasked>
__global__ void __launch_bounds__(kScanThreads) meshEmitFacesKernel(int W, size_t n, const uint8_t* __restrict__ quadBits,
                                                                    const unsigned* __restrict__ tileFaces,
                                                                    const unsigned* __restrict__ newIndex,
                                                                    uint32_t* __restrict__ faces) {
  unsigned running = tileFaces[blockIdx.x];
#pragma unroll 1
  for (int round = 0; round < kScanItems; ++round) {
    const size_t i = (size_t)blockIdx.x * kScanTile + (size_t)round * kScanThreads + threadIdx.x;
    const unsigned bits = i < n ? quadBits[i] : 0u;
    unsigned total;
    unsigned at = running + blockExclusive((unsigned)__popc(bits), &total);
    running += total;
    if (!bits) continue;
    const size_t corner[4] = {i, i + 1, i + (size_t)W, i + (size_t)W + 1};
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      if (!((bits >> t) & 1u)) continue;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const size_t v = corner[triangleCorner(t, c)];
        faces[(size_t)at * 3 + c] = kMasked ? newIndex[v] : (unsigned)v;
      }
      ++at;
    }
  }
}

// getFaces' wrap (MeshUtil.h:285-293): after the quad faces, two faces per row pair join the last and the first column
__global__ void eqrWrapFacesKernel(int W, int H, size_t first, uint32_t* __restrict__ faces) {
  const int y = blockIdx.x * blockDim.x + threadIdx.x;
  if (y >= H - 1) return;
  const unsigned base = (unsigned)y * W, w = (unsigned)W;
  uint32_t* f = faces + (first + 2 * (size_t)y) * 3;
  f[0] = base + w, f[1] = base, f[2] = base + w - 1;
  f[3] = base + w - 1, f[4] = base + 2 * w - 1, f[5] = base + w;
}

}  // namespace derp
