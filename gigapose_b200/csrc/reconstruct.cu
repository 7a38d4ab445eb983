// Row f17: reconstruction of an object from its onboarding RGB-D frames, for the depth refiners of model-free runs.
// The frames' depth images are fused into a truncated signed distance volume in the object frame (gp_tsdf_fuse) and
// its zero surface is extracted by marching tetrahedra (gp_tsdf_extract_count / gp_tsdf_extract_emit).  The host
// (gigapose_b200/reconstruct.py) chooses the box and streams the frames.
//
// Contract (the file is compiled with -fmad=false: every fp32 operation below rounds once, in the order written):
//  Grid.  A dense [Z,Y,X] array of (tsdf, weight) f32 pairs over an axis-aligned box of the object frame; the caller
//   zeroes it before the first frame.  Voxel (x, y, z) has centre c = (o_x + (x + 0.5) s, ...) per axis: the index is
//   converted to f32, 0.5 added, multiplied by s, added to o.
//  Fusion.  Frames are applied in the given order.  Frame f has D f32 [H,W] (the depth in the unit of the poses,
//   0 = missing), a u8 mask [H,W], K f32 [3,3] whose last row is (0, 0, 1), and the object -> camera pose [R | t] f32.
//   Per voxel and frame:
//     x_c = ((R_r0 c_x + R_r1 c_y) + R_r2 c_z) + t_r for r = 0, 1, 2; skip the frame when z = x_c[2] <= 0.
//     u = ((K00 x + K01 y) + K02 z) / z, v = (K11 y + K12 z) / z; the pixel is (rint(u), rint(v)), round half to
//     even, pixel (i, j) centred at (i, j); skip the frame when it lies outside [0, W) x [0, H).
//     With D = D[row, col] > 0 and the mask set: sdf = D - z; when sdf >= -mu the value is min(1, sdf / mu).
//     With D > 0, the mask clear and z < D - mu: the value is +1 (free space, carving the background; a voxel behind
//     an occluder is not carved).  Anything else: no update.
//     Update: tsdf <- (tsdf w + value) / (w + 1), then w <- w + 1.
//   A voxel's result depends on its own frame sequence only: fusion is deterministic and bit-identical between runs.
//  Extraction.  Marching tetrahedra between the voxel centres.  Cube (x, y, z) spans grid points (x..x+1, y..y+1,
//   z..z+1); corner code k = dx + 2 dy + 4 dz.  The Freudenthal split cuts each cube into 6 tetrahedra sharing the
//   diagonal 0 -> 7: for the axis permutation (a, b, c), in the order (x,y,z), (x,z,y), (y,x,z), (y,z,x), (z,x,y),
//   (z,y,x), the corners are 0, e_a, e_a + e_b, 7.  Every tetrahedron edge joins a grid point p to p + d with d a
//   non-zero 0/1 vector (direction code d = dx + 2 dy + 4 dz, 1..7), so neighbouring cubes share their edges and the
//   surface is watertight by construction.
//   A corner is inside when tsdf < 0.  A tetrahedron emits nothing when a corner has weight 0, when an edge has the
//   ends +1 and -1 exactly (a truncation step, not a surface), or when its corners are all inside or all outside.
//   Otherwise one triangle (one corner apart) or two (two and two), on the edges whose ends differ.
//   Vertices: one per grid edge (p, d) that an emitting tetrahedron crosses, at c_p + t (c_{p+d} - c_p) per axis with
//   t = v_p / (v_p - v_{p+d}) (tsdf values; the centres as above, the difference, the product and the sum rounded
//   once each).  Vertex order: by p row-major, then by d; face order: by cube row-major, then tetrahedron, then the
//   triangles of its case.  With tetrahedron corners numbered 0..3 as listed above: one corner a apart from the other
//   three gives one triangle on the edges a-o for the others o, starting at the lowest o; two inside corners a < b and
//   two outside c < d give the quad a-c, a-d, b-d, b-c as the triangles {a-c, a-d, b-d} and {a-c, b-d, b-c}, each
//   starting at a-c.  Every triangle is wound so that its normal (v1 - v0) x (v2 - v0) points from the inside to the
//   outside.
#include <math.h>
#include <stdio.h>

#include "../../include/gigapose_b200.h"
#include "gigapose_kernels.h"

using gp::fail;

namespace {

constexpr int kThreads = 256;
constexpr int kGroup = 32;                   // frames per fusion launch; their matrices travel by value
constexpr int kScanItems = 4;                // elements per thread of the scan
constexpr int kScanBlock = kThreads * kScanItems;

struct FrameParams {
  float R[kGroup][9];
  float t[kGroup][3];
  float K[kGroup][5];                        // K00, K01, K02, K11, K12
};

struct Box {
  int nx, ny, nz;
  float o[3], s;
};

__device__ __forceinline__ float centre(float o, int i, float s) { return o + ((float)i + 0.5f) * s; }

__global__ void __launch_bounds__(kThreads)
fuse_kernel(Box b, float mu, int H, int W, int n, int frame_base, const float* __restrict__ depth,
            const uint8_t* __restrict__ masks, FrameParams fp, float2* __restrict__ grid) {
  const long long total = (long long)b.nx * b.ny * b.nz;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int x = (int)(idx % b.nx), y = (int)((idx / b.nx) % b.ny), z = (int)(idx / ((long long)b.nx * b.ny));
  const float cx = centre(b.o[0], x, b.s), cy = centre(b.o[1], y, b.s), cz = centre(b.o[2], z, b.s);
  float2 g = grid[idx];
  const size_t plane = (size_t)H * W;
  for (int f = 0; f < n; ++f) {
    const float* R = fp.R[f];
    const float* t = fp.t[f];
    const float px = ((R[0] * cx + R[1] * cy) + R[2] * cz) + t[0];
    const float py = ((R[3] * cx + R[4] * cy) + R[5] * cz) + t[1];
    const float pz = ((R[6] * cx + R[7] * cy) + R[8] * cz) + t[2];
    if (!(pz > 0.f)) continue;
    const float* K = fp.K[f];
    const float u = ((K[0] * px + K[1] * py) + K[2] * pz) / pz;
    const float v = (K[3] * py + K[4] * pz) / pz;
    const float ru = rintf(u), rv = rintf(v);
    if (!(ru >= 0.f && ru < (float)W && rv >= 0.f && rv < (float)H)) continue;
    const size_t pix = (size_t)(frame_base + f) * plane + (size_t)(int)rv * W + (int)ru;
    const float D = depth[pix];
    if (!(D > 0.f)) continue;
    float value;
    if (masks[pix]) {
      const float sdf = D - pz;
      if (!(sdf >= -mu)) continue;
      value = fminf(1.f, sdf / mu);
    } else {
      if (!(pz < D - mu)) continue;
      value = 1.f;
    }
    g.x = (g.x * g.y + value) / (g.y + 1.f);
    g.y = g.y + 1.f;
  }
  grid[idx] = g;
}

// ---------------------------------------------------------------------------------------------------- tetrahedra
__device__ __constant__ int kPerm[6][3] = {{0, 1, 2}, {0, 2, 1}, {1, 0, 2}, {1, 2, 0}, {2, 0, 1}, {2, 1, 0}};
__device__ __constant__ int kOdd[6] = {0, 1, 1, 0, 0, 1};

// corner codes of tetrahedron `k` of a cube
__device__ __forceinline__ void tet_corners(int k, int c[4]) {
  c[0] = 0;
  c[1] = 1 << kPerm[k][0];
  c[2] = c[1] | (1 << kPerm[k][1]);
  c[3] = 7;
}

// The triangles of tetrahedron `k` given the cube's corner values: 0, 1 or 2; tri[j] = the 3 edges (as pairs of
// tetrahedron corner indices i < j, packed i * 4 + j) of triangle j, wound outward.
__device__ __forceinline__ int tet_case(int k, const float2 val[8], int tri[2][3]) {
  int c[4];
  tet_corners(k, c);
  int in = 0;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 g = val[c[i]];
    if (!(g.y > 0.f)) return 0;
    if (g.x < 0.f) in |= 1 << i;
  }
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = i + 1; j < 4; ++j) {
      const float a = val[c[i]].x, b = val[c[j]].x;
      if ((a == 1.f && b == -1.f) || (a == -1.f && b == 1.f)) return 0;
    }
  const int cnt = __popc(in);
  if (cnt == 0 || cnt == 4) return 0;
  const auto edge = [](int i, int j) { return i < j ? i * 4 + j : j * 4 + i; };
  bool flip = kOdd[k];
  if (cnt == 1 || cnt == 3) {
    const int lone_bits = cnt == 1 ? in : (~in & 15);
    const int a = __ffs(lone_bits) - 1;
    int o[3], m = 0;
    for (int i = 0; i < 4; ++i)
      if (i != a) o[m++] = i;
    if (a & 1) { const int tmp = o[1]; o[1] = o[2]; o[2] = tmp; }
    if (cnt == 3) flip = !flip;                                       // the lone corner is outside
    tri[0][0] = edge(a, o[0]);
    tri[0][1] = flip ? edge(a, o[2]) : edge(a, o[1]);
    tri[0][2] = flip ? edge(a, o[1]) : edge(a, o[2]);
    return 1;
  }
  int ins[2], outs[2], ni = 0, no = 0;
  for (int i = 0; i < 4; ++i) {
    if (in >> i & 1) ins[ni++] = i;
    else outs[no++] = i;
  }
  // parity of the permutation (a, b, c, d) = (ins, outs)
  const int p[4] = {ins[0], ins[1], outs[0], outs[1]};
  int inv = 0;
  for (int i = 0; i < 4; ++i)
    for (int j = i + 1; j < 4; ++j) inv += p[i] > p[j];
  if (inv & 1) flip = !flip;
  const int q[4] = {edge(ins[0], outs[0]), edge(ins[0], outs[1]), edge(ins[1], outs[1]), edge(ins[1], outs[0])};
  tri[0][0] = q[0]; tri[0][1] = flip ? q[2] : q[1]; tri[0][2] = flip ? q[1] : q[2];
  tri[1][0] = q[0]; tri[1][1] = flip ? q[3] : q[2]; tri[1][2] = flip ? q[2] : q[3];
  return 2;
}

__device__ __forceinline__ void load_cube(const float2* __restrict__ grid, const Box& b, int x, int y, int z,
                                          float2 val[8]) {
#pragma unroll
  for (int k = 0; k < 8; ++k)
    val[k] = grid[((size_t)(z + (k >> 2 & 1)) * b.ny + (y + (k >> 1 & 1))) * b.nx + (x + (k & 1))];
}

__device__ __forceinline__ size_t corner_index(const Box& b, int x, int y, int z, int code) {
  return ((size_t)(z + (code >> 2 & 1)) * b.ny + (y + (code >> 1 & 1))) * b.nx + (x + (code & 1));
}

// count pass: marks the crossed edges of emitting tetrahedra (bit d of edges[p]) and counts each cube's triangles
__global__ void __launch_bounds__(kThreads)
mark_kernel(Box b, const float2* __restrict__ grid, unsigned* __restrict__ edges, int* __restrict__ face_count) {
  const long long total = (long long)b.nx * b.ny * b.nz;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int x = (int)(idx % b.nx), y = (int)((idx / b.nx) % b.ny), z = (int)(idx / ((long long)b.nx * b.ny));
  int faces = 0;
  if (x + 1 < b.nx && y + 1 < b.ny && z + 1 < b.nz) {
    float2 val[8];
    load_cube(grid, b, x, y, z, val);
    for (int k = 0; k < 6; ++k) {
      int tri[2][3];
      const int nt = tet_case(k, val, tri);
      if (!nt) continue;
      faces += nt;
      int c[4];
      tet_corners(k, c);
      for (int t = 0; t < nt; ++t)
        for (int e = 0; e < 3; ++e) {
          const int i = tri[t][e] >> 2, j = tri[t][e] & 3;
          atomicOr(edges + corner_index(b, x, y, z, c[i]), 1u << (c[i] ^ c[j]));
        }
    }
  }
  face_count[idx] = faces;
}

__global__ void __launch_bounds__(kThreads)
edge_count_kernel(long long total, const unsigned* __restrict__ edges, int* __restrict__ vertex_count) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx < total) vertex_count[idx] = __popc(edges[idx]);
}

// ---------------------------------------------------------------------------------------------------- scan
// exclusive scan of n ints in place, in three launches: block sums, a one-block scan of the block sums (which also
// writes the total to *total), and the per-block scans with their offsets
__global__ void __launch_bounds__(kThreads) scan_sums_kernel(long long n, const int* __restrict__ a, int* __restrict__ sums) {
  __shared__ int red[kThreads / 32];
  const long long base = (long long)blockIdx.x * kScanBlock;
  int s = 0;
#pragma unroll
  for (int i = 0; i < kScanItems; ++i) {
    const long long j = base + (long long)threadIdx.x * kScanItems + i;
    if (j < n) s += a[j];
  }
  for (int d = 16; d; d >>= 1) s += __shfl_xor_sync(0xffffffffu, s, d);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    int t = 0;
    for (int w = 0; w < kThreads / 32; ++w) t += red[w];
    sums[blockIdx.x] = t;
  }
}

// block-wide exclusive scan of one int per thread; returns the thread's prefix and sets *block_total
__device__ __forceinline__ int block_exclusive(int v, int* block_total) {
  __shared__ int warp_sums[kThreads / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int incl = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const int o = __shfl_up_sync(0xffffffffu, incl, d);
    if (lane >= d) incl += o;
  }
  if (lane == 31) warp_sums[warp] = incl;
  __syncthreads();
  int before = 0, total = 0;
  for (int w = 0; w < kThreads / 32; ++w) {
    if (w < warp) before += warp_sums[w];
    total += warp_sums[w];
  }
  __syncthreads();
  *block_total = total;
  return before + incl - v;
}

__global__ void __launch_bounds__(kThreads) scan_block_sums_kernel(int nb, int* __restrict__ sums, long long* __restrict__ total) {
  int carry = 0;
  for (int base = 0; base < nb; base += kThreads) {
    const int j = base + threadIdx.x;
    const int v = j < nb ? sums[j] : 0;
    int chunk;
    const int ex = block_exclusive(v, &chunk);
    if (j < nb) sums[j] = carry + ex;
    carry += chunk;
  }
  if (threadIdx.x == 0) *total = carry;
}

__global__ void __launch_bounds__(kThreads) scan_apply_kernel(long long n, int* __restrict__ a, const int* __restrict__ sums) {
  const long long base = (long long)blockIdx.x * kScanBlock + (long long)threadIdx.x * kScanItems;
  int v[kScanItems], s = 0;
#pragma unroll
  for (int i = 0; i < kScanItems; ++i) {
    v[i] = base + i < n ? a[base + i] : 0;
    s += v[i];
  }
  int unused;
  int run = sums[blockIdx.x] + block_exclusive(s, &unused);
#pragma unroll
  for (int i = 0; i < kScanItems; ++i) {
    if (base + i < n) a[base + i] = run;
    run += v[i];
  }
}

// ---------------------------------------------------------------------------------------------------- emit
__device__ __forceinline__ int vertex_id(const unsigned* __restrict__ edges, const int* __restrict__ vbase, size_t p,
                                         int d) {
  return vbase[p] + __popc(edges[p] & ((1u << d) - 1u));
}

__global__ void __launch_bounds__(kThreads)
vertex_kernel(Box b, const float2* __restrict__ grid, const unsigned* __restrict__ edges, const int* __restrict__ vbase,
              float* __restrict__ vertices) {
  const long long total = (long long)b.nx * b.ny * b.nz;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const unsigned m = edges[idx];
  if (!m) return;
  const int x = (int)(idx % b.nx), y = (int)((idx / b.nx) % b.ny), z = (int)(idx / ((long long)b.nx * b.ny));
  const float v0 = grid[idx].x;
  const int p0[3] = {x, y, z};
  int out = vbase[idx];
  for (int d = 1; d < 8; ++d) {
    if (!(m >> d & 1)) continue;
    const float v1 = grid[corner_index(b, x, y, z, d)].x;
    const float t = v0 / (v0 - v1);
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const float c0 = centre(b.o[a], p0[a], b.s);
      float pos = c0;
      if (d >> a & 1) {
        const float c1 = centre(b.o[a], p0[a] + 1, b.s);
        pos = c0 + t * (c1 - c0);
      }
      vertices[3 * (size_t)out + a] = pos;
    }
    ++out;
  }
}

__global__ void __launch_bounds__(kThreads)
face_kernel(Box b, const float2* __restrict__ grid, const unsigned* __restrict__ edges, const int* __restrict__ vbase,
            const int* __restrict__ fbase, int* __restrict__ faces) {
  const long long total = (long long)b.nx * b.ny * b.nz;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int x = (int)(idx % b.nx), y = (int)((idx / b.nx) % b.ny), z = (int)(idx / ((long long)b.nx * b.ny));
  if (!(x + 1 < b.nx && y + 1 < b.ny && z + 1 < b.nz)) return;
  float2 val[8];
  load_cube(grid, b, x, y, z, val);
  int out = fbase[idx];
  for (int k = 0; k < 6; ++k) {
    int tri[2][3];
    const int nt = tet_case(k, val, tri);
    int c[4];
    tet_corners(k, c);
    for (int t = 0; t < nt; ++t) {
      for (int e = 0; e < 3; ++e) {
        const int i = tri[t][e] >> 2, j = tri[t][e] & 3;
        faces[3 * (size_t)out + e] = vertex_id(edges, vbase, corner_index(b, x, y, z, c[i]), c[i] ^ c[j]);
      }
      ++out;
    }
  }
}

// ---------------------------------------------------------------------------------------------------- host
int check_box(int nx, int ny, int nz, const float* origin, float voxel, int min_side) {
  if (nx < min_side || ny < min_side || nz < min_side)
    return fail(GP_ERR_INVALID, "grid %d x %d x %d: every side must be at least %d", nx, ny, nz, min_side);
  // 12 triangles per cube at most: face and vertex counts and indices stay within int32
  if ((long long)nx * ny * nz > GP_TSDF_MAX_VOXELS)
    return fail(GP_ERR_INVALID, "grid %d x %d x %d exceeds GP_TSDF_MAX_VOXELS = %d voxels", nx, ny, nz,
                GP_TSDF_MAX_VOXELS);
  if (!origin) return fail(GP_ERR_INVALID, "null origin");
  for (int a = 0; a < 3; ++a)
    if (!isfinite(origin[a])) return fail(GP_ERR_INVALID, "origin[%d] is not finite", a);
  if (!(voxel > 0.f) || !isfinite(voxel)) return fail(GP_ERR_INVALID, "voxel size %g must be positive and finite", voxel);
  return GP_OK;
}

Box make_box(int nx, int ny, int nz, const float* origin, float voxel) {
  Box b;
  b.nx = nx; b.ny = ny; b.nz = nz;
  for (int a = 0; a < 3; ++a) b.o[a] = origin[a];
  b.s = voxel;
  return b;
}

int blocks_for(long long n) { return (int)((n + kThreads - 1) / kThreads); }

struct Workspace {
  unsigned* edges;
  int* vbase;
  int* fbase;
  int* sums;
  long long* totals;
};

Workspace carve(void* base, long long total) {
  gp::Carver c(base);
  Workspace w;
  w.edges = c.take<unsigned>(total);
  w.vbase = c.take<int>(total);
  w.fbase = c.take<int>(total);
  w.sums = c.take<int>((total + kScanBlock - 1) / kScanBlock);
  w.totals = c.take<long long>(2);
  return w;
}

size_t workspace_bytes(long long total) {
  gp::Carver c(nullptr);
  c.take<unsigned>(total);
  c.take<int>(total);
  c.take<int>(total);
  c.take<int>((total + kScanBlock - 1) / kScanBlock);
  c.take<long long>(2);
  return c.off;
}

int scan(long long n, int* a, int* sums, long long* total, cudaStream_t s) {
  const int nb = (int)((n + kScanBlock - 1) / kScanBlock);
  GP_CUDA(gp::launch_ex(scan_sums_kernel, nb, kThreads, 0, s, 1, false, n, a, sums));
  GP_CUDA(gp::launch_ex(scan_block_sums_kernel, 1, kThreads, 0, s, 1, false, nb, sums, total));
  GP_CUDA(gp::launch_ex(scan_apply_kernel, nb, kThreads, 0, s, 1, false, n, a, sums));
  return GP_OK;
}

}  // namespace

extern "C" int gp_tsdf_fuse(int nx, int ny, int nz, const float* origin, float voxel, float trunc, int n_frames,
                            int height, int width, const float* depth, const uint8_t* masks, const float* K,
                            const float* poses, float* grid, void* stream) {
  if (const int rc = check_box(nx, ny, nz, origin, voxel, 1)) return rc;
  if (!(trunc > 0.f) || !isfinite(trunc)) return fail(GP_ERR_INVALID, "truncation %g must be positive and finite", trunc);
  if (n_frames < 0 || height < 1 || width < 1)
    return fail(GP_ERR_INVALID, "bad frame shape: %d frames of %d x %d", n_frames, height, width);
  if (height > (1 << 24) || width > (1 << 24)) return fail(GP_ERR_INVALID, "frame side over 2^24 px");
  if (!grid) return fail(GP_ERR_INVALID, "null grid");
  if (n_frames == 0) return GP_OK;
  if (!depth || !masks || !K || !poses) return fail(GP_ERR_INVALID, "null argument");
  for (int f = 0; f < n_frames; ++f) {
    const float* k = K + 9 * (size_t)f;
    const float* p = poses + 16 * (size_t)f;
    for (int i = 0; i < 9; ++i)
      if (!isfinite(k[i])) return fail(GP_ERR_INVALID, "frame %d: K holds a non-finite value", f);
    if (k[3] != 0.f || k[6] != 0.f || k[7] != 0.f || k[8] != 1.f)
      return fail(GP_ERR_INVALID, "frame %d: K must have the rows (K10, K20, K21, K22) = (0, 0, 0, 1)", f);
    for (int i = 0; i < 12; ++i)
      if (!isfinite(p[i])) return fail(GP_ERR_INVALID, "frame %d: the pose holds a non-finite value", f);
  }
  const Box b = make_box(nx, ny, nz, origin, voxel);
  const long long total = (long long)nx * ny * nz;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  for (int f0 = 0; f0 < n_frames; f0 += kGroup) {
    const int g = n_frames - f0 < kGroup ? n_frames - f0 : kGroup;
    FrameParams fp = {};
    for (int f = 0; f < g; ++f) {
      const float* k = K + 9 * (size_t)(f0 + f);
      const float* p = poses + 16 * (size_t)(f0 + f);
      for (int r = 0; r < 3; ++r) {
        for (int c = 0; c < 3; ++c) fp.R[f][3 * r + c] = p[4 * r + c];
        fp.t[f][r] = p[4 * r + 3];
      }
      fp.K[f][0] = k[0]; fp.K[f][1] = k[1]; fp.K[f][2] = k[2]; fp.K[f][3] = k[4]; fp.K[f][4] = k[5];
    }
    GP_CUDA(gp::launch_ex(fuse_kernel, blocks_for(total), kThreads, 0, s, 1, false, b, trunc, height, width, g, f0,
                          depth, masks, fp, reinterpret_cast<float2*>(grid)));
  }
  return GP_OK;
}

extern "C" int gp_tsdf_extract_query_sizes(int nx, int ny, int nz, size_t* workspace_bytes_out) {
  const float o[3] = {0.f, 0.f, 0.f};
  if (const int rc = check_box(nx, ny, nz, o, 1.f, 2)) return rc;
  if (!workspace_bytes_out) return fail(GP_ERR_INVALID, "null argument");
  *workspace_bytes_out = workspace_bytes((long long)nx * ny * nz);
  return GP_OK;
}

extern "C" int gp_tsdf_extract_count(int nx, int ny, int nz, const float* grid, void* workspace, int64_t* counts,
                                     void* stream) {
  const float o[3] = {0.f, 0.f, 0.f};
  if (const int rc = check_box(nx, ny, nz, o, 1.f, 2)) return rc;
  if (!grid || !workspace || !counts) return fail(GP_ERR_INVALID, "null argument");
  const long long total = (long long)nx * ny * nz;
  const Box b = make_box(nx, ny, nz, o, 1.f);
  const Workspace w = carve(workspace, total);
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  GP_CUDA(cudaMemsetAsync(w.edges, 0, (size_t)total * sizeof(unsigned), s));
  GP_CUDA(gp::launch_ex(mark_kernel, blocks_for(total), kThreads, 0, s, 1, false, b,
                        reinterpret_cast<const float2*>(grid), w.edges, w.fbase));
  GP_CUDA(gp::launch_ex(edge_count_kernel, blocks_for(total), kThreads, 0, s, 1, false, total, w.edges, w.vbase));
  if (const int rc = scan(total, w.vbase, w.sums, w.totals, s)) return rc;
  if (const int rc = scan(total, w.fbase, w.sums, w.totals + 1, s)) return rc;
  GP_CUDA(cudaMemcpyAsync(counts, w.totals, 2 * sizeof(long long), cudaMemcpyDeviceToDevice, s));
  return GP_OK;
}

extern "C" int gp_tsdf_extract_emit(int nx, int ny, int nz, const float* origin, float voxel, const float* grid,
                                    const void* workspace, float* vertices, int32_t* faces, void* stream) {
  if (const int rc = check_box(nx, ny, nz, origin, voxel, 2)) return rc;
  if (!grid || !workspace || !vertices || !faces) return fail(GP_ERR_INVALID, "null argument");
  const long long total = (long long)nx * ny * nz;
  const Box b = make_box(nx, ny, nz, origin, voxel);
  const Workspace w = carve(const_cast<void*>(workspace), total);
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  GP_CUDA(gp::launch_ex(vertex_kernel, blocks_for(total), kThreads, 0, s, 1, false, b,
                        reinterpret_cast<const float2*>(grid), w.edges, w.vbase, vertices));
  GP_CUDA(gp::launch_ex(face_kernel, blocks_for(total), kThreads, 0, s, 1, false, b,
                        reinterpret_cast<const float2*>(grid), w.edges, w.vbase, w.fbase, faces));
  return GP_OK;
}
