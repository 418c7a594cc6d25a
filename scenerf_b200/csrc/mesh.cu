// Mesh extraction from a TSDF volume: marching cubes at level 0 on the device, the get_mesh / get_point_cloud of the
// reference's TSDFVolume (scenerf/data/utils/fusion.py:333-379, skimage's marching_cubes_lewiner there).
//
// Algorithm (DESIGN.md 6.6; numpy statement in oracle/mesh_oracle.py, held to bit for bit):
//   count   one thread per grid point p: the 3-bit mask of p's crossed owned edges (+x, +y, +z; a corner is inside iff
//           its value is < 0, masked-out voxels read 1.0) and the triangle count of the cell whose lowest corner is p;
//   scan    deterministic exclusive scan of both counts (tile scan, scan of tile totals, add back): vertex ids and the
//           first face of every cell, in C order, with no atomics;
//   verts   one thread per grid point: position p + t e_axis (t = f0 / (f0 - f1)), world coordinates, colour at the
//           rounded index, lerped central-difference gradient as the normal;
//   faces   one thread per cell: re-trace the cell's polygon loops and triangulate them.
// Cell topology comes from a polygon tracer instead of a case table: every face with two crossed edges gets one
// segment, every face with four crossed edges gets two, paired by the asymptotic decider on the face's corners in
// global-axis order (so the two cells of a face decide bit for bit alike).  Segments are directed so that the loops
// have normals toward increasing values.
//
// Cell numbering: corner c has offset (c & 1, c >> 1 & 1, c >> 2 & 1); edge e runs along axis e >> 2 from the corner
// whose two other bits, lower axis first, are e & 3.  Loops are packed as 4-bit edge ids in a 64-bit word so that no
// per-thread array needs local memory.
#include "kernels.cuh"

namespace srf {
namespace {

constexpr int kScanThreads = 256;
constexpr int kScanItems = 8;
constexpr int kScanTile = kScanThreads * kScanItems;
constexpr int kTotalsThreads = 1024;

struct Grid {
  int X, Y, Z;
  long long n, sx, sy;    // strides of x and y (z is contiguous)
};

__device__ __forceinline__ float mval(const float* __restrict__ tsdf, const unsigned char* __restrict__ mask, long long i) {
  return (mask && !mask[i]) ? 1.0f : tsdf[i];
}

__device__ __forceinline__ int edge_of(int axis, int corner) {
  const int o1 = axis == 0 ? 1 : 0, o2 = axis == 2 ? 1 : 2;
  return axis * 4 + (((corner >> o1) & 1) | (((corner >> o2) & 1) << 1));
}

__device__ __forceinline__ int edge_origin(int e) {
  const int a = e >> 2, j = e & 3, o1 = a == 0 ? 1 : 0, o2 = a == 2 ? 1 : 2;
  return ((j & 1) << o1) | ((j >> 1) << o2);
}

// Bit n set when edge e lies on the cell's high face of axis n (the face shared with the next cell along n).
__device__ __forceinline__ int high_faces(int e) { return edge_origin(e); }

__device__ __forceinline__ int nib(unsigned long long w, int k) { return (int)((w >> (4 * k)) & 15ull); }

__device__ __forceinline__ void load_cell(const float* __restrict__ tsdf, const unsigned char* __restrict__ mask,
                                          const Grid& g, long long i, float (&v)[8]) {
#pragma unroll
  for (int c = 0; c < 8; ++c) v[c] = mval(tsdf, mask, i + (c & 1) * g.sx + ((c >> 1) & 1) * g.sy + ((c >> 2) & 1));
}

// The cell's directed segments as a successor table nxt (edge -> next edge of its loop, 4 bits each); returns the
// 12-bit set of crossed edges.
__device__ __forceinline__ unsigned trace_cell(const float (&v)[8], unsigned long long& nxt) {
  unsigned inside = 0;
#pragma unroll
  for (int c = 0; c < 8; ++c) inside |= (v[c] < 0.0f ? 1u : 0u) << c;
  nxt = 0;
  unsigned crossed = 0;
  if (inside == 0 || inside == 255) return 0;
#pragma unroll
  for (int n = 0; n < 3; ++n) {
#pragma unroll
    for (int s = 0; s < 2; ++s) {
      const int U = n == 0 ? 1 : 0, V = n == 2 ? 1 : 2, base = s << n;
      const int q0 = base, q1 = base | 1 << U, q2 = base | 1 << U | 1 << V, q3 = base | 1 << V;   // (u0v0) (u1v0) (u1v1) (u0v1)
      const int e_ab = edge_of(U, q0), e_bc = edge_of(V, q1), e_cd = edge_of(U, q3), e_da = edge_of(V, q0);
      // counter-clockwise seen from outside the cell: q0 q1 q2 q3 turns about U x V, which is +n for n = 0, 2
      const bool fwd = (n != 1) == (s == 1);
      const int W[4] = {q0, fwd ? q1 : q3, q2, fwd ? q3 : q1};
      const int E[4] = {fwd ? e_ab : e_da, fwd ? e_bc : e_cd, fwd ? e_cd : e_bc, fwd ? e_da : e_ab};   // E[k]: W[k] -> W[k+1]
      unsigned cr = 0;
#pragma unroll
      for (int k = 0; k < 4; ++k) cr |= (((inside >> W[k]) ^ (inside >> W[(k + 1) & 3])) & 1u) << k;
      if (!cr) continue;
      bool cut_outside = false;
      if (cr == 15u) {
        // asymptotic decider, a=f(u0,v0) b=f(u1,v0) c=f(u1,v1) d=f(u0,v1), no contraction into FMAs
        const float a = v[q0], b = v[q1], c = v[q2], d = v[q3];
        const float det = __fsub_rn(__fmul_rn(a, c), __fmul_rn(b, d));
        const float den = __fsub_rn(__fsub_rn(__fadd_rn(a, c), b), d);
        cut_outside = (det < 0.0f && den > 0.0f) || (det > 0.0f && den < 0.0f);
      }
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        if (!((cr >> k) & 1u)) continue;
        crossed |= 1u << E[k];
        if ((inside >> W[k]) & 1u) continue;                  // only steps that enter the inside start a segment
        int m;
        if (cut_outside) {
          m = (k + 3) & 3;
        } else {
          m = (k + 1) & 3;
          if (!((cr >> m) & 1u)) m = (m + 1) & 3;
          if (!((cr >> m) & 1u)) m = (m + 1) & 3;
        }
        int em = E[0];
#pragma unroll
        for (int j = 1; j < 4; ++j) em = m == j ? E[j] : em;
        nxt |= (unsigned long long)em << (4 * E[k]);
      }
    }
  }
  return crossed;
}

__device__ __forceinline__ int loop_count(unsigned crossed, unsigned long long nxt) {
  int loops = 0;
  while (crossed) {
    const int e0 = __ffs(crossed) - 1;
    int e = e0;
    do {
      crossed &= ~(1u << e);
      e = nib(nxt, e);
    } while (e != e0);
    ++loops;
  }
  return loops;
}

__global__ void mesh_count_kernel(const float* __restrict__ tsdf, const unsigned char* __restrict__ mask, const Grid g,
                                  unsigned char* __restrict__ emask, int* __restrict__ vcount, int* __restrict__ tcount) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= g.n) return;
  const int z = (int)(i % g.Z), y = (int)((i / g.Z) % g.Y), x = (int)(i / g.sx);
  const bool in0 = mval(tsdf, mask, i) < 0.0f;
  unsigned em = 0;
  if (x + 1 < g.X && (mval(tsdf, mask, i + g.sx) < 0.0f) != in0) em |= 1u;
  if (y + 1 < g.Y && (mval(tsdf, mask, i + g.sy) < 0.0f) != in0) em |= 2u;
  if (z + 1 < g.Z && (mval(tsdf, mask, i + 1) < 0.0f) != in0) em |= 4u;
  emask[i] = (unsigned char)em;
  vcount[i] = __popc(em);
  int tris = 0;
  if (x + 1 < g.X && y + 1 < g.Y && z + 1 < g.Z) {
    float v[8];
    load_cell(tsdf, mask, g, i, v);
    unsigned long long nxt;
    const unsigned crossed = trace_cell(v, nxt);
    if (crossed) tris = __popc(crossed) - 2 * loop_count(crossed, nxt);   // a loop of k edges gives k - 2 triangles
  }
  tcount[i] = tris;
}

// Exclusive scan of one value per thread over the block; *total gets the block's sum.  s: 33 ints of shared memory.
__device__ __forceinline__ int block_exclusive_scan(int v, int* s, int* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  int inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int u = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += u;
  }
  if (lane == 31) s[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    const int w = lane < nwarps ? s[lane] : 0;
    int winc = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int u = __shfl_up_sync(0xffffffffu, winc, o);
      if (lane >= o) winc += u;
    }
    if (lane < nwarps) s[lane] = winc - w;
    if (lane == 31) s[32] = winc;
  }
  __syncthreads();
  const int out = inc - v + s[warp];
  *total = s[32];
  __syncthreads();                        // s is reused by the caller's next scan
  return out;
}

// blockIdx.y selects the array (0 vertices, 1 triangles); each block scans one tile in place and writes its total to
// tot[y * (ntiles + 1) + tile].
__global__ void __launch_bounds__(kScanThreads) scan_tiles_kernel(int* __restrict__ a0, int* __restrict__ a1, long long n,
                                                                  int* __restrict__ tot, int ntiles) {
  __shared__ int s[33];
  int* a = blockIdx.y ? a1 : a0;
  const long long base = (long long)blockIdx.x * kScanTile + (long long)threadIdx.x * kScanItems;
  int x[kScanItems];
  int sum = 0;
#pragma unroll
  for (int k = 0; k < kScanItems; ++k) {
    x[k] = base + k < n ? a[base + k] : 0;
    sum += x[k];
  }
  int total;
  int run = block_exclusive_scan(sum, s, &total);
#pragma unroll
  for (int k = 0; k < kScanItems; ++k) {
    if (base + k < n) a[base + k] = run;
    run += x[k];
  }
  if (threadIdx.x == 0) tot[blockIdx.y * (ntiles + 1) + blockIdx.x] = total;
}

// One block per array: exclusive scan of the tile totals in place, the grand total at index ntiles.
__global__ void __launch_bounds__(kTotalsThreads) scan_totals_kernel(int* __restrict__ tot, int ntiles) {
  __shared__ int s[33];
  int* t = tot + blockIdx.y * (ntiles + 1);
  int carry = 0;
  for (int base = 0; base < ntiles; base += kTotalsThreads) {
    const int j = base + threadIdx.x;
    const int v = j < ntiles ? t[j] : 0;
    int total;
    const int ex = block_exclusive_scan(v, s, &total);
    if (j < ntiles) t[j] = carry + ex;
    carry += total;
  }
  if (threadIdx.x == 0) t[ntiles] = carry;
}

__global__ void __launch_bounds__(kScanThreads) scan_add_kernel(int* __restrict__ a0, int* __restrict__ a1, long long n,
                                                                const int* __restrict__ tot, int ntiles) {
  if (blockIdx.x == 0) return;
  int* a = blockIdx.y ? a1 : a0;
  const int off = tot[blockIdx.y * (ntiles + 1) + blockIdx.x];
  const long long base = (long long)blockIdx.x * kScanTile + (long long)threadIdx.x * kScanItems;
#pragma unroll
  for (int k = 0; k < kScanItems; ++k)
    if (base + k < n) a[base + k] += off;
}

// np.gradient(edge_order=1) along axis k at grid point i (coordinate c of dim D, stride st)
__device__ __forceinline__ float grad1(const float* __restrict__ tsdf, const unsigned char* __restrict__ mask, long long i,
                                       int c, int D, long long st) {
  if (c == 0) return __fsub_rn(mval(tsdf, mask, i + st), mval(tsdf, mask, i));
  if (c == D - 1) return __fsub_rn(mval(tsdf, mask, i), mval(tsdf, mask, i - st));
  return __fmul_rn(__fsub_rn(mval(tsdf, mask, i + st), mval(tsdf, mask, i - st)), 0.5f);
}

struct EmitParams {
  Grid g;
  float origin[3];
  float voxel;                            // float32(voxel_size)
};

__global__ void mesh_verts_kernel(const __grid_constant__ EmitParams q, const float* __restrict__ tsdf,
                                  const float* __restrict__ color, const unsigned char* __restrict__ mask,
                                  const unsigned char* __restrict__ emask, const int* __restrict__ vscan,
                                  float* __restrict__ verts, float* __restrict__ normals, unsigned char* __restrict__ colors) {
  const Grid& g = q.g;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= g.n) return;
  const unsigned em = emask[i];
  if (!em) return;
  const int z = (int)(i % g.Z), y = (int)((i / g.Z) % g.Y), x = (int)(i / g.sx);
  const float f0 = mval(tsdf, mask, i);
  long long id = vscan[i];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    if (!((em >> a) & 1u)) continue;
    const long long st = a == 0 ? g.sx : a == 1 ? g.sy : 1;
    const float f1 = mval(tsdf, mask, i + st);
    const float t = __fdiv_rn(f0, __fsub_rn(f0, f1));
    float p[3] = {(float)x, (float)y, (float)z};
    p[a] = __fadd_rn(p[a], t);
#pragma unroll
    for (int k = 0; k < 3; ++k) verts[id * 3 + k] = __fadd_rn(__fmul_rn(p[k], q.voxel), q.origin[k]);
    if (colors) {
      // fusion.py:342,346-351: colour of the voxel at the rounded (half to even) index, b*65536 + g*256 + r unfolded
      const long long ci = (long long)rintf(p[0]) * g.sx + (long long)rintf(p[1]) * g.sy + (long long)rintf(p[2]);
      const float rgb = color[ci];
      const float cb = floorf(__fdiv_rn(rgb, 65536.0f));
      const float hi = __fsub_rn(rgb, __fmul_rn(cb, 65536.0f));
      const float cg = floorf(__fdiv_rn(hi, 256.0f));
      const float cr = __fsub_rn(hi, __fmul_rn(cg, 256.0f));
      colors[id * 3 + 0] = (unsigned char)(int)floorf(cr);
      colors[id * 3 + 1] = (unsigned char)(int)cg;
      colors[id * 3 + 2] = (unsigned char)(int)cb;
    }
    if (normals) {
      const int c1[3] = {x + (a == 0), y + (a == 1), z + (a == 2)};
      const int c0[3] = {x, y, z};
      const int D[3] = {g.X, g.Y, g.Z};
      const long long S[3] = {g.sx, g.sy, 1};
      float nv[3];
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const float g0 = grad1(tsdf, mask, i, c0[k], D[k], S[k]);
        const float g1 = grad1(tsdf, mask, i + st, c1[k], D[k], S[k]);
        nv[k] = __fadd_rn(g0, __fmul_rn(t, __fsub_rn(g1, g0)));
      }
      const float len = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(nv[0], nv[0]), __fmul_rn(nv[1], nv[1])), __fmul_rn(nv[2], nv[2])));
#pragma unroll
      for (int k = 0; k < 3; ++k) normals[id * 3 + k] = len > 0.0f ? __fdiv_rn(nv[k], len) : 0.0f;
    }
    ++id;
  }
}

__device__ __forceinline__ int vertex_id(const Grid& g, long long cell, int e, const unsigned char* __restrict__ emask,
                                         const int* __restrict__ vscan) {
  const int o = edge_origin(e), a = e >> 2;
  const long long p = cell + (o & 1) * g.sx + ((o >> 1) & 1) * g.sy + ((o >> 2) & 1);
  return vscan[p] + __popc(emask[p] & ((1u << a) - 1u));
}

// Loops start at their lowest edge.  Triangulation: ear clipping that takes, at each step, the first ear
// (prev, cur, next) with cur = L[1], L[2], ..., L[n-1], L[0] whose diagonal (prev, next) does not lie on a high face of
// the cell; this is the fan from L[0] whenever all of its diagonals qualify.  A diagonal on a cell face is also an edge
// of the neighbouring cell's polygons; allowing them on low faces only keeps the two cells of a face from both drawing it.
__global__ void mesh_faces_kernel(const float* __restrict__ tsdf, const unsigned char* __restrict__ mask, const Grid g,
                                  const unsigned char* __restrict__ emask, const int* __restrict__ vscan,
                                  const int* __restrict__ tscan, int* __restrict__ faces) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= g.n) return;
  const int z = (int)(i % g.Z), y = (int)((i / g.Z) % g.Y), x = (int)(i / g.sx);
  if (x + 1 >= g.X || y + 1 >= g.Y || z + 1 >= g.Z) return;
  float v[8];
  load_cell(tsdf, mask, g, i, v);
  unsigned long long nxt;
  unsigned todo = trace_cell(v, nxt);
  long long f = tscan[i];
  while (todo) {
    const int e0 = __ffs(todo) - 1;
    unsigned long long L = 0;
    int n = 0, e = e0;
    do {
      L |= (unsigned long long)e << (4 * n);
      ++n;
      todo &= ~(1u << e);
      e = nib(nxt, e);
    } while (e != e0);
    while (n > 3) {
      int pick = 1;
      for (int s = 1; s <= n; ++s) {
        const int c = s == n ? 0 : s;
        const int pv = nib(L, c == 0 ? n - 1 : c - 1), nx = nib(L, c + 1 == n ? 0 : c + 1);
        if (!(high_faces(pv) & high_faces(nx))) {
          pick = c;
          break;
        }
      }
      const int pv = nib(L, pick == 0 ? n - 1 : pick - 1), nx = nib(L, pick + 1 == n ? 0 : pick + 1);
      faces[f * 3 + 0] = vertex_id(g, i, pv, emask, vscan);
      faces[f * 3 + 1] = vertex_id(g, i, nib(L, pick), emask, vscan);
      faces[f * 3 + 2] = vertex_id(g, i, nx, emask, vscan);
      ++f;
      const unsigned long long low = L & ((1ull << (4 * pick)) - 1ull);
      L = low | ((L >> (4 * (pick + 1))) << (4 * pick));
      --n;
    }
    faces[f * 3 + 0] = vertex_id(g, i, nib(L, 0), emask, vscan);
    faces[f * 3 + 1] = vertex_id(g, i, nib(L, 1), emask, vscan);
    faces[f * 3 + 2] = vertex_id(g, i, nib(L, 2), emask, vscan);
    ++f;
  }
}

Grid make_grid(const int* dims) {
  Grid g;
  g.X = dims[0]; g.Y = dims[1]; g.Z = dims[2];
  g.sy = g.Z;
  g.sx = (long long)g.Y * g.Z;
  g.n = (long long)g.X * g.sx;
  return g;
}

struct MeshWs {
  int* vscan;
  int* tscan;
  unsigned char* emask;
  int* tot;
  int ntiles;
};

inline size_t al256(size_t x) { return (x + 255) & ~(size_t)255; }

MeshWs carve(const Grid& g, void* ws) {
  MeshWs w;
  unsigned char* b = static_cast<unsigned char*>(ws);
  w.ntiles = (int)((g.n + kScanTile - 1) / kScanTile);
  w.vscan = reinterpret_cast<int*>(b);
  b += al256(g.n * sizeof(int));
  w.tscan = reinterpret_cast<int*>(b);
  b += al256(g.n * sizeof(int));
  w.emask = b;
  b += al256(g.n);
  w.tot = reinterpret_cast<int*>(b);
  return w;
}

}  // namespace

size_t mesh_workspace_bytes(const int* dims) {
  const Grid g = make_grid(dims);
  const long long ntiles = (g.n + kScanTile - 1) / kScanTile;
  return 2 * al256(g.n * sizeof(int)) + al256(g.n) + al256(2 * (ntiles + 1) * sizeof(int));
}

void launch_mesh_count(const float* tsdf, const unsigned char* mask, const int* dims, void* ws, cudaStream_t st) {
  const Grid g = make_grid(dims);
  const MeshWs w = carve(g, ws);
  const unsigned blocks = (unsigned)((g.n + 255) / 256);
  mesh_count_kernel<<<blocks, 256, 0, st>>>(tsdf, mask, g, w.emask, w.vscan, w.tscan);
  scan_tiles_kernel<<<dim3(w.ntiles, 2), kScanThreads, 0, st>>>(w.vscan, w.tscan, g.n, w.tot, w.ntiles);
  scan_totals_kernel<<<dim3(1, 2), kTotalsThreads, 0, st>>>(w.tot, w.ntiles);
  scan_add_kernel<<<dim3(w.ntiles, 2), kScanThreads, 0, st>>>(w.vscan, w.tscan, g.n, w.tot, w.ntiles);
}

cudaError_t mesh_read_totals(const int* dims, const void* ws, int* n_verts, int* n_tris, cudaStream_t st) {
  const MeshWs w = carve(make_grid(dims), const_cast<void*>(ws));
  cudaMemcpyAsync(n_verts, w.tot + w.ntiles, sizeof(int), cudaMemcpyDeviceToHost, st);
  cudaMemcpyAsync(n_tris, w.tot + 2 * w.ntiles + 1, sizeof(int), cudaMemcpyDeviceToHost, st);
  return cudaStreamSynchronize(st);
}

void launch_mesh_emit(const float* tsdf, const float* color, const unsigned char* mask, const int* dims, const float* origin,
                      double voxel_size, const void* ws, float* verts, float* normals, unsigned char* colors, int* faces,
                      cudaStream_t st) {
  EmitParams q;
  q.g = make_grid(dims);
  for (int k = 0; k < 3; ++k) q.origin[k] = origin[k];
  q.voxel = (float)voxel_size;
  const MeshWs w = carve(q.g, const_cast<void*>(ws));
  const unsigned blocks = (unsigned)((q.g.n + 255) / 256);
  mesh_verts_kernel<<<blocks, 256, 0, st>>>(q, tsdf, color, mask, w.emask, w.vscan, verts, normals, colors);
  if (faces) mesh_faces_kernel<<<blocks, 256, 0, st>>>(tsdf, mask, q.g, w.emask, w.vscan, w.tscan, faces);
}

}  // namespace srf
