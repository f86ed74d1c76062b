// Object point clouds on the GPU (sm_90a): mask erosion, masked unprojection in row-major order, DBSCAN largest cluster.
//
// Reference: vlfm/mapping/object_point_cloud_map.py
//   _extract_object_cloud :143-163   cv2.erode(mask*255, None, iterations=k) -> valid depth (0 -> 1, metres, float32)
//                                    -> get_point_cloud (vlfm/utils/geometry_utils.py:216-236, np.where order)
//                                    -> get_random_subarray (host: numpy's global RNG, see mapping/object_point_cloud_map.py)
//                                    -> open3d_dbscan_filtering :192-219 (Open3D cluster_dbscan(eps=0.2, min_points=100),
//                                       points of the largest non-noise cluster in input order)
// The spec of every step is oracle/object_map_oracle.py.
//
//  C1 object_erode_count_kernel   one warp per image row: (2k+1)^2 erosion (the image border does not erode: cv2's default
//                                 border value for erosion is +inf) -> eroded byte mask + per-row pixel count
//  C2 object_row_scan_kernel      exclusive scan of the row counts (one block), total -> d_count
//  C3 object_unproject_kernel     one warp per row: points (z, -x, -y) float64 written at row offset + ballot rank
//  D1 dbscan_adjacency_kernel     N x N radius test in float64 (dx^2 + dy^2, + dz^2; <= eps^2) -> bit matrix + neighbour counts
//  D2 dbscan_union_kernel         union-find (atomicMin) over core-core adjacencies: root = lowest core index of the component,
//                                 which is also the order in which Open3D numbers the clusters
//  D3 dbscan_label_kernel         cores take their root; a border point takes the LOWEST root among its core neighbours (the first
//                                 cluster that reaches it); cluster sizes by atomicAdd
//  D4 dbscan_select_kernel        largest cluster (ties: lowest root, like np.argmax over np.unique) -> stable compaction
#include <math.h>

#include "common.cuh"

namespace vlfm {

__global__ void __launch_bounds__(256)
object_erode_count_kernel(const uint8_t* __restrict__ mask, int H, int W, int k, uint8_t* __restrict__ eroded, int* __restrict__ row_count) {
  const int lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
  for (int y = blockIdx.x * wpb + (threadIdx.x >> 5); y < H; y += gridDim.x * wpb) {
    int cnt = 0;
    for (int x0 = 0; x0 < W; x0 += 32) {
      const int x = x0 + lane;
      bool keep = false;
      if (x < W) {
        keep = true;
        for (int dy = -k; dy <= k && keep; ++dy) {
          const int yy = y + dy;
          if ((unsigned)yy >= (unsigned)H) continue;
          for (int dx = -k; dx <= k; ++dx) {
            const int xx = x + dx;
            if ((unsigned)xx >= (unsigned)W) continue;
            if (mask[(size_t)yy * W + xx] == 0) { keep = false; break; }
          }
        }
        eroded[(size_t)y * W + x] = keep ? 255 : 0;
      }
      cnt += __popc(__ballot_sync(0xffffffffu, keep));
    }
    if (lane == 0) row_count[y] = cnt;
  }
}

__global__ void __launch_bounds__(1024) object_row_scan_kernel(const int* __restrict__ row_count, int H, int* __restrict__ row_off, int* __restrict__ total) {
  __shared__ int s[1024];
  __shared__ int carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int base = 0; base < H; base += 1024) {
    const int i = base + threadIdx.x;
    const int v = i < H ? row_count[i] : 0;
    s[threadIdx.x] = v;
    __syncthreads();
    for (int o = 1; o < 1024; o <<= 1) {
      const int t = threadIdx.x >= o ? s[threadIdx.x - o] : 0;
      __syncthreads();
      s[threadIdx.x] += t;
      __syncthreads();
    }
    if (i < H) row_off[i] = carry + s[threadIdx.x] - v;
    __syncthreads();
    if (threadIdx.x == 1023) carry += s[1023];
    __syncthreads();
  }
  if (threadIdx.x == 0) *total = carry;
}

__global__ void __launch_bounds__(256)
object_unproject_kernel(const float* __restrict__ depth, const uint8_t* __restrict__ eroded, int H, int W, float dscale, float doff, double fx,
                        double fy, const int* __restrict__ row_off, double* __restrict__ pts, int cap) {
  const int lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
  for (int y = blockIdx.x * wpb + (threadIdx.x >> 5); y < H; y += gridDim.x * wpb) {
    int off = row_off[y];
    for (int x0 = 0; x0 < W; x0 += 32) {
      const int x = x0 + lane;
      const bool keep = x < W && eroded[(size_t)y * W + x] != 0;
      const unsigned m = __ballot_sync(0xffffffffu, keep);
      if (keep) {
        const int o = off + __popc(m & ((1u << lane) - 1));
        if (o < cap) {
          float d = depth[(size_t)y * W + x];
          if (d == 0.f) d = 1.f;                                      // :157 holes are far
          const float z32 = __fadd_rn(__fmul_rn(d, dscale), doff);     // :158 float32
          const double z = (double)z32;
          const double xc = __ddiv_rn(__dmul_rn((double)(x - W / 2), z), fx);   // geometry_utils.py:230-231 (int64 * float32 -> float64)
          const double yc = __ddiv_rn(__dmul_rn((double)(y - H / 2), z), fy);
          pts[3 * (size_t)o + 0] = z; pts[3 * (size_t)o + 1] = -xc; pts[3 * (size_t)o + 2] = -yc;
        }
      }
      off += __popc(m);
    }
  }
}

// optional gather (the host's np.random.choice indices): dst[i] = src[idx[i]]
__global__ void object_gather_kernel(const double* __restrict__ src, const int* __restrict__ idx, int n, double* __restrict__ dst) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int j = idx[i];
    dst[3 * (size_t)i] = src[3 * (size_t)j]; dst[3 * (size_t)i + 1] = src[3 * (size_t)j + 1]; dst[3 * (size_t)i + 2] = src[3 * (size_t)j + 2];
  }
}

// ---------------------------------------------------------------------------------------------- DBSCAN ----
// one block per point i; threads stride over j; adjacency words built with ballots
__global__ void __launch_bounds__(256)
dbscan_adjacency_kernel(const double* __restrict__ pts, int n, double eps2, uint32_t* __restrict__ adj, int wpr, int* __restrict__ nbr_count) {
  const int i = blockIdx.x;
  if (i >= n) return;
  const double xi = pts[3 * (size_t)i], yi = pts[3 * (size_t)i + 1], zi = pts[3 * (size_t)i + 2];
  __shared__ int s_cnt;
  if (threadIdx.x == 0) s_cnt = 0;
  __syncthreads();
  int cnt = 0;
  for (int j0 = 0; j0 < wpr * 32; j0 += blockDim.x) {
    const int j = j0 + threadIdx.x;
    bool in = false;
    if (j < n) {
      const double dx = xi - pts[3 * (size_t)j], dy = yi - pts[3 * (size_t)j + 1], dz = zi - pts[3 * (size_t)j + 2];
      const double d2 = __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
      in = d2 <= eps2;
    }
    const unsigned m = __ballot_sync(0xffffffffu, in);
    if ((threadIdx.x & 31) == 0 && (j >> 5) < wpr) { adj[(size_t)i * wpr + (j >> 5)] = m; cnt += __popc(m); }
  }
  if ((threadIdx.x & 31) == 0) atomicAdd(&s_cnt, cnt);
  __syncthreads();
  if (threadIdx.x == 0) nbr_count[i] = s_cnt;
}

__device__ __forceinline__ int db_find(int* L, int i) {
  while (true) { const int p = *reinterpret_cast<volatile int*>(&L[i]); if (p == i) return i; i = p; }
}
__device__ __forceinline__ void db_union(int* L, int a, int b) {
  while (true) {
    a = db_find(L, a); b = db_find(L, b);
    if (a == b) return;
    if (a < b) { const int t = a; a = b; b = t; }
    const int old = atomicMin(&L[a], b);
    if (old == a) return;
    a = old;
  }
}
__global__ void dbscan_init_kernel(const int* __restrict__ nbr_count, int n, int min_points, int* __restrict__ root, int* __restrict__ size) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    root[i] = nbr_count[i] >= min_points ? i : -1;       // cores are their own root; -1 = not core
    size[i] = 0;
  }
}
// one warp per core point i: union with every core neighbour j < i
__global__ void __launch_bounds__(256)
dbscan_union_kernel(const uint32_t* __restrict__ adj, int wpr, int n, int* __restrict__ root) {
  const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (i >= n || root[i] < 0) return;
  for (int w = lane; w * 32 < i; w += 32) {
    uint32_t m = adj[(size_t)i * wpr + w];
    while (m) {
      const int j = w * 32 + __ffs(m) - 1;
      m &= m - 1;
      if (j < i && *reinterpret_cast<volatile int*>(&root[j]) >= 0) db_union(root, i, j);
    }
  }
}
__global__ void dbscan_flatten_kernel(int n, int* __restrict__ root) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    if (root[i] >= 0) root[i] = db_find(root, i);
}
// label[i]: cluster root (lowest core index of the cluster) or -1 (noise)
__global__ void __launch_bounds__(256)
dbscan_label_kernel(const uint32_t* __restrict__ adj, int wpr, int n, const int* __restrict__ root, int* __restrict__ label, int* __restrict__ size) {
  const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (i >= n) return;
  int best = 0x7fffffff;
  if (root[i] >= 0) best = root[i];
  else {
    for (int w = lane; w < wpr; w += 32) {
      uint32_t m = adj[(size_t)i * wpr + w];
      while (m) {
        const int j = w * 32 + __ffs(m) - 1;
        m &= m - 1;
        const int r = j < n ? root[j] : -1;
        if (r >= 0 && r < best) best = r;
      }
    }
    for (int o = 16; o; o >>= 1) best = min(best, __shfl_xor_sync(0xffffffffu, best, o));
  }
  if (lane == 0) {
    const int l = best == 0x7fffffff ? -1 : best;
    label[i] = l;
    if (l >= 0) atomicAdd(&size[l], 1);
  }
}
// one block: largest cluster (first maximum in ascending root order), then a stable compaction of its points
__global__ void __launch_bounds__(1024)
dbscan_select_kernel(const double* __restrict__ pts, const int* __restrict__ label, const int* __restrict__ size, int n, double* __restrict__ out,
                     int* __restrict__ out_count) {
  __shared__ unsigned long long s_best;      // (size << 32) | (0xffffffff - root): max picks the largest size, then the lowest root
  __shared__ int s_scan[1024];
  __shared__ int s_carry;
  if (threadIdx.x == 0) { s_best = 0ull; s_carry = 0; }
  __syncthreads();
  unsigned long long b = 0ull;
  for (int i = threadIdx.x; i < n; i += 1024) {
    const int sz = size[i];
    if (sz > 0) { const unsigned long long v = ((unsigned long long)(unsigned)sz << 32) | (unsigned long long)(0xffffffffu - (unsigned)i); if (v > b) b = v; }
  }
  atomicMax(&s_best, b);
  __syncthreads();
  if (s_best == 0ull) { if (threadIdx.x == 0) *out_count = 0; return; }
  const int best = (int)(0xffffffffu - (unsigned)(s_best & 0xffffffffull));
  for (int base = 0; base < n; base += 1024) {
    const int i = base + threadIdx.x;
    const int v = (i < n && label[i] == best) ? 1 : 0;
    s_scan[threadIdx.x] = v;
    __syncthreads();
    for (int o = 1; o < 1024; o <<= 1) {
      const int t = threadIdx.x >= o ? s_scan[threadIdx.x - o] : 0;
      __syncthreads();
      s_scan[threadIdx.x] += t;
      __syncthreads();
    }
    if (v) {
      const int o = s_carry + s_scan[threadIdx.x] - 1;
      out[3 * (size_t)o] = pts[3 * (size_t)i]; out[3 * (size_t)o + 1] = pts[3 * (size_t)i + 1]; out[3 * (size_t)o + 2] = pts[3 * (size_t)i + 2];
    }
    __syncthreads();
    if (threadIdx.x == 1023) s_carry += s_scan[1023];
    __syncthreads();
  }
  if (threadIdx.x == 0) *out_count = s_carry;
}

}  // namespace vlfm

using namespace vlfm;

// Replaces ObjectPointCloudMap._extract_object_cloud up to (not including) the random subsample
// (vlfm/mapping/object_point_cloud_map.py:153-159): d_points [cap,3] float64 in np.where order, *d_count = number of points
// (may exceed cap: the caller checks).  d_scratch: H*W bytes + 2*H ints.
extern "C" int vlfm_object_cloud_extract(const float* d_depth, const uint8_t* d_mask, int H, int W, int erosion_iterations, float depth_scale,
                                         float depth_offset, double fx, double fy, double* d_points, int cap, int32_t* d_count,
                                         void* d_scratch, size_t scratch_bytes, void* stream) {
  const size_t need = (((size_t)H * W + 255) & ~(size_t)255) + (size_t)2 * H * 4 + 256;
  if (!d_depth || !d_mask || !d_points || !d_count || !d_scratch || H < 1 || W < 1 || erosion_iterations < 0 || erosion_iterations > 16 ||
      cap < 1 || scratch_bytes < need) { set_error("vlfm_object_cloud_extract: bad argument (scratch %zu < %zu)", scratch_bytes, need); return VLFM_E_INVALID; }
  cudaStream_t st = (cudaStream_t)stream;
  uint8_t* eroded = (uint8_t*)d_scratch;
  int* row_count = (int*)(eroded + (((size_t)H * W + 255) & ~(size_t)255));
  int* row_off = row_count + H;
  const int blocks = (H + 7) / 8;
  object_erode_count_kernel<<<blocks, 256, 0, st>>>(d_mask, H, W, erosion_iterations, eroded, row_count);
  object_row_scan_kernel<<<1, 1024, 0, st>>>(row_count, H, row_off, d_count);
  object_unproject_kernel<<<blocks, 256, 0, st>>>(d_depth, eroded, H, W, depth_scale, depth_offset, fx, fy, row_off, d_points, cap);
  VLFM_CHECK_LAUNCH("vlfm_object_cloud_extract");
  count_launch(3);
  return VLFM_OK;
}

extern "C" int vlfm_dbscan_workspace_bytes(int n, size_t* bytes) {
  if (!bytes || n < 0) { set_error("vlfm_dbscan_workspace_bytes: bad argument"); return VLFM_E_INVALID; }
  const size_t wpr = ((size_t)n + 31) / 32;
  *bytes = (size_t)n * wpr * 4 + (size_t)4 * n * 4 + 1024;
  return VLFM_OK;
}

// Replaces open3d_dbscan_filtering (vlfm/mapping/object_point_cloud_map.py:192-219): d_out [<= n, 3] = points of the largest
// DBSCAN cluster in input order, *d_out_count = its size (0: only noise).  d_gather (optional, int32[n]): the points are
// d_points[d_gather[i]] (the host's random subsample) instead of d_points[i].
extern "C" int vlfm_dbscan_largest_cluster(const double* d_points, const int32_t* d_gather, int n, double eps, int min_points, double* d_gathered,
                                           double* d_out, int32_t* d_out_count, void* d_workspace, size_t workspace_bytes, void* stream) {
  size_t need = 0;
  vlfm_dbscan_workspace_bytes(n, &need);
  if (!d_points || !d_out || !d_out_count || !d_workspace || n < 1 || n > 65535 || min_points < 1 || workspace_bytes < need || (d_gather && !d_gathered)) {
    set_error("vlfm_dbscan_largest_cluster: bad argument (1 <= n <= 65535; workspace %zu < %zu)", workspace_bytes, need); return VLFM_E_INVALID; }
  cudaStream_t st = (cudaStream_t)stream;
  const int wpr = (n + 31) / 32;
  uint32_t* adj = (uint32_t*)d_workspace;
  int* nbr = (int*)(adj + (size_t)n * wpr);
  int* root = nbr + n;
  int* label = root + n;
  int* size = label + n;
  const double* pts = d_points;
  const int nb = (n + 255) / 256;
  if (d_gather) { object_gather_kernel<<<nb, 256, 0, st>>>(d_points, d_gather, n, d_gathered); pts = d_gathered; }
  dbscan_adjacency_kernel<<<n, 256, 0, st>>>(pts, n, eps * eps, adj, wpr, nbr);
  dbscan_init_kernel<<<nb, 256, 0, st>>>(nbr, n, min_points, root, size);
  dbscan_union_kernel<<<(n + 7) / 8, 256, 0, st>>>(adj, wpr, n, root);
  dbscan_flatten_kernel<<<nb, 256, 0, st>>>(n, root);
  dbscan_label_kernel<<<(n + 7) / 8, 256, 0, st>>>(adj, wpr, n, root, label, size);
  dbscan_select_kernel<<<1, 1024, 0, st>>>(pts, label, size, n, d_out, d_out_count);
  VLFM_CHECK_LAUNCH("vlfm_dbscan_largest_cluster");
  count_launch(d_gather ? 7 : 6);
  return VLFM_OK;
}
