// Triangle-mesh closest-hit tracing for stage II (replaces the third-party `raytracing.RayTracer` the reference calls at
// network/renderer.py:676,720): a host-side BVH build (init time, once per mesh) and a one-thread-per-ray stack traversal.
//
// Layout: nodes are 32-byte records in depth-first order (left child = index + 1) so a node is two 16-byte loads;
// triangles are stored re-ordered by leaf as (v0, e1, e2) float4 triples, the form Moeller-Trumbore consumes.
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstdint>
#include <vector>

#include "bvh_traverse.cuh"
#include "common.cuh"

namespace nero {

struct BvhNode {      // 32 B
  float lo[3];
  int a;              // inner: index of the right child;  leaf: first triangle
  float hi[3];
  int count;          // 0 = inner node, >0 = leaf with `count` triangles
};

namespace {
struct BuildTri { float c[3]; float lo[3]; float hi[3]; int id; };

struct Builder {
  std::vector<BuildTri>& t;
  std::vector<BvhNode>& nodes;
  int leaf_size;
  int build(int first, int last, int depth = 0) {   // [first, last)
    const int me = int(nodes.size());
    nodes.emplace_back();
    float lo[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, hi[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
    float clo[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, chi[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
    for (int i = first; i < last; ++i)
      for (int k = 0; k < 3; ++k) {
        lo[k] = std::min(lo[k], t[i].lo[k]); hi[k] = std::max(hi[k], t[i].hi[k]);
        clo[k] = std::min(clo[k], t[i].c[k]); chi[k] = std::max(chi[k], t[i].c[k]);
      }
    for (int k = 0; k < 3; ++k) { nodes[me].lo[k] = lo[k]; nodes[me].hi[k] = hi[k]; }
    const int n = last - first;
    int axis = 0;
    for (int k = 1; k < 3; ++k) if (chi[k] - clo[k] > chi[axis] - clo[axis]) axis = k;
    if (n <= leaf_size || !(chi[axis] > clo[axis])) {
      nodes[me].a = first; nodes[me].count = n;
      return me;
    }
    // binned surface-area heuristic along the widest centroid axis, median fallback
    const int NB = 16;
    int cnt[NB] = {0};
    float blo[NB][3], bhi[NB][3];
    for (int b = 0; b < NB; ++b) for (int k = 0; k < 3; ++k) { blo[b][k] = FLT_MAX; bhi[b][k] = -FLT_MAX; }
    const float scale = NB / (chi[axis] - clo[axis]);
    auto bin_of = [&](const BuildTri& x) { return std::min(NB - 1, std::max(0, int((x.c[axis] - clo[axis]) * scale))); };
    for (int i = first; i < last; ++i) {
      const int b = bin_of(t[i]);
      cnt[b]++;
      for (int k = 0; k < 3; ++k) { blo[b][k] = std::min(blo[b][k], t[i].lo[k]); bhi[b][k] = std::max(bhi[b][k], t[i].hi[k]); }
    }
    auto area = [](const float* l, const float* h) {
      const float dx = h[0] - l[0], dy = h[1] - l[1], dz = h[2] - l[2];
      return (dx < 0 || dy < 0 || dz < 0) ? 0.f : 2.f * (dx * dy + dy * dz + dz * dx);
    };
    float la[NB], ra[NB];
    int lc[NB], rc[NB];
    {
      float l[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, h[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
      int c = 0;
      for (int b = 0; b < NB; ++b) {
        for (int k = 0; k < 3; ++k) { l[k] = std::min(l[k], blo[b][k]); h[k] = std::max(h[k], bhi[b][k]); }
        c += cnt[b]; lc[b] = c; la[b] = area(l, h);
      }
      float l2[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, h2[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
      c = 0;
      for (int b = NB - 1; b >= 0; --b) {
        for (int k = 0; k < 3; ++k) { l2[k] = std::min(l2[k], blo[b][k]); h2[k] = std::max(h2[k], bhi[b][k]); }
        c += cnt[b]; rc[b] = c; ra[b] = area(l2, h2);
      }
    }
    int best = -1;
    float best_cost = FLT_MAX;
    for (int b = 0; b + 1 < NB; ++b) {
      if (lc[b] == 0 || rc[b + 1] == 0) continue;
      const float cost = la[b] * lc[b] + ra[b + 1] * rc[b + 1];
      if (cost < best_cost) { best_cost = cost; best = b; }
    }
    int mid;
    if (best >= 0 && depth < 28) {   // beyond that depth only balanced splits: bounds the traversal stack
      mid = int(std::partition(t.begin() + first, t.begin() + last, [&](const BuildTri& x) { return bin_of(x) <= best; }) - t.begin());
    } else {
      mid = first + n / 2;
      std::nth_element(t.begin() + first, t.begin() + mid, t.begin() + last,
                       [&](const BuildTri& x, const BuildTri& y) { return x.c[axis] < y.c[axis]; });
    }
    if (mid == first || mid == last) mid = first + n / 2;
    nodes[me].count = 0;
    build(first, mid, depth + 1);
    const int right = build(mid, last, depth + 1);
    nodes[me].a = right;
    return me;
  }
};
}  // namespace

// Host build.  verts [V,3] fp32, tris [T,3] int32 (host memory).  Outputs (host memory, caller-allocated):
//   nodes_out  [2T] x 32 B, tri_out [T] x 3 float4 (v0, e1, e2; w unused), tri_id_out [T] original triangle index.
extern "C" int nero_bvh_build_host(const float* verts, int V, const int* tris, int T, void* nodes_out, float* tri_out, int* tri_id_out,
                                   int* n_nodes) {
  if (!verts || !tris || !nodes_out || !tri_out || !tri_id_out || !n_nodes) return NERO_ERR_ARG;
  if (T <= 0 || V <= 0) return NERO_ERR_ARG;
  std::vector<BuildTri> t(T);
  for (int i = 0; i < T; ++i) {
    for (int k = 0; k < 3; ++k) {
      if (tris[i * 3 + k] < 0 || tris[i * 3 + k] >= V) return NERO_ERR_ARG;
    }
    const float* a = verts + 3 * tris[i * 3], *b = verts + 3 * tris[i * 3 + 1], *c = verts + 3 * tris[i * 3 + 2];
    for (int k = 0; k < 3; ++k) {
      t[i].lo[k] = std::min(a[k], std::min(b[k], c[k]));
      t[i].hi[k] = std::max(a[k], std::max(b[k], c[k]));
      t[i].c[k] = (a[k] + b[k] + c[k]) * (1.0f / 3.0f);
    }
    t[i].id = i;
  }
  std::vector<BvhNode> nodes;
  nodes.reserve(2 * size_t(T));
  Builder bl{t, nodes, 4};
  bl.build(0, T);
  std::copy(nodes.begin(), nodes.end(), static_cast<BvhNode*>(nodes_out));
  *n_nodes = int(nodes.size());
  for (int i = 0; i < T; ++i) {
    const int id = t[i].id;
    const float* a = verts + 3 * tris[id * 3], *b = verts + 3 * tris[id * 3 + 1], *c = verts + 3 * tris[id * 3 + 2];
    float* o = tri_out + size_t(i) * 12;
    for (int k = 0; k < 3; ++k) { o[k] = a[k]; o[4 + k] = b[k] - a[k]; o[8 + k] = c[k] - a[k]; }
    o[3] = o[7] = o[11] = 0.f;
    tri_id_out[i] = id;
  }
  return NERO_OK;
}

struct TraceParams {
  const BvhNode* nodes; const float4* tris; int n_rays;
  const float* org; int ldo; const float* dir; int ldd;
  float4* pos_depth;   // (hit position, depth); depth = miss_depth when nothing is hit
  float4* nrm_hit;     // (normal, hit flag 0/1); flip_normalize: -normalize(face normal) as renderer.py:722-723
  float miss_depth; int flip;
};

__global__ void bvh_trace_kernel(const TraceParams q) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= q.n_rays) return;
  const float ox = q.org[size_t(i) * q.ldo], oy = q.org[size_t(i) * q.ldo + 1], oz = q.org[size_t(i) * q.ldo + 2];
  const float dx = q.dir[size_t(i) * q.ldd], dy = q.dir[size_t(i) * q.ldd + 1], dz = q.dir[size_t(i) * q.ldd + 2];
  const BvhHit h = bvh_traverse<false>(reinterpret_cast<const float4*>(q.nodes), q.tris, ox, oy, oz, dx, dy, dz, q.miss_depth);
  const float best = h.t;
  const int best_tri = h.tri;
  float nx = 0.f, ny = 0.f, nz = 0.f;
  if (best_tri >= 0) {
    const float4 e1 = __ldg(q.tris + 3 * best_tri + 1), e2 = __ldg(q.tris + 3 * best_tri + 2);
    nx = e1.y * e2.z - e1.z * e2.y; ny = e1.z * e2.x - e1.x * e2.z; nz = e1.x * e2.y - e1.y * e2.x;
    const float inv = (q.flip ? -1.0f : 1.0f) / fmaxf(sqrtf(nx * nx + ny * ny + nz * nz), 1e-12f);
    nx *= inv; ny *= inv; nz *= inv;
  }
  q.pos_depth[i] = make_float4(ox + best * dx, oy + best * dy, oz + best * dz, best);
  q.nrm_hit[i] = make_float4(nx, ny, nz, best_tri >= 0 ? 1.0f : 0.0f);
}

extern "C" int nero_bvh_trace(const void* nodes, const float* tris, int n_rays, const float* org, int ldo, const float* dir, int ldd,
                              float* pos_depth, float* nrm_hit, float miss_depth, int flip, void* stream) {
  if (!nodes || !tris || (n_rays > 0 && (!org || !dir || !pos_depth || !nrm_hit))) return NERO_ERR_ARG;
  if (n_rays <= 0) return NERO_OK;
  const TraceParams q{reinterpret_cast<const BvhNode*>(nodes), reinterpret_cast<const float4*>(tris), n_rays, org, ldo, dir, ldd,
                      reinterpret_cast<float4*>(pos_depth), reinterpret_cast<float4*>(nrm_hit), miss_depth, flip};
  bvh_trace_kernel<<<(n_rays + 127) / 128, 128, 0, (cudaStream_t)stream>>>(q);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

}  // namespace nero
