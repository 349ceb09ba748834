// UV atlas unwrapping on the host: the replacement of the reference's xatlas call (extract_materials_texture_map.py:75-82).
// Init-time host code of the library, like nero_bvh_build_host; it runs without a GPU.  Its charts and layout are its
// own, not xatlas's (DESIGN.md section 2).
//
// Charts.  Two triangles are neighbours iff they share an edge used by exactly those two triangles, in opposite directions.
// Seeds are taken in ascending triangle order and grow breadth-first (edges in vertex order).  A neighbour joins when its
// unit normal lies within 60 degrees of the seed's and its orthographic projection onto the plane normal to the seed
// overlaps no triangle already in the chart.  Projections are snapped to integers below 2^29 so the orientation tests are
// exact in int64; a per-chart grid finds the candidates.  Charts are therefore injective by construction.  Zero-area and
// non-manifold triangles end up in charts of their own (a zero normal is outside every cone).
//
// Layout.  Each chart is turned to the principal axes of its vertices and shelf-packed by decreasing rectangle height
// (ties: chart index) at one texel density for all charts, with `gutter` texels between charts and from the border.  The
// density is the largest that fits, found by bisection.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <unordered_map>
#include <vector>

#include "common.cuh"
#include "../../include/nero_texmap.h"

namespace nero {

namespace {

struct P2 {
  long long x, y;
};

inline long long orient(const P2& a, const P2& b, const P2& c) {
  return (b.x - a.x) * (c.y - a.y) - (b.y - a.y) * (c.x - a.x);
}

// interiors of two positively oriented triangles are disjoint iff an edge line of one weakly separates the other
bool overlap(const P2* a, const P2* b) {
  for (int pass = 0; pass < 2; ++pass) {
    const P2* p = pass ? b : a;
    const P2* q = pass ? a : b;
    for (int e = 0; e < 3; ++e) {
      const P2& u = p[e];
      const P2& v = p[(e + 1) % 3];
      if (orient(u, v, q[0]) <= 0 && orient(u, v, q[1]) <= 0 && orient(u, v, q[2]) <= 0) return false;
    }
  }
  return true;
}

struct Chart {
  std::vector<int> tris;    // in the order they joined
  double w = 0, h = 0;      // rectangle in world units after the rotation
};

struct Unwrapper {
  const float* verts;
  const int* tris;
  int V, T;
  std::vector<int> adj;            // [3T] neighbour across edge (v_e, v_e+1) or -1
  std::vector<double> nrm;         // [3T] unit normals, zero for zero-area triangles
  std::vector<P2> proj;            // [3T] projected, snapped vertices of each triangle in its chart's frame
  std::vector<int> chart_of;
  std::vector<Chart> charts;
  double scale = 1.0;              // world -> snapped projection units
  double cell = 1.0;               // grid cell in snapped units

  void adjacency() {
    struct E {
      long long key;
      int t, e, fwd;
    };
    std::vector<E> es;
    es.reserve(3 * size_t(T));
    for (int t = 0; t < T; ++t)
      for (int e = 0; e < 3; ++e) {
        const int a = tris[3 * t + e], b = tris[3 * t + (e + 1) % 3];
        if (a == b) continue;
        es.push_back({(long long)std::min(a, b) * V + std::max(a, b), t, e, a < b ? 1 : 0});
      }
    std::sort(es.begin(), es.end(), [](const E& p, const E& q) {
      return p.key != q.key ? p.key < q.key : (p.t != q.t ? p.t < q.t : p.e < q.e);
    });
    adj.assign(3 * size_t(T), -1);
    for (size_t i = 0; i < es.size();) {
      size_t j = i;
      while (j < es.size() && es[j].key == es[i].key) ++j;
      if (j - i == 2 && es[i].fwd != es[i + 1].fwd && es[i].t != es[i + 1].t) {
        adj[3 * size_t(es[i].t) + es[i].e] = es[i + 1].t;
        adj[3 * size_t(es[i + 1].t) + es[i + 1].e] = es[i].t;
      }
      i = j;
    }
  }

  void normals() {
    nrm.assign(3 * size_t(T), 0.0);
    double rmax = 0.0, elen = 0.0;
    for (int t = 0; t < T; ++t) {
      const float* p[3];
      for (int k = 0; k < 3; ++k) p[k] = verts + 3 * size_t(tris[3 * t + k]);
      double e1[3], e2[3];
      for (int k = 0; k < 3; ++k) {
        e1[k] = double(p[1][k]) - p[0][k];
        e2[k] = double(p[2][k]) - p[0][k];
        for (int m = 0; m < 3; ++m) rmax = std::max(rmax, std::fabs(double(p[m][k])));
      }
      elen += std::sqrt(e1[0] * e1[0] + e1[1] * e1[1] + e1[2] * e1[2]);
      const double n[3] = {e1[1] * e2[2] - e1[2] * e2[1], e1[2] * e2[0] - e1[0] * e2[2], e1[0] * e2[1] - e1[1] * e2[0]};
      const double l = std::sqrt(n[0] * n[0] + n[1] * n[1] + n[2] * n[2]);
      if (l > 0.0 && std::isfinite(l))
        for (int k = 0; k < 3; ++k) nrm[3 * size_t(t) + k] = n[k] / l;
    }
    // |projection| <= |p| <= sqrt(3) max|coordinate|: snapped values stay below 2^29, products of differences below 2^61
    scale = rmax > 0.0 ? std::ldexp(1.0, 29) / (std::sqrt(3.0) * rmax * (1.0 + 1e-9)) : 1.0;
    cell = std::max(1.0, 2.0 * elen / std::max(T, 1) * scale);
  }

  static void frame(const double* n, double* u, double* v) {
    const double a[3] = {std::fabs(n[0]) < 0.9 ? 1.0 : 0.0, std::fabs(n[0]) < 0.9 ? 0.0 : 1.0, 0.0};
    double c[3] = {n[1] * a[2] - n[2] * a[1], n[2] * a[0] - n[0] * a[2], n[0] * a[1] - n[1] * a[0]};
    const double l = std::sqrt(c[0] * c[0] + c[1] * c[1] + c[2] * c[2]);
    for (int k = 0; k < 3; ++k) u[k] = c[k] / l;
    v[0] = n[1] * u[2] - n[2] * u[1];
    v[1] = n[2] * u[0] - n[0] * u[2];
    v[2] = n[0] * u[1] - n[1] * u[0];
  }

  void project(int t, const double* u, const double* v, P2* out) const {
    for (int k = 0; k < 3; ++k) {
      const float* p = verts + 3 * size_t(tris[3 * t + k]);
      out[k].x = std::llround((double(p[0]) * u[0] + double(p[1]) * u[1] + double(p[2]) * u[2]) * scale);
      out[k].y = std::llround((double(p[0]) * v[0] + double(p[1]) * v[1] + double(p[2]) * v[2]) * scale);
    }
  }

  void grow() {
    const double cos_cone = 0.5;   // 60 degrees
    chart_of.assign(T, -1);
    proj.resize(3 * size_t(T));
    std::unordered_map<uint64_t, std::vector<int>> grid;
    std::vector<int> big, stamp(T, -1);
    std::vector<int> queue;
    int visit = 0;
    auto box = [&](const P2* p, long long* b) {
      b[0] = (long long)std::floor(std::min(p[0].x, std::min(p[1].x, p[2].x)) / cell);
      b[1] = (long long)std::floor(std::min(p[0].y, std::min(p[1].y, p[2].y)) / cell);
      b[2] = (long long)std::floor(std::max(p[0].x, std::max(p[1].x, p[2].x)) / cell);
      b[3] = (long long)std::floor(std::max(p[0].y, std::max(p[1].y, p[2].y)) / cell);
    };
    auto key = [](long long cx, long long cy) { return (uint64_t(uint32_t(cx)) << 32) | uint64_t(uint32_t(cy)); };
    auto insert = [&](int t) {
      long long b[4];
      box(&proj[3 * size_t(t)], b);
      if ((b[2] - b[0] + 1) * (b[3] - b[1] + 1) > 4096) {
        big.push_back(t);
        return;
      }
      for (long long cy = b[1]; cy <= b[3]; ++cy)
        for (long long cx = b[0]; cx <= b[2]; ++cx) grid[key(cx, cy)].push_back(t);
    };
    auto clashes = [&](const P2* p) {
      ++visit;
      for (int o : big)
        if (overlap(p, &proj[3 * size_t(o)])) return true;
      long long b[4];
      box(p, b);
      if ((b[2] - b[0] + 1) * (b[3] - b[1] + 1) > 4096) {   // a large candidate: test the whole chart
        for (const auto& kv : grid)
          for (int o : kv.second)
            if (stamp[o] != visit && (stamp[o] = visit, overlap(p, &proj[3 * size_t(o)]))) return true;
        return false;
      }
      for (long long cy = b[1]; cy <= b[3]; ++cy)
        for (long long cx = b[0]; cx <= b[2]; ++cx) {
          const auto it = grid.find(key(cx, cy));
          if (it == grid.end()) continue;
          for (int o : it->second)
            if (stamp[o] != visit && (stamp[o] = visit, overlap(p, &proj[3 * size_t(o)]))) return true;
        }
      return false;
    };
    for (int seed = 0; seed < T; ++seed) {
      if (chart_of[seed] >= 0) continue;
      const int c = int(charts.size());
      charts.emplace_back();
      Chart& ch = charts.back();
      grid.clear();
      big.clear();
      const double* ns = &nrm[3 * size_t(seed)];
      const bool flat = ns[0] == 0.0 && ns[1] == 0.0 && ns[2] == 0.0;
      const double zn[3] = {0.0, 0.0, 1.0};
      double u[3], v[3];
      frame(flat ? zn : ns, u, v);
      project(seed, u, v, &proj[3 * size_t(seed)]);
      chart_of[seed] = c;
      ch.tris.push_back(seed);
      if (flat) continue;
      insert(seed);
      queue.assign(1, seed);
      for (size_t qi = 0; qi < queue.size(); ++qi) {
        const int t = queue[qi];
        for (int e = 0; e < 3; ++e) {
          const int nb = adj[3 * size_t(t) + e];
          if (nb < 0 || chart_of[nb] >= 0) continue;
          const double* nn = &nrm[3 * size_t(nb)];
          if (nn[0] * ns[0] + nn[1] * ns[1] + nn[2] * ns[2] < cos_cone) continue;
          P2 p[3];
          project(nb, u, v, p);
          if (orient(p[0], p[1], p[2]) <= 0 || clashes(p)) continue;
          std::copy(p, p + 3, &proj[3 * size_t(nb)]);
          chart_of[nb] = c;
          ch.tris.push_back(nb);
          insert(nb);
          queue.push_back(nb);
        }
      }
    }
  }
};

}  // namespace

extern "C" int nero_uv_atlas_host(const float* verts, int V, const int* tris, int T, int width, int height, int gutter, float* vt_out,
                                  int* ft_out, int* n_uv, int* n_charts) {
  if (!verts || !tris || !vt_out || !ft_out || !n_uv || !n_charts || V <= 0 || T <= 0) return NERO_ERR_ARG;
  if (width < 1 || height < 1 || gutter < 0 || 2 * gutter >= std::min(width, height)) return NERO_ERR_ARG;
  for (long long i = 0; i < 3LL * T; ++i)
    if (tris[i] < 0 || tris[i] >= V) return NERO_ERR_ARG;
  for (long long i = 0; i < 3LL * V; ++i)
    if (!std::isfinite(verts[i])) return NERO_ERR_ARG;
  Unwrapper U{verts, tris, V, T};
  U.adjacency();
  U.normals();
  U.grow();
  const int C = int(U.charts.size());
  // chart-local coordinates (world units) turned to the principal axes of the chart's vertices, shifted to start at 0
  std::vector<int> uv_of(V, -1), uv_stamp(V, -1);
  std::vector<double> lx, ly;               // per uv vertex
  std::vector<int> uv_chart;
  for (int c = 0; c < C; ++c) {
    const Chart& ch = U.charts[c];
    const size_t first = lx.size();
    for (int t : ch.tris)
      for (int k = 0; k < 3; ++k) {
        const int vi = tris[3 * t + k];
        if (uv_stamp[vi] != c) {
          uv_stamp[vi] = c;
          uv_of[vi] = int(lx.size());
          lx.push_back(double(U.proj[3 * size_t(t) + k].x) / U.scale);
          ly.push_back(double(U.proj[3 * size_t(t) + k].y) / U.scale);
          uv_chart.push_back(c);
        }
        ft_out[3 * size_t(t) + k] = uv_of[vi];
      }
    const size_t n = lx.size() - first;
    double mx = 0, my = 0;
    for (size_t i = first; i < lx.size(); ++i) mx += lx[i], my += ly[i];
    mx /= double(n), my /= double(n);
    double cxx = 0, cyy = 0, cxy = 0;
    for (size_t i = first; i < lx.size(); ++i) {
      const double dx = lx[i] - mx, dy = ly[i] - my;
      cxx += dx * dx, cyy += dy * dy, cxy += dx * dy;
    }
    const double th = 0.5 * std::atan2(2.0 * cxy, cxx - cyy), co = std::cos(th), si = std::sin(th);
    double x0 = INFINITY, y0 = INFINITY, x1 = -INFINITY, y1 = -INFINITY;
    for (size_t i = first; i < lx.size(); ++i) {
      const double dx = lx[i] - mx, dy = ly[i] - my;
      lx[i] = co * dx + si * dy;
      ly[i] = -si * dx + co * dy;
      x0 = std::min(x0, lx[i]), x1 = std::max(x1, lx[i]), y0 = std::min(y0, ly[i]), y1 = std::max(y1, ly[i]);
    }
    for (size_t i = first; i < lx.size(); ++i) lx[i] -= x0, ly[i] -= y0;
    U.charts[c].w = x1 - x0;
    U.charts[c].h = y1 - y0;
  }
  std::vector<int> order(C);
  for (int c = 0; c < C; ++c) order[c] = c;
  std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return U.charts[a].h > U.charts[b].h; });
  // shelf packing at density s (texels per world unit); positions are whole texels
  std::vector<double> px(C), py(C);
  const double g = gutter;
  auto pack = [&](double s) {
    double x = g, y = g, shelf = 0.0;
    for (int c : order) {
      const double w = s * U.charts[c].w, h = s * U.charts[c].h;
      if (x + w > width - g && x > g) {
        y = std::ceil(y + shelf) + g;
        x = g;
        shelf = 0.0;
      }
      if (x + w > width - g || y + h > height - g) return false;
      px[c] = x, py[c] = y;
      shelf = std::max(shelf, h);
      x = std::ceil(x + w) + g;
    }
    return true;
  };
  double area = 0.0;
  for (const Chart& ch : U.charts) area += ch.w * ch.h;
  double lo = 0.0, hi = area > 0.0 ? std::sqrt(double(width) * height / area) : 1.0;
  if (!pack(lo)) return NERO_ERR_ARG;   // more charts than the atlas holds
  for (int it = 0; it < 64 && pack(hi); ++it) hi *= 2.0;   // long thin charts: the area bound need not be an upper bound
  for (int it = 0; it < 60; ++it) {
    const double mid = 0.5 * (lo + hi);
    (pack(mid) ? lo : hi) = mid;
  }
  pack(lo);
  for (size_t i = 0; i < lx.size(); ++i) {
    const int c = uv_chart[i];
    vt_out[2 * i] = float((px[c] + lo * lx[i]) / width);
    vt_out[2 * i + 1] = float((py[c] + lo * ly[i]) / height);
  }
  *n_uv = int(lx.size());
  *n_charts = C;
  return NERO_OK;
}

}  // namespace nero
