// Mesh simplification of ConvertToBinary (source/mesh_stream/ConvertToBinary.cpp:186-203): quadric-error edge contraction
// after Garland & Heckbert as source/render/MeshSimplifier.cpp runs it — sweeps over the face list in order, contracting
// every edge whose cost is under a percentile threshold, with immediate in-place updates of the neighbourhood.  Each
// contraction reads the state the previous one left (vertex positions, quadrics, face costs, touched / deleted flags), so
// the reference's result is defined by that sequential order and the stage is host code here exactly as it is there
// (kThreads = 1 in the reference's call); the GPU delivers the mesh it starts from (derp_mesh.cuh) in double precision.
//
// What this version does NOT repeat of the reference's work (same result, tests/test_mesh.py against the reference's own code
// on 100+ meshes): attempts that are known to fail again, and the per-sweep passes of sweeps that cannot contract anything
// — see run() and the `failed` / `stamped` members.
//
// Arithmetic conventions (they decide threshold comparisons, hence the output): IEEE double, no FMA contraction,
// 3-term sums left to right, cross product and 3 x 3 determinant in the textbook cofactor order Eigen's fixed-size
// kernels use.  Checked against the reference's own MeshSimplifier.cpp compiled into oracle/_ref (tests/test_mesh.py).
#pragma once

#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <limits>
#include <map>
#include <set>
#include <vector>

namespace derp {
namespace simplify {

struct V3 {
  double x, y, z;
};
inline V3 sub(const V3& a, const V3& b) { return V3{a.x - b.x, a.y - b.y, a.z - b.z}; }
inline double dot(const V3& a, const V3& b) { return (a.x * b.x + a.y * b.y) + a.z * b.z; }
inline V3 cross(const V3& a, const V3& b) { return V3{a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; }
inline V3 unit(const V3& a) {
  const double n = std::sqrt(dot(a, a));
  return n > 0 ? V3{a.x / n, a.y / n, a.z / n} : a;
}

struct Quadric {  // symmetric 4 x 4, stored in full like the reference's Matrix4d (sums are element-wise either way)
  double m[4][4];
};
inline void addInto(Quadric& a, const Quadric& b) {
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) a.m[i][j] = a.m[i][j] + b.m[i][j];
}
inline double det3(const double a[3][3]) {
  auto term = [&](int i, int j, int k) { return a[0][i] * (a[1][j] * a[2][k] - a[1][k] * a[2][j]); };
  return term(0, 1, 2) - term(1, 0, 2) + term(2, 0, 1);
}
// v^T Q v for homogeneous v = (x, y, z, 1), symmetric Q (MeshSimplifier.cpp computeFastError: same term order)
inline double quadricError(const Quadric& q, const V3& v) {
  return q.m[0][0] * v.x * v.x + 2 * q.m[0][1] * v.x * v.y + 2 * q.m[0][2] * v.x * v.z + 2 * q.m[0][3] * v.x +
      q.m[1][1] * v.y * v.y + 2 * q.m[1][2] * v.y * v.z + 2 * q.m[1][3] * v.y + q.m[2][2] * v.z * v.z +
      2 * q.m[2][3] * v.z + q.m[3][3];
}

class Mesh {
 public:
  struct Vertex {
    V3 p{0, 0, 0};
    Quadric q{};
    bool boundary = false;
  };
  struct Face {  // (the plane quadric of a face is only needed to seed the vertex quadrics: it is not kept here,
                 // which makes the per-sweep compaction of the face list three times lighter than the reference's)
    int v[3];
    V3 normal{0, 0, 0};
  };
  std::vector<Vertex> verts;
  std::vector<Face> faces;
  // what the sweeps scan, apart from the face records: 3 edge costs per face (edge j = v[j] -> v[j + 1]) and the flags
  // faces around every vertex as of the start of the sweep, ascending (the reference rebuilds its per-vertex lists once per
  // sweep and does not update them inside it): one flat array + offsets
  std::vector<int> around0, aroundAt;
  struct FaceRange {
    const int *first, *last;
    const int* begin() const { return first; }
    const int* end() const { return last; }
    size_t size() const { return (size_t)(last - first); }
  };
  FaceRange facesOf(int v) const { return FaceRange{around0.data() + aroundAt[v], around0.data() + aroundAt[v + 1]}; }
  std::vector<double> cost;
  std::vector<uint8_t> flag;
  enum : uint8_t { kDeleted = 1, kTouched = 2 };
  // Memory of failed attempts.  Whether edge a-b can be contracted is a pure function of the two vertexes (position, quadric,
  // boundary flag, face lists) and of the faces around them (vertex ids, normals, deleted flags, positions of their
  // vertexes) — the closed 1-rings of a and b.  A contraction x <- y changes exactly the closed 1-rings of x and y, so it
  // stamps every vertex of every face around x and y; an edge that failed after `failed[e] - 1` contractions still fails as
  // long as neither end has been stamped since.  The reference tries such edges again in every sweep (a failed attempt has
  // no side effects, so skipping it changes nothing): on torn meshes that is where its time goes.
  // whether the boundary rules admit the edge at all (MeshSimplifier.cpp:512-521: both ends on the boundary or neither, and
  // boundary edges only when asked to remove them): a property of the two end points' boundary flags, refreshed with the
  // costs; kept per edge so that the sweeps do not have to fetch two vertex records to find out
  std::vector<uint8_t> admissible;
  bool removeBoundary = false;
  std::vector<uint32_t> failed;   // per edge (3 per face): 1 + number of contractions done when it last failed, 0 = not known
  std::vector<uint32_t> stamped;  // per vertex: number of the last contraction that touched its closed 1-ring
  uint32_t contractions = 0;
  // MeshSimplifier's isEquiError: false divides every cost by the squared norm of the contraction target
  // (MeshSimplifier.cpp:165-169), for meshes in rig coordinates, where the same error matters less further away
  bool equiError = true;

  // xyz: 3 doubles per vertex; idx: 3 indices per face
  Mesh(const double* xyz, size_t nv, const uint32_t* idx, size_t nf, bool isEquiError = true) : verts(nv), faces(nf), cost(3 * nf), flag(nf, 0), admissible(3 * nf, 1), failed(3 * nf, 0), stamped(nv, 0), equiError(isEquiError) {
    for (size_t i = 0; i < nv; ++i) verts[i].p = V3{xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]};
    for (size_t i = 0; i < nf; ++i)
      for (int j = 0; j < 3; ++j) faces[i].v[j] = (int)idx[3 * i + j];
  }

  // optimal position of the vertex an edge contracts to, and the cost of contracting there (computeError)
  double contraction(const Vertex& a, const Vertex& b, V3* target) const {
    const double e = quadricContraction(a, b, target);
    return equiError ? e : e / dot(*target, *target);
  }
  double quadricContraction(const Vertex& a, const Vertex& b, V3* target) const {
    Quadric q = a.q;
    addInto(q, b.q);
    double top[3][3];
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) top[i][j] = q.m[i][j];
    const double det = det3(top);
    if (det != 0 && !(a.boundary && b.boundary)) {
      // Cramer: the first three entries of the last column of the inverse of [top | q14 q24 q34; 0 0 0 1]
      const double mx[3][3] = {{q.m[0][1], q.m[0][2], q.m[0][3]}, {q.m[1][1], q.m[1][2], q.m[1][3]}, {q.m[2][1], q.m[2][2], q.m[2][3]}};
      const double my[3][3] = {{q.m[0][0], q.m[0][2], q.m[0][3]}, {q.m[1][0], q.m[1][2], q.m[1][3]}, {q.m[2][0], q.m[2][2], q.m[2][3]}};
      const double mz[3][3] = {{q.m[0][0], q.m[0][1], q.m[0][3]}, {q.m[1][0], q.m[1][1], q.m[1][3]}, {q.m[2][0], q.m[2][1], q.m[2][3]}};
      const double inv = 1 / det;
      *target = V3{(-det3(mx)) * inv, det3(my) * inv, (-det3(mz)) * inv};
      return quadricError(q, *target);
    }
    const V3 cand[3] = {a.p, b.p, V3{(a.p.x + b.p.x) / 2, (a.p.y + b.p.y) / 2, (a.p.z + b.p.z) / 2}};
    int best = 0;
    double err[3];
    for (int k = 0; k < 3; ++k) {
      err[k] = quadricError(q, cand[k]);
      if (err[k] < err[best]) best = k;  // std::min_element: first of equal minima
    }
    *target = cand[best];
    return err[best];
  }

  void initialQuadrics() {
    for (Face& f : faces) {  // face order = accumulation order of the vertex quadrics, as in the reference
      const V3 &p0 = verts[f.v[0]].p, &p1 = verts[f.v[1]].p, &p2 = verts[f.v[2]].p;
      const V3 n = unit(cross(sub(p1, p0), sub(p2, p0)));
      f.normal = n;
      const double plane[4] = {n.x, n.y, n.z, -dot(n, p0)};
      Quadric q;
      for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) q.m[i][j] = plane[i] * plane[j];
      for (int j = 0; j < 3; ++j) addInto(verts[f.v[j]].q, q);
    }
    for (size_t fi = 0; fi < faces.size(); ++fi) refreshCosts(fi);
  }
  void refreshCosts(size_t fi) {
    const Face& f = faces[fi];
    for (int j = 0; j < 3; ++j) {
      V3 unused;
      const Vertex &a = verts[f.v[j]], &b = verts[f.v[(j + 1) % 3]];
      cost[3 * fi + j] = contraction(a, b, &unused);
      admissible[3 * fi + j] = a.boundary == b.boundary && (removeBoundary || !(a.boundary || b.boundary));
    }
  }
  void dropDeletedFaces() {
    size_t keep = 0;
    for (size_t fi = 0; fi < faces.size(); ++fi) {
      if (flag[fi] & kDeleted) continue;
      if (keep != fi) {
        faces[keep] = faces[fi];
        for (int j = 0; j < 3; ++j) cost[3 * keep + j] = cost[3 * fi + j];
        for (int j = 0; j < 3; ++j) failed[3 * keep + j] = failed[3 * fi + j];
        for (int j = 0; j < 3; ++j) admissible[3 * keep + j] = admissible[3 * fi + j];
      }
      ++keep;
    }
    faces.resize(keep);
    cost.resize(3 * keep);
    failed.resize(3 * keep);
    admissible.resize(3 * keep);
    flag.assign(keep, 0);
  }
  void rebuildIncidence() {
    aroundAt.assign(verts.size() + 1, 0);
    for (const Face& f : faces)
      for (int j = 0; j < 3; ++j) ++aroundAt[f.v[j] + 1];
    for (size_t v = 0; v < verts.size(); ++v) aroundAt[v + 1] += aroundAt[v];
    around0.resize(3 * faces.size());
    std::vector<int> fill(aroundAt.begin(), aroundAt.end() - 1);
    for (size_t i = 0; i < faces.size(); ++i)
      for (int j = 0; j < 3; ++j) around0[fill[faces[i].v[j]]++] = (int)i;
  }
  std::vector<int> sharedFaces(int a, int b) const {
    std::vector<int> out;
    for (int fa : facesOf(a))
      for (int fb : facesOf(b))
        if (fa == fb) out.push_back(fa);
    return out;
  }
  // a vertex is on the boundary when an edge at it has a single face (identifySubBoundaries, whole range in one thread)
  void markBoundaries() {
    for (Vertex& v : verts) v.boundary = false;
    std::vector<std::pair<int, int>> near;
    for (int i = 0; i < (int)verts.size(); ++i) {
      if (verts[i].boundary) continue;
      if (facesOf(i).size() == 1) {
        verts[i].boundary = true;
        continue;
      }
      bool border = false;
      // neighbours of i with the number of faces they share with it (= how often they occur among the vertexes of i's
      // faces: a face has three different vertexes); the reference looks every neighbour up once, in this order
      near.clear();
      for (int fi : facesOf(i))
        for (int j = 0; j < 3; ++j) {
          const int o = faces[fi].v[j];
          if (o == i) continue;
          size_t k = 0;
          while (k < near.size() && near[k].first != o) ++k;
          if (k == near.size())
            near.emplace_back(o, 1);
          else
            ++near[k].second;
        }
      for (const std::pair<int, int>& n : near)
        if (facesOf(n.first).size() == 1 || n.second == 1) {
          verts[n.first].boundary = true;
          border = true;
        }
      if (border) verts[i].boundary = true;
    }
  }
  // getThreshold: the cost at rank strictness * (number of costs - 1).  The reference copies the costs and calls
  // std::nth_element; the value at a rank does not depend on how it is found, so this is a two-level radix selection on
  // the order-preserving integer image of the doubles (one counting pass over 16 bits, then nth_element inside the one
  // bucket that holds the rank).  NaN costs have no rank: then the reference's call is reproduced literally.
  double costPercentile(float strictness) const {
    const size_t n = cost.size();  // called right after the compaction: every face is live
    const int at = strictness * (n - 1);  // float * size_t -> float -> int, as written in getThreshold
    auto key = [](double d) {
      uint64_t u;
      std::memcpy(&u, &d, 8);
      return (u >> 63) ? ~u : (u | 0x8000000000000000ull);  // negatives reversed below the positives
    };
    std::vector<uint32_t> count(65536, 0);
    bool nan = false;
    for (size_t i = 0; i < n; ++i) {
      const double c = cost[i];
      nan |= c != c;
      ++count[key(c) >> 48];
    }
    if (nan) {
      std::vector<double> all(cost);
      std::nth_element(all.begin(), all.begin() + at, all.end());
      return all[at];
    }
    size_t below = 0;
    uint32_t bucket = 0;
    for (;; ++bucket) {
      if (below + count[bucket] > (size_t)at) break;
      below += count[bucket];
    }
    std::vector<double> in;
    in.reserve(count[bucket]);
    for (size_t i = 0; i < n; ++i)
      if ((key(cost[i]) >> 48) == bucket) in.push_back(cost[i]);
    std::nth_element(in.begin(), in.begin() + ((size_t)at - below), in.end());
    return in[(size_t)at - below];
  }
  // would moving vertex a (edge a-b contracting) to p flip the normal of a face around a?
  bool flips(const V3& p, int a, int b) {
    for (int fi : facesOf(a)) {
      if (flag[fi] & kDeleted) continue;
      const Face& f = faces[fi];
      int at = 0;
      for (int j = 0; j < 3; ++j)
        if (f.v[j] == a) {
          at = j;
          break;
        }
      const int i0 = f.v[(at + 1) % 3], i1 = f.v[(at + 2) % 3];
      if (i0 == b || i1 == b) continue;  // a face of the contracting edge itself
      const V3 e0 = unit(sub(verts[i0].p, p)), e1 = unit(sub(verts[i1].p, p));
      if (dot(unit(cross(e0, e1)), f.normal) < 0) return true;
    }
    return false;
  }
  void contract(int a, int b, const V3& p) {  // vertex a becomes the merged vertex
    verts[a].p = p;
    addInto(verts[a].q, verts[b].q);
    const FaceRange fa = facesOf(a), fb = facesOf(b);
    std::vector<int> around(fa.begin(), fa.end());
    around.insert(around.end(), fb.begin(), fb.end());
    ++contractions;
    stamped[b] = contractions;
    for (int fi : around)  // before b is renamed to a; the faces the edge shared (just deleted) count: their third vertex
      for (int j = 0; j < 3; ++j) stamped[faces[fi].v[j]] = contractions;  // loses a face
    for (int fi : around) {
      if (flag[fi] & kDeleted) continue;
      Face& f = faces[fi];
      for (int j = 0; j < 3; ++j)
        if (f.v[j] == a || f.v[j] == b) {
          f.v[j] = a;
          flag[fi] |= kTouched;
          break;
        }
      refreshCosts(fi);
    }
  }
  void compact() {
    std::vector<char> live(verts.size(), 0);
    dropDeletedFaces();
    for (const Face& f : faces)
      for (int j = 0; j < 3; ++j) live[f.v[j]] = 1;
    std::vector<int> renumber(verts.size(), -1);
    int next = 0;
    for (size_t i = 0; i < verts.size(); ++i)
      if (live[i]) {
        renumber[i] = next;
        verts[next++].p = verts[i].p;
      }
    verts.resize(next);
    for (Face& f : faces)
      for (int j = 0; j < 3; ++j) f.v[j] = renumber[f.v[j]];
  }

  // one attempt at contracting edge j of face fi (MeshSimplifier.cpp:519-553); true if it was contracted.  A failed attempt
  // changes nothing.
  bool tryEdge(size_t fi, int j, int* gone) {
    if (!admissible[3 * fi + j]) return false;
    const int a = faces[fi].v[j], b = faces[fi].v[(j + 1) % 3];
    uint32_t& memo = failed[3 * fi + j];
    if (memo > stamped[a] && memo > stamped[b]) return false;  // failed before, and nothing around it has changed since
    V3 p;
    contraction(verts[a], verts[b], &p);
    if (flips(p, a, b) || flips(p, b, a)) {
      memo = contractions + 1;
      return false;
    }
    const std::vector<int> shared = sharedFaces(a, b);
    for (int s : shared) flag[s] |= kDeleted;
    *gone += (int)shared.size();
    contract(a, b, p);
    return true;
  }
  // a sweep over the faces from `from` on: every edge whose cost is under the threshold is tried, in order
  void sweepFrom(size_t from, double threshold, int facesIn, int facesOut, int* gone) {
    for (size_t fi = from; fi < faces.size(); ++fi) {
      // by index: contract() may not grow `faces`, but it writes through references into it
      if (flag[fi]) continue;  // deleted, or touched in this sweep
      for (int j = 0; j < 3; ++j) {
        if (cost[3 * fi + j] > threshold) continue;
        if (tryEdge(fi, j, gone)) break;
      }
      if (facesIn - *gone <= facesOut) break;
    }
  }

  // MeshSimplifier::simplify.  The reference runs sweep after sweep: compaction, incidence lists, threshold (a percentile
  // of the edge costs after a sweep that contracted something, the previous threshold times 2, 4, 6, ... after one that
  // did not, until it overflows to inf), then the pass over the faces.  Sweeps that contract nothing are the bulk on torn
  // meshes (boundary edges are kept, so the target is out of reach and the loop only ends at inf: hundreds of sweeps), and
  // they are where this version does less work for the same result: such a sweep leaves the mesh as it found it, every
  // edge it tried failed for reasons that do not depend on the threshold, and a failed attempt has no side effects — so
  // the following sweeps need no compaction, no incidence rebuild and no pass over the faces, only attempts at the edges
  // their larger thresholds newly admit, in face order.  One pass sorts those edges into the sweeps that will admit them.
  void run(int facesOut, float strictness, bool removeBoundaryEdges) {
    initialQuadrics();
    const int facesIn = (int)faces.size();
    int gone = 0, stuck = 0, iteration = 0;
    double threshold = 0;
    bool done = false;
    while (!done && (int)faces.size() > facesOut) {
      // ---- a sweep after a change (or the first one): the reference's sweep as it is
      dropDeletedFaces();
      rebuildIncidence();
      if (iteration == 0) {
        markBoundaries();
        removeBoundary = removeBoundaryEdges;
        for (size_t fi = 0; fi < faces.size(); ++fi)
          for (int j = 0; j < 3; ++j) {
            const Vertex &a = verts[faces[fi].v[j]], &b = verts[faces[fi].v[(j + 1) % 3]];
            admissible[3 * fi + j] = a.boundary == b.boundary && (removeBoundary || !(a.boundary || b.boundary));
          }
      }
      threshold = costPercentile(strictness);
      stuck = 0;
      int gonePrev = gone;
      sweepFrom(0, threshold, facesIn, facesOut, &gone);
      ++iteration;
      if (gone != gonePrev) continue;
      if (!((int)faces.size() > facesOut)) break;  // the reference tests its loop condition before every sweep

      // ---- nothing was contracted: the sweeps that follow, until one contracts something or the threshold overflows.
      // No face is deleted or touched here (the compaction cleared the flags and nothing has happened since).
      std::vector<double> levels;  // thresholds of the coming sweeps, computed the way the reference computes them
      {
        double t = threshold;
        int s = stuck;
        do {
          t *= 2 * ++s;
          levels.push_back(t);
        } while (!std::isinf(t) && t != 0 && t == t && levels.size() < 4096);
      }
      // A threshold of exactly 0 (exactly planar patches: constant-disparity regions) or NaN never grows: the reference's
      // loop spins forever there (MeshSimplifier.cpp:483-493, reproduced with its own code in tests/test_mesh.py).  Nothing
      // more can be contracted under the reference's rules, so stop with the mesh as it is.
      if (!(levels[0] != 0) || levels[0] != levels[0]) break;
      // edges not tried yet (cost above the last threshold; NaN costs pass every threshold test and were tried), filed under
      // the first coming sweep that admits them; the pass runs in face order, so every list is in face order
      std::vector<std::vector<uint32_t>> admitted(levels.size());
      for (size_t fi = 0; fi < faces.size(); ++fi)
        for (int j = 0; j < 3; ++j) {
          const double c = cost[3 * fi + j];
          if (!(c > threshold) || !admissible[3 * fi + j]) continue;
          const size_t k = std::lower_bound(levels.begin(), levels.end(), c) - levels.begin();  // first level >= c
          if (k + 1 < levels.size()) admitted[k].push_back((uint32_t)(3 * fi + j));  // the last level is inf: the loop ends there
        }
      size_t pending = 0;
      for (const auto& list : admitted) pending += list.size();
      for (size_t k = 0; k < levels.size(); ++k) {
        threshold = levels[k];
        ++stuck;
        if (std::isinf(threshold) || pending == 0) {  // the reference's loop ends at inf; with nothing left to try the sweeps
          done = true;                                // up to there change nothing
          break;
        }
        gonePrev = gone;
        bool contracted = false;
        for (uint32_t e : admitted[k]) {
          const size_t fi = e / 3;
          if (!tryEdge(fi, (int)(e % 3), &gone)) continue;
          contracted = true;  // the mesh moved: the rest of this sweep is an ordinary one (what failed before may succeed now)
          if (facesIn - gone > facesOut) sweepFrom(fi + 1, threshold, facesIn, facesOut, &gone);
          break;
        }
        pending -= admitted[k].size();
        ++iteration;
        if (contracted) break;
      }
    }
    compact();
  }
};

}  // namespace simplify
}  // namespace derp
