// mjb_ccd.cuh -- general convex collision (GJK + EPA) for analytic convex geoms, one lane per geom pair.
//
// Replaces /root/reference/mujoco_warp/_src/collision_gjk.py: :115 support, :281-594 distance sub-algorithm (S1D / S2D / S3D),
// :635 gjk, :1021-1286 polytope construction, :1319 _epa, :947 _epa_witness, :2303 _inflate, :2350 gjk_phase,
// :2421 epa_phase, :2076 multicontact (sphere, capsule, ellipsoid, cylinder, box; meshes and height fields are not built).
// The EPA polytope lives in a per-lane slice of shared memory supplied by the caller; the multi-contact clipping of box
// pairs reuses that slice for its polygon buffers once EPA has finished.
#pragma once
#include "mjb_colliders.cuh"
#include "mjb_math.cuh"
#include "mjb_types.cuh"

#define CCD_FLOAT_MAX 1e30f
#define CCD_MINVAL 1e-15f
#define CCD_MIN_DIST2 1e-10f
#define CCD_MIN_DIST3 1e-10f
#define CCD_MIN_DIST4 1e-17f
#define CCD_MAX_EPAFACES 5
#define CCD_MAX_EPAHORIZON 24
#define CCD_FACE_DELETED 0x80000000u
#define CCD_FACE_INVALID 0x40000000u
#define CCD_MIN_EPATOL 1e-7f
#define CCD_MINVAL2 1e-30f
#define CCD_FACE_TOL 0.99999872f       // cos(0.0016)
#define CCD_EDGE_TOL 0.00159999931f    // sin(0.0016)
#define CCD_INTERSECT_TOL 0.0000003f
// CCD_MESH = 1 adds mesh geoms (hull-vertex support function with a cached start vertex, mesh multi-contact).  The product library carries
// both builds of the collision kernel: k_collision.cu without it (models without mesh geoms keep the lean box / analytic code and its small
// stack), k_collision_mesh.cu with it; tests/host_harness also builds this header with it on the host.
// CCD_MESH = 2 is the same mesh code for hulls past the fixed buffers of CCD_MESH = 1 (npolygonmax > 32 or nmeshdegmax > 16): the multi-contact
// buffers are a per-lane slice of scratch the caller passes in (CcdClip), sized from the model at run time, so no per-lane array grows with the
// model (k_collision_mesh_large.cu, k_sensor_collision_large.cu).
#ifndef CCD_MESH
#define CCD_MESH 0
#endif
#if CCD_MESH == 2
#define CCD_VSHIFT 16
#define CCD_VMASK 0xFFFF
#define CCD_FLOAT_MIN -1e30f
#define CCD_DEGREES(n) (n)          // the candidate buffers hold every polygon at a vertex
#define CCD_POLY_FITS(n) true       // and every hull polygon
#define CCD_QUAD_GUARD(np) (np)     // a walk around a polygon of np vertices takes at most np steps
#define CCD_CLIPCAP clipcap         // twice the largest polygon (collision_convex.py:1229-1236)
#define CCD_CLIPCAP_PARAM , int clipcap
#define CCD_CLIPCAP_ARG , clipcap
#define CCD_CLIP_PARAM , CcdClip mc
#define CCD_CLIP_ARG , mc
// one lane's multi-contact scratch: buf holds mesh_clip_words(maxpoly, maxdeg) floats (mjb_types.cuh)
struct CcdClip { float* buf; int maxpoly, maxdeg; };
#elif CCD_MESH
#define CCD_VSHIFT 16        // support-vertex ids of the two geoms packed in one word: mesh vertex ids need 16 bits each
#define CCD_VMASK 0xFFFF
#define CCD_MAXDEG 16        // hull polygons meeting at one mesh vertex (model nmeshdegmax)
#define CCD_MAXPOLY 32       // vertices of one hull polygon (model npolygonmax)
#define CCD_CLIPCAP (2 * CCD_MAXPOLY)
#define CCD_FLOAT_MIN -1e30f
#else
#define CCD_VSHIFT 4         // box corner ids
#define CCD_VMASK 15
#define CCD_MAXDEG 3
#define CCD_MAXPOLY 4
#define CCD_CLIPCAP 8
#endif
#if CCD_MESH != 2
#define CCD_DEGREES(n) min(n, CCD_MAXDEG)
#define CCD_POLY_FITS(n) ((n) <= CCD_MAXPOLY)
#define CCD_QUAD_GUARD(np) 64
#define CCD_CLIPCAP_PARAM
#define CCD_CLIPCAP_ARG
#define CCD_CLIP_PARAM
#define CCD_CLIP_ARG
#endif

// Geom-type pairs the reference routes to the convex path (collision_driver.py:47-81), analytic geoms only, in table order.
// Box-box is convex unless the nativeccd disable flag routes it to the primitive box_box.
#if CCD_MESH
// with mesh geoms: the reference's full table order (sphere-mesh after sphere-ellipsoid, ... mesh-mesh last)
#define CCD_NRANK 15
static __host__ __device__ inline int convex_rank(int t1, int t2, bool nativeccd) {
  if (t1 == GEOM_SPHERE && t2 == GEOM_ELLIPSOID) return 0;
  if (t1 == GEOM_SPHERE && t2 == GEOM_MESH) return 1;
  if (t1 == GEOM_CAPSULE && t2 == GEOM_ELLIPSOID) return 2;
  if (t1 == GEOM_CAPSULE && t2 == GEOM_CYLINDER) return 3;
  if (t1 == GEOM_CAPSULE && t2 == GEOM_MESH) return 4;
  if (t1 == GEOM_ELLIPSOID && t2 == GEOM_ELLIPSOID) return 5;
  if (t1 == GEOM_ELLIPSOID && t2 == GEOM_CYLINDER) return 6;
  if (t1 == GEOM_ELLIPSOID && t2 == GEOM_BOX) return 7;
  if (t1 == GEOM_ELLIPSOID && t2 == GEOM_MESH) return 8;
  if (t1 == GEOM_CYLINDER && t2 == GEOM_CYLINDER) return 9;
  if (t1 == GEOM_CYLINDER && t2 == GEOM_BOX) return 10;
  if (t1 == GEOM_CYLINDER && t2 == GEOM_MESH) return 11;
  if (t1 == GEOM_BOX && t2 == GEOM_BOX && nativeccd) return 12;
  if (t1 == GEOM_BOX && t2 == GEOM_MESH) return 13;
  if (t1 == GEOM_MESH && t2 == GEOM_MESH) return 14;
  return -1;
}
#else
#define CCD_NRANK 9
static __host__ __device__ inline int convex_rank(int t1, int t2, bool nativeccd) {
  if (t1 == GEOM_SPHERE && t2 == GEOM_ELLIPSOID) return 0;
  if (t1 == GEOM_CAPSULE && t2 == GEOM_ELLIPSOID) return 1;
  if (t1 == GEOM_CAPSULE && t2 == GEOM_CYLINDER) return 2;
  if (t1 == GEOM_ELLIPSOID && t2 == GEOM_ELLIPSOID) return 3;
  if (t1 == GEOM_ELLIPSOID && t2 == GEOM_CYLINDER) return 4;
  if (t1 == GEOM_ELLIPSOID && t2 == GEOM_BOX) return 5;
  if (t1 == GEOM_CYLINDER && t2 == GEOM_CYLINDER) return 6;
  if (t1 == GEOM_CYLINDER && t2 == GEOM_BOX) return 7;
  if (t1 == GEOM_BOX && t2 == GEOM_BOX && nativeccd) return 8;
  return -1;
}
#endif

#if CCD_MESH
// mesh geoms carry their vertex block, hull graph (nullptr: exhaustive search) and hull polygon tables, already offset to the mesh
// (collision_core.py Geom); index = cached support vertex (vertex id, or hull-local id for the hill climb; -1: none)
struct CGeom {
  v3 pos; const float* rot; v3 size; float margin; int type;
  mutable int index; int vertnum, polynum;
  const float *vert, *polynormal;
  const int *graph, *polyvertadr, *polyvertnum, *polyvert, *polymapadr, *polymapnum, *polymap;
};
#define CCD_CACHE , true
#else
struct CGeom { v3 pos; const float* rot; v3 size; float margin; int type; };
#define CCD_CACHE
#endif
struct GjkRes { bool separated; int dim; float dist; v3 x1, x2, s[4], s1[4], s2[4]; int vi[4]; };  // vi: box corner ids, geom1 | geom2 << 4
// words of shared memory one lane's polytope needs: vertices (2 per support pair), faces, face projections, squared norms, horizon
static __host__ __device__ inline int ccd_scratch_words(int iterations) {
  return 3 * (10 + 2 * iterations) + 5 * (6 + CCD_MAX_EPAFACES * iterations) + CCD_MAX_EPAHORIZON + (5 + iterations);
}
struct Polytope {
  int status, nvert, nface, nhorizon, maxface;
  v3 center;
  float* vert;       // 3 * (10 + 2 it)
  unsigned* face;    // maxface
  float* face_pr;    // 3 * maxface
  float* face_norm2; // maxface
  int* horizon;      // CCD_MAX_EPAHORIZON
  int* vidx;         // 5 + it: box corner ids of each support pair (geom1 | geom2 << 4)
};

#if CCD_MESH
// collision_core.py:60-140 geom(): a mesh geom carries its asset's vertex block, hull graph and hull polygon tables
static __device__ __forceinline__ void fill_mesh(const ModelDev& m, int g, CGeom& c) {
  c.index = -1; c.vertnum = 0; c.polynum = 0; c.vert = nullptr; c.polynormal = nullptr; c.graph = nullptr;
  c.polyvertadr = c.polyvertnum = c.polyvert = c.polymapadr = c.polymapnum = c.polymap = nullptr;
  if (c.type != GEOM_MESH) return;
  const int id = m.geom_dataid[g];
  if (id < 0) return;
  const int vadr = m.mesh_vertadr[id], padr = m.mesh_polyadr[id];
  c.vert = m.mesh_vert + 3 * vadr; c.vertnum = m.mesh_vertnum[id];
  c.graph = m.mesh_graphadr[id] >= 0 ? m.mesh_graph + m.mesh_graphadr[id] : nullptr;
  c.polynum = m.mesh_polynum[id]; c.polynormal = m.mesh_polynormal + 3 * padr;
  c.polyvertadr = m.mesh_polyvertadr + padr; c.polyvertnum = m.mesh_polyvertnum + padr; c.polyvert = m.mesh_polyvert;
  c.polymapadr = m.mesh_polymapadr + vadr; c.polymapnum = m.mesh_polymapnum + vadr; c.polymap = m.mesh_polymap;
}

#endif

static __device__ __forceinline__ float csign(float x) { return x < 0.f ? -1.f : 1.f; }  // wp.sign(0) = +1

#if CCD_MESH
// :154-194 support vertex of a mesh in its own frame.  cache: remember the vertex for the geom's next query (GJK / EPA main loops)
static __device__ v3 mesh_support_local(const CGeom& g, v3 ld, int* vindex, bool cache) {
  const int cached = g.index;
  v3 res = mk3(0.f, 0.f, 0.f);
  int cidx = -1, vid = -1;
  float max_dist = CCD_FLOAT_MIN;
  if (!g.graph || g.vertnum < 10) {
    if (cached > -1) { cidx = cached; res = ld3(g.vert + 3 * cached); max_dist = dot(res, ld); }
    for (int i = 0; i < g.vertnum; i++) {
      const v3 p = ld3(g.vert + 3 * i);
      const float dd = dot(p, ld);
      if (dd > max_dist) { max_dist = dd; res = p; cidx = i; }
    }
    vid = cidx;
  } else {
    const int numvert = g.graph[0];
    const int *vert_edgeadr = g.graph + 2, *vert_globalid = g.graph + 2 + numvert, *edge_localid = g.graph + 2 + 2 * numvert;
    int prev = -1, imax = cached > -1 ? cached : 0;
    max_dist = dot(ld, ld3(g.vert + 3 * vert_globalid[imax]));
    while (imax != prev) {
      prev = imax;
      int i = vert_edgeadr[imax], subidx = edge_localid[i];
      while (subidx >= 0) {
        const float dd = dot(ld, ld3(g.vert + 3 * vert_globalid[subidx]));
        if (dd > max_dist) { imax = subidx; max_dist = dd; }
        i++; subidx = edge_localid[i];
      }
    }
    cidx = imax; vid = vert_globalid[imax];
    res = ld3(g.vert + 3 * vid);
  }
  if (vindex) *vindex = vid;
  if (cache) g.index = cidx;
  return res;
}
static __device__ v3 ccd_support(const CGeom& g, v3 dir, int* vindex = nullptr, bool cache = false) {
#else
static __device__ v3 ccd_support(const CGeom& g, v3 dir, int* vindex = nullptr) {
#endif
  if (g.type == GEOM_SPHERE) return g.pos + dir * (g.size.x + 0.5f * g.margin);
  const v3 ld = mat_t_vec(g.rot, dir);
  v3 res = mk3(0.f, 0.f, 0.f);
  if (g.type == GEOM_BOX) {
    res = mk3(csign(ld.x) * g.size.x, csign(ld.y) * g.size.y, csign(ld.z) * g.size.z);
    if (vindex) *vindex = (ld.x >= 0.f ? 1 : 0) | (ld.y >= 0.f ? 2 : 0) | (ld.z >= 0.f ? 4 : 0);  // :128-137 corner id
  }
  else if (g.type == GEOM_CAPSULE) { res = ld * g.size.x; res.z += csign(ld.z) * g.size.y; }
  else if (g.type == GEOM_ELLIPSOID) res = cw_mul(normalize(cw_mul(ld, g.size)), g.size);
  else if (g.type == GEOM_CYLINDER) {
    const float d = sqrtf(ld.x * ld.x + ld.y * ld.y);
    if (d > CCD_MINVAL) { const float scl = g.size.x / d; res.x = ld.x * scl; res.y = ld.y * scl; }
    res.z = csign(ld.z) * g.size.y;
  }
#if CCD_MESH
  else if (g.type == GEOM_MESH) res = mesh_support_local(g, ld, vindex, cache);
#endif
  v3 out = matvec(g.rot, res) + g.pos;
  if (g.margin > 0.f) out = out + dir * (0.5f * g.margin);
  return out;
}

static __device__ __forceinline__ float det3(v3 a, v3 b, v3 c) { return dot(a, cross(b, c)); }
static __device__ __forceinline__ int same_sign(float a, float b) { return (a > 0.f && b > 0.f) ? 1 : ((a < 0.f && b < 0.f) ? -1 : 0); }
static __device__ __forceinline__ v3 project_origin_line(v3 v1, v3 v2) {
  const v3 diff = v2 - v1;
  return v2 + diff * (-(dot(v2, diff) / dot(diff, diff)));
}
static __device__ int project_origin_plane(v3 v1, v3 v2, v3 v3_, v3* o) {
  const v3 d21 = v2 - v1, d31 = v3_ - v1, d32 = v3_ - v2;
  *o = mk3(0.f, 0.f, 0.f);
  v3 n = cross(d32, d21);
  float nv = dot(n, v2), nn = dot(n, n);
  if (nn == 0.f) return 1;
  if (nv != 0.f && nn > CCD_MINVAL) { *o = n * (nv / nn); return 0; }
  n = cross(d21, d31); nv = dot(n, v1); nn = dot(n, n);
  if (nn == 0.f) return 1;
  if (nv != 0.f && nn > CCD_MINVAL) { *o = n * (nv / nn); return 0; }
  n = cross(d31, d32); nv = dot(n, v3_); nn = dot(n, n);
  *o = n * (nv / nn);
  return 0;
}
static __device__ void S1D(v3 s1, v3 s2, float* l) {
  const v3 po = project_origin_line(s1, s2);
  float mu_max = s1.x - s2.x;
  int index = 0;
  float mu = s1.y - s2.y;
  if (fabsf(mu) >= fabsf(mu_max)) { mu_max = mu; index = 1; }
  mu = s1.z - s2.z;
  if (fabsf(mu) >= fabsf(mu_max)) { mu_max = mu; index = 2; }
  const float C1 = comp(po, index) - comp(s2, index), C2 = comp(s1, index) - comp(po, index);
  if (same_sign(mu_max, C1) && same_sign(mu_max, C2)) { l[0] = C1 / mu_max; l[1] = C2 / mu_max; return; }
  l[0] = 0.f; l[1] = 1.f;
}
// signed areas of (p, s2, s3), (p, s1, s3), (p, s1, s2) in the projection that drops the axis with the largest minor; returns that minor
static __device__ float tri_cofactors(v3 s1, v3 s2, v3 s3, v3 p, float* C) {
  const float M14 = s2.y * s3.z - s2.z * s3.y - s1.y * s3.z + s1.z * s3.y + s1.y * s2.z - s1.z * s2.y;
  const float M24 = s2.x * s3.z - s2.z * s3.x - s1.x * s3.z + s1.z * s3.x + s1.x * s2.z - s1.z * s2.x;
  const float M34 = s2.x * s3.y - s2.y * s3.x - s1.x * s3.y + s1.y * s3.x + s1.x * s2.y - s1.y * s2.x;
  const float mu1 = fabsf(M14), mu2 = fabsf(M24), mu3 = fabsf(M34);
  float Mmax; int x, y;
  if (mu1 >= mu2 && mu1 >= mu3) { Mmax = M14; x = 1; y = 2; } else if (mu2 >= mu3) { Mmax = M24; x = 0; y = 2; } else { Mmax = M34; x = 0; y = 1; }
  const float px = comp(p, x), py = comp(p, y), ax = comp(s1, x), ay = comp(s1, y), bx = comp(s2, x), by = comp(s2, y), cx = comp(s3, x), cy = comp(s3, y);
  C[0] = px * by + py * cx + bx * cy - px * cy - py * bx - cx * by;
  C[1] = px * cy + py * ax + cx * ay - px * ay - py * cx - ax * cy;
  C[2] = px * ay + py * bx + ax * by - px * by - py * ax - bx * ay;
  return Mmax;
}
static __device__ void S2D(v3 s1, v3 s2, v3 s3, float* l) {
  v3 po;
  if (project_origin_plane(s1, s2, s3, &po)) { S1D(s1, s2, l); l[2] = 0.f; return; }
  float C[3];
  const float Mmax = tri_cofactors(s1, s2, s3, po, C);
  const int c1 = same_sign(Mmax, C[0]), c2 = same_sign(Mmax, C[1]), c3 = same_sign(Mmax, C[2]);
  if (c1 && c2 && c3) { l[0] = C[0] / Mmax; l[1] = C[1] / Mmax; l[2] = C[2] / Mmax; return; }
  float dmin = CCD_FLOAT_MAX, sub[2];
  l[0] = l[1] = l[2] = 0.f;
  if (!c1) { S1D(s2, s3, sub); const v3 x = s2 * sub[0] + s3 * sub[1]; l[0] = 0.f; l[1] = sub[0]; l[2] = sub[1]; dmin = dot(x, x); }
  if (!c2) { S1D(s1, s3, sub); const v3 x = s1 * sub[0] + s3 * sub[1]; const float d = dot(x, x); if (d < dmin) { l[0] = sub[0]; l[1] = 0.f; l[2] = sub[1]; dmin = d; } }
  if (!c3) { S1D(s1, s2, sub); const v3 x = s1 * sub[0] + s2 * sub[1]; const float d = dot(x, x); if (d < dmin) { l[0] = sub[0]; l[1] = sub[1]; l[2] = 0.f; } }
}
static __device__ void S3D(v3 s1, v3 s2, v3 s3, v3 s4, float* l) {
  const float C41 = -det3(s2, s3, s4), C42 = det3(s1, s3, s4), C43 = -det3(s1, s2, s4), C44 = det3(s1, s2, s3);
  const float m_det = C41 + C42 + C43 + C44;
  const int c1 = same_sign(m_det, C41), c2 = same_sign(m_det, C42), c3 = same_sign(m_det, C43), c4 = same_sign(m_det, C44);
  if (c1 && c2 && c3 && c4) { l[0] = C41 / m_det; l[1] = C42 / m_det; l[2] = C43 / m_det; l[3] = C44 / m_det; return; }
  float dmin = CCD_FLOAT_MAX, sub[3];
  l[0] = l[1] = l[2] = l[3] = 0.f;
  if (!c1) { S2D(s2, s3, s4, sub); const v3 x = s2 * sub[0] + s3 * sub[1] + s4 * sub[2]; l[0] = 0.f; l[1] = sub[0]; l[2] = sub[1]; l[3] = sub[2]; dmin = dot(x, x); }
  if (!c2) { S2D(s1, s3, s4, sub); const v3 x = s1 * sub[0] + s3 * sub[1] + s4 * sub[2]; const float d = dot(x, x); if (d < dmin) { l[0] = sub[0]; l[1] = 0.f; l[2] = sub[1]; l[3] = sub[2]; dmin = d; } }
  if (!c3) { S2D(s1, s2, s4, sub); const v3 x = s1 * sub[0] + s2 * sub[1] + s4 * sub[2]; const float d = dot(x, x); if (d < dmin) { l[0] = sub[0]; l[1] = sub[1]; l[2] = 0.f; l[3] = sub[2]; dmin = d; } }
  if (!c4) { S2D(s1, s2, s3, sub); const v3 x = s1 * sub[0] + s2 * sub[1] + s3 * sub[2]; const float d = dot(x, x); if (d < dmin) { l[0] = sub[0]; l[1] = sub[1]; l[2] = sub[2]; l[3] = 0.f; } }
}
static __device__ __forceinline__ v3 lin_comb(int n, const float* l, const v3* m) {
  v3 o = m[0] * l[0];
  for (int k = 1; k < n; k++) o = o + m[k] * l[k];
  return o;
}

// collision_gjk.py:635; discrete (box pairs without margin) drops the tolerances and tracks box corner ids (:662-663)
static __device__ void ccd_gjk(float tolerance, int iterations, const CGeom& g1, const CGeom& g2, float cutoff, bool discrete, GjkRes& r) {
  float lmbda[4] = {1.f, 0.f, 0.f, 0.f};
  const float epsilon = discrete ? 0.f : 0.5f * tolerance * tolerance, min_norm = discrete ? CCD_MINVAL : tolerance;
  int n = 0;
  v3 x_k = g1.pos - g2.pos;
  float xnorm = sqrtf(dot(x_k, x_k)), xnorm_prev = 0.f;
  r.separated = false; r.dim = 0; r.dist = 0.f; r.x1 = r.x2 = mk3(0.f, 0.f, 0.f);
#pragma unroll 1
  for (int it = 0; it < iterations; it++) {
    if (xnorm < min_norm || fabsf(xnorm_prev - xnorm) < CCD_MINVAL) break;
    v3 dir_neg = x_k * (1.0f / xnorm);
    if (discrete && xnorm < 1e-4f) {  // :609-627 the search direction is noisy near the origin: rebuild it from the simplex
      if (n == 2) {
        const v3 edge = r.s[1] - r.s[0];
        const float en2 = dot(edge, edge);
        if (en2 > CCD_MINVAL2) {
          dir_neg = dir_neg - edge * (dot(dir_neg, edge) / en2);
          const float dn = length(dir_neg);
          if (dn > CCD_MINVAL) dir_neg = dir_neg * (1.0f / dn);
        }
      } else if (n == 3) {
        const v3 nrm = cross(r.s[1] - r.s[0], r.s[2] - r.s[0]);
        const float nn = length(nrm);
        if (nn > CCD_MINVAL) dir_neg = nrm * (csign(dot(dir_neg, nrm)) / nn);
      }
    }
    int i1 = 0, i2 = 0;
    r.s1[n] = ccd_support(g1, dir_neg * -1.0f, &i1 CCD_CACHE);
    r.s2[n] = ccd_support(g2, dir_neg, &i2 CCD_CACHE);
    r.vi[n] = i1 | (i2 << CCD_VSHIFT);
    r.s[n] = r.s1[n] - r.s2[n];
    if (dot(x_k, x_k - r.s[n]) < epsilon) break;
    const float lower = dot(x_k, r.s[n]);
    if (cutoff == 0.f) { if (lower > 0.f) { r.separated = true; r.dist = CCD_FLOAT_MAX; return; } }
    else if (cutoff < CCD_FLOAT_MAX) { if (lower > 0.f && lower >= cutoff * xnorm) { r.separated = true; r.dist = CCD_FLOAT_MAX; return; } }
    if (n == 3) S3D(r.s[0], r.s[1], r.s[2], r.s[3], lmbda);
    else if (n == 2) { S2D(r.s[0], r.s[1], r.s[2], lmbda); lmbda[3] = 0.f; }
    else if (n == 1) { S1D(r.s[0], r.s[1], lmbda); lmbda[2] = lmbda[3] = 0.f; }
    else { lmbda[0] = 1.f; lmbda[1] = lmbda[2] = lmbda[3] = 0.f; }
    n = 0;
#pragma unroll
    for (int i = 0; i < 4; i++) {
      if (lmbda[i] == 0.f) continue;
      r.s[n] = r.s[i]; r.s1[n] = r.s1[i]; r.s2[n] = r.s2[i]; r.vi[n] = r.vi[i]; lmbda[n] = lmbda[i];
      n++;
    }
    if (n < 1) break;
    x_k = lin_comb(n, lmbda, r.s);
    xnorm_prev = xnorm;
    xnorm = sqrtf(dot(x_k, x_k));
    if (n == 4) break;
  }
  if (n == 0) { r.x1 = g1.pos; r.x2 = g2.pos; } else { r.x1 = lin_comb(n, lmbda, r.s1); r.x2 = lin_comb(n, lmbda, r.s2); }
  if (xnorm > 0.f) {
    const v3 dir = x_k * (1.0f / xnorm);
    r.separated = dot(x_k, ccd_support(g1, dir * -1.0f) - ccd_support(g2, dir)) > 0.f;
  }
  r.dist = (n == 4 && !r.separated) ? 0.f : xnorm;
  r.dim = n;
}

static __device__ __forceinline__ v3 pt_v1(const Polytope& pt, int v) { return ld3(pt.vert + 6 * v); }
static __device__ __forceinline__ v3 pt_v2(const Polytope& pt, int v) { return ld3(pt.vert + 6 * v + 3); }
static __device__ __forceinline__ v3 pt_mink(const Polytope& pt, int v) { return pt_v1(pt, v) - pt_v2(pt, v); }
static __device__ bool same_side(v3 p0, v3 p1, v3 p2, v3 p3) {
  const v3 n = cross(p1 - p0, p2 - p0);
  const float d1 = dot(n, p3 - p0), d2 = dot(n, p0 * -1.0f);
  return (d1 > 0.f && d2 > 0.f) || (d1 < 0.f && d2 < 0.f);
}
static __device__ bool test_tetra(v3 p0, v3 p1, v3 p2, v3 p3) {
  return same_side(p0, p1, p2, p3) && same_side(p1, p2, p3, p0) && same_side(p2, p3, p0, p1) && same_side(p3, p0, p1, p2);
}
static __device__ bool tri_point_intersect(v3 v1, v3 v2, v3 v3_, v3 p) {
  float C[3];
  const float Mmax = tri_cofactors(v1, v2, v3_, p, C);
  const float l1 = C[0] / Mmax, l2 = C[1] / Mmax, l3 = C[2] / Mmax;
  if (l1 < 0.f || l2 < 0.f || l3 < 0.f) return false;
  return length(v1 * l1 + v2 * l2 + v3_ * l3 - p) < CCD_MINVAL;
}
static __device__ float attach_face(Polytope& pt, int idx, int v1, int v2, int v3_) {
  if (pt.nface == pt.maxface) return 0.f;
  const v3 p1 = pt_mink(pt, v1), p2 = pt_mink(pt, v2), p3 = pt_mink(pt, v3_);
  v3 r;
  if (project_origin_plane(p3, p2, p1, &r)) return 0.f;
  if (dot(r, p1 - pt.center) < 0.f) r = r * -1.0f;
  pt.face[idx] = (unsigned)(v1 + (v2 << 10) + (v3_ << 20));
  st3(pt.face_pr + 3 * idx, r);
  const float n2 = dot(r, r);
  pt.face_norm2[idx] = n2;
  return n2;
}
static __device__ void epa_support(Polytope& pt, int idx, const CGeom& g1, const CGeom& g2, v3 dir) {
  int i1 = 0, i2 = 0;
  st3(pt.vert + 6 * idx, ccd_support(g1, dir, &i1));
  st3(pt.vert + 6 * idx + 3, ccd_support(g2, dir * -1.0f, &i2));
  pt.vidx[idx] = i1 | (i2 << CCD_VSHIFT);
}
#if CCD_MESH
static __device__ void epa_support_cached(Polytope& pt, int idx, const CGeom& g1, const CGeom& g2, v3 dir) {  // :1372-1373 the cached vertices follow the expansion
  int i1 = 0, i2 = 0;
  st3(pt.vert + 6 * idx, ccd_support(g1, dir, &i1, true));
  st3(pt.vert + 6 * idx + 3, ccd_support(g2, dir * -1.0f, &i2, true));
  pt.vidx[idx] = i1 | (i2 << CCD_VSHIFT);
}
#else
#define epa_support_cached epa_support
#endif
static __device__ void replace_simplex3(const Polytope& pt, int v1, int v2, int v3_, GjkRes& r) {
  const int v[3] = {v1, v2, v3_};
  for (int k = 0; k < 3; k++) { r.s1[k] = pt_v1(pt, v[k]); r.s2[k] = pt_v2(pt, v[k]); r.s[k] = r.s1[k] - r.s2[k]; r.vi[k] = pt.vidx[v[k]]; }
}
static __device__ void load_simplex(Polytope& pt, const GjkRes& r, int n) {
  for (int k = 0; k < n; k++) { st3(pt.vert + 6 * k, r.s1[k]); st3(pt.vert + 6 * k + 3, r.s2[k]); pt.vidx[k] = r.vi[k]; }
}
static __device__ void polytope2(Polytope& pt, GjkRes& r, const CGeom& g1, const CGeom& g2) {
  const v3 diff = r.s[1] - r.s[0];
  pt.center = (r.s[0] + r.s[1]) * 0.5f;
  float value = CCD_FLOAT_MAX;
  int index = 0;
  for (int i = 0; i < 3; i++) if (fabsf(comp(diff, i)) < value) { value = fabsf(comp(diff, i)); index = i; }
  v3 e = mk3(0.f, 0.f, 0.f);
  setcomp(e, index, 1.0f);
  const v3 d1 = cross(e, diff);
  float R[9];
  { const float n = length(diff), u1 = diff.x / n, u2 = diff.y / n, u3 = diff.z / n, s = 0.86602540378f, c = -0.5f;  // rotation by 120 degrees (:885)
    R[0] = c + u1 * u1 * (1.f - c); R[1] = u1 * u2 * (1.f - c) - u3 * s; R[2] = u1 * u3 * (1.f - c) + u2 * s;
    R[3] = u2 * u1 * (1.f - c) + u3 * s; R[4] = c + u2 * u2 * (1.f - c); R[5] = u2 * u3 * (1.f - c) - u1 * s;
    R[6] = u1 * u3 * (1.f - c) - u2 * s; R[7] = u2 * u3 * (1.f - c) + u1 * s; R[8] = c + u3 * u3 * (1.f - c); }
  const v3 d2 = matvec(R, d1), d3 = matvec(R, d2);
  load_simplex(pt, r, 2);
  epa_support(pt, 2, g1, g2, d1 * (1.0f / length(d1)));
  epa_support(pt, 3, g1, g2, d2 * (1.0f / length(d2)));
  epa_support(pt, 4, g1, g2, d3 * (1.0f / length(d3)));
  const int F[6][3] = {{0, 2, 3}, {0, 4, 2}, {0, 3, 4}, {1, 3, 2}, {1, 2, 4}, {1, 4, 3}};
  for (int f = 0; f < 6; f++)
    if (attach_face(pt, f, F[f][0], F[f][1], F[f][2]) < CCD_MIN_DIST2) { pt.status = -1; replace_simplex3(pt, F[f][0], F[f][1], F[f][2], r); return; }
  {  // the hexahedron must enclose the segment (:907 _ray_triangle)
    const v3 v1 = r.s[0], a = pt_mink(pt, 2) - v1, b = pt_mink(pt, 3) - v1, c = pt_mink(pt, 4) - v1, d = r.s[1] - v1;
    const float vol1 = det3(a, b, d), vol2 = det3(b, c, d), vol3 = det3(c, a, d);
    if (!((vol1 >= 0.f && vol2 >= 0.f && vol3 >= 0.f) || (vol1 <= 0.f && vol2 <= 0.f && vol3 <= 0.f))) { pt.status = 1; return; }
  }
  pt.nvert = 5; pt.nface = 6; pt.status = 0;
}
static __device__ void polytope3(Polytope& pt, const GjkRes& r, const CGeom& g1, const CGeom& g2) {
  pt.center = (r.s[0] + r.s[1] + r.s[2]) * (1.0f / 3.0f);
  v3 n = cross(r.s[1] - r.s[0], r.s[2] - r.s[0]);
  const float norm = length(n);
  if (norm < CCD_MINVAL) { pt.status = 2; return; }
  n = n * (1.0f / norm);
  load_simplex(pt, r, 3);
  epa_support(pt, 3, g1, g2, n * -1.0f);
  epa_support(pt, 4, g1, g2, n);
  const v3 v1 = r.s[0], v2 = r.s[1], v3_ = r.s[2], v4 = pt_mink(pt, 3), v5 = pt_mink(pt, 4);
  if (tri_point_intersect(v1, v2, v3_, v4)) { pt.status = 3; return; }
  if (tri_point_intersect(v1, v2, v3_, v5)) { pt.status = 4; return; }
  if (r.dist > 1e-5f && !test_tetra(v1, v2, v3_, v4) && !test_tetra(v1, v2, v3_, v5)) { pt.status = 5; return; }
  const int F[6][3] = {{4, 0, 1}, {4, 2, 0}, {4, 1, 2}, {3, 1, 0}, {3, 0, 2}, {3, 2, 1}};
  for (int f = 0; f < 6; f++) if (attach_face(pt, f, F[f][0], F[f][1], F[f][2]) < CCD_MIN_DIST3) { pt.status = 6 + f; return; }
  pt.nvert = 5; pt.nface = 6; pt.status = 0;
}
static __device__ void polytope4(Polytope& pt, GjkRes& r) {
  pt.center = (r.s[0] + r.s[1] + r.s[2] + r.s[3]) * 0.25f;
  load_simplex(pt, r, 4);
  const int F[4][3] = {{0, 1, 2}, {0, 3, 1}, {0, 2, 3}, {3, 2, 1}};
  float dist[4];
  int idx = 0;
  for (int f = 0; f < 4; f++) {
    dist[f] = attach_face(pt, f, F[f][0], F[f][1], F[f][2]);
    if (dist[f] < CCD_MIN_DIST4) { pt.status = -1; replace_simplex3(pt, F[f][0], F[f][1], F[f][2], r); return; }
    if (f == 1) idx = dist[0] < dist[1] ? 0 : 1;
    else if (f > 1) idx = dist[f] < dist[idx] ? f : idx;
  }
  if (!test_tetra(r.s[0], r.s[1], r.s[2], r.s[3])) {
    if (dist[idx] > CCD_MINVAL) { pt.status = 12; return; }
    pt.status = -1;
    replace_simplex3(pt, F[idx][0], F[idx][1], F[idx][2], r);
    return;
  }
  pt.nvert = 4; pt.nface = 4; pt.status = 0;
}
static __device__ int add_edge(Polytope& pt, int e1, int e2) {
  const int n = pt.nhorizon;
  if (n < 0) return -1;
  const int edge = (min(e1, e2) << 10) | max(e1, e2);
  for (int i = 0; i < n; i++) if (edge == pt.horizon[i]) { pt.horizon[i] = pt.horizon[n - 1]; return n - 1; }
  if (n == CCD_MAX_EPAHORIZON) return -1;
  pt.horizon[n] = edge;
  return n + 1;
}
// :1319 _epa + :947 witness points; returns the closest face index or -1
static __device__ int ccd_epa(float tolerance, int iterations, Polytope& pt, const CGeom& g1, const CGeom& g2, bool discrete, float* dist, v3* x1, v3* x2, bool* ovf) {
  float upper = CCD_FLOAT_MAX, upper2 = CCD_FLOAT_MAX;
  const float epsilon = discrete ? CCD_MIN_EPATOL : tolerance;
  int idx = -1, pidx = -1, nvalid = pt.nface;
  iterations = min(iterations, 1000);
#pragma unroll 1
  for (int it = 0; it < iterations; it++) {
    pidx = idx; idx = -1;
    float lower2 = CCD_FLOAT_MAX;
    for (int i = 0; i < pt.nface; i++) if (!(pt.face[i] & (CCD_FACE_DELETED | CCD_FACE_INVALID)) && pt.face_norm2[i] < lower2) { idx = i; lower2 = pt.face_norm2[i]; }
    if (lower2 > upper2 || idx < 0) { idx = pidx; break; }
    if (lower2 <= 0.f) break;
    const float lower = sqrtf(lower2);
    const int wi = pt.nvert;
    const v3 fp = ld3(pt.face_pr + 3 * idx);
    epa_support_cached(pt, wi, g1, g2, fp * (1.0f / lower));
    const v3 w = pt_mink(pt, wi);
    pt.nvert++;
    const float upper_k = dot(fp, w) / lower;
    if (upper_k < upper) { upper = upper_k; upper2 = upper * upper; }
    if (upper - lower < epsilon) break;
    if (discrete) {  // :1377-1385 a repeated support point ends the expansion
      bool rep = false;
      for (int i = 0; i < wi; i++) if (pt.vidx[i] == pt.vidx[wi]) { rep = true; break; }
      if (rep) break;
    }
    nvalid--;
    pt.face[idx] |= CCD_FACE_DELETED;
    { const unsigned f = pt.face[idx]; const int a = f & 0x3FF, b = (f >> 10) & 0x3FF, c = (f >> 20) & 0x3FF;
      pt.nhorizon = add_edge(pt, a, b); pt.nhorizon = add_edge(pt, b, c); pt.nhorizon = add_edge(pt, c, a); }
    if (pt.nhorizon == -1) { *ovf = true; idx = -1; break; }
    for (int i = 0; i < pt.nface; i++) {
      if (pt.face[i] & CCD_FACE_DELETED) continue;
      if (dot(ld3(pt.face_pr + 3 * i), w) - pt.face_norm2[i] > 1e-10f) {
        if (!(pt.face[i] & CCD_FACE_INVALID)) nvalid--;
        pt.face[i] |= CCD_FACE_DELETED;
        const unsigned f = pt.face[i]; const int a = f & 0x3FF, b = (f >> 10) & 0x3FF, c = (f >> 20) & 0x3FF;
        pt.nhorizon = add_edge(pt, a, b); pt.nhorizon = add_edge(pt, b, c); pt.nhorizon = add_edge(pt, c, a);
        if (pt.nhorizon == -1) { *ovf = true; idx = -1; break; }
      }
    }
    for (int i = 0; i < pt.nhorizon; i++) {
      const int e = pt.horizon[i];
      const float dist2 = attach_face(pt, pt.nface, wi, e & 0x3FF, (e >> 10) & 0x3FF);
      if (dist2 == 0.f) { idx = -1; break; }
      pt.nface++;
      if (dist2 >= lower2 && dist2 <= upper2) nvalid++; else pt.face[pt.nface - 1] |= CCD_FACE_INVALID;
    }
    if (nvalid == 0 || idx == -1) break;
    pt.nhorizon = 0;
  }
  if (idx > -1) {
    const unsigned f = pt.face[idx]; const int a = f & 0x3FF, b = (f >> 10) & 0x3FF, c = (f >> 20) & 0x3FF;
    float C[3];
    const float Mmax = tri_cofactors(pt_mink(pt, a), pt_mink(pt, b), pt_mink(pt, c), ld3(pt.face_pr + 3 * idx), C);
    const float l1 = C[0] / Mmax, l2 = C[1] / Mmax, l3 = C[2] / Mmax;
    *x2 = pt_v2(pt, a) * l1 + pt_v2(pt, b) * l2 + pt_v2(pt, c) * l3;
    *x1 = pt_v1(pt, a) * l1 + pt_v1(pt, b) * l2 + pt_v1(pt, c) * l3;
    *dist = -sqrtf(pt.face_norm2[idx]);
    return idx;
  }
  *dist = 0.f; *x1 = *x2 = mk3(0.f, 0.f, 0.f);
  return -1;
}

// ---- multi-contact recovery for box pairs (collision_gjk.py:1503 _feature_dim, :1703-1888 box normals / edges / faces,
// :1916-2056 polygon clipping, :2076 multicontact; mesh branches not built)
struct BoxFeat { int dim, idx[3]; v3 v0, v1; };
static __device__ BoxFeat feature_dim(const Polytope& pt, const int* face, int which) {
  BoxFeat f;
  const int sh = which ? CCD_VSHIFT : 0;
  const int a = (pt.vidx[face[0]] >> sh) & CCD_VMASK, b = (pt.vidx[face[1]] >> sh) & CCD_VMASK, c = (pt.vidx[face[2]] >> sh) & CCD_VMASK;
  f.idx[0] = a; f.idx[1] = b; f.idx[2] = c;
  f.v0 = ld3(pt.vert + 6 * face[0] + 3 * which);
  f.v1 = ld3(pt.vert + 6 * face[1] + 3 * which);
  if (a != b) { f.dim = (c == a || c == b) ? 2 : 3; return f; }
  f.idx[1] = c; f.v1 = ld3(pt.vert + 6 * face[2] + 3 * which);
  f.dim = a != c ? 2 : 1;
  return f;
}
static __device__ __forceinline__ v3 box_face_normal(int i) { return mk3(i == 0 ? 1.f : (i == 1 ? -1.f : 0.f), i == 2 ? 1.f : (i == 3 ? -1.f : 0.f), i == 4 ? 1.f : (i == 5 ? -1.f : 0.f)); }
static __device__ int box_normals2(const float* mat, v3 n, v3* nout, int* iout) {
  const v3 ln = normalize(mat_t_vec(mat, n));
  for (int i = 0; i < 6; i++) if (dot(ln, box_face_normal(i)) > CCD_FACE_TOL) { nout[0] = matvec(mat, box_face_normal(i)); iout[0] = i; return 1; }
  return 0;
}
static __device__ __forceinline__ float bit_axis(int a, int b, int c, int bit) {  // +1 when every corner has the bit, -1 when none has it
  return (float)(((a & bit) && (b & bit) && (c & bit)) ? 1 : 0) - (float)((!(a & bit) && !(b & bit) && !(c & bit)) ? 1 : 0);
}
static __device__ int box_normals(const BoxFeat& f, const float* mat, v3 dir, v3* nout, int* iout) {
  const int v1 = f.idx[0], v2 = f.idx[1], v3i = f.idx[2];
  if (f.dim == 3) {
    int c = 0;
    const float x = bit_axis(v1, v2, v3i, 1), y = bit_axis(v1, v2, v3i, 2), z = bit_axis(v1, v2, v3i, 4);
    nout[0] = matvec(mat, mk3(x, y, z));
    if (x != 0.f) iout[c++] = 0;
    if (y != 0.f) iout[c++] = 2;
    if (z != 0.f) iout[c++] = 4;
    if (x + y + z == -1.f) iout[0] = iout[0] + 1;
    if (c == 1) return 1;
    return box_normals2(mat, dir, nout, iout);
  }
  if (f.dim == 2) {
    int c = 0;
    const float x = bit_axis(v1, v2, v2, 1), y = bit_axis(v1, v2, v2, 2), z = bit_axis(v1, v2, v2, 4);
    if (x != 0.f) { nout[c] = matvec(mat, mk3(x, 0.f, 0.f)); iout[c] = x > 0.f ? 0 : 1; c++; }
    if (y != 0.f) { nout[c] = matvec(mat, mk3(0.f, y, 0.f)); iout[c] = y > 0.f ? 2 : 3; c++; }
    if (z != 0.f) { nout[c] = matvec(mat, mk3(0.f, 0.f, z)); iout[c] = z > 0.f ? 4 : 5; c++; }
    if (c == 1 || c == 2) return c;  // 1: diagonal of a face, 2: an edge of the box
    return box_normals2(mat, dir, nout, iout);
  }
  if (f.dim == 1) {
    const float x = (v1 & 1) ? 1.f : -1.f, y = (v1 & 2) ? 1.f : -1.f, z = (v1 & 4) ? 1.f : -1.f;
    nout[0] = matvec(mat, mk3(x, 0.f, 0.f)); nout[1] = matvec(mat, mk3(0.f, y, 0.f)); nout[2] = matvec(mat, mk3(0.f, 0.f, z));
    iout[0] = x > 0.f ? 0 : 1; iout[1] = y > 0.f ? 2 : 3; iout[2] = z > 0.f ? 4 : 5;
    return 3;
  }
  return 0;
}
static __device__ int box_edge_normals(const BoxFeat& f, const CGeom& g, v3* nout, v3* endvert) {
  if (f.dim == 2) { endvert[0] = f.v1; nout[0] = normalize(f.v1 - f.v0); return 1; }
  if (f.dim == 1) {
    const int vi = f.idx[0];
    const float x = (vi & 1) ? g.size.x : -g.size.x, y = (vi & 2) ? g.size.y : -g.size.y, z = (vi & 4) ? g.size.z : -g.size.z;
    endvert[0] = matvec(g.rot, mk3(-x, y, z)) + g.pos; nout[0] = normalize(endvert[0] - f.v0);
    endvert[1] = matvec(g.rot, mk3(x, -y, z)) + g.pos; nout[1] = normalize(endvert[1] - f.v0);
    endvert[2] = matvec(g.rot, mk3(x, y, -z)) + g.pos; nout[2] = normalize(endvert[2] - f.v0);
    return 3;
  }
  return 0;
}
static __device__ int box_face(const CGeom& g, int idx, v3* face) {
  if (idx < 0 || idx > 5) return 0;
  // corner k of face idx, as signs of (x, y, z): one byte per face, bit (3 k + axis)
  const float sx = g.size.x, sy = g.size.y, sz = g.size.z;
  v3 l[4];
  switch (idx) {
    case 0: l[0] = mk3(sx, sy, sz); l[1] = mk3(sx, sy, -sz); l[2] = mk3(sx, -sy, -sz); l[3] = mk3(sx, -sy, sz); break;
    case 1: l[0] = mk3(-sx, sy, -sz); l[1] = mk3(-sx, sy, sz); l[2] = mk3(-sx, -sy, sz); l[3] = mk3(-sx, -sy, -sz); break;
    case 2: l[0] = mk3(-sx, sy, -sz); l[1] = mk3(sx, sy, -sz); l[2] = mk3(sx, sy, sz); l[3] = mk3(-sx, sy, sz); break;
    case 3: l[0] = mk3(-sx, -sy, sz); l[1] = mk3(sx, -sy, sz); l[2] = mk3(sx, -sy, -sz); l[3] = mk3(-sx, -sy, -sz); break;
    case 4: l[0] = mk3(-sx, sy, sz); l[1] = mk3(sx, sy, sz); l[2] = mk3(sx, -sy, sz); l[3] = mk3(-sx, -sy, sz); break;
    default: l[0] = mk3(sx, sy, -sz); l[1] = mk3(-sx, sy, -sz); l[2] = mk3(-sx, -sy, -sz); l[3] = mk3(sx, -sy, -sz); break;
  }
  for (int k = 0; k < 4; k++) face[k] = matvec(g.rot, l[k]) + g.pos;
  return 4;
}
static __device__ __forceinline__ float area4(v3 a, v3 b, v3 c, v3 d) { return 0.5f * length(cross(a - d, d - b) + cross(b - c, c - a)); }
static __device__ void polygon_quad(const float* poly, int np, int* res) {  // :1463 maximum-area quadrilateral of a convex polygon
  int b = 1, c = 2, d = 3;
  res[0] = 0; res[1] = b; res[2] = c; res[3] = d;
  float m = area4(ld3(poly), ld3(poly + 3 * b), ld3(poly + 3 * c), ld3(poly + 3 * d));
  for (int a = 0; a < np; a++) {
    for (int guard = 0; guard < CCD_QUAD_GUARD(np); guard++) {
      float mn = area4(ld3(poly + 3 * a), ld3(poly + 3 * b), ld3(poly + 3 * c), ld3(poly + 3 * ((d + 1) % np)));
      if (mn <= m) break;
      m = mn; d = (d + 1) % np; res[0] = a; res[1] = b; res[2] = c; res[3] = d;
      for (int g2 = 0; g2 < CCD_QUAD_GUARD(np); g2++) {
        mn = area4(ld3(poly + 3 * a), ld3(poly + 3 * b), ld3(poly + 3 * ((c + 1) % np)), ld3(poly + 3 * d));
        if (mn <= m) break;
        m = mn; c = (c + 1) % np; res[0] = a; res[1] = b; res[2] = c; res[3] = d;
      }
      for (int g3 = 0; g3 < CCD_QUAD_GUARD(np); g3++) {
        mn = area4(ld3(poly + 3 * a), ld3(poly + 3 * ((b + 1) % np)), ld3(poly + 3 * c), ld3(poly + 3 * d));
        if (mn <= m) break;
        m = mn; b = (b + 1) % np; res[0] = a; res[1] = b; res[2] = c; res[3] = d;
      }
    }
    if (b == a) { b = (b + 1) % np; if (c == b) { c = (c + 1) % np; if (d == c) d = (d + 1) % np; } }
  }
}
// :1941 clip polygon face2 against the side planes of face1 (extruded along n).  witness2 lies on the clipped polygon,
// witness1 = witness2 - dir.  buf: two polygons of CCD_CLIPCAP vertices.
static __device__ int polygon_clip(const v3* face1, int nface1, const v3* face2, int nface2, v3 n, v3 dir, float* buf, v3* w1, v3* w2 CCD_CLIPCAP_PARAM) {
  if (nface1 < 3) return 0;
  float* poly = buf;
  float* clip = buf + 3 * CCD_CLIPCAP;
  int np = nface2, nc = 0;
  for (int i = 0; i < nface2; i++) st3(poly + 3 * i, face2[i]);
  for (int e = 0; e < nface1; e++) {
    const v3 a = face1[e], b = face1[(e + 1) % nface1];
    const v3 pn = cross(b - a, (a + n) - a);  // :1916 _plane_normal
    const float pd = dot(pn, a);
    for (int i = 0; i < np; i++) {
      const v3 P = ld3(poly + 3 * i), Q = ld3(poly + 3 * ((i + 1) % np));
      const bool in1 = dot(P - a, pn) > -1e-10f, in2 = dot(Q - a, pn) > -1e-10f;
      if (!in1 && !in2) continue;
      if (in1 && in2) { if (nc < CCD_CLIPCAP) st3(clip + 3 * nc, Q); nc++; continue; }
      const v3 pq = Q - P;
      const float dt = dot(pn, pq);
      float t = fabsf(dt) < 1e-10f ? CCD_FLOAT_MAX : (pd - dot(pn, P)) / dt;
      if (t > -CCD_INTERSECT_TOL && t < 1.f + CCD_INTERSECT_TOL) {
        t = fminf(fmaxf(t, 0.f), 1.f);
        if (nc < CCD_CLIPCAP) st3(clip + 3 * nc, P + pq * t);
        nc++;
      }
      if (in2) { if (nc < CCD_CLIPCAP) st3(clip + 3 * nc, Q); nc++; }
    }
    float* tmp = poly; poly = clip; clip = tmp;
    np = min(nc, CCD_CLIPCAP); nc = 0;
  }
  if (np < 1) return 0;
  if (nface2 == 2 && np > 2) {  // an edge: keep the two points farthest apart
    int b1 = 0, b2 = 1;
    float maxd = 0.f;
    for (int i = 0; i < np; i++) for (int j = i + 1; j < np; j++) {
      const v3 df = ld3(poly + 3 * j) - ld3(poly + 3 * i);
      const float d2 = dot(df, df);
      if (d2 > maxd) { maxd = d2; b1 = i; b2 = j; }
    }
    w2[0] = ld3(poly + 3 * b1); w1[0] = w2[0] - dir; w2[1] = ld3(poly + 3 * b2); w1[1] = w2[1] - dir;
    return 2;
  }
  if (np > 4) {
    int q[4];
    polygon_quad(poly, np, q);
    for (int i = 0; i < 4; i++) { w2[i] = ld3(poly + 3 * q[i]); w1[i] = w2[i] - dir; }
    return 4;
  }
  for (int i = 0; i < np; i++) { w2[i] = ld3(poly + 3 * i); w1[i] = w2[i] - dir; }
  return np;
}
#if CCD_MESH
// :1556-1581 common polygon ids of two vertices' polygon lists (at most two)
static __device__ int mesh_intersect(const int* a1, int n1, const int* a2, int n2, int* res) {
  int count = 0;
  for (int i = 0; i < n1; i++) for (int j = 0; j < n2; j++) if (a1[i] == a2[j]) { res[count++] = a1[i]; if (count == 2) return 2; }
  return count;
}
// :1585-1651 candidate hull-polygon normals of a mesh feature given by up to three vertices
static __device__ int mesh_normals(const BoxFeat& f, const CGeom& g, v3* nout, int* iout) {
  const int* m1 = g.polymap + g.polymapadr[f.idx[0]];
  const int n1 = g.polymapnum[f.idx[0]];
  if (f.dim == 3) {
    int e[2], ff[2];
    int n = mesh_intersect(m1, n1, g.polymap + g.polymapadr[f.idx[1]], g.polymapnum[f.idx[1]], e);
    if (n == 0) return 0;
    n = mesh_intersect(e, n, g.polymap + g.polymapadr[f.idx[2]], g.polymapnum[f.idx[2]], ff);
    if (n == 0) return 0;
    nout[0] = matvec(g.rot, ld3(g.polynormal + 3 * ff[0])); iout[0] = ff[0];
    return 1;
  }
  if (f.dim == 2) {
    int e[2];
    const int n = mesh_intersect(m1, n1, g.polymap + g.polymapadr[f.idx[1]], g.polymapnum[f.idx[1]], e);
    for (int i = 0; i < n; i++) { nout[i] = matvec(g.rot, ld3(g.polynormal + 3 * e[i])); iout[i] = e[i]; }
    return n;
  }
  if (f.dim == 1) {
    const int n = CCD_DEGREES(n1);
    for (int i = 0; i < n; i++) { nout[i] = matvec(g.rot, ld3(g.polynormal + 3 * m1[i])); iout[i] = m1[i]; }
    return n;
  }
  return 0;
}
// :1656-1699 edge directions of a mesh feature: the edge itself, or the edge entering the vertex in each of its polygons
static __device__ int mesh_edge_normals(const BoxFeat& f, const CGeom& g, v3* nout, v3* endvert) {
  if (f.dim == 2) { endvert[0] = f.v1; nout[0] = normalize(f.v1 - f.v0); return 1; }
  if (f.dim == 1) {
    const int v1i = f.idx[0];
    const int* m1 = g.polymap + g.polymapadr[v1i];
    const int n = CCD_DEGREES(g.polymapnum[v1i]);
    for (int i = 0; i < n; i++) {
      const int adr = g.polyvertadr[m1[i]], nvert = g.polyvertnum[m1[i]];
      for (int j = 0; j < nvert; j++)
        if (g.polyvert[adr + j] == v1i) {
          const int k = j == 0 ? nvert - 1 : j - 1;
          endvert[i] = matvec(g.rot, ld3(g.vert + 3 * g.polyvert[adr + k])) + g.pos;
          nout[i] = normalize(endvert[i] - f.v0);
        }
    }
    return n;
  }
  return 0;
}
// :1891-1912 a hull polygon in world coordinates, vertex order reversed
static __device__ int mesh_face(const CGeom& g, int idx, v3* face) {
  const int adr = g.polyvertadr[idx], nvert = g.polyvertnum[idx];
  if (!CCD_POLY_FITS(nvert)) return 0;
  int j = 0;
  for (int i = nvert - 1; i >= 0; i--, j++) face[j] = matvec(g.rot, ld3(g.vert + 3 * g.polyvert[adr + i])) + g.pos;
  return nvert;
}
#define CCD_NORMALS(f, g, dir, n, idx) ((g).type == GEOM_BOX ? box_normals(f, (g).rot, dir, n, idx) : mesh_normals(f, g, n, idx))
#define CCD_EDGE_NORMALS(f, g, n, ev) ((g).type == GEOM_BOX ? box_edge_normals(f, g, n, ev) : mesh_edge_normals(f, g, n, ev))
#define CCD_FACE(g, idx, face) ((g).type == GEOM_BOX ? box_face(g, idx, face) : mesh_face(g, idx, face))
#else
#define CCD_NORMALS(f, g, dir, n, idx) box_normals(f, (g).rot, dir, n, idx)
#define CCD_EDGE_NORMALS(f, g, n, ev) box_edge_normals(f, g, n, ev)
#define CCD_FACE(g, idx, face) box_face(g, idx, face)
#endif
#if CCD_MESH == 2
#define CCD_MC_BUF const CcdClip& mc
#else
#define CCD_MC_BUF float* buf
#endif
// :2076 for two boxes (CCD_MESH: boxes and meshes).  Overwrites the witness arrays (4 each) and returns the contact count; buf must not alias
// pt.vert / pt.vidx.
static __device__ int ccd_multicontact(const Polytope& pt, int epa_face, const CGeom& g1, const CGeom& g2, CCD_MC_BUF, v3* w1, v3* w2) {
  const v3 x1 = w1[0], x2 = w2[0];
  for (int k = 1; k < 4; k++) w1[k] = w2[k] = mk3(0.f, 0.f, 0.f);
  const unsigned fw = pt.face[epa_face];
  const int face[3] = {(int)(fw & 0x3FF), (int)((fw >> 10) & 0x3FF), (int)((fw >> 20) & 0x3FF)};
  const BoxFeat f1 = feature_dim(pt, face, 0), f2 = feature_dim(pt, face, 1);
  const v3 ev1 = ld3(pt.vert + 6 * face[0]), ev2 = ld3(pt.vert + 6 * face[0] + 3);
  const v3 dir = x2 - x1;
#if CCD_MESH == 2
  // the buffers in the lane's scratch, in mesh_clip_words order; maxdeg / maxpoly are the model's, at least a box's 3 / 4
  const int maxdeg = mc.maxdeg, clipcap = 2 * mc.maxpoly;
  v3 *n1 = reinterpret_cast<v3*>(mc.buf), *n2 = n1 + maxdeg, *endvert = n2 + maxdeg, *face1 = endvert + maxdeg, *face2 = face1 + mc.maxpoly;
  int *idx1 = reinterpret_cast<int*>(face2 + mc.maxpoly), *idx2 = idx1 + maxdeg;
  float* buf = reinterpret_cast<float*>(idx2 + maxdeg);
  for (int k = 0; k < maxdeg; k++) { idx1[k] = idx2[k] = 0; n1[k] = n2[k] = endvert[k] = mk3(0.f, 0.f, 0.f); }
#else
  v3 n1[CCD_MAXDEG], n2[CCD_MAXDEG], endvert[CCD_MAXDEG];
#if CCD_MESH
  int idx1[CCD_MAXDEG], idx2[CCD_MAXDEG];
  for (int k = 0; k < CCD_MAXDEG; k++) idx1[k] = idx2[k] = 0;
#else
  int idx1[3] = {0, 0, 0}, idx2[3] = {0, 0, 0};
#endif
  for (int k = 0; k < CCD_MAXDEG; k++) n1[k] = n2[k] = endvert[k] = mk3(0.f, 0.f, 0.f);
#endif
  int nn1 = CCD_NORMALS(f1, g1, dir * -1.0f, n1, idx1), nn2 = CCD_NORMALS(f2, g2, dir, n2, idx2);
  bool edge1 = false, edge2 = false, found = false;
  int ri = 0, rj = 0;
  for (int i = 0; i < nn1 && !found; i++) for (int j = 0; j < nn2; j++) if (dot(n1[i], n2[j]) < -CCD_FACE_TOL) { ri = i; rj = j; found = true; break; }
  if (!found) {
    if (f1.dim < 3 && f1.dim <= f2.dim) {  // edge of geom1 against a face of geom2
      nn1 = CCD_EDGE_NORMALS(f1, g1, n1, endvert);
      for (int i = 0; i < nn2 && !found; i++) for (int j = 0; j < nn1; j++) if (fabsf(dot(n1[j], n2[i])) < CCD_EDGE_TOL) { ri = j; rj = i; found = true; break; }
      if (!found) return 1;
      edge1 = true;
    } else if (f2.dim < 3) {  // face of geom1 against an edge of geom2
      nn2 = CCD_EDGE_NORMALS(f2, g2, n2, endvert);
      for (int i = 0; i < nn1 && !found; i++) for (int j = 0; j < nn2; j++) if (fabsf(dot(n2[j], n1[i])) < CCD_EDGE_TOL) { ri = j; rj = i; found = true; break; }
      if (!found) return 1;
      edge2 = true;
    } else return 1;
  }
#if CCD_MESH != 2
  v3 face1[CCD_MAXPOLY], face2[CCD_MAXPOLY];
#endif
  int nface1, nface2;
  if (edge1) { face1[0] = ev1; face1[1] = endvert[ri]; nface1 = 2; } else nface1 = CCD_FACE(g1, edge2 ? idx1[rj] : idx1[ri], face1);
  if (edge2) { face2[0] = ev2; face2[1] = endvert[ri]; nface2 = 2; } else nface2 = CCD_FACE(g2, idx2[rj], face2);
  const float dl = length(dir);
  if (edge1) return polygon_clip(face2, nface2, face1, nface1, n2[rj], n2[rj] * -dl, buf, w2, w1 CCD_CLIPCAP_ARG);  // roles flipped, witnesses flipped back
  if (edge2) return polygon_clip(face1, nface1, face2, nface2, n1[rj], n1[rj] * -dl, buf, w1, w2 CCD_CLIPCAP_ARG);
  return polygon_clip(face1, nface1, face2, nface2, n1[ri], n2[rj] * dl, buf, w1, w2 CCD_CLIPCAP_ARG);
}

// gjk_phase (:2350) + epa_phase (:2421) + multicontact for box pairs.  Returns the number of contacts (0..4, witnesses in
// w1 / w2, 4 each); *dist is relative to the margin-inflated shapes.  CCD_MESH = 2: mc is the lane's multi-contact scratch.
static __device__ __noinline__ int ccd_pair(float tolerance, float cutoff, int gjk_iterations, int epa_iterations, CGeom g1, CGeom g2, float* scratch, float* dist, v3* w1, v3* w2, bool* ovf CCD_CLIP_PARAM) {
  const CGeom o1 = g1, o2 = g2;
  float full1 = 0.f, full2 = 0.f, size1 = 0.f, size2 = 0.f;
#if CCD_MESH
  const bool disc1 = g1.type == GEOM_BOX || g1.type == GEOM_MESH, disc2 = g2.type == GEOM_BOX || g2.type == GEOM_MESH;
  const bool boxes = disc1 && disc2 && g1.margin == 0.f && g2.margin == 0.f;  // :109 _discrete_geoms
#else
  const bool boxes = g1.type == GEOM_BOX && g2.type == GEOM_BOX && g1.margin == 0.f && g2.margin == 0.f;  // :109 _discrete_geoms
#endif
  GjkRes r;
  if (g1.type == GEOM_SPHERE || g1.type == GEOM_CAPSULE) { size1 = g1.size.x; full1 = size1 + 0.5f * g1.margin; g1.margin = 0.f; g1.size.x = 0.f; }
  if (g2.type == GEOM_SPHERE || g2.type == GEOM_CAPSULE) { size2 = g2.size.x; full2 = size2 + 0.5f * g2.margin; g2.margin = 0.f; g2.size.x = 0.f; }
  if (size1 + size2 > 0.f) {
    cutoff += full1 + full2;
    ccd_gjk(tolerance, gjk_iterations, g1, g2, cutoff, boxes, r);
    if (r.dist > tolerance) {
      w1[0] = r.x1; w2[0] = r.x2;
      if (r.dist == CCD_FLOAT_MAX) { *dist = r.dist; return 1; }
      const v3 n = normalize(w2[0] - w1[0]);  // :2303 _inflate
      if (full1 > 0.f) w1[0] = w1[0] + n * full1;
      if (full2 > 0.f) w2[0] = w2[0] - n * full2;
      *dist = r.dist - (full1 + full2);
      return 1;
    }
#if CCD_MESH
    { const int c1 = g1.index, c2 = g2.index; g1 = o1; g2 = o2; g1.index = c1; g2.index = c2; }  // :2392-2403 the cached support vertices stay
#else
    g1 = o1; g2 = o2;
#endif
    cutoff -= full1 + full2;
  }
  ccd_gjk(tolerance, gjk_iterations, g1, g2, cutoff, boxes, r);
  if (r.dist > tolerance || r.dim < 2 || r.separated) { *dist = r.dist; w1[0] = r.x1; w2[0] = r.x2; return 1; }
  Polytope pt;
  const int maxvert = 10 + 2 * epa_iterations;
  pt.maxface = 6 + CCD_MAX_EPAFACES * epa_iterations;
  pt.status = 0; pt.nvert = 0; pt.nface = 0; pt.nhorizon = 0;
  pt.vert = scratch;
  pt.face = (unsigned*)(scratch + 3 * maxvert);
  pt.face_pr = scratch + 3 * maxvert + pt.maxface;
  pt.face_norm2 = pt.face_pr + 3 * pt.maxface;
  pt.horizon = (int*)(pt.face_norm2 + pt.maxface);
  pt.vidx = pt.horizon + CCD_MAX_EPAHORIZON;
  if (r.dim == 2) { polytope2(pt, r, g1, g2); if (pt.status == -1) r.dim = 3; }
  else if (r.dim == 4) { polytope4(pt, r); if (pt.status == -1) r.dim = 3; }
  if (r.dim == 3) { pt.status = 0; polytope3(pt, r, g1, g2); }
  if (pt.status) { *dist = r.dist; w1[0] = r.x1; w2[0] = r.x2; return 1; }
  const int fidx = ccd_epa(tolerance, epa_iterations, pt, g1, g2, boxes, dist, &w1[0], &w2[0], ovf);
  if (fidx == -1) { *dist = CCD_FLOAT_MAX; return 0; }
#if CCD_MESH == 2
  if (boxes && (g1.type != GEOM_MESH || g1.polynum > 0) && (g2.type != GEOM_MESH || g2.polynum > 0)) return ccd_multicontact(pt, fidx, g1, g2, mc, w1, w2);
#elif CCD_MESH
  if (boxes && (g1.type != GEOM_MESH || g1.polynum > 0) && (g2.type != GEOM_MESH || g2.polynum > 0)) {  // a mesh without polygon data keeps one contact
    float clipbuf[2 * 3 * CCD_CLIPCAP];
    return ccd_multicontact(pt, fidx, g1, g2, clipbuf, w1, w2);
  }
#else
  if (boxes) return ccd_multicontact(pt, fidx, g1, g2, pt.face_pr, w1, w2);  // face_pr (>= 108 words) is free once EPA is done
#endif
  return 1;
}

#if CCD_MESH
// collision_primitive.py:52-277 plane_convex for a mesh: up to four well-spread hull vertices that lie (nearly) deepest below the plane.
// pass 0: deepest vertex a; 1: farthest from a; 2: farthest from the line a-b; 3: farthest from the triangle's other two edges -- candidates
// restricted to vertices within 1e-3 of the deepest.  Exhaustive over the vertex block, or hill climbing on the hull graph.
#define PM_HUGE 1e6f
static __device__ __forceinline__ float pm_support(v3 ppl, v3 v, v3 n) { return dot(ppl - v, n); }
static __device__ __forceinline__ float pm_score(int pass, v3 v, v3 a, v3 b, v3 ab, v3 ac, v3 bc, float sup, float threshold) {
  const float mask = sup > threshold ? 0.f : -PM_HUGE;
  if (pass == 1) { const v3 df = a - v; return dot(df, df) + mask; }
  if (pass == 2) return fabsf(dot(a - v, ab)) + mask;
  return (fabsf(dot(a - v, ac)) + mask) + (fabsf(dot(b - v, bc)) + mask);
}
static __device__ int plane_mesh(v3 n_world, v3 plane_pos, const CGeom& c, float* dist, v3* pos) {
  int idx[4] = {-1, -1, -1, -1};
  for (int i = 0; i < 4; i++) { dist[i] = MJ_MAXVAL; pos[i] = mk3(0.f, 0.f, 0.f); }
  const v3 ppl = mat_t_vec(c.rot, plane_pos - c.pos), n = mat_t_vec(c.rot, n_world);
  v3 a = mk3(0.f, 0.f, 0.f), b = a, cc = a, ab = a, ac = a, bc = a;
  if (!c.graph || c.vertnum < 10) {
    float max_support = -PM_HUGE;
    for (int i = 0; i < c.vertnum; i++) { const v3 v = ld3(c.vert + 3 * i); const float s = pm_support(ppl, v, n); if (s > max_support) { max_support = s; idx[0] = i; a = v; } }
    if (max_support < 0.f) return 0;
    const float threshold = max_support - 1e-3f;
    for (int pass = 1; pass < 4; pass++) {
      float best = -PM_HUGE;
      v3 pick = mk3(0.f, 0.f, 0.f);
      for (int i = 0; i < c.vertnum; i++) {
        const v3 v = ld3(c.vert + 3 * i);
        const float dd = pm_score(pass, v, a, b, ab, ac, bc, pm_support(ppl, v, n), threshold);
        if (dd > best) { idx[pass] = i; best = dd; pick = v; }
      }
      if (pass == 1) { b = pick; ab = cross(n, a - b); }
      else if (pass == 2) { cc = pick; ac = cross(n, a - cc); bc = cross(n, b - cc); }
    }
  } else {
    const int numvert = c.graph[0];
    const int *vert_edgeadr = c.graph + 2, *vert_globalid = c.graph + 2 + numvert, *edge_localid = c.graph + 2 + 2 * numvert;
    float max_support = -PM_HUGE;
    int prev, imax = 0;
    for (;;) {  // hill climb to the deepest vertex
      prev = imax;
      for (int i = vert_edgeadr[imax]; edge_localid[i] >= 0; i++) {
        const int sub = edge_localid[i];
        const float s = pm_support(ppl, ld3(c.vert + 3 * vert_globalid[sub]), n);
        if (s > max_support) { max_support = s; imax = sub; }
      }
      if (imax == prev) break;
    }
    const float threshold = fmaxf(0.f, max_support - 1e-3f);
    float best = -PM_HUGE;
    for (;;) {
      prev = imax;
      for (int i = vert_edgeadr[imax]; edge_localid[i] >= 0; i++) {
        const int sub = edge_localid[i];
        const float s = pm_support(ppl, ld3(c.vert + 3 * vert_globalid[sub]), n);
        const float dd = s > threshold ? s : -PM_HUGE;
        if (dd > best) { best = dd; imax = sub; }
      }
      if (imax == prev) break;
    }
    a = ld3(c.vert + 3 * vert_globalid[imax]); idx[0] = vert_globalid[imax];
    for (int pass = 1; pass < 4; pass++) {
      best = -PM_HUGE;
      for (;;) {
        prev = imax;
        for (int i = vert_edgeadr[imax]; edge_localid[i] >= 0; i++) {
          const int sub = edge_localid[i];
          const v3 v = ld3(c.vert + 3 * vert_globalid[sub]);
          const float dd = pm_score(pass, v, a, b, ab, ac, bc, pm_support(ppl, v, n), threshold);
          if (dd > best) { best = dd; imax = sub; }
        }
        if (imax == prev) break;
      }
      idx[pass] = vert_globalid[imax];
      const v3 pick = ld3(c.vert + 3 * vert_globalid[imax]);
      if (pass == 1) { b = pick; ab = cross(n, a - b); }
      else if (pass == 2) { cc = pick; ac = cross(n, a - cc); bc = cross(n, b - cc); }
    }
  }
  int count = 0;
  for (int i = 3; i >= 0; i--) {  // unique vertices, last first
    int uniq = 0;
    for (int j = 0; j <= i; j++) if (idx[j] == idx[i]) uniq++;
    if (uniq != 1) continue;
    const v3 v = ld3(c.vert + 3 * idx[i]);
    const float dd = -pm_support(ppl, v, n);
    pos[count] = c.pos + matvec(c.rot, v) - n_world * (0.5f * dd);
    dist[count] = dd;
    count++;
  }
  return count;
}
#endif
