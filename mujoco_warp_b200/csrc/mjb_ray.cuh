// mjb_ray.cuh -- intersection of one ray with one geom (fp32), and the closest-hit scan over a world's geoms, shared by k_ray (mjw.ray / mjw.rays),
// the rangefinder sensor (k_sensor_rangefinder) and the touch sensor (k_sensor).
//
// Restates the reference's ray.py (/root/reference/mujoco_warp/_src/ray.py) in its operation order: :33 _ray_map, :53 _ray_eliminate,
// :106 _ray_quad, :129 _orthogonal_basis, :155 _ray_triangle, :214 ray_plane, :238 ray_sphere, :255 ray_capsule, :329 ray_ellipsoid,
// :360 ray_cylinder, :421 ray_box, :629 ray_mesh, :799 ray_geom.  Every routine returns the distance along `vec` (in units of |vec|)
// to the first intersection, -1 if none; with NORMAL it also writes the world-frame surface normal there (zero on a miss).  The
// distance-only instances (NORMAL = false) are the arithmetic the touch sensor has always done.
//
// Scalar code, one ray per thread: compiles as plain host C++ too (tests/host_harness/ray_host.cpp).
#pragma once
#include "mjb_math.cuh"
#include "mjb_types.cuh"

static __device__ __forceinline__ float ray_comp3(v3 v, int i) { return i == 0 ? v.x : (i == 1 ? v.y : v.z); }
static __device__ __forceinline__ v3 ray_zero3() { return mk3(0.f, 0.f, 0.f); }

// :33 _ray_map: ray in the geom frame (mat^T (pnt - pos), mat^T vec)
static __device__ __forceinline__ v3 ray_mat_t_vec(const float* m, v3 v) {
  return mk3(m[0] * v.x + m[3] * v.y + m[6] * v.z, m[1] * v.x + m[4] * v.y + m[7] * v.z, m[2] * v.x + m[5] * v.y + m[8] * v.z);
}

// :106 _ray_quad: smallest non-negative root of a x^2 + 2 b x + c = 0 (both roots in x2), -1 if none
static __device__ float ray_quad(float a, float b, float c, float* x2) {
  float det = b * b - a * c;
  x2[0] = x2[1] = -1.f;
  if (det < MJ_MINVAL) return -1.f;
  det = sqrtf(det);
  const float den = a != 0.f ? 1.0f / a : 0.f;
  x2[0] = (-b - det) * den; x2[1] = (-b + det) * den;
  return x2[0] >= 0.f ? x2[0] : (x2[1] >= 0.f ? x2[1] : -1.f);
}

// :238
template <bool NORMAL>
static __device__ float ray_sphere(v3 pos, float dist_sqr, v3 pnt, v3 vec, v3* normal) {
  const v3 dif = pnt - pos;
  float xx[2];
  const float sol = ray_quad(dot(vec, vec), dot(vec, dif), dot(dif, dif) - dist_sqr, xx);
  if (NORMAL && sol >= 0.f) *normal = normalize(pnt + vec * sol - pos);
  return sol;
}

// :214 (size x / y <= 0: infinite in that direction)
template <bool NORMAL>
static __device__ __forceinline__ float ray_plane(const float* mat, v3 size, v3 lpnt, v3 lvec, v3* normal) {
  if (lvec.z > -MJ_MINVAL) return -1.f;  // not pointing at the front face
  const float x = -lpnt.z / lvec.z;
  if (x < 0.f) return -1.f;
  const float p0 = lpnt.x + x * lvec.x, p1 = lpnt.y + x * lvec.y;
  if ((size.x <= 0.f || fabsf(p0) <= size.x) && (size.y <= 0.f || fabsf(p1) <= size.y)) {
    if (NORMAL) *normal = mk3(mat[2], mat[5], mat[8]);
    return x;
  }
  return -1.f;
}

// :255 (after the bounding-sphere test)
template <bool NORMAL>
static __device__ __forceinline__ float ray_capsule(const float* mat, v3 size, v3 lpnt, v3 lvec, v3* normal) {
  float xx[2];
  float x = -1.f;
  int part = 0;  // -1 bottom cap, 0 cylinder, 1 top cap
  const float sq = size.x * size.x;
  float a = lvec.x * lvec.x + lvec.y * lvec.y, b = lvec.x * lpnt.x + lvec.y * lpnt.y, c = lpnt.x * lpnt.x + lpnt.y * lpnt.y - sq;
  const float sol = ray_quad(a, b, c, xx);
  if (sol >= 0.f && fabsf(lpnt.z + sol * lvec.z) <= size.y) if (x < 0.f || sol < x) x = sol;
  v3 ldif = mk3(lpnt.x, lpnt.y, lpnt.z - size.y);
  a += lvec.z * lvec.z; b = dot(lvec, ldif); c = dot(ldif, ldif) - sq;
  ray_quad(a, b, c, xx);
  for (int i = 0; i < 2; i++) if (xx[i] >= 0.f && lpnt.z + xx[i] * lvec.z >= size.y) if (x < 0.f || xx[i] < x) { x = xx[i]; part = 1; }
  ldif.z = lpnt.z + size.y;
  b = dot(lvec, ldif); c = dot(ldif, ldif) - sq;
  ray_quad(a, b, c, xx);
  for (int i = 0; i < 2; i++) if (xx[i] >= 0.f && lpnt.z + xx[i] * lvec.z <= -size.y) if (x < 0.f || xx[i] < x) { x = xx[i]; part = -1; }
  if (NORMAL && x >= 0.f) {
    const v3 n = mk3(lpnt.x + lvec.x * x, lpnt.y + lvec.y * x, part == 0 ? 0.f : lpnt.z + lvec.z * x - size.y * (float)part);
    *normal = matvec(mat, normalize(n));
  }
  return x;
}

// :329
template <bool NORMAL>
static __device__ __forceinline__ float ray_ellipsoid(const float* mat, v3 size, v3 lpnt, v3 lvec, v3* normal) {
  float xx[2];
  const v3 si = mk3(size.x != 0.f ? 1.0f / (size.x * size.x) : 0.f, size.y != 0.f ? 1.0f / (size.y * size.y) : 0.f, size.z != 0.f ? 1.0f / (size.z * size.z) : 0.f);
  const v3 sv = mk3(si.x * lvec.x, si.y * lvec.y, si.z * lvec.z), sp = mk3(si.x * lpnt.x, si.y * lpnt.y, si.z * lpnt.z);
  const float sol = ray_quad(dot(sv, lvec), dot(sv, lpnt), dot(sp, lpnt) - 1.0f, xx);
  if (NORMAL && sol >= 0.f) {
    const v3 l = lpnt + lvec * sol;
    *normal = matvec(mat, normalize(mk3(si.x * l.x, si.y * l.y, si.z * l.z)));
  }
  return sol;
}

// :360 (after the bounding-sphere test)
template <bool NORMAL>
static __device__ __forceinline__ float ray_cylinder(const float* mat, v3 size, v3 lpnt, v3 lvec, v3* normal) {
  float xx[2];
  float x = -1.f;
  int part = 0;  // -1 bottom, 0 side, 1 top
  if (fabsf(lvec.z) > MJ_MINVAL)
    for (int side = -1; side <= 1; side += 2) {
      const float sol = ((float)side * size.y - lpnt.z) / lvec.z;
      if (sol >= 0.f) {
        const float p0 = lpnt.x + sol * lvec.x, p1 = lpnt.y + sol * lvec.y;
        if (p0 * p0 + p1 * p1 <= size.x * size.x) if (x < 0.f || sol < x) { x = sol; part = side; }
      }
    }
  const float a = lvec.x * lvec.x + lvec.y * lvec.y, b = lvec.x * lpnt.x + lvec.y * lpnt.y, c = lpnt.x * lpnt.x + lpnt.y * lpnt.y - size.x * size.x;
  const float sol = ray_quad(a, b, c, xx);
  if (sol >= 0.f && fabsf(lpnt.z + sol * lvec.z) <= size.y) if (x < 0.f || sol < x) { x = sol; part = 0; }
  if (NORMAL && x >= 0.f) {
    const v3 n = part == 0 ? normalize(mk3(lpnt.x + lvec.x * x, lpnt.y + lvec.y * x, 0.f)) : mk3(0.f, 0.f, (float)part);
    *normal = matvec(mat, n);
  }
  return x;
}

// :421 in the geom frame (after the bounding-sphere test)
template <bool NORMAL>
static __device__ __forceinline__ float ray_box_local(const float* mat, v3 size, v3 lpnt, v3 lvec, v3* normal) {
  float x = -1.f;
  int face_axis = -1;
  float face_side = 0.f;
  for (int i = 0; i < 3; i++) {
    const float lv = ray_comp3(lvec, i);
    if (fabsf(lv) <= MJ_MINVAL) continue;
    for (int side = -1; side <= 1; side += 2) {
      const float sol = ((float)side * ray_comp3(size, i) - ray_comp3(lpnt, i)) / lv;
      if (sol < 0.f) continue;
      const int id0 = i == 0 ? 1 : 0, id1 = i == 2 ? 1 : 2;
      const float p0 = ray_comp3(lpnt, id0) + sol * ray_comp3(lvec, id0), p1 = ray_comp3(lpnt, id1) + sol * ray_comp3(lvec, id1);
      if (fabsf(p0) <= ray_comp3(size, id0) && fabsf(p1) <= ray_comp3(size, id1)) if (x < 0.f || sol < x) { x = sol; face_axis = i; face_side = (float)side; }
    }
  }
  if (NORMAL && x >= 0.f) *normal = matcol(mat, face_axis) * face_side;  // mat @ (face_side e_axis)
  return x;
}

// :421 with its bounding-sphere test (the mesh pre-test of :629)
template <bool NORMAL>
static __device__ __forceinline__ float ray_box(v3 pos, const float* mat, v3 size, v3 pnt, v3 vec, v3* normal) {
  if (ray_sphere<false>(pos, dot(size, size), pnt, vec, nullptr) < 0.f) return -1.f;
  return ray_box_local<NORMAL>(mat, size, ray_mat_t_vec(mat, pnt - pos), ray_mat_t_vec(mat, vec), normal);
}

// :799 ray_geom for the primitive types (plane, sphere, capsule, ellipsoid, cylinder, box); -1 for any other type
template <bool NORMAL>
static __device__ __forceinline__ float ray_geom(v3 pos, const float* mat, v3 size, v3 pnt, v3 vec, int type, v3* normal) {
  if (NORMAL) *normal = ray_zero3();
  if (type == GEOM_SPHERE) return ray_sphere<NORMAL>(pos, size.x * size.x, pnt, vec, normal);
  const v3 lpnt = ray_mat_t_vec(mat, pnt - pos), lvec = ray_mat_t_vec(mat, vec);
  if (type == GEOM_CAPSULE) {
    const float ssz = size.x + size.y;
    if (ray_sphere<false>(pos, ssz * ssz, pnt, vec, nullptr) < 0.f) return -1.f;
    return ray_capsule<NORMAL>(mat, size, lpnt, lvec, normal);
  }
  if (type == GEOM_ELLIPSOID) return ray_ellipsoid<NORMAL>(mat, size, lpnt, lvec, normal);
  if (type == GEOM_CYLINDER) {
    if (ray_sphere<false>(pos, size.x * size.x + size.y * size.y, pnt, vec, nullptr) < 0.f) return -1.f;
    return ray_cylinder<NORMAL>(mat, size, lpnt, lvec, normal);
  }
  if (type == GEOM_BOX) {
    if (ray_sphere<false>(pos, dot(size, size), pnt, vec, nullptr) < 0.f) return -1.f;
    return ray_box_local<NORMAL>(mat, size, lpnt, lvec, normal);
  }
  if (type == GEOM_PLANE) return ray_plane<NORMAL>(mat, size, lpnt, lvec, normal);
  return -1.f;
}

// :129 _orthogonal_basis: two unit vectors orthogonal to the unit vector v (Duff et al. 2017)
static __device__ __forceinline__ void ray_orthogonal_basis(v3 v, v3* b0, v3* b1) {
  const float sign = v.z >= 0.f ? 1.f : -1.f;
  const float a = -1.0f / (sign + v.z);
  const float b = v.x * v.y * a;
  *b0 = mk3(1.0f + sign * v.x * v.x * a, sign * b, -sign * v.x);
  *b1 = mk3(b, sign + v.y * v.y * a, -v.y);
}

// :155 _ray_triangle (triangle and ray in one frame; b0, b1 span the plane normal to the ray); the normal is only valid on a hit
static __device__ __forceinline__ float ray_triangle(v3 v0, v3 v1, v3 v2, v3 pnt, v3 vec, v3 b0, v3 b1, v3* normal) {
  v3 dif0 = v0 - pnt, dif1 = v1 - pnt, dif2 = v2 - pnt;
  const float p00 = dot(dif0, b0), p01 = dot(dif0, b1), p10 = dot(dif1, b0), p11 = dot(dif1, b1), p20 = dot(dif2, b0), p21 = dot(dif2, b1);
  // reject if all three lie on one side of either axis
  if ((p00 > 0.f && p10 > 0.f && p20 > 0.f) || (p00 < 0.f && p10 < 0.f && p20 < 0.f) || (p01 > 0.f && p11 > 0.f && p21 > 0.f) ||
      (p01 < 0.f && p11 < 0.f && p21 < 0.f))
    return -1.f;
  // is the origin inside the planar projection: A = (p0 - p2, p1 - p2), solve A t = -p2
  const float A00 = p00 - p20, A10 = p10 - p20, A01 = p01 - p21, A11 = p11 - p21;
  const float bb0 = -p20, bb1 = -p21;
  const float det = A00 * A11 - A10 * A01;
  if (fabsf(det) < MJ_MINVAL) return -1.f;
  const float t0 = (A11 * bb0 - A10 * bb1) / det, t1 = (-A01 * bb0 + A00 * bb1) / det;
  if (t0 < 0.f || t1 < 0.f || t0 + t1 > 1.0f) return -1.f;
  // intersect with the triangle's plane
  dif0 = v0 - v2; dif1 = v1 - v2; dif2 = pnt - v2;
  const v3 nrm = cross(dif0, dif1);
  const float denom = dot(vec, nrm);
  if (fabsf(denom) < MJ_MINVAL) return -1.f;
  const float dist = -dot(dif2, nrm) / denom;
  *normal = normalize(nrm);
  return dist >= 0.f ? dist : -1.f;
}

// :629 ray_mesh after its bounding-box test: every triangle of faces [f0, f1) of the mesh whose vertices start at `vert`
static __device__ __forceinline__ float ray_mesh_faces(const int* __restrict__ face, int f0, int f1, const float* __restrict__ vert, v3 pos, const float* mat,
                                                       v3 pnt, v3 vec, v3* normal) {
  const v3 lpnt = ray_mat_t_vec(mat, pnt - pos), lvec = ray_mat_t_vec(mat, vec);
  v3 b0, b1;
  ray_orthogonal_basis(lvec, &b0, &b1);
  float x = -1.f;
  v3 n = ray_zero3();
#pragma unroll 1
  for (int i = f0; i < f1; i++) {
    const int* f = face + 3 * i;
    v3 nt;
    const float dist = ray_triangle(ld3(vert + 3 * f[0]), ld3(vert + 3 * f[1]), ld3(vert + 3 * f[2]), lpnt, lvec, b0, b1, &nt);
    if (dist >= 0.f && (x < 0.f || dist < x)) { x = dist; n = nt; }
  }
  *normal = matvec(mat, n);
  return x;
}

// face range of mesh `id`: [mesh_faceadr[id], mesh_faceadr[id + 1] or nmeshface)
static __device__ __forceinline__ void ray_mesh_range(const ModelDev& m, int id, int* f0, int* f1) {
  *f0 = m.mesh_faceadr[id];
  *f1 = id + 1 < m.nmesh ? m.mesh_faceadr[id + 1] : m.nmeshface;
}

// :629 ray_mesh
static __device__ __forceinline__ float ray_mesh(const ModelDev& m, int id, v3 pos, const float* mat, v3 size, v3 pnt, v3 vec, v3* normal) {
  *normal = ray_zero3();
  if (ray_box<false>(pos, mat, size, pnt, vec, nullptr) < 0.f) return -1.f;
  int f0, f1;
  ray_mesh_range(m, id, &f0, &f1);
  return ray_mesh_faces(m.mesh_face, f0, f1, m.mesh_vert + 3 * m.mesh_vertadr[id], pos, mat, pnt, vec, normal);
}

// :53 _ray_eliminate: true if geom g is excluded from the ray (its body, invisible geom or material, static, or group filter).
// `m` is the model as the ray's world sees it (geom_rgba / mat_rgba of the world's batch entry).
struct RayFilter { int geomgroup[6]; int flg_static; };
static __device__ __forceinline__ bool ray_eliminate(const ModelDev& m, int g, const RayFilter& f, int bodyexclude) {
  const int body = m.geom_bodyid[g], matid = m.geom_matid[g];
  if (body == bodyexclude) return true;
  if (matid < 0 && m.geom_rgba[4 * g + 3] == 0.f) return true;
  if (matid >= 0 && m.mat_rgba[4 * matid + 3] == 0.f) return true;
  if (!f.flg_static && m.body_weldid[body] == 0) return true;
  const int* gg = f.geomgroup;
  if (gg[0] == -1 && gg[1] == -1 && gg[2] == -1 && gg[3] == -1 && gg[4] == -1 && gg[5] == -1) return false;
  const int grp = min(5, max(0, m.geom_group[g]));
  return gg[grp] == 0;
}

// :822 _ray_geom_mesh (without height fields): one geom of one world, eliminated geoms miss
static __device__ __forceinline__ float ray_world_geom(const ModelDev& m, const float* geom_xpos, const float* geom_xmat, int g, const RayFilter& f, int bodyexclude,
                                                       v3 pnt, v3 vec, v3* normal) {
  *normal = ray_zero3();
  if (ray_eliminate(m, g, f, bodyexclude)) return -1.f;
  const v3 pos = ld3(geom_xpos + 3 * g), size = ld3(m.geom_size + 3 * g);
  const float* mat = geom_xmat + 9 * g;
  if (m.geom_type[g] == GEOM_MESH) return ray_mesh(m, m.geom_dataid[g], pos, mat, size, pnt, vec, normal);
  return ray_geom<true>(pos, mat, size, pnt, vec, m.geom_type[g], normal);
}

// The warp vote of the scan below; compiled as host C++ each ray is its own warp
static __device__ __forceinline__ bool ray_warp_any(bool v) {
#ifdef __CUDA_ARCH__
  return __any_sync(FULL_MASK, v);
#else
  return v;
#endif
}

// :907 _ray's closest-hit scan for one ray of world geoms (geom_xpos / geom_xmat of the world), shared by k_ray and k_sensor_rangefinder.
// Every lane of the warp must call it (`live` false for lanes past the last ray, which keep the warp-wide vote of the mesh path
// complete): geoms are visited in ascending order and the closest hit is replaced only on a strictly smaller distance, so ties go to
// the lowest geom id.  Returns the distance (-1 on a miss), with the geom id (-1) and world-frame normal (zero) of the hit.
// MESH: the model has meshes (the triangle path is compiled in); `m` is the model as the ray's world sees it.
template <bool MESH>
static __device__ __forceinline__ float ray_scan(const ModelDev& m, const float* xpos, const float* xmat, const RayFilter& filter, int bodyexclude, bool live,
                                                 v3 p, v3 v, int* geomid, v3* normal) {
  float best = MJ_MAXVAL;
  int best_g = -1;
  v3 best_n = ray_zero3();
#pragma unroll 1
  for (int g = 0; g < m.ngeom; g++) {
    const bool skip = !live || ray_eliminate(m, g, filter, bodyexclude);
    const int type = m.geom_type[g];
    const v3 pos = ld3(xpos + 3 * g), size = ld3(m.geom_size + 3 * g);
    const float* mat = xmat + 9 * g;
    float x = -1.f;
    v3 n = ray_zero3();
    if (MESH && type == GEOM_MESH) {
      // ray.py:646 bounding-box test; the warp skips the triangles when no lane's ray enters the box
      const bool inbox = !skip && ray_box<false>(pos, mat, size, p, v, nullptr) >= 0.f;
      if (ray_warp_any(inbox) && inbox) {
        const int id = m.geom_dataid[g];
        int f0, f1;
        ray_mesh_range(m, id, &f0, &f1);
        x = ray_mesh_faces(m.mesh_face, f0, f1, m.mesh_vert + 3 * m.mesh_vertadr[id], pos, mat, p, v, &n);
      }
    } else if (!skip) {
      x = ray_geom<true>(pos, mat, size, p, v, type, &n);
    }
    if (x >= 0.f && x < best) { best = x; best_g = g; best_n = n; }
  }
  *geomid = best_g;
  *normal = best_n;
  return best_g >= 0 ? best : -1.f;
}
