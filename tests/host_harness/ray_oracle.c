/* ray_oracle.c -- TEST INFRASTRUCTURE ONLY: a plain-C restatement of the reference's ray casting (ray.py:33-1011: _ray_map,
 * _ray_eliminate, _ray_quad, _orthogonal_basis, _ray_triangle, ray_plane / sphere / capsule / ellipsoid / cylinder / box / mesh,
 * ray_geom and the closest-hit scan of _ray), written independently of the CUDA header mujoco_warp_b200/csrc/mjb_ray.cuh.
 * real = double by default; -DORC_FLOAT builds the fp32 twin.  The geom poses are arguments (no kinematics is run), so a test can
 * feed it the GPU's own geom_xpos / geom_xmat and compare only the ray arithmetic.  OpenMP over worlds. */
#include <math.h>
#include <string.h>

#ifdef ORC_FLOAT
typedef float real;
#else
typedef double real;
#endif

#define MINVAL ((real)1e-15)
#define MAXVAL ((real)1e10)
enum { PLANE = 0, SPHERE = 2, CAPSULE = 3, ELLIPSOID = 4, CYLINDER = 5, BOX = 6, MESH = 7 };

int ray_oracle_sizeof_real(void) { return (int)sizeof(real); }

static real dot3(const real* a, const real* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }
static void zero3(real* a) { a[0] = a[1] = a[2] = 0; }
static void normalize3(real* a) {
  const real l = (real)sqrt((double)dot3(a, a));
  if (l > 0) { a[0] /= l; a[1] /= l; a[2] /= l; } else zero3(a);
}
static void mat_vec(const real* m, const real* v, real* o) {  /* o = m v (row-major) */
  real r[3];
  for (int i = 0; i < 3; i++) r[i] = m[3 * i] * v[0] + m[3 * i + 1] * v[1] + m[3 * i + 2] * v[2];
  memcpy(o, r, sizeof r);
}
static void mat_t_vec(const real* m, const real* v, real* o) {  /* o = m^T v */
  real r[3];
  for (int i = 0; i < 3; i++) r[i] = m[i] * v[0] + m[3 + i] * v[1] + m[6 + i] * v[2];
  memcpy(o, r, sizeof r);
}
static void ray_map(const real* pos, const real* mat, const real* pnt, const real* vec, real* lpnt, real* lvec) {
  real d[3] = {pnt[0] - pos[0], pnt[1] - pos[1], pnt[2] - pos[2]};
  mat_t_vec(mat, d, lpnt);
  mat_t_vec(mat, vec, lvec);
}
static real quad(real a, real b, real c, real* x) {
  real det = b * b - a * c;
  x[0] = x[1] = -1;
  if (det < MINVAL) return -1;
  det = (real)sqrt((double)det);
  const real den = a != 0 ? (real)1 / a : 0;
  x[0] = (-b - det) * den;
  x[1] = (-b + det) * den;
  if (x[0] >= 0) return x[0];
  if (x[1] >= 0) return x[1];
  return -1;
}
static real sphere(const real* pos, real r2, const real* pnt, const real* vec, real* n) {
  real dif[3] = {pnt[0] - pos[0], pnt[1] - pos[1], pnt[2] - pos[2]}, x[2];
  const real sol = quad(dot3(vec, vec), dot3(vec, dif), dot3(dif, dif) - r2, x);
  zero3(n);
  if (sol >= 0) {
    for (int i = 0; i < 3; i++) n[i] = pnt[i] + vec[i] * sol - pos[i];
    normalize3(n);
  }
  return sol;
}
static real plane(const real* pos, const real* mat, const real* size, const real* pnt, const real* vec, real* n) {
  real lp[3], lv[3];
  ray_map(pos, mat, pnt, vec, lp, lv);
  zero3(n);
  if (lv[2] > -MINVAL) return -1;
  const real x = -lp[2] / lv[2];
  if (x < 0) return -1;
  const real p0 = lp[0] + x * lv[0], p1 = lp[1] + x * lv[1];
  if ((size[0] <= 0 || fabs(p0) <= size[0]) && (size[1] <= 0 || fabs(p1) <= size[1])) {
    n[0] = mat[2]; n[1] = mat[5]; n[2] = mat[8];
    return x;
  }
  return -1;
}
static real capsule(const real* pos, const real* mat, const real* size, const real* pnt, const real* vec, real* n) {
  const real ssz = size[0] + size[1];
  if (sphere(pos, ssz * ssz, pnt, vec, n) < 0) { zero3(n); return -1; }
  zero3(n);
  real lp[3], lv[3], xx[2];
  ray_map(pos, mat, pnt, vec, lp, lv);
  real x = -1;
  int part = 0;
  const real sq = size[0] * size[0];
  real a = lv[0] * lv[0] + lv[1] * lv[1], b = lv[0] * lp[0] + lv[1] * lp[1], c = lp[0] * lp[0] + lp[1] * lp[1] - sq;
  const real sol = quad(a, b, c, xx);
  if (sol >= 0 && fabs(lp[2] + sol * lv[2]) <= size[1] && (x < 0 || sol < x)) x = sol;
  real ld[3] = {lp[0], lp[1], lp[2] - size[1]};
  a += lv[2] * lv[2];
  b = dot3(lv, ld);
  c = dot3(ld, ld) - sq;
  quad(a, b, c, xx);
  for (int i = 0; i < 2; i++)
    if (xx[i] >= 0 && lp[2] + xx[i] * lv[2] >= size[1] && (x < 0 || xx[i] < x)) { x = xx[i]; part = 1; }
  ld[2] = lp[2] + size[1];
  b = dot3(lv, ld);
  c = dot3(ld, ld) - sq;
  quad(a, b, c, xx);
  for (int i = 0; i < 2; i++)
    if (xx[i] >= 0 && lp[2] + xx[i] * lv[2] <= -size[1] && (x < 0 || xx[i] < x)) { x = xx[i]; part = -1; }
  if (x >= 0) {
    real l[3] = {lp[0] + lv[0] * x, lp[1] + lv[1] * x, part == 0 ? 0 : lp[2] + lv[2] * x - size[1] * (real)part};
    normalize3(l);
    mat_vec(mat, l, n);
  }
  return x;
}
static real ellipsoid(const real* pos, const real* mat, const real* size, const real* pnt, const real* vec, real* n) {
  real lp[3], lv[3], xx[2], s[3], sv[3], sp[3];
  ray_map(pos, mat, pnt, vec, lp, lv);
  for (int i = 0; i < 3; i++) {
    const real q = size[i] * size[i];
    s[i] = q != 0 ? (real)1 / q : 0;
    sv[i] = s[i] * lv[i];
    sp[i] = s[i] * lp[i];
  }
  const real sol = quad(dot3(sv, lv), dot3(sv, lp), dot3(sp, lp) - 1, xx);
  zero3(n);
  if (sol >= 0) {
    real g[3];
    for (int i = 0; i < 3; i++) g[i] = s[i] * (lp[i] + lv[i] * sol);
    normalize3(g);
    mat_vec(mat, g, n);
  }
  return sol;
}
static real cylinder(const real* pos, const real* mat, const real* size, const real* pnt, const real* vec, real* n) {
  if (sphere(pos, size[0] * size[0] + size[1] * size[1], pnt, vec, n) < 0) { zero3(n); return -1; }
  zero3(n);
  real lp[3], lv[3], xx[2];
  ray_map(pos, mat, pnt, vec, lp, lv);
  real x = -1;
  int part = 0;
  if (fabs(lv[2]) > MINVAL)
    for (int side = -1; side <= 1; side += 2) {
      const real sol = ((real)side * size[1] - lp[2]) / lv[2];
      if (sol >= 0) {
        const real p0 = lp[0] + sol * lv[0], p1 = lp[1] + sol * lv[1];
        if (p0 * p0 + p1 * p1 <= size[0] * size[0] && (x < 0 || sol < x)) { x = sol; part = side; }
      }
    }
  const real a = lv[0] * lv[0] + lv[1] * lv[1], b = lv[0] * lp[0] + lv[1] * lp[1], c = lp[0] * lp[0] + lp[1] * lp[1] - size[0] * size[0];
  const real sol = quad(a, b, c, xx);
  if (sol >= 0 && fabs(lp[2] + sol * lv[2]) <= size[1] && (x < 0 || sol < x)) { x = sol; part = 0; }
  if (x >= 0) {
    real l[3] = {0, 0, (real)part};
    if (part == 0) { l[0] = lp[0] + lv[0] * x; l[1] = lp[1] + lv[1] * x; l[2] = 0; normalize3(l); }
    mat_vec(mat, l, n);
  }
  return x;
}
static real box(const real* pos, const real* mat, const real* size, const real* pnt, const real* vec, real* n) {
  if (sphere(pos, dot3(size, size), pnt, vec, n) < 0) { zero3(n); return -1; }
  zero3(n);
  real lp[3], lv[3];
  ray_map(pos, mat, pnt, vec, lp, lv);
  real x = -1;
  int axis = -1, fside = 0;
  for (int i = 0; i < 3; i++) {
    if (!(fabs(lv[i]) > MINVAL)) continue;
    for (int side = -1; side <= 1; side += 2) {
      const real sol = ((real)side * size[i] - lp[i]) / lv[i];
      if (sol < 0) continue;
      const int i0 = i == 0 ? 1 : 0, i1 = i == 2 ? 1 : 2;
      const real p0 = lp[i0] + sol * lv[i0], p1 = lp[i1] + sol * lv[i1];
      if (fabs(p0) <= size[i0] && fabs(p1) <= size[i1] && (x < 0 || sol < x)) { x = sol; axis = i; fside = side; }
    }
  }
  if (x >= 0) {
    real l[3] = {0, 0, 0};
    l[axis] = (real)fside;
    mat_vec(mat, l, n);
  }
  return x;
}
static real triangle(const real* v0, const real* v1, const real* v2, const real* pnt, const real* vec, const real* b0, const real* b1, real* n) {
  real d0[3], d1[3], d2[3];
  for (int i = 0; i < 3; i++) { d0[i] = v0[i] - pnt[i]; d1[i] = v1[i] - pnt[i]; d2[i] = v2[i] - pnt[i]; }
  const real p00 = dot3(d0, b0), p01 = dot3(d0, b1), p10 = dot3(d1, b0), p11 = dot3(d1, b1), p20 = dot3(d2, b0), p21 = dot3(d2, b1);
  if ((p00 > 0 && p10 > 0 && p20 > 0) || (p00 < 0 && p10 < 0 && p20 < 0) || (p01 > 0 && p11 > 0 && p21 > 0) || (p01 < 0 && p11 < 0 && p21 < 0)) return -1;
  const real A00 = p00 - p20, A10 = p10 - p20, A01 = p01 - p21, A11 = p11 - p21, bb0 = -p20, bb1 = -p21;
  const real det = A00 * A11 - A10 * A01;
  if (fabs(det) < MINVAL) return -1;
  const real t0 = (A11 * bb0 - A10 * bb1) / det, t1 = (-A01 * bb0 + A00 * bb1) / det;
  if (t0 < 0 || t1 < 0 || t0 + t1 > 1) return -1;
  real e0[3], e1[3], e2[3], nrm[3];
  for (int i = 0; i < 3; i++) { e0[i] = v0[i] - v2[i]; e1[i] = v1[i] - v2[i]; e2[i] = pnt[i] - v2[i]; }
  nrm[0] = e0[1] * e1[2] - e0[2] * e1[1];
  nrm[1] = e0[2] * e1[0] - e0[0] * e1[2];
  nrm[2] = e0[0] * e1[1] - e0[1] * e1[0];
  const real denom = dot3(vec, nrm);
  if (fabs(denom) < MINVAL) return -1;
  const real dist = -dot3(e2, nrm) / denom;
  memcpy(n, nrm, sizeof nrm);
  normalize3(n);
  return dist >= 0 ? dist : -1;
}

typedef struct {
  int ngeom, nmesh, nmeshface;
  const int *geom_type, *geom_bodyid, *body_weldid, *geom_group, *geom_matid, *geom_dataid, *mesh_vertadr, *mesh_faceadr, *mesh_face;
  const real *geom_size, *geom_rgba, *mat_rgba, *mesh_vert;
} RayModel;

static real mesh(const RayModel* m, int id, const real* pos, const real* mat, const real* size, const real* pnt, const real* vec, real* n) {
  zero3(n);
  if (box(pos, mat, size, pnt, vec, n) < 0) { zero3(n); return -1; }
  real lp[3], lv[3], b0[3], b1[3], best[3] = {0, 0, 0};
  ray_map(pos, mat, pnt, vec, lp, lv);
  const real sign = lv[2] >= 0 ? 1 : -1, a = -1 / (sign + lv[2]), b = lv[0] * lv[1] * a;
  b0[0] = 1 + sign * lv[0] * lv[0] * a; b0[1] = sign * b; b0[2] = -sign * lv[0];
  b1[0] = b; b1[1] = sign + lv[1] * lv[1] * a; b1[2] = -lv[1];
  const real* vert = m->mesh_vert + 3 * m->mesh_vertadr[id];
  const int f0 = m->mesh_faceadr[id], f1 = id + 1 < m->nmesh ? m->mesh_faceadr[id + 1] : m->nmeshface;
  real x = -1;
  for (int f = f0; f < f1; f++) {
    real nt[3];
    const int* F = m->mesh_face + 3 * f;
    const real d = triangle(vert + 3 * F[0], vert + 3 * F[1], vert + 3 * F[2], lp, lv, b0, b1, nt);
    if (d >= 0 && (x < 0 || d < x)) { x = d; memcpy(best, nt, sizeof best); }
  }
  mat_vec(mat, best, n);
  return x;
}

static int eliminate(const RayModel* m, int g, const int* gg, int flg_static, int bodyexclude) {
  const int body = m->geom_bodyid[g], matid = m->geom_matid[g];
  if (body == bodyexclude) return 1;
  if (matid < 0 && m->geom_rgba[4 * g + 3] == 0) return 1;
  if (matid >= 0 && m->mat_rgba[4 * matid + 3] == 0) return 1;
  if (!flg_static && m->body_weldid[body] == 0) return 1;
  int all = 1;
  for (int k = 0; k < 6; k++) all &= gg[k] == -1;
  if (all) return 0;
  int grp = m->geom_group[g];
  grp = grp < 0 ? 0 : (grp > 5 ? 5 : grp);
  return gg[grp] == 0;
}

/* ray.py:907 _ray over nworld worlds and nray rays: pnt / vec (pnt_nbatch, nray, 3), geom_xpos (nworld, ngeom, 3), geom_xmat
 * (nworld, ngeom, 9); outputs dist / geomid (nworld, nray), normal (nworld, nray, 3).  Model tables are shared by all worlds. */
void ray_oracle_rays(int ngeom, int nmesh, int nmeshface, const int* geom_type, const int* geom_bodyid, const int* body_weldid, const int* geom_group,
                     const int* geom_matid, const int* geom_dataid, const real* geom_size, const real* geom_rgba, const real* mat_rgba,
                     const int* mesh_vertadr, const int* mesh_faceadr, const int* mesh_face, const real* mesh_vert, int nworld, const real* geom_xpos,
                     const real* geom_xmat, int nray, int pnt_nbatch, const real* pnt, const real* vec, const int* geomgroup, int flg_static,
                     const int* bodyexclude, real* dist, int* geomid, real* normal) {
  const RayModel m = {ngeom, nmesh, nmeshface, geom_type, geom_bodyid, body_weldid, geom_group, geom_matid, geom_dataid, mesh_vertadr, mesh_faceadr,
                      mesh_face, geom_size, geom_rgba, mat_rgba, mesh_vert};
#pragma omp parallel for schedule(dynamic, 16)
  for (long i = 0; i < (long)nworld * nray; i++) {
    const int w = (int)(i / nray), r = (int)(i % nray);
    const real* p = pnt + 3 * ((long)(pnt_nbatch == 1 ? 0 : w) * nray + r);
    const real* v = vec + 3 * ((long)(pnt_nbatch == 1 ? 0 : w) * nray + r);
    real best = MAXVAL, bn[3] = {0, 0, 0};
    int bg = -1;
    for (int g = 0; g < ngeom; g++) {
      if (eliminate(&m, g, geomgroup, flg_static, bodyexclude[r])) continue;
      const real* pos = geom_xpos + 3 * ((long)w * ngeom + g);
      const real* mat = geom_xmat + 9 * ((long)w * ngeom + g);
      const real* size = geom_size + 3 * g;
      real n[3], x;
      switch (geom_type[g]) {
        case PLANE: x = plane(pos, mat, size, p, v, n); break;
        case SPHERE: x = sphere(pos, size[0] * size[0], p, v, n); break;
        case CAPSULE: x = capsule(pos, mat, size, p, v, n); break;
        case ELLIPSOID: x = ellipsoid(pos, mat, size, p, v, n); break;
        case CYLINDER: x = cylinder(pos, mat, size, p, v, n); break;
        case BOX: x = box(pos, mat, size, p, v, n); break;
        case MESH: x = mesh(&m, geom_dataid[g], pos, mat, size, p, v, n); break;
        default: x = -1;
      }
      if (x >= 0 && x < best) { best = x; bg = g; memcpy(bn, n, sizeof bn); }
    }
    dist[i] = bg >= 0 ? best : -1;
    geomid[i] = bg;
    memcpy(normal + 3 * i, bn, sizeof bn);
  }
}
