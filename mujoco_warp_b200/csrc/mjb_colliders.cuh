// mjb_colliders.cuh -- box / cylinder / ellipsoid primitive pair functions (device).
//
// Replaces /root/reference/mujoco_warp/_src/collision_primitive_core.py:305 plane_ellipsoid, :336 plane_box,
// :387 sphere_cylinder, :459 plane_cylinder, :588 box_box (+ :556 _compute_rotmore), :1043 sphere_box, :1098 capsule_box.
// One lane evaluates one geom pair; results go to per-lane arrays (dist = MJB_MAXVAL for unpopulated slots), the caller
// applies write_contact's `dist < margin + gap` filter and stages the survivors in pair order.
#pragma once
#include "mjb_math.cuh"

#define MJB_MAXVAL 1e10f

static __device__ __forceinline__ v3 mat_t_vec(const float* m, v3 v) {  // m^T v
  return mk3(m[0] * v.x + m[3] * v.y + m[6] * v.z, m[1] * v.x + m[4] * v.y + m[7] * v.z, m[2] * v.x + m[5] * v.y + m[8] * v.z);
}
static __device__ __forceinline__ void mat_mul33(const float* a, const float* b, float* c) {
#pragma unroll
  for (int i = 0; i < 3; i++)
#pragma unroll
    for (int j = 0; j < 3; j++) c[3 * i + j] = a[3 * i] * b[j] + a[3 * i + 1] * b[3 + j] + a[3 * i + 2] * b[6 + j];
}
static __device__ __forceinline__ void mat_t33(const float* a, float* t) {
#pragma unroll
  for (int i = 0; i < 3; i++)
#pragma unroll
    for (int j = 0; j < 3; j++) t[3 * i + j] = a[3 * j + i];
}
static __device__ __forceinline__ float comp(v3 a, int i) { return i == 0 ? a.x : (i == 1 ? a.y : a.z); }
static __device__ __forceinline__ void setcomp(v3& a, int i, float x) { if (i == 0) a.x = x; else if (i == 1) a.y = x; else a.z = x; }
static __device__ __forceinline__ v3 cw_mul(v3 a, v3 b) { return mk3(a.x * b.x, a.y * b.y, a.z * b.z); }
static __device__ __forceinline__ v3 vabs(v3 a) { return mk3(fabsf(a.x), fabsf(a.y), fabsf(a.z)); }

static __device__ __forceinline__ float col_plane_sphere(v3 n, v3 ppos, v3 spos, float r, v3* pos) {
  const float dist = dot(spos - ppos, n) - r;
  *pos = spos - n * (r + 0.5f * dist);
  return dist;
}
static __device__ __forceinline__ float col_sphere_sphere(v3 pos1, float r1, v3 pos2, float r2, v3* pos, v3* n) {
  const v3 dir = pos2 - pos1;
  float dist = length(dir);
  *n = dist == 0.f ? mk3(1.f, 0.f, 0.f) : dir * (1.0f / dist);
  dist -= r1 + r2;
  *pos = pos1 + *n * (r1 + 0.5f * dist);
  return dist;
}

// collision_primitive_core.py capsule_capsule for the collision sensors, the arithmetic k_collision inlines: the closest segment points, or up to two end points of
// (nearly) parallel segments; only contacts within `margin` are produced (dist INFINITY otherwise)
static __device__ __forceinline__ void capsule_capsule(v3 pos1, v3 ax1, v3 size1, v3 pos2, v3 ax2, v3 size2, float margin, float* cd, v3* cp, v3* cn) {
  const v3 axis1 = ax1 * size1.y, axis2 = ax2 * size2.y, dif = pos1 - pos2;
  const float ma = dot(axis1, axis1), mb = -dot(axis1, axis2), mc = dot(axis2, axis2), u = -dot(axis1, dif), v = dot(axis2, dif);
  const float det = ma * mc - mb * mb;
  v3 p, n;
  if (fabsf(det) >= MJ_MINVAL) {
    const float inv = 1.0f / det;
    float x1 = (mc * u - mb * v) * inv, x2 = (ma * v - mb * u) * inv;
    if (x1 > 1.f) { x1 = 1.f; x2 = (v - mb) / mc; } else if (x1 < -1.f) { x1 = -1.f; x2 = (v + mb) / mc; }
    if (x2 > 1.f) { x2 = 1.f; x1 = clampf((u - mb) / ma, -1.f, 1.f); } else if (x2 < -1.f) { x2 = -1.f; x1 = clampf((u + mb) / ma, -1.f, 1.f); }
    const float dist = col_sphere_sphere(pos1 + axis1 * x1, size1.x, pos2 + axis2 * x2, size2.x, &p, &n);
    if (dist <= margin) { cd[0] = dist; cp[0] = p; cn[0] = n; }
    return;
  }
  int cc = 0;
  float dist = col_sphere_sphere(pos1 + axis1, size1.x, pos2 + axis2 * clampf((v - mb) / mc, -1.f, 1.f), size2.x, &p, &n);
  if (dist <= margin) { cd[cc] = dist; cp[cc] = p; cn[cc] = n; cc++; }
  dist = col_sphere_sphere(pos1 - axis1, size1.x, pos2 + axis2 * clampf((v + mb) / mc, -1.f, 1.f), size2.x, &p, &n);
  if (dist <= margin) { cd[cc] = dist; cp[cc] = p; cn[cc] = n; cc++; }
  if (cc < 2) {
    dist = col_sphere_sphere(pos1 + axis1 * clampf((u - mb) / ma, -1.f, 1.f), size1.x, pos2 + axis2, size2.x, &p, &n);
    if (dist <= margin) { cd[cc] = dist; cp[cc] = p; cn[cc] = n; cc++; }
  }
  if (cc < 2) {
    dist = col_sphere_sphere(pos1 + axis1 * clampf((u + mb) / ma, -1.f, 1.f), size1.x, pos2 - axis2, size2.x, &p, &n);
    if (dist <= margin) { cd[cc] = dist; cp[cc] = p; cn[cc] = n; }
  }
}

static __device__ __forceinline__ float plane_ellipsoid(v3 n, v3 ppos, v3 epos, const float* erot, v3 esize, v3* pos) {
  const v3 sup = normalize(cw_mul(mat_t_vec(erot, n), esize)) * -1.0f;
  v3 p = epos + matvec(erot, cw_mul(sup, esize));
  const float dist = dot(n, p - ppos);
  *pos = p - n * (dist * 0.5f);
  return dist;
}

static __device__ __forceinline__ void plane_box(v3 n, v3 ppos, v3 bpos, const float* brot, v3 bsize, float* dist, v3* pos) {
  const float center_dist = dot(bpos - ppos, n);
#pragma unroll
  for (int i = 0; i < 8; i++) {
    const v3 corner = matvec(brot, mk3((i & 1) ? bsize.x : -bsize.x, (i & 2) ? bsize.y : -bsize.y, (i & 4) ? bsize.z : -bsize.z));
    const float cdist = center_dist + dot(n, corner);
    dist[i] = cdist;
    pos[i] = corner + bpos - n * (0.5f * cdist);
  }
}

static __device__ __forceinline__ float sphere_cylinder(v3 spos, float sr, v3 cpos, v3 caxis, float cr, float chh, v3* pos, v3* nrm) {
  const v3 vec = spos - cpos;
  const float x = dot(vec, caxis);
  const v3 a_proj = caxis * x, p_proj = vec - a_proj;
  const float p_sqr = dot(p_proj, p_proj);
  bool side = fabsf(x) < chh, cap = p_sqr < cr * cr;
  if (side && cap) {
    if (chh - fabsf(x) < cr - sqrtf(p_sqr)) side = false; else cap = false;
  }
  if (side) return col_sphere_sphere(spos, sr, cpos + a_proj, cr, pos, nrm);
  if (cap) {
    const float sgn = x > 0.f ? 1.f : -1.f;
    const v3 pn = caxis * sgn;
    const float dist = col_plane_sphere(pn, cpos + pn * chh, spos, sr, pos);
    *nrm = pn * -1.0f;
    return dist;
  }
  const float inv_len = safe_div(1.0f, sqrtf(p_sqr)), sgn = x < 0.f ? -1.f : 1.f;  // wp.sign(0) = +1
  return col_sphere_sphere(spos, sr, cpos + caxis * (sgn * chh) + p_proj * (cr * inv_len), 0.f, pos, nrm);
}

static __device__ __forceinline__ void plane_cylinder(v3 n, v3 ppos, v3 center, v3 caxis, float cr, float chh, float* dist, v3* pos) {
  v3 axis = caxis;
  float prjaxis = dot(n, axis);
  if (prjaxis > 0.f) { axis = axis * -1.0f; prjaxis = -prjaxis; }
  const float dist0 = dot(center - ppos, n);
  v3 vec = axis * prjaxis - n;
  const float len_sqr = dot(vec, vec);
  vec = len_sqr >= 1e-12f ? vec * safe_div(cr, sqrtf(len_sqr)) : mk3(cr, 0.f, 0.f);
  const float prjvec = dot(vec, n);
  axis = axis * chh;
  prjaxis *= chh;
  const float dist1 = dist0 + prjaxis + prjvec, dist2 = dist0 - prjaxis + prjvec, dist3 = dist0 + prjaxis - 0.5f * prjvec;
  dist[0] = dist1; pos[0] = center + vec + axis - n * (dist1 * 0.5f);
  dist[1] = dist2; pos[1] = center + vec - axis - n * (dist2 * 0.5f);
  const v3 vec1 = normalize(cross(vec, axis)) * (cr * sqrtf(3.0f) * 0.5f);
  dist[2] = dist3; pos[2] = center + vec1 + axis - vec * 0.5f - n * (dist3 * 0.5f);
  dist[3] = dist3; pos[3] = center - vec1 + axis - vec * 0.5f - n * (dist3 * 0.5f);
}

static __device__ __noinline__ float sphere_box(v3 spos, float sr, v3 bpos, const float* brot, v3 bsize, v3* cpos, v3* nrm) {
  const v3 center = mat_t_vec(brot, spos - bpos);
  const v3 clamped = mk3(fmaxf(-bsize.x, fminf(bsize.x, center.x)), fmaxf(-bsize.y, fminf(bsize.y, center.y)), fmaxf(-bsize.z, fminf(bsize.z, center.z)));
  const v3 dif = clamped - center;
  const float dist = length(dif);
  v3 pos;
  float cdist;
  if (dist <= MJ_MINVAL) {  // centre inside the box: leave through the nearest face
    float closest = 2.0f * (bsize.x + bsize.y + bsize.z);
    int k = 0;
#pragma unroll
    for (int i = 0; i < 6; i++) {
      const float face_dist = fabsf(((i & 1) ? 1.0f : -1.0f) * comp(bsize, i >> 1) - comp(center, i >> 1));
      if (closest > face_dist) { closest = face_dist; k = i; }
    }
    v3 nearest = mk3(0.f, 0.f, 0.f);
    setcomp(nearest, k >> 1, (k & 1) ? -1.0f : 1.0f);
    pos = center + nearest * ((sr - closest) * 0.5f);
    *nrm = matvec(brot, nearest);
    cdist = -closest - sr;
  } else {
    const v3 dir = dif * (1.0f / dist);
    pos = (clamped + center + dir * sr) * 0.5f;
    *nrm = matvec(brot, dir);
    cdist = dist - sr;
  }
  *cpos = bpos + matvec(brot, pos);
  return cdist;
}

// closest-feature search between the capsule segment and the box (faces, then the 12 edges), an optional second point
// further along the segment, and one sphere-box test per point
static __device__ __noinline__ void capsule_box(v3 cpos_in, v3 caxis, float crad, float chl, v3 bpos, const float* brot, v3 bsize, float* dist, v3* cpos, v3* cnrm) {
  const v3 pos = mat_t_vec(brot, cpos_in - bpos), axis = mat_t_vec(brot, caxis), halfaxis = axis * chl;
  const int axisdir = (halfaxis.x > 0.f ? 1 : 0) + (halfaxis.y > 0.f ? 2 : 0) + (halfaxis.z > 0.f ? 4 : 0);
  float bestdist = 1.0e32f, bestsegmentpos = -12.f, bestboxpos = 0.f;
  int cltype = -4, clface = -12, clcorner = -123, cledge = -123;
#pragma unroll 1
  for (int i = -1; i <= 1; i += 2) {
    const v3 tip = pos + halfaxis * (float)i;
    v3 bp = tip;
    int n_out = 0, ax_out = -1;
#pragma unroll
    for (int j = 0; j < 3; j++) {
      const float s = comp(bsize, j), t = comp(bp, j);
      if (t < -s) { n_out++; ax_out = j; setcomp(bp, j, -s); }
      else if (t > s) { n_out++; ax_out = j; setcomp(bp, j, s); }
    }
    if (n_out > 1) continue;
    const v3 dd = bp - tip;
    const float ds = dot(dd, dd);
    if (ds < bestdist) { bestdist = ds; bestsegmentpos = (float)i; cltype = -2 + i; clface = ax_out; }
  }
#pragma unroll 1
  for (int i = 0; i < 8; i++) {
#pragma unroll 1
    for (int j = 0; j < 3; j++) {
      if (i & (1 << j)) continue;
      v3 box_pt = mk3((i & 1) ? bsize.x : -bsize.x, (i & 2) ? bsize.y : -bsize.y, (i & 4) ? bsize.z : -bsize.z);
      setcomp(box_pt, j, 0.f);
      v3 dif = box_pt - pos;
      const float sj = comp(bsize, j), hj = comp(halfaxis, j);
      const float u = -sj * comp(dif, j), v = dot(halfaxis, dif), ma = sj * sj, mb = -sj * hj, mc = chl * chl, det = ma * mc - mb * mb;
      if (fabsf(det) < MJ_MINVAL) continue;
      const float idet = 1.0f / det;
      float x1 = (mc * u - mb * v) * idet, x2 = (ma * v - mb * u) * idet;
      int s1 = 1, s2 = 1;
      if (x1 > 1.f) { x1 = 1.f; s1 = 2; x2 = safe_div(v - mb, mc); }
      else if (x1 < -1.f) { x1 = -1.f; s1 = 0; x2 = safe_div(v + mb, mc); }
      const bool over = x2 > 1.f;
      if (over || x2 < -1.f) {
        if (over) { x2 = 1.f; s2 = 2; x1 = safe_div(u - mb, ma); } else { x2 = -1.f; s2 = 0; x1 = safe_div(u + mb, ma); }
        if (x1 > 1.f) { x1 = 1.f; s1 = 2; } else if (x1 < -1.f) { x1 = -1.f; s1 = 0; }
      }
      dif = dif - halfaxis * x2;
      setcomp(dif, j, comp(dif, j) + sj * x1);
      const int ct = s1 * 3 + s2;
      const float dsq = dot(dif, dif);
      if (dsq < bestdist - MJ_MINVAL) {
        bestdist = dsq; bestsegmentpos = x2; bestboxpos = x1;
        clcorner = i + (1 << j) * (ct / 6); cledge = j; cltype = ct;
      }
    }
  }
  dist[0] = MJB_MAXVAL; dist[1] = MJB_MAXVAL;
  if (cltype == -4) return;
  float secondpos = -4.f;
  if (cltype >= 0 && cltype / 3 != 1) {  // a box corner is closest
    int c1 = axisdir ^ clcorner;
    if (c1 != 0 && c1 != 7) {
      int mul = 1;
      if (!(c1 == 1 || c1 == 2 || c1 == 4)) { mul = -1; c1 = 7 - c1; }
      const int ax = c1 == 1 ? 0 : (c1 == 2 ? 1 : 2), ax1 = (ax + 1) % 3, ax2 = (ax + 2) % 3;
      if (comp(axis, ax) * comp(axis, ax) > 0.5f) {
        const float mm = 2.0f * safe_div(comp(bsize, ax), fabsf(comp(halfaxis, ax)));
        secondpos = fminf(1.0f - (float)mul * bestsegmentpos, mm);
      } else {
        const float mm = 2.0f * fminf(safe_div(comp(bsize, ax1), fabsf(comp(halfaxis, ax1))), safe_div(comp(bsize, ax2), fabsf(comp(halfaxis, ax2))));
        secondpos = -fminf(1.0f + (float)mul * bestsegmentpos, mm);
      }
      secondpos *= (float)mul;
    }
  } else if (cltype >= 0) {  // the interior of a box edge is closest
    int c1 = axisdir ^ clcorner;
    c1 &= 7 - (1 << cledge);
    if (c1 == 1 || c1 == 2 || c1 == 4) {
      const int ax = cledge;
      int ax1 = (cledge + 1) % 3, ax2 = (cledge + 2) % 3, mul;
      if (fabsf(comp(axis, ax1)) > fabsf(comp(axis, ax2))) ax1 = ax2;
      ax2 = 3 - ax - ax1;
      if (c1 & (1 << ax2)) { mul = 1; secondpos = 1.0f - bestsegmentpos; } else { mul = -1; secondpos = 1.0f + bestsegmentpos; }
      float e1 = 2.0f * safe_div(comp(bsize, ax2), fabsf(comp(halfaxis, ax2)));
      secondpos = fminf(e1, secondpos);
      const float e2 = (((axisdir & (1 << ax)) != 0) == ((c1 & (1 << ax2)) != 0)) ? 1.0f - bestboxpos : 1.0f + bestboxpos;
      e1 = comp(bsize, ax) * safe_div(e2, fabsf(comp(halfaxis, ax)));
      secondpos = fminf(e1, secondpos) * (float)mul;
    }
  } else if (clface != -1) {  // a tip over a face: second point at the other end, clamped to the face outline
    const int mul = cltype == -3 ? 1 : -1;
    secondpos = 2.0f;
    const v3 tmp1 = pos - halfaxis * (float)mul;
#pragma unroll
    for (int i = 0; i < 3; i++) {
      if (i == clface) continue;
      const float ha_r = safe_div((float)mul, comp(halfaxis, i));
      float e1 = (comp(bsize, i) - comp(tmp1, i)) * ha_r;
      if (0.f < e1 && e1 < secondpos) secondpos = e1;
      e1 = (-comp(bsize, i) - comp(tmp1, i)) * ha_r;
      if (0.f < e1 && e1 < secondpos) secondpos = e1;
    }
    secondpos *= (float)mul;
  }
  dist[0] = sphere_box(matvec(brot, pos + halfaxis * bestsegmentpos) + bpos, crad, bpos, brot, bsize, &cpos[0], &cnrm[0]);
  if (secondpos > -3.f) dist[1] = sphere_box(matvec(brot, pos + halfaxis * (secondpos + bestsegmentpos)) + bpos, crad, bpos, brot, bsize, &cpos[1], &cnrm[1]);
}

static __device__ __forceinline__ void rotmore_of(int face, float* r) {
#pragma unroll
  for (int i = 0; i < 9; i++) r[i] = 0.f;
  if (face == 0) { r[2] = -1.f; r[4] = 1.f; r[6] = 1.f; }
  else if (face == 1) { r[0] = 1.f; r[5] = -1.f; r[7] = 1.f; }
  else if (face == 2) { r[0] = 1.f; r[4] = 1.f; r[8] = 1.f; }
  else if (face == 3) { r[2] = 1.f; r[4] = 1.f; r[6] = -1.f; }
  else if (face == 4) { r[0] = 1.f; r[5] = 1.f; r[7] = -1.f; }
  else { r[0] = -1.f; r[4] = 1.f; r[8] = -1.f; }
}
static __device__ __forceinline__ v3 row3(const float* m, int i) { return mk3(m[3 * i], m[3 * i + 1], m[3 * i + 2]); }

// 15-axis separating-axis search, then clipping of the incident face (face-vertex case) or of box2's closest face against
// box1's (edge-edge case); at most 8 contacts sharing one normal.  Returns the contact count.
static __device__ __noinline__ int box_box(v3 pos1, const float* rot1, v3 size1, v3 pos2, const float* rot2, v3 size2, float margin, float* cdist, v3* cpos, v3* cnormal) {
  const v3 pos21 = mat_t_vec(rot1, pos2 - pos1), pos12 = mat_t_vec(rot2, pos1 - pos2);
  float rot1T[9], rot21[9], rot12[9], rot21abs[9], rot12abs[9];
  mat_t33(rot1, rot1T);
  mat_mul33(rot1T, rot2, rot21);
  mat_t33(rot21, rot12);
  for (int i = 0; i < 9; i++) rot21abs[i] = fabsf(rot21[i]);
  mat_t33(rot21abs, rot12abs);
  const v3 plen2 = matvec(rot21abs, size2), plen1 = matvec(rot12abs, size1);
  float separation = margin + 3.0f * (size1.x + size2.x) + 3.0f * (size1.y + size2.y) + 3.0f * (size1.z + size2.z);
  int axis_code = -1;
#pragma unroll
  for (int i = 0; i < 3; i++) {
    const float c1 = -fabsf(comp(pos21, i)) + comp(size1, i) + comp(plen2, i), c2 = -fabsf(comp(pos12, i)) + comp(size2, i) + comp(plen1, i);
    if (c1 < -margin || c2 < -margin) return 0;
    if (c1 < separation) { separation = c1; axis_code = i + 3 * (comp(pos21, i) < 0.f ? 1 : 0); }
    if (c2 < separation) { separation = c2; axis_code = i + 3 * (comp(pos12, i) < 0.f ? 1 : 0) + 6; }
  }
  v3 clnorm = mk3(0.f, 0.f, 0.f);
  bool inv = false;
  int cle1 = 0, cle2 = 0;
#pragma unroll 1
  for (int i = 0; i < 3; i++) {
#pragma unroll 1
    for (int j = 0; j < 3; j++) {
      const v3 a = row3(rot12, j);
      v3 ca = i == 0 ? mk3(0.f, -a.z, a.y) : (i == 1 ? mk3(a.z, 0.f, -a.x) : mk3(-a.y, a.x, 0.f));
      const float cl = length(ca);
      if (cl < MJ_MINVAL) continue;
      ca = ca * (1.0f / cl);
      const float box_dist = dot(pos21, ca);
      float c3 = 0.f;
      for (int k = 0; k < 3; k++) {
        if (k != i) c3 += comp(size1, k) * fabsf(comp(ca, k));
        if (k != j) c3 += comp(size2, k) * rot21abs[3 * i + (3 - k - j)] / cl;
      }
      c3 -= fabsf(box_dist);
      if (c3 < -margin) return 0;
      if (c3 < separation * (1.0f - 1e-12f)) {
        separation = c3; cle1 = 0; cle2 = 0;
        for (int k = 0; k < 3; k++) {
          if (k != i && ((comp(ca, k) > 0.f) != (box_dist < 0.f))) cle1 += 1 << k;
          if (k != j && (((rot21[3 * i + (3 - k - j)] > 0.f) != (box_dist < 0.f)) != ((k - j + 3) % 3 == 1))) cle2 += 1 << k;
        }
        axis_code = 12 + i * 3 + j;
        clnorm = ca;
        inv = box_dist < 0.f;
      }
    }
  }
  if (axis_code == -1) return 0;
  v3 points[8];
  float depth[8], rotmore[9], rmT[9], rw[9], hz;
  v3 pw, normal;
  int n = 0;
  if (axis_code < 12) {
    const int face_idx = axis_code % 6, box_idx = axis_code / 6;
    rotmore_of(face_idx, rotmore);
    float r[9], rt[9];
    mat_mul33(rotmore, box_idx ? rot12 : rot21, r);
    mat_t33(r, rt);
    v3 p = matvec(rotmore, box_idx ? pos12 : pos21);
    const v3 ss = vabs(matvec(rotmore, box_idx ? size2 : size1)), s = box_idx ? size1 : size2;
    const float lx = ss.x, ly = ss.y;
    hz = ss.z;
    p.z -= hz;
    int clcorner = 0;
    for (int i = 0; i < 3; i++) if (r[6 + i] < 0.f) clcorner += 1 << i;
    v3 lp = p;
    for (int i = 0; i < 3; i++) lp = lp + row3(rt, i) * (comp(s, i) * ((clcorner & (1 << i)) ? 1.0f : -1.0f));
    int dirs = 0;
    v3 cn1 = mk3(0.f, 0.f, 0.f), cn2 = cn1;
    for (int i = 0; i < 3; i++) {
      if (fabsf(r[6 + i]) < 0.5f) {
        const v3 cn = row3(rt, i) * (comp(s, i) * ((clcorner & (1 << i)) ? -2.0f : 2.0f));
        if (dirs == 0) cn1 = cn; else cn2 = cn;
        dirs++;
      }
    }
    const int kk = dirs * dirs;
#pragma unroll 1
    for (int i = 0; i < kk; i++) {
#pragma unroll 1
      for (int q = 0; q < 2; q++) {
        const v3 lav = lp + (i < 2 ? mk3(0.f, 0.f, 0.f) : (i == 2 ? cn1 : cn2)), lbv = (i == 0 || i == 3) ? cn1 : cn2;
        const float lbq = comp(lbv, q);
        if (fabsf(lbq) > MJ_MINVAL) {
          const float br = 1.0f / lbq;
          for (int j = -1; j <= 1; j += 2) {
            const float l = comp(ss, q) * (float)j, c1 = (l - comp(lav, q)) * br;
            if (c1 < 0.f || c1 > 1.f) continue;
            const float c2 = comp(lav, 1 - q) + comp(lbv, 1 - q) * c1;
            if (fabsf(c2) > comp(ss, 1 - q)) continue;
            if (n < 8) { points[n] = lav + lbv * c1; n++; }
          }
        }
      }
    }
    if (dirs == 2) {
      const float ax = cn1.x, bx = cn2.x, ay = cn1.y, by = cn2.y, C = safe_div(1.0f, ax * by - bx * ay);
      for (int i = 0; i < 4; i++) {
        const float llx = (i / 2) ? lx : -lx, lly = (i % 2) ? ly : -ly, x = llx - lp.x, y = lly - lp.y;
        const float u = (x * by - y * bx) * C, v = (y * ax - x * ay) * C;
        if (u > 0.f && v > 0.f && u < 1.f && v < 1.f && n < 8) { points[n] = mk3(llx, lly, lp.z + u * cn1.z + v * cn2.z); n++; }
      }
    }
    for (int i = 0; i < (1 << dirs); i++) {
      const v3 t = lp + cn1 * (float)(i & 1) + cn2 * (float)((i & 2) != 0);
      if (t.x > -lx && t.x < lx && t.y > -ly && t.y < ly && n < 8) { points[n] = t; n++; }
    }
    const int m = n;
    n = 0;
    for (int i = 0; i < m; i++) {
      if (points[i].z > margin) continue;
      if (i != n) points[n] = points[i];
      depth[n] = points[n].z;
      points[n].z *= 0.5f;
      n++;
    }
    mat_t33(rotmore, rmT);
    mat_mul33(box_idx ? rot2 : rot1, rmT, rw);
    pw = box_idx ? pos2 : pos1;
    normal = matcol(rw, 2) * (box_idx ? -1.0f : 1.0f);
  } else {
    const int edge1 = (axis_code - 12) / 3, edge2 = (axis_code - 12) % 3;
    int ax1 = 1 - (edge2 & 1), ax2 = 2 - (edge2 & 2), pax1 = 1 - (edge1 & 1), pax2 = 2 - (edge1 & 2);
    if (rot21abs[3 * edge1 + ax1] < rot21abs[3 * edge1 + ax2]) { const int t = ax1; ax1 = ax2; ax2 = t; }
    if (rot12abs[3 * edge2 + pax1] < rot12abs[3 * edge2 + pax2]) { const int t = pax1; pax1 = pax2; pax2 = t; }
    rotmore_of((cle1 & (1 << pax2)) ? pax2 : pax2 + 3, rotmore);
    float r[9], rt[9];
    v3 p = matvec(rotmore, pos21);
    const v3 rnorm = matvec(rotmore, clnorm);
    mat_mul33(rotmore, rot21, r);
    mat_t33(r, rt);
    mat_t33(rotmore, rmT);
    const v3 s = vabs(matvec(rmT, size1));
    const float lx = s.x, ly = s.y;
    hz = s.z;
    p.z -= hz;
    const float sg1 = (cle2 & (1 << ax1)) ? 1.0f : -1.0f, sg2 = (cle2 & (1 << ax2)) ? 1.0f : -1.0f;
    const v3 t1 = row3(rt, ax1) * (comp(size2, ax1) * sg1), t2 = row3(rt, ax2) * (comp(size2, ax2) * sg2), te = row3(rt, edge2) * comp(size2, edge2);
    points[0] = p + t1 + t2 + te; points[1] = p + t1 + t2 - te;
    points[2] = p - t1 + t2 + te; points[3] = p - t1 + t2 - te;
    const v3 axi_lp = points[0], axi_cn1 = points[1] - points[0], axi_cn2 = points[2] - points[0];
    if (fabsf(rnorm.z) < MJ_MINVAL) return 0;
    const float sgn = inv ? -1.0f : 1.0f, innorm = sgn / rnorm.z;
    v3 pu[4];
    for (int i = 0; i < 4; i++) {
      pu[i] = points[i];
      points[i] = points[i] - rnorm * (points[i].z * sgn * innorm);
    }
    const v3 pts_lp = points[0], pts_cn1 = points[1] - points[0], pts_cn2 = points[2] - points[0];
    n = 0;
#pragma unroll 1
    for (int i = 0; i < 4; i++) {
#pragma unroll 1
      for (int q = 0; q < 2; q++) {
        const v3 poff = i < 2 ? mk3(0.f, 0.f, 0.f) : (i == 2 ? pts_cn1 : pts_cn2), pdir = (i == 0 || i == 3) ? pts_cn1 : pts_cn2;
        const float la = comp(pts_lp, q) + comp(poff, q), lb = comp(pdir, q), lc = comp(pts_lp, 1 - q) + comp(poff, 1 - q), ld = comp(pdir, 1 - q);
        const v3 lua = axi_lp + (i < 2 ? mk3(0.f, 0.f, 0.f) : (i == 2 ? axi_cn1 : axi_cn2)), lub = (i == 0 || i == 3) ? axi_cn1 : axi_cn2;
        if (fabsf(lb) > MJ_MINVAL) {
          const float br = 1.0f / lb;
          for (int j = -1; j <= 1; j += 2) {
            if (n == 8) break;
            const float l = comp(s, q) * (float)j, c1 = (l - la) * br;
            if (c1 < 0.f || c1 > 1.f) continue;
            const float c2 = lc + ld * c1;
            if (fabsf(c2) > comp(s, 1 - q)) continue;
            if ((lua.z + lub.z * c1) * innorm > margin) continue;
            v3 pt = lua * 0.5f + lub * (c1 * 0.5f);
            setcomp(pt, q, comp(pt, q) + 0.5f * l);
            setcomp(pt, 1 - q, comp(pt, 1 - q) + 0.5f * c2);
            points[n] = pt;
            depth[n] = pt.z * innorm * 2.0f;
            n++;
          }
        }
      }
    }
    const int nl = n;
    const float ax = pts_cn1.x, bx = pts_cn2.x, ay = pts_cn1.y, by = pts_cn2.y, C = safe_div(1.0f, ax * by - bx * ay);
    for (int i = 0; i < 4; i++) {
      if (n == 8) break;
      const float llx = (i / 2) ? lx : -lx, lly = (i % 2) ? ly : -ly, x = llx - pts_lp.x, y = lly - pts_lp.y;
      float u = (x * by - y * bx) * C, v = (y * ax - x * ay) * C;
      if (nl == 0) { if ((u < 0.f || u > 1.f) && (v < 0.f || v > 1.f)) continue; }
      else if (u < 0.f || v < 0.f || u > 1.f || v > 1.f) continue;
      u = clampf(u, 0.f, 1.f); v = clampf(v, 0.f, 1.f);
      const v3 vtmp = pu[0] * (1.0f - u - v) + pu[1] * u + pu[2] * v, pt = mk3(llx, lly, 0.f), dv = pt - vtmp;
      const float tc1 = dot(dv, dv);
      if (vtmp.z > 0.f && tc1 > margin * margin) continue;
      points[n] = (pt + vtmp) * 0.5f;
      depth[n] = sqrtf(tc1) * (vtmp.z < 0.f ? -1.0f : 1.0f);
      n++;
    }
    const int nf = n;
    for (int i = 0; i < 4; i++) {
      if (n >= 8) break;
      const float x = pu[i].x, y = pu[i].y;
      if (nl == 0 && nf != 0) { if ((x < -lx || x > lx) && (y < -ly || y > ly)) continue; }
      else if (x < -lx || x > lx || y < -ly || y > ly) continue;
      float c1 = 0.f;
      v3 tp = mk3(x, y, 0.f);
      for (int j = 0; j < 2; j++) {
        const float pj = comp(pu[i], j), sj = comp(s, j);
        if (pj < -sj) { c1 += (pj + sj) * (pj + sj); setcomp(tp, j, -sj * 0.5f); }
        else if (pj > sj) { c1 += (pj - sj) * (pj - sj); setcomp(tp, j, sj * 0.5f); }
      }
      c1 += pu[i].z * innorm * pu[i].z * innorm;
      if (pu[i].z > 0.f && c1 > margin * margin) continue;
      points[n] = (tp + pu[i]) * 0.5f;
      depth[n] = sqrtf(c1) * (pu[i].z < 0.f ? -1.0f : 1.0f);
      n++;
    }
    mat_mul33(rot1, rmT, rw);
    pw = pos1;
    normal = matvec(rw, rnorm) * sgn;
  }
  for (int i = 0; i < n; i++) {
    points[i].z += hz;
    cpos[i] = matvec(rw, points[i]) + pw;
    cdist[i] = depth[i];
  }
  *cnormal = normal;
  return n;
}
