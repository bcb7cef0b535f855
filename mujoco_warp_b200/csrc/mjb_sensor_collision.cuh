// mjb_sensor_collision.cuh -- distance / normal / fromto sensors of one world: the geom pairs' colliders and the per-sensor reduction.
//
// Replaces (reference, /root/reference/mujoco_warp/_src/): the sensor pairs' pass through the narrowphase (collision_primitive.py wrappers,
// collision_convex.py:814-818 with cutoff 1e32, collision_core.py:259-291 write_contact of ContactType.SENSOR contacts), sensor.py:759
// _sensor_collision (the witness points pos -/+ 0.5 dist normal) and sensor.py:642-718 (the reduction, flip and cutoff rules).  Every pair
// runs the collider the reference routes its geom types to and reports every contact that collider writes; nothing reaches the contact pool.
//
// Scalar code, one geom pair or one sensor per thread.  Needs the CCD_MESH build of mjb_ccd.cuh (1, or 2 with the lane's multi-contact scratch).
#pragma once
#include "mjb_ccd.cuh"
#include "mjb_colliders.cuh"
#include "mjb_math.cuh"
#include "mjb_types.cuh"

constexpr int SC_WORDS = 7;       // per geom pair: distance, witness point on the first and on the second geom (narrowphase order)
constexpr int SC_PAIR_WORDS = 4;  // sensor_collision_pair row: geom1, geom2, explicit <pair> id or -1, EPA scratch slot or -1

// One sensor pair (g1, g2 in narrowphase order, pid its explicit <pair> or -1) at the world's geom poses: every contact of its collider
// (at most 8), reduced to the first one of least distance.  out[SC_WORDS]: that distance (INFINITY if the collider produced nothing) and
// its witness points pos -/+ 0.5 dist normal.  scratch: ccd_scratch_words(epa_iterations) floats for EPA.  Returns whether EPA ran out
// of horizon edges (OVF_EPA_HORIZON, as k_collision reports it).
static __device__ bool sensor_pair(const ModelDev& m, const float* gxpos, const float* gxmat, int g1, int g2, int pid, int epa_iterations, float* scratch,
                                   float* out CCD_CLIP_PARAM) {
  float cd[8];
  v3 cp[8], cn[8];
  for (int k = 0; k < 8; k++) { cd[k] = INFINITY; cp[k] = mk3(0.f, 0.f, 0.f); cn[k] = mk3(1.f, 0.f, 0.f); }
  const int t1 = m.geom_type[g1], t2 = m.geom_type[g2];
  const float margin = pid > -1 ? m.pair_margin[pid] : m.geom_margin[g1] + m.geom_margin[g2];
  const v3 pos1 = ld3(gxpos + 3 * g1), pos2 = ld3(gxpos + 3 * g2);
  const float *rot1 = gxmat + 9 * g1, *rot2 = gxmat + 9 * g2;
  const v3 ax1 = matcol(rot1, 2), ax2 = matcol(rot2, 2);
  const v3 size1 = ld3(m.geom_size + 3 * g1), size2 = ld3(m.geom_size + 3 * g2);
  const bool nativeccd = !(m.disableflags & DSBL_NATIVECCD);
  bool eovf = false;
  if (t1 == GEOM_PLANE) {
    if (t2 == GEOM_SPHERE) {
      cd[0] = col_plane_sphere(ax1, pos1, pos2, size2.x, &cp[0]);
    } else if (t2 == GEOM_CAPSULE) {
      const v3 seg = ax2 * size2.y;
      cd[0] = col_plane_sphere(ax1, pos1, pos2 + seg, size2.x, &cp[0]);
      cd[1] = col_plane_sphere(ax1, pos1, pos2 - seg, size2.x, &cp[1]);
    } else if (t2 == GEOM_ELLIPSOID) {
      cd[0] = plane_ellipsoid(ax1, pos1, pos2, rot2, size2, &cp[0]);
    } else if (t2 == GEOM_CYLINDER) {
      plane_cylinder(ax1, pos1, pos2, ax2, size2.x, size2.y, cd, cp);
    } else if (t2 == GEOM_BOX) {
      plane_box(ax1, pos1, pos2, rot2, size2, cd, cp);
    } else if (t2 == GEOM_MESH) {
      CGeom c;
      c.pos = pos2; c.rot = rot2; c.size = size2; c.margin = 0.f; c.type = GEOM_MESH;
      fill_mesh(m, g2, c);
      plane_mesh(ax1, pos1, c, cd, cp);
    }
    for (int k = 0; k < 8; k++) cn[k] = ax1;
  } else if (t1 == GEOM_SPHERE && t2 == GEOM_SPHERE) {
    cd[0] = col_sphere_sphere(pos1, size1.x, pos2, size2.x, &cp[0], &cn[0]);
  } else if (t1 == GEOM_SPHERE && t2 == GEOM_CAPSULE) {
    const v3 seg = ax2 * size2.y;
    cd[0] = col_sphere_sphere(pos1, size1.x, closest_segment_point(pos2 - seg, pos2 + seg, pos1), size2.x, &cp[0], &cn[0]);
  } else if (t1 == GEOM_SPHERE && t2 == GEOM_CYLINDER) {
    cd[0] = sphere_cylinder(pos1, size1.x, pos2, ax2, size2.x, size2.y, &cp[0], &cn[0]);
  } else if (t1 == GEOM_SPHERE && t2 == GEOM_BOX) {
    cd[0] = sphere_box(pos1, size1.x, pos2, rot2, size2, &cp[0], &cn[0]);
  } else if (t1 == GEOM_CAPSULE && t2 == GEOM_CAPSULE) {
    capsule_capsule(pos1, ax1, size1, pos2, ax2, size2, margin, cd, cp, cn);
  } else if (t1 == GEOM_CAPSULE && t2 == GEOM_BOX) {
    capsule_box(pos1, ax1, size1.x, size1.y, pos2, rot2, size2, cd, cp, cn);
  } else if (t1 == GEOM_BOX && t2 == GEOM_BOX && !nativeccd) {
    v3 nn;
    const int nc = box_box(pos1, rot1, size1, pos2, rot2, size2, margin, cd, cp, &nn);
    for (int k = 0; k < 8; k++) { cn[k] = nn; if (k >= nc) cd[k] = INFINITY; }
  } else {  // GJK / EPA (collision_convex.py:814-818): cutoff 1e32, so a separated pair still reports its distance
    CGeom a, b;
    a.pos = pos1; a.rot = rot1; a.size = size1; a.margin = margin; a.type = t1;
    b.pos = pos2; b.rot = rot2; b.size = size2; b.margin = margin; b.type = t2;
    fill_mesh(m, g1, a); fill_mesh(m, g2, b);
    float dist = 0.f;
    v3 w1[4], w2[4];
    w1[0] = w2[0] = mk3(0.f, 0.f, 0.f);
    const int nc = ccd_pair(m.ccd_tolerance, 1.0e32f, m.ccd_iterations, epa_iterations, a, b, scratch, &dist, w1, w2, &eovf CCD_CLIP_ARG);
    dist += margin;
    const v3 nrm = dist <= margin ? w1[0] - w2[0] : w2[0] - w1[0];
    for (int k = 0; k < nc; k++) { cd[k] = dist; cp[k] = (w1[k] + w2[k]) * 0.5f; cn[k] = nrm; }
  }
  int best = -1;
  float bd = INFINITY;
  for (int k = 0; k < 8; k++)
    if (cd[k] < bd) { bd = cd[k]; best = k; }
  out[0] = bd;
  if (best < 0) { for (int k = 1; k < SC_WORDS; k++) out[k] = 0.f; return eovf; }
  const v3 n = normalize(cn[best]);  // the contact frame's first row (make_frame)
  st3(out + 1, cp[best] - n * (0.5f * bd));
  st3(out + 4, cp[best] + n * (0.5f * bd));
  return eovf;
}

// sensor.py:642-718 for collision sensor i (of c.nsensorcollision_sensor): the pairs' results `pairs` (nsensorcollision x SC_WORDS) in
// the sensor's loop order, geom1 outer and geom2 inner, the first strict minimum below the cutoff wins; then the flip rule, the cutoff
// rule and the cutoff clamp of _write_scalar / _write_vector (REAL data to [-cutoff, cutoff]; fromto, whose points are positions, is exempt:
// sensor.py:72, :101).  Writes the sensor's slots of `out`.
static __device__ void sensor_collision_reduce(const ModelDev& m, const SensorCollisionDev& c, int i, const float* pairs, float* out) {
  const int s = c.sensor_collision_id[i], type = m.sensor_type[s];
  const float cutoff = m.sensor_cutoff[s];
  float dist = cutoff;
  const float* best = nullptr;
  bool flip = false;
  for (int e = c.sensor_collision_adr[i]; e < c.sensor_collision_adr[i + 1]; e++) {
    const float* p = pairs + SC_WORDS * c.sensor_collision_start_adr[e];
    if (p[0] < dist) { dist = p[0]; best = p; flip = c.sensor_collision_flip[e] != 0; }
  }
  float v[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (type == SENS_GEOMDIST) {
    v[0] = dist;
  } else if (best && dist <= cutoff) {  // no pair below the cutoff: zero normal and fromto
    const v3 p1 = ld3(best + 1), p2 = ld3(best + 4);
    if (type == SENS_GEOMNORMAL) {
      const v3 n = normalize(p2 - p1) * (flip ? -1.0f : 1.0f);
      v[0] = n.x; v[1] = n.y; v[2] = n.z;
    } else {
      st3(v, flip ? p2 : p1); st3(v + 3, flip ? p1 : p2);
    }
  }
  const int dt = m.sensor_datatype[s], adr = m.sensor_adr[s];
  for (int k = 0; k < m.sensor_dim[s]; k++) {
    float x = v[k];
    if (cutoff > 0.f && dt == 0 && type != SENS_GEOMFROMTO) x = fminf(fmaxf(x, -cutoff), cutoff);
    out[adr + k] = x;
  }
}
