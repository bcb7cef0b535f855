// mjb_sensor_contact.cuh -- the <contact> sensor of one world: which contacts match, their order, and what each slot reports.
//
// Replaces (reference, /root/reference/mujoco_warp/_src/): support.py:326-397 contact_force_fn (the contact-frame force decode),
// util_misc.py:676 inside_geom (the site volume), sensor.py:2315 _check_match and :2334-2471 _contact_match (side matching and the
// direction), sensor.py:1810-2010 (slot contents and the netforce reduction).  The match order and the sort are k_sensor_contact's
// (k_sensor_contact.cu): matches in pool order, sorted by (criterion, pool index).
//
// Plain functions of one contact or one slot, plus the in-place sort of the stored matches, which takes its lane and lane count as
// arguments.  The same source also compiles as host C++: tests/host_harness/sensor_contact_host.cpp runs it on the CPU against the fp64
// restatement of tests/contact_sensor_oracle.py.
#pragma once
#include "mjb_math.cuh"
#include "mjb_types.cuh"

// sensor_intprm[0] bits, in MuJoCo's order, and the reductions of sensor_intprm[1]
enum { CSD_FOUND = 1, CSD_FORCE = 2, CSD_TORQUE = 4, CSD_DIST = 8, CSD_POS = 16, CSD_NORMAL = 32, CSD_TANGENT = 64 };
enum { CSR_NONE = 0, CSR_MINDIST = 1, CSR_MAXFORCE = 2, CSR_NETFORCE = 3 };

// floats of one slot: found 1, force 3, torque 3, dist 1, pos 3, normal 3, tangent 3
__device__ __forceinline__ int contact_slot_size(int dataspec) {
  return ((dataspec & CSD_FOUND) ? 1 : 0) + ((dataspec & CSD_FORCE) ? 3 : 0) + ((dataspec & CSD_TORQUE) ? 3 : 0) + ((dataspec & CSD_DIST) ? 1 : 0) +
         ((dataspec & CSD_POS) ? 3 : 0) + ((dataspec & CSD_NORMAL) ? 3 : 0) + ((dataspec & CSD_TANGENT) ? 3 : 0);
}

// The 6D force / torque of one contact in its contact frame (support.py:326-397, no adhesion: adhesion actuators are refused).
// force: the world's efc_force row; adr: the contact's efc_address row; mu: its friction.  Pyramidal rows are decoded from the
// pyramid edges, elliptic rows are the components themselves.  Rows cut by njmax (address -1, or past njmax) read as zero force.
__device__ __forceinline__ void contact_force_decode(int cone, int njmax, const float* force, const int* adr, const float* mu, int dim, float* f) {
  for (int k = 0; k < 6; k++) f[k] = 0.f;
  if (adr[0] < 0) return;
  if (cone == CONE_PYRAMIDAL) {
    if (dim == 1) { f[0] = adr[0] < njmax ? force[adr[0]] : 0.f; return; }
    for (int i = 0; i < dim - 1; i++) {
      const int a = 2 * i + adr[0];
      const float d1 = a < njmax ? force[a] : 0.f, d2 = a + 1 < njmax ? force[a + 1] : 0.f;
      f[0] += d1 + d2;
      f[i + 1] = (d1 - d2) * mu[i];
    }
  } else {
    for (int i = 0; i < dim; i++) if (adr[i] >= 0 && adr[i] < njmax) f[i] = force[adr[i]];
  }
}

// util_misc.py:676 inside_geom: the point p strictly inside the site's primitive (sphere, capsule, ellipsoid, cylinder, box)
__device__ __forceinline__ bool contact_inside_site(v3 pos, const float* mat, v3 size, int type, v3 p) {
  const v3 v = p - pos;
  if (type == GEOM_SPHERE) return dot(v, v) < size.x * size.x;
  const v3 l = mk3(mat[0] * v.x + mat[3] * v.y + mat[6] * v.z, mat[1] * v.x + mat[4] * v.y + mat[7] * v.z, mat[2] * v.x + mat[5] * v.y + mat[8] * v.z);
  if (type == GEOM_CAPSULE) {
    const float z = l.z - fminf(fmaxf(l.z, -size.y), size.y);
    return l.x * l.x + l.y * l.y + z * z < size.x * size.x;
  }
  if (type == GEOM_ELLIPSOID) {
    const v3 s = mk3(l.x / size.x, l.y / size.y, l.z / size.z);
    return dot(s, s) < 1.0f;
  }
  if (type == GEOM_CYLINDER) return fabsf(l.z) < size.y && l.x * l.x + l.y * l.y < size.x * size.x;
  if (type == GEOM_BOX) return fabsf(l.x) < size.x && fabsf(l.y) < size.y && fabsf(l.z) < size.z;
  if (type == GEOM_PLANE) return l.z < 0.f;
  return false;
}

// sensor.py:2315 _check_match: one side of the sensor against one side of the contact.  No object and a site (whose volume test
// already passed) match anything; a subtree matches every body below it.
__device__ __forceinline__ bool contact_side_match(const int* body_parentid, int body, int geom, int type, int id) {
  if (type == 0 || type == OBJ_SITE) return true;
  if (type == OBJ_GEOM) return id == geom;
  if (type == OBJ_BODY) return id == body;
  if (type == OBJ_XBODY) {
    while (body > id) body = body_parentid[body];
    return body == id;
  }
  return false;
}

// sensor.py:2398-2436: 0 if the contact between geoms g1 (body b1) and g2 (body b2) does not match the sensor's sides, else the direction
// +1 / -1 the slot's force z, torque z, normal and tangent are multiplied by (-1 when the sensor's first side is the contact's second)
__device__ __forceinline__ int contact_match_dir(const int* body_parentid, int otype, int oid, int rtype, int rid, int g1, int b1, int g2, int b2) {
  if (otype == 0 && rtype == 0) return 1;
  const bool m11 = contact_side_match(body_parentid, b1, g1, otype, oid), m12 = contact_side_match(body_parentid, b2, g2, otype, oid);
  const bool m21 = contact_side_match(body_parentid, b1, g1, rtype, rid), m22 = contact_side_match(body_parentid, b2, g2, rtype, rid);
  if ((!m11 && !m12) || (!m21 && !m22)) return 0;
  if (otype != 0 && rtype != 0) {
    const bool regular = m11 && m22, reverse = m12 && m21;
    if (!regular && !reverse) return 0;
    return (reverse && !regular) ? -1 : 1;
  }
  if (otype != 0) return m11 ? 1 : -1;
  return m22 ? 1 : -1;
}

// sensor.py:1955-2004: one slot of a matched contact.  f: its contact_force_decode; frame: its contact frame (rows normal, tangent, ...).
__device__ __forceinline__ void contact_slot_write(int dataspec, int nmatch, float dir, const float* f, float dist, const float* pos, const float* frame, float* out) {
  int a = 0;
  if (dataspec & CSD_FOUND) out[a++] = (float)nmatch;
  if (dataspec & CSD_FORCE) { out[a] = f[0]; out[a + 1] = f[1]; out[a + 2] = dir * f[2]; a += 3; }
  if (dataspec & CSD_TORQUE) { out[a] = f[3]; out[a + 1] = f[4]; out[a + 2] = dir * f[5]; a += 3; }
  if (dataspec & CSD_DIST) out[a++] = dist;
  if (dataspec & CSD_POS) { out[a] = pos[0]; out[a + 1] = pos[1]; out[a + 2] = pos[2]; a += 3; }
  if (dataspec & CSD_NORMAL) { out[a] = dir * frame[0]; out[a + 1] = dir * frame[1]; out[a + 2] = dir * frame[2]; a += 3; }
  if (dataspec & CSD_TANGENT) { out[a] = dir * frame[3]; out[a + 1] = dir * frame[4]; out[a + 2] = dir * frame[5]; }
}

// netforce (sensor.py:1857-1945), one contact's part of the sums acc[10]: |force| weight (0), weight * pos (1-3), the world-frame force
// times dir (4-6) and the world-frame torque times dir plus pos x that force (7-9), all about the origin
enum { CNF_WORDS = 10 };
__device__ __forceinline__ void contact_netforce_add(float dir, const float* f, const float* pos, const float* R, float* acc) {
  const float w = sqrtf(f[0] * f[0] + f[1] * f[1] + f[2] * f[2]);
  acc[0] += w;
  for (int k = 0; k < 3; k++) acc[1 + k] += w * pos[k];
  const v3 fg = mk3(R[0] * f[0] + R[3] * f[1] + R[6] * f[2], R[1] * f[0] + R[4] * f[1] + R[7] * f[2], R[2] * f[0] + R[5] * f[1] + R[8] * f[2]) * dir;
  const v3 tg = mk3(R[0] * f[3] + R[3] * f[4] + R[6] * f[5], R[1] * f[3] + R[4] * f[4] + R[7] * f[5], R[2] * f[3] + R[5] * f[4] + R[8] * f[5]) * dir;
  const v3 t = tg + cross(ld3(pos), fg);
  acc[4] += fg.x; acc[5] += fg.y; acc[6] += fg.z;
  acc[7] += t.x; acc[8] += t.y; acc[9] += t.z;
}
// the netforce slot from the sums: the force-weighted centroid, the net force, the net torque about the centroid, dist 0, normal
// (1, 0, 0) and tangent (0, 1, 0)
__device__ __forceinline__ void contact_netforce_write(int dataspec, int nmatch, const float* acc, float* out) {
  const float inv = 1.0f / fmaxf(acc[0], MJ_MINVAL);
  const v3 c = mk3(acc[1] * inv, acc[2] * inv, acc[3] * inv), fn = ld3(acc + 4), t = ld3(acc + 7) - cross(c, fn);
  int a = 0;
  if (dataspec & CSD_FOUND) out[a++] = (float)nmatch;
  if (dataspec & CSD_FORCE) { st3(out + a, fn); a += 3; }
  if (dataspec & CSD_TORQUE) { st3(out + a, t); a += 3; }
  if (dataspec & CSD_DIST) out[a++] = 0.f;
  if (dataspec & CSD_POS) { st3(out + a, c); a += 3; }
  if (dataspec & CSD_NORMAL) { out[a] = 1.f; out[a + 1] = 0.f; out[a + 2] = 0.f; a += 3; }
  if (dataspec & CSD_TANGENT) { out[a] = 0.f; out[a + 1] = 1.f; out[a + 2] = 0.f; }
}

// the stored match i goes after match j: larger criterion, or an equal one and a later pool index
__device__ __forceinline__ bool contact_after(const int* cid, const float* crit, int i, int j) {
  return crit[i] > crit[j] || (crit[i] == crit[j] && cid[i] > cid[j]);
}
// Sorts the n stored matches (cid, crit, dir) by (criterion, pool index), ascending.  A bitonic network over the next power of two, in
// the form whose comparators all put the smaller key at the lower index: the first comparator of each merge pairs i with the mirrored
// index of its block, the others pair i with i + k.  Positions at or past n stand for +infinity, so a comparator that reaches one never
// swaps and is skipped.  Lanes lane, lane + nlane, ... take the comparators of one step; sync() separates the steps.
template <typename Sync>
__device__ __forceinline__ void contact_sort(int* cid, float* crit, float* dir, int n, int lane, int nlane, Sync sync) {
  int P = 1;
  while (P < n) P <<= 1;
  for (int size = 2; size <= P; size <<= 1) {
    for (int k = size >> 1; k > 0; k >>= 1) {
      for (int p = lane; p < (P >> 1); p += nlane) {
        int i, j;
        if (k == (size >> 1)) { const int b = p / k, o = p % k; i = b * size + o; j = b * size + size - 1 - o; }
        else { i = (p / k) * 2 * k + p % k; j = i + k; }
        if (j < n && contact_after(cid, crit, i, j)) {
          const int c = cid[i]; cid[i] = cid[j]; cid[j] = c;
          const float r = crit[i]; crit[i] = crit[j]; crit[j] = r;
          const float s = dir[i]; dir[i] = dir[j]; dir[j] = s;
        }
      }
      sync();
    }
  }
}
