// mjb_sensor_extra.cuh -- the magnetometer, camprojection, insidesite and tendon actuator-force sensors of one world, one sensor at a time.
//
// Replaces (reference, /root/reference/mujoco_warp/_src/): sensor.py:117 _magnetometer, :131 _cam_projection, :719-746 (insidesite's
// object position; the site volume is util_misc.py:676 inside_geom, shared with the contact sensor as contact_inside_site) and
// :1598 _tendon_actuator_force.  The tendon limit sensors are the joint-limit scan of k_sensor.cu with the other constraint type.
//
// Plain functions of one sensor; k_sensor.cu's EXTRA build calls them.  The same source also compiles as host C++:
// tests/host_harness/sensor_extra_host.cpp runs it on the CPU against the reference's fixtures.
#pragma once
#include "mjb_math.cuh"
#include "mjb_sensor_contact.cuh"
#include "mjb_types.cuh"

// sensor.py:117: the field opt.magnetic in the site frame
__device__ __forceinline__ v3 sensor_magnetometer(const float* site_xmat, v3 magnetic) {
  const float* R = site_xmat;
  return mk3(R[0] * magnetic.x + R[3] * magnetic.y + R[6] * magnetic.z, R[1] * magnetic.x + R[4] * magnetic.y + R[7] * magnetic.z,
             R[2] * magnetic.x + R[5] * magnetic.y + R[8] * magnetic.z);
}

// sensor.py:131: the pixel coordinates of the site's position in the camera's image.  Focal lengths come from the intrinsic focal
// lengths over the sensor size when both sensor sizes are non-zero, else from fovy; a target in the camera's plane has its depth
// clamped to +-MJ_MINVAL.
__device__ __forceinline__ void sensor_camprojection(v3 target, v3 cam_pos, const float* cam_mat, float fovy, const float* intrinsic, const float* sensorsize,
                                                     const int* res, float* out) {
  const v3 dif = target - cam_pos;
  const float* R = cam_mat;
  const v3 v = mk3(R[0] * dif.x + R[3] * dif.y + R[6] * dif.z, R[1] * dif.x + R[4] * dif.y + R[7] * dif.z, R[2] * dif.x + R[5] * dif.y + R[8] * dif.z);
  const float rx = (float)res[0], ry = (float)res[1];
  float fx, fy;
  if (sensorsize[0] != 0.f && sensorsize[1] != 0.f) {
    fx = intrinsic[0] / (sensorsize[0] + MJ_MINVAL) * rx;
    fy = intrinsic[1] / (sensorsize[1] + MJ_MINVAL) * ry;
  } else {
    fx = fy = 0.5f / tanf(fovy * (3.14159265358979323846f / 360.0f)) * ry;
  }
  float denom = v.z;
  if (fabsf(denom) < MJ_MINVAL) denom = fminf(fmaxf(denom, -MJ_MINVAL), MJ_MINVAL);
  out[0] = -fx * v.x / denom + 0.5f * rx;
  out[1] = fy * v.y / denom + 0.5f * ry;
}

// sensor.py:719-741: the point insidesite tests.  A body's point is its center of mass, or its subtree's for a body without mass whose
// subtree has some (xipos is then the static frame origin); xbody is the frame origin.  pos: the object's position array of the
// sensor's objtype (xipos for body, xpos for xbody, geom_xpos, site_xpos, cam_xpos), subtree_com: the body's subtree com.
__device__ __forceinline__ v3 sensor_inside_point(int objtype, int objid, const float* pos, const float* subtree_com, float body_mass, float body_subtreemass) {
  if (objtype == OBJ_BODY && objid > 0 && body_mass < MJ_MINVAL && body_subtreemass >= MJ_MINVAL) return ld3(subtree_com);
  return ld3(pos);
}

// sensor.py:1598: the force of the actuators that drive the tendon, summed in actuator index order (the reference adds atomically, in
// no fixed order; this sum is the same in every run)
__device__ __forceinline__ float sensor_tendon_actfrc(int nu, const int* trntype, const int* trnid, const float* actuator_force, int tendon) {
  float s = 0.f;
#pragma unroll 1
  for (int a = 0; a < nu; a++)
    if (trntype[a] == TRN_TENDON && trnid[2 * a] == tendon) s += actuator_force[a];
  return s;
}
