// mjb_history.cuh -- the ring buffers of actuator and sensor delays: one buffer of one world, [user, cursor, times[n], values[n * dim]].
//
// Replaces (reference, /root/reference/mujoco_warp/_src/history.py): :27 _history_physical_index, :33 _history_find_index (circular
// binary search), :77 / :156 _history_read_scalar / _vector (zero-order hold, linear, Catmull-Rom), :255 / :306 _history_insert_scalar /
// _vector (exact-match replace, replace-oldest, advance the cursor, out-of-order shift) and the interval rule of :447-456 / :499-507.
// Plain functions of a buffer pointer (no warp intrinsics, no shared memory), kept in a header so that the same source also compiles
// as host C++: tests/host_harness/history_host.cpp replays the reference's read / insert vectors through THIS code on the CPU.
#pragma once
#include "mjb_types.cuh"

// logical index (0 oldest, n - 1 newest) -> slot
__device__ __forceinline__ int hist_phys(int cursor, int n, int logical) { return (cursor + 1 + logical) % n; }

// The smallest logical i with times[i] >= t: 0 if t <= the oldest time, n if t > the newest.
__device__ __forceinline__ int hist_find(const float* buf, int n, int cursor, float t) {
  const float* times = buf + 2;
  if (t <= times[hist_phys(cursor, n, 0)]) return 0;
  if (t > times[hist_phys(cursor, n, n - 1)]) return n;
  int lo = 0, hi = n - 1;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (times[hist_phys(cursor, n, mid)] < t) lo = mid;
    else hi = mid;
  }
  return hi;
}

// The value (dim floats) at time t into out; interp 0 zero-order hold, 1 linear, 2 cubic (Catmull-Rom, slopes 0 at the ends).
// Times within 1e-6 of the oldest / newest sample or of a sample in between read that sample.
__device__ __forceinline__ void hist_read(const float* buf, int n, int dim, float t, int interp, float* out) {
  const int cursor = (int)buf[1];
  const float* times = buf + 2;
  const float* vals = buf + 2 + n;
  const int p_old = hist_phys(cursor, n, 0), p_new = hist_phys(cursor, n, n - 1);
  int p = -1;
  if (t <= times[p_old] + 1e-6f) p = p_old;
  else if (t >= times[p_new] - 1e-6f) p = p_new;
  const int i = p < 0 ? hist_find(buf, n, cursor, t) : 0;
  if (p < 0 && fabsf(t - times[hist_phys(cursor, n, i)]) < 1e-6f) p = hist_phys(cursor, n, i);
  if (p < 0 && interp == 0) p = hist_phys(cursor, n, i - 1);
  if (p >= 0) {
    for (int k = 0; k < dim; k++) out[k] = vals[p * dim + k];
    return;
  }
  const int lo = hist_phys(cursor, n, i - 1), hi = hist_phys(cursor, n, i);
  const float dt = times[hi] - times[lo], alpha = (t - times[lo]) / dt;
  if (interp == 1) {
    for (int k = 0; k < dim; k++) {
      const float v_lo = vals[lo * dim + k], v_hi = vals[hi * dim + k];
      out[k] = v_lo + alpha * (v_hi - v_lo);
    }
    return;
  }
  const float a2 = alpha * alpha, a3 = a2 * alpha;
  const float h00 = 2.0f * a3 - 3.0f * a2 + 1.0f, h10 = a3 - 2.0f * a2 + alpha, h01 = -2.0f * a3 + 3.0f * a2, h11 = a3 - a2;
  const int lo_prev = i > 1 ? hist_phys(cursor, n, i - 2) : -1, hi_next = i < n - 1 ? hist_phys(cursor, n, i + 1) : -1;
  for (int k = 0; k < dim; k++) {
    const float v_lo = vals[lo * dim + k], v_hi = vals[hi * dim + k];
    const float m_lo = lo_prev >= 0 ? (v_hi - vals[lo_prev * dim + k]) / (times[hi] - times[lo_prev]) : 0.0f;
    const float m_hi = hi_next >= 0 ? (vals[hi_next * dim + k] - v_lo) / (times[hi_next] - times[lo]) : 0.0f;
    out[k] = h00 * v_lo + h10 * dt * m_lo + h01 * v_hi + h11 * dt * m_hi;
  }
}

// Inserts value (dim floats) at time t: replaces a sample within 1e-6 of t, else replaces the oldest when t is older, else advances
// the cursor when t is newer, else shifts the older samples down one slot and inserts in time order.
__device__ __forceinline__ void hist_insert(float* buf, int n, int dim, float t, const float* value) {
  int cursor = (int)buf[1];
  float* times = buf + 2;
  float* vals = buf + 2 + n;
  const int i = hist_find(buf, n, cursor, t);
  int slot = -1;
  if (i < n && fabsf(t - times[hist_phys(cursor, n, i)]) < 1e-6f) slot = hist_phys(cursor, n, i);
  if (slot < 0) {
    if (i == 0) {
      slot = hist_phys(cursor, n, 0);
    } else if (i == n) {
      cursor = (cursor + 1) % n;
      buf[1] = (float)cursor;
      slot = cursor;
    } else {
      for (int j = 0; j < i - 1; j++) {
        const int src = hist_phys(cursor, n, j + 1), dst = hist_phys(cursor, n, j);
        times[dst] = times[src];
        for (int k = 0; k < dim; k++) vals[dst * dim + k] = vals[src * dim + k];
      }
      slot = hist_phys(cursor, n, i - 1);
    }
    times[slot] = t;
  }
  for (int k = 0; k < dim; k++) vals[slot * dim + k] = value[k];
}

// One sensor of one world after its stage computed `data` (dim floats, sensordata): the reported value becomes the one read at
// t - delay (delay > 0), or the held one while an interval sensor is not due (user slot + period > t); then the fresh value is inserted
// at t, for an interval sensor only when it is due, advancing the user slot by one period.  `fresh` holds the fresh value meanwhile.
__device__ __forceinline__ void hist_sensor(float* buf, int n, int dim, int interp, float delay, float period, float t, float* data, float* fresh) {
  for (int k = 0; k < dim; k++) fresh[k] = data[k];
  if (delay > 0.0f) hist_read(buf, n, dim, t - delay, interp, data);
  else if (period > 0.0f && buf[0] + period > t) hist_read(buf, n, dim, t, interp, data);
  if (period > 0.0f) {
    const float prev = buf[0];
    if (prev + period > t) return;
    buf[0] = prev + period;
  }
  hist_insert(buf, n, dim, t, fresh);
}
