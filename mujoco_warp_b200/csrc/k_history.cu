// k_history.cu -- actuator and sensor delays: one thread per (world, actuator) or (world, delayed sensor) over the ring buffers of
// mjb_history.cuh.
//
// Replaces (reference, /root/reference/mujoco_warp/_src/history.py): :361 _read_ctrl_delayed_kernel (forward.py:1162, fwd_actuation),
// :391 _insert_ctrl_history_kernel (forward.py:320, _advance), :416 / :460 the sensor delay + insert pair of apply_sensor_delay (sensor.py
// :956, :1502, :2765), and the kernels of the public read_ctrl / read_sensor / init_ctrl_history / init_sensor_history (:600-925).
// apply_sensor_delay copies sensordata, overwrites it and inserts the copy, in three launches; here each sensor's thread keeps its
// fresh value in registers between the read and the insert, which is the same order because every buffer belongs to one sensor.
#include "mjb_history.cuh"
#include "mjb_launch.cuh"
#include "mjb_types.cuh"

namespace {

constexpr int kMaxSensorDim = 6;  // the widest sensor this build compiles (fromto)

__global__ void k_history_ctrl_read(const __grid_constant__ ModelDev m, const __grid_constant__ DataDev d, const __grid_constant__ HistoryDev h) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= d.wn * m.nu) return;
  const int w = d.w0 + idx / m.nu, u = idx % m.nu;
  const size_t wu = (size_t)w * m.nu + u;
  const int n = h.actuator_history[2 * u];
  const float delay = h.actuator_delay[u];
  float v = d.ctrl[wu];
  if (n > 0 && delay != 0.0f) hist_read(h.history + (size_t)w * h.nhistory + h.actuator_historyadr[u], n, 1, d.time[w] - delay, h.actuator_history[2 * u + 1], &v);
  h.ctrl_delayed[wu] = v;
}

__global__ void k_history_ctrl_insert(const __grid_constant__ ModelDev m, const __grid_constant__ DataDev d, const __grid_constant__ HistoryDev h) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= d.wn * m.nu) return;
  const int w = d.w0 + idx / m.nu, u = idx % m.nu;
  const int n = h.actuator_history[2 * u];
  if (n == 0) return;
  hist_insert(h.history + (size_t)w * h.nhistory + h.actuator_historyadr[u], n, 1, d.time[w], d.ctrl + (size_t)w * m.nu + u);
}

__global__ void k_history_sensor(const __grid_constant__ ModelDev m, const __grid_constant__ DataDev d, const __grid_constant__ HistoryDev h, int stages) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= d.wn * h.nsensor_history) return;
  const int w = d.w0 + idx / h.nsensor_history, s = h.sensor_history_id[idx % h.nsensor_history];
  const int stage = m.sensor_needstage[s];
  if (stage < 1 || !(stages & (1 << (stage - 1)))) return;
  float fresh[kMaxSensorDim];
  hist_sensor(h.history + (size_t)w * h.nhistory + h.sensor_historyadr[s], h.sensor_history[2 * s], m.sensor_dim[s], h.sensor_history[2 * s + 1], h.sensor_delay[s],
              h.sensor_interval[2 * s], d.time[w], d.sensordata + (size_t)w * m.nsensordata + m.sensor_adr[s], fresh);
}

// history.py:600-752: one actuator's (dim 1) or sensor's value at time[w] - delay; the current value when it has no buffer
__global__ void k_history_read(const __grid_constant__ ModelDev m, const __grid_constant__ DataDev d, const __grid_constant__ HistoryDev h, int sensor, int id,
                               const float* __restrict__ time, int interp, float* __restrict__ result) {
  const int w = blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= d.nworld) return;
  const int* hist = (sensor ? h.sensor_history : h.actuator_history) + 2 * id;
  const int dim = sensor ? m.sensor_dim[id] : 1;
  const float* cur = sensor ? d.sensordata + (size_t)w * m.nsensordata + m.sensor_adr[id] : d.ctrl + (size_t)w * m.nu + id;
  float* out = result + (size_t)w * dim;
  if (hist[0] == 0) {
    for (int k = 0; k < dim; k++) out[k] = cur[k];
    return;
  }
  const float delay = sensor ? h.sensor_delay[id] : h.actuator_delay[id];
  const int adr = sensor ? h.sensor_historyadr[id] : h.actuator_historyadr[id];
  hist_read(h.history + (size_t)w * h.nhistory + adr, hist[0], dim, time[w] - delay, interp < 0 ? hist[1] : interp, out);
}

// history.py:755-925: one buffer of every world from times (or -MJ_MAXVAL stamps) and values, newest last (cursor n - 1); the user slot
// is set to phase[w] for a sensor and kept for an actuator
__global__ void k_history_init(const __grid_constant__ ModelDev m, const __grid_constant__ DataDev d, const __grid_constant__ HistoryDev h, int sensor, int id,
                               const float* __restrict__ times, const float* __restrict__ values, const float* __restrict__ phase) {
  const int w = blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= d.nworld) return;
  const int n = (sensor ? h.sensor_history : h.actuator_history)[2 * id];
  const int dim = sensor ? m.sensor_dim[id] : 1;
  float* buf = h.history + (size_t)w * h.nhistory + (sensor ? h.sensor_historyadr[id] : h.actuator_historyadr[id]);
  if (sensor) buf[0] = phase[w];
  buf[1] = (float)(n - 1);
  for (int i = 0; i < n; i++) {
    buf[2 + i] = times ? times[i] : -MJ_MAXVAL;
    for (int k = 0; k < dim; k++) buf[2 + n + i * dim + k] = values[(size_t)w * n * dim + i * dim + k];
  }
}

}  // namespace

cudaError_t launch_history_ctrl_read(const ModelDev& m, const DataDev& d, const HistoryDev& h, cudaStream_t s) {
  const int n = d.wn * m.nu;
  return launch(k_history_ctrl_read, (n + 127) / 128, 128, 0, s, m, d, h);
}
cudaError_t launch_history_ctrl_insert(const ModelDev& m, const DataDev& d, const HistoryDev& h, cudaStream_t s) {
  const int n = d.wn * m.nu;
  return launch(k_history_ctrl_insert, (n + 127) / 128, 128, 0, s, m, d, h);
}
cudaError_t launch_history_sensor(const ModelDev& m, const DataDev& d, const HistoryDev& h, int stages, cudaStream_t s) {
  const int n = d.wn * h.nsensor_history;
  return launch(k_history_sensor, (n + 127) / 128, 128, 0, s, m, d, h, stages);
}
cudaError_t launch_history_read(const ModelDev& m, const DataDev& d, const HistoryDev& h, int sensor, int id, const float* time, int interp, float* result, cudaStream_t s) {
  return launch(k_history_read, (d.nworld + 127) / 128, 128, 0, s, m, d, h, sensor, id, time, interp, result);
}
cudaError_t launch_history_init(const ModelDev& m, const DataDev& d, const HistoryDev& h, int sensor, int id, const float* times, const float* values, const float* phase,
                                cudaStream_t s) {
  return launch(k_history_init, (d.nworld + 127) / 128, 128, 0, s, m, d, h, sensor, id, times, values, phase);
}
