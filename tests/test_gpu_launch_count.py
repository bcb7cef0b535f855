"""mjb_last_launch_count (bench.py's gpu_launches) against the kernels the same call puts into a CUDA graph.

Every kernel goes through one launch helper that counts it, so the count is the number of kernels the call launched: no more for
calls that launch nothing, no less for the kernels only some models need (k_next_act, k_implicit, k_efc_csr, k_sensor).  Memsets
are not kernels and are not counted.  The reference count is the number of kernel nodes of a graph captured from the call: it is
exact, where a torch.profiler trace of a call this short was seen to miss all of its kernel records."""
import pytest
import torch

from tests.test_oracle_golden_pipeline import load_scene

pytestmark = pytest.mark.gpu


def _captured_kernels(call):
  from cuda.bindings import driver as cu

  torch.cuda.synchronize()
  g = torch.cuda.CUDAGraph(keep_graph=True)
  with torch.cuda.graph(g):
    call()
  graph = cu.CUgraph(g.raw_cuda_graph())
  err, _, n = cu.cuGraphGetNodes(graph, 0)
  assert err == cu.CUresult.CUDA_SUCCESS, err
  err, nodes, n = cu.cuGraphGetNodes(graph, n)
  assert err == cu.CUresult.CUDA_SUCCESS, err
  types = [cu.cuGraphNodeGetType(node)[1] for node in nodes[:n]]
  return sum(t == cu.CUgraphNodeType.CU_GRAPH_NODE_TYPE_KERNEL for t in types)


def _model_data(scene, nworld):
  import mujoco_warp_b200 as mjw

  mjm = load_scene(scene)
  m = mjw.put_model(mjm)
  return mjw, m, mjw.make_data(mjm, nworld=nworld, m=m)


@pytest.mark.parametrize("scene,nworld,expected", [
  ("humanoid", 8, 6),
  ("humanoid", 2048, 12),  # two world halves on internal streams
  ("actuators", 8, None),  # na > 0, Euler: k_next_act after the integrator
  ("actuators_implicit", 8, None),  # k_implicit, k_euler, k_next_act
  ("sensors", 8, None),
  ("g1", 8, None),  # sparse (k_efc_csr) and sensors
  ("mixed_rk4", 8, None),  # four forward passes and four Runge-Kutta stages
])
def test_step_launch_count_matches_kernels_launched(built, scene, nworld, expected):
  mjw, m, d = _model_data(scene, nworld)
  mjw.step(m, d)  # first launches configure the kernel instances
  kernels = _captured_kernels(lambda: mjw.step(m, d))
  assert mjw.last_launch_count() == kernels
  if expected is not None:
    assert kernels == expected


def test_calls_that_launch_nothing_count_zero(built):
  mjw, m, d = _model_data("humanoid", 8)
  ids, force = torch.zeros(0, dtype=torch.int32, device="cuda"), torch.zeros((0, 6), dtype=torch.float32, device="cuda")
  mjw.step(m, d)
  calls = {"sensor_pos (no sensors)": lambda: mjw.sensor_pos(m, d), "contact_force (no ids)": lambda: mjw.contact_force(m, d, ids, False, force)}
  _, m_b, d_b = _model_data("boxes", 8)
  assert m_b.nu == 0
  calls["ctrl_noise (nu = 0)"] = lambda: mjw.ctrl_noise(m_b, d_b, 0)
  for name, call in calls.items():
    kernels = _captured_kernels(call)
    assert kernels == 0 and mjw.last_launch_count() == 0, (name, kernels, mjw.last_launch_count())
