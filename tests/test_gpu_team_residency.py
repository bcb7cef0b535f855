"""Residency of the two team kernels in the benchmark configuration.

k_position and k_velocity are latency bound: their time is the number of residency rounds (waves of blocks that fit on the SMs
at once) times one world's dependent chain (DESIGN.md §3).  For the humanoid at 8192 worlds, every world must be resident at
once, as the occupancy API reports it for the launch shape the library picks."""
import pytest
import torch

from tests import util

pytestmark = pytest.mark.gpu

NWORLD, NCONMAX, NJMAX = 8192, 24, 64


def test_bench_config_fits_one_residency_round(built):
  import mujoco_warp_b200 as mjw

  mjm = mjw.mjcf.load_any(util.HUMANOID)
  m = mjw.put_model(mjm)
  d = mjw.make_data(mjm, nworld=NWORLD, nconmax=NCONMAX, njmax=NJMAX, m=m)
  sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
  res = mjw.team_residency(m, d)
  assert set(res) == {"position", "velocity"}
  for kernel, per_sm in res.items():
    assert per_sm * sms >= NWORLD, f"k_{kernel}: {per_sm} worlds per SM x {sms} SMs < {NWORLD} worlds, so more than one round"
