"""CPU tests of the host side of energy: the MJCF compiler's energy sensors, option validation, the sensor table put_model derives,
and the put_model / make_data registration of the energy fields against a stub of the C library."""
import numpy as np
import pytest

from mujoco_warp_b200._src import constants as C
from tests import energy_scenes


def test_compiler_emits_the_energy_sensors():
  from mujoco_warp_b200._src import mjcf

  mjm = mjcf.load_string(energy_scenes.joints_xml(sensors=True))
  names = mjm.names.sensor
  for name, typ, cutoff in (("pot", C.SENS_E_POTENTIAL, 0.0), ("kin", C.SENS_E_KINETIC, 0.0), ("pot_cut", C.SENS_E_POTENTIAL, 0.5), ("kin_cut", C.SENS_E_KINETIC, 0.05)):
    s = names.index(name)
    assert mjm.sensor_type[s] == typ and mjm.sensor_dim[s] == 1 and mjm.sensor_datatype[s] == 0 and mjm.sensor_needstage[s] == 1, name
    assert mjm.sensor_objtype[s] == C.OBJ_UNKNOWN and mjm.sensor_objid[s] == -1 and mjm.sensor_cutoff[s] == cutoff, name
  assert list(mjm.sensor_adr) == [0, 1, 2, 3, 4, 5] and mjm.nsensordata == 6
  assert not mjm.sensor_unsupported


def test_validate_accepts_energy_and_names_the_refused_flags():
  from mujoco_warp_b200._src import io as mio
  from mujoco_warp_b200._src import mjcf

  xml = energy_scenes.joints_xml()
  mjm = mjcf.load_string(xml.replace("<option ", '<option><flag energy="enable"/></option><option '))
  assert int(mjm.opt.enableflags) & C.ENBL_ENERGY
  mio._validate(mjm)
  for flag in ("override", "fwdinv", "sleep"):
    bad = mjcf.load_string(xml.replace("<option ", f'<option><flag energy="enable" {flag}="enable"/></option><option '))
    with pytest.raises(NotImplementedError, match=flag):
      mio._validate(bad)


def test_derive_tables_lists_the_energy_sensors():
  from mujoco_warp_b200._src import io as mio
  from mujoco_warp_b200._src import mjcf

  t = mio.derive_tables(mjcf.load_string(energy_scenes.joints_xml(sensors=True)))
  assert t["sensor_energy_adr"].tolist() == [1, 2, 3, 4] and t["sensor_e_potential"] and t["sensor_e_kinetic"]
  t = mio.derive_tables(mjcf.load_string(energy_scenes.joints_xml()))
  assert t["sensor_energy_adr"].tolist() == [] and not t["sensor_e_potential"] and not t["sensor_e_kinetic"]
  t = mio.derive_tables(mjcf.load_string(energy_scenes.joints_xml(sensors=True).replace('<e_kinetic name="kin"/>', "").replace('<e_kinetic name="kin_cut" cutoff="0.05"/>', "")))
  assert t["sensor_energy_adr"].tolist() == [1, 2] and t["sensor_e_potential"] and not t["sensor_e_kinetic"]


@pytest.mark.parametrize("scene", ["sensors_on", "tendon", "humanoid"])
def test_put_model_and_make_data_host_path(monkeypatch, scene):
  """put_model / make_data for an energy scene against a stub of the C library: the sensor table, its counts and Data.energy are
  registered by name."""
  import torch

  from mujoco_warp_b200._src import _lib
  from mujoco_warp_b200._src import io as mio

  calls = []

  class Stub:
    def __getattr__(self, name):
      def f(*a):
        calls.append((name, a))
        return 1 if name in ("mjb_model_create", "mjb_data_create") else 0

      return f

  monkeypatch.setattr(mio, "_require_cuda", lambda: torch.device("cpu"))
  monkeypatch.setattr(_lib, "lib", lambda: Stub())
  mjm = energy_scenes.load(scene)
  m = mio.put_model(mjm, batch_sizes={f: 3 for f in energy_scenes.per_world_inputs(scene, mjm)})
  d = mio.make_data(mjm, nworld=3, nconmax=8, njmax=32, m=m)
  ints = {a[1].decode(): a[2] for n, a in calls if n == "mjb_model_set_int"}
  arrays = {a[1].decode() for n, a in calls if n == "mjb_model_set_array_batched"}
  data = {a[1].decode() for n, a in calls if n == "mjb_data_set_array"}
  nsens = 4 if scene.startswith("sensors") else 0
  assert ints["nsensor_energy"] == nsens and ints["sensor_e_potential"] == int(nsens > 0) and ints["sensor_e_kinetic"] == int(nsens > 0)
  assert ints["enableflags"] & C.ENBL_ENERGY
  assert "sensor_energy_adr" in arrays and "energy" in data
  assert d.energy.shape == (3, 2) and len(m.sensor_energy_adr) == nsens
  assert np.array_equal(m.sensor_energy_adr.numpy(), np.arange(1, 1 + nsens))
