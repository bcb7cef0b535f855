"""Distance / normal / fromto sensors without a GPU: what the MJCF compiler emits for them, and put_model's sensor-pair tables."""
import numpy as np
import pytest

from mujoco_warp_b200._src import constants as C
from mujoco_warp_b200._src import io, mjcf
from tests import sensor_collision_scenes as scenes


def _one(tag, attrs):
  return mjcf.load_string(f"""
<mujoco>
  <worldbody>
    <geom name="floor" type="plane" size="1 1 .1"/>
    <body name="a" pos="0 0 1"><freejoint/><geom name="ga" type="sphere" size=".1"/><geom name="ga2" type="box" size=".1 .1 .1"/></body>
  </worldbody>
  <sensor><{tag} {attrs}/></sensor>
</mujoco>""")


@pytest.mark.parametrize("tag,stype,dim,datatype", [("distance", C.SENS_GEOMDIST, 1, 0), ("normal", C.SENS_GEOMNORMAL, 3, 2), ("fromto", C.SENS_GEOMFROMTO, 6, 0)])
@pytest.mark.parametrize("attrs,obj,ref", [('geom1="floor" geom2="ga"', (C.OBJ_GEOM, 0), (C.OBJ_GEOM, 1)), ('body1="a" geom2="floor"', (C.OBJ_BODY, 1), (C.OBJ_GEOM, 0)),
                                           ('geom1="ga2" body2="a"', (C.OBJ_GEOM, 2), (C.OBJ_BODY, 1))])
def test_compiler_emits_collision_sensors(tag, stype, dim, datatype, attrs, obj, ref):
  mjm = _one(tag, attrs + ' cutoff="0.5"')
  assert mjm.nsensor == 1 and not mjm.sensor_unsupported
  assert (mjm.sensor_type[0], mjm.sensor_dim[0], mjm.sensor_datatype[0], mjm.sensor_needstage[0], mjm.sensor_adr[0]) == (stype, dim, datatype, 1, 0)
  assert (mjm.sensor_objtype[0], mjm.sensor_objid[0]) == obj
  assert (mjm.sensor_reftype[0], mjm.sensor_refid[0]) == ref
  assert mjm.sensor_cutoff[0] == 0.5 and mjm.nsensordata == dim


@pytest.mark.parametrize("attrs", ['geom1="floor"', 'geom1="floor" body1="a" geom2="ga"', 'geom1="floor" geom2="ga" body2="a"', 'body2="a"'])
def test_compiler_refuses_ambiguous_sides(attrs):
  with pytest.raises(ValueError, match="distance sensor 'sensor0'"):
    _one("distance", attrs)


def test_sensor_data_addresses_follow_the_sensor_order():
  mjm = mjcf.load_string(scenes.spheres_xml())
  assert list(mjm.sensor_dim) == [1, 3, 6, 1, 3, 6, 1, 6, 3]
  np.testing.assert_array_equal(mjm.sensor_adr, np.concatenate(([0], np.cumsum(mjm.sensor_dim)[:-1])))


def test_tables_unique_pairs_in_first_seen_order():
  # geoms: obj0 = 0, obj1 = 1, objobj0 = 2, objobj1 = 3 (sphere, sphere, box, capsule)
  mjm = mjcf.load_string(scenes.pair_xml())
  t = io.derive_tables(mjm)
  sc = io._sensor_collision_tables(mjm, t)
  # per sensor tag: geom obj0/obj1 both orders (x2 cutoffs), geom obj0 / body objobj, body obj1 / body objobj; the tags repeat the same pairs
  per_tag = [0, 0, 0, 0,  1, 2, 1, 2, 1, 2, 1, 2,  3, 4, 3, 4, 3, 4, 3, 4]
  assert sc["nsensorcollision"] == 5
  np.testing.assert_array_equal(sc["sensor_collision_start_adr"], per_tag * 3)
  # narrowphase order: geom types ascending (the spheres 0 and 1 come before the box 2 and the capsule 3)
  np.testing.assert_array_equal(sc["sensor_collision_pair"], [[0, 1, -1, -1], [0, 2, -1, -1], [0, 3, -1, -1], [1, 2, -1, -1], [1, 3, -1, -1]])
  np.testing.assert_array_equal(sc["sensor_collision_id"], np.arange(36))
  counts = [1, 1, 1, 1, 2, 2, 2, 2, 2, 2, 2, 2] * 3
  np.testing.assert_array_equal(sc["sensor_collision_adr"], np.concatenate(([0], np.cumsum(counts))))
  # flip: geom1 comes second in narrowphase order (higher type, or the same type and the higher id)
  flip_tag = [0, 1, 0, 1,  0, 0, 1, 1, 0, 0, 1, 1,  0, 0, 1, 1, 0, 0, 1, 1]
  np.testing.assert_array_equal(sc["sensor_collision_flip"], flip_tag * 3)
  assert sc["nsensorcollision_ccd"] == 0  # sphere-box, sphere-capsule and sphere-sphere are primitive pairs


def test_tables_leave_the_contact_pairs_alone():
  with_sensors = mjcf.load_string(scenes.spheres_xml(contact=True))
  without = mjcf.load_string(scenes.spheres_xml(contact=True, sensors=False))
  a, b = io.derive_tables(with_sensors), io.derive_tables(without)
  for k in ("nxn_geom_pair", "nxn_pairid", "nxn_geom_pair_filtered", "nxn_pairid_filtered"):
    np.testing.assert_array_equal(a[k], b[k])
  assert (a["nxn_pairid"][:, 1] == -1).all()
  assert io._sensor_collision_tables(without, b)["nsensorcollision"] == 0


def test_convex_pairs_and_box_box():
  mjm = mjcf.load_string(scenes.pair_xml("ellipsoid", "cylinder", "box", "box"))
  sc = io._sensor_collision_tables(mjm, io.derive_tables(mjm))
  # ellipsoid-cylinder, ellipsoid-box, cylinder-box run GJK / EPA (ranks 0, 1, 2 in first-seen order); the box-box pair too
  np.testing.assert_array_equal(sc["sensor_collision_pair"][:, 3], [0, 1, 2, 3, 4])
  assert sc["nsensorcollision_ccd"] == 5 and sc["sensor_collision_epa_iterations"] == 35
  mjm = mjcf.load_string(scenes.pair_xml("box", "box", "box", "box"))
  sc = io._sensor_collision_tables(mjm, io.derive_tables(mjm))
  assert sc["nsensorcollision_ccd"] == 5 and sc["sensor_collision_epa_iterations"] == 16  # every convex pair is box-box
  mjm = mjcf.load_string(scenes.pair_xml("box", "box", "box", "box", nativeccd=False))
  assert io._sensor_collision_tables(mjm, io.derive_tables(mjm))["nsensorcollision_ccd"] == 0  # the primitive box_box


def test_pairs_without_a_collider_are_refused_by_name():
  mjm = mjcf.load_string("""
<mujoco>
  <worldbody>
    <geom name="p1" type="plane" size="1 1 .1"/>
    <geom name="p2" type="plane" size="1 1 .1" pos="0 0 1"/>
  </worldbody>
  <sensor><distance geom1="p1" geom2="p2"/></sensor>
</mujoco>""")
  with pytest.raises(NotImplementedError, match="plane and plane"):
    io._sensor_collision_tables(mjm, io.derive_tables(mjm))
