"""The team-kernel scenes (tests/team_scenes.py) stay in their shared-memory layout regimes: checked from the compiled model's sizes,
without a GPU, so that a scene that drifts out of its regime (and would no longer reach the kernel instance or layout branch its GPU
test is there for) fails here."""
import pytest

from mujoco_warp_b200._src import mjcf
from tests import team_scenes as T


@pytest.mark.parametrize("scene", sorted(T.SCENES))
def test_scene_stays_in_its_regime(scene):
  xml, regime, pos_lanes, vel_lanes, instance = T.SCENES[scene]
  T.check(mjcf.load_string(xml), regime, pos_lanes, vel_lanes, instance)


@pytest.mark.parametrize("scene", sorted(T.FLUID))
def test_padded_fluid_scene_reaches_its_lanes(scene):
  base, xml, regime, vel_lanes, nbody0 = T.FLUID[scene]
  T.check(mjcf.load_string(xml), regime, None, vel_lanes, "fluid")


def test_scenes_cover_every_lane_count_of_every_instance():
  pos = {s[2] for s in T.SCENES.values()}
  vel = {(s[4], s[3]) for s in T.SCENES.values()} | {("fluid", f[3]) for f in T.FLUID.values()}
  assert pos == {8, 16, 32}
  assert vel == {(i, l) for i in ("plain", "pext", "fluid") for l in (8, 16, 32)}, sorted(vel)


def test_layout_restatement_matches_the_documented_humanoid_footprint():
  from tests import util

  mjm = mjcf.load_any(util.HUMANOID)  # DESIGN.md §3: 852 / 792 words per humanoid world
  assert (T.pos_words(mjm)["words"], T.vel_words(mjm)["words"]) == (852, 792)
  assert T.lanes(852) == T.lanes(792) == 8
