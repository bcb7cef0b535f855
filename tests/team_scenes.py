"""MJCF scenes that pin the team kernels (k_position, k_velocity, k_velocity_fluid) to one shared-memory layout regime each.

The team kernels give each world LPW lanes (8, 16 or 32, mjb_team.cuh team_shape) from the words of shared memory one world needs
(k_position.cu pos_layout, k_velocity.cu vel_layout), and those layouts have size-dependent branches.  `pos_words` / `vel_words`
restate the two layouts from the compiled model's sizes, and every scene asserts, from those sizes alone, the inequality that
defines its regime and the lanes per world it must run at -- so a scene that drifts out of its regime fails on the CPU.

No scene has contacts, joint limits or equality constraints (every geom has contype = conaffinity = 0): nefc = 0, and forward's
qacc is qacc_smooth.  Every joint of a long chain has armature >= 0.01, except in `ill` (the ill-conditioned chain).
"""
from mujoco_warp_b200._src import constants as C
from tests import fluid_scenes

MREG = 32  # entries of M per lane that k_velocity prefetches into registers (k_velocity_body.cuh)
BLOCK_MAX = 200 * 1024  # mjb_team.cuh team_shape: a block's bytes; 8 lanes per world while four worlds fit in half of it


def _pad(n):
  return (n + 3) & ~3


def qld_total(mjm):
  return sum(int(n) * int(n) for n in mjm.tree_dofnum)


def pos_words(mjm):
  """k_position's words per world and which region sets them: "tree" (body fields + arena), "geoms" (geom poses from xipos on)
  or "M" (M after the crb * cdof scratch); "arena_qpos" is whether qpos (not 9 nbody) sizes the arena."""
  nb, nj, ng, nv, nq = mjm.nbody, mjm.njnt, mjm.ngeom, mjm.nv, mjm.nq
  xipos = _pad(3 * nb) + _pad(4 * nb)
  tree = xipos + _pad(3 * nb) + 2 * _pad(3 * nj) + _pad(3 * nb) + max(_pad(nq), _pad(9 * nb))
  geoms = xipos + _pad(3 * ng) + _pad(9 * ng)
  M = _pad(6 * nv) + _pad(int(mjm.nC))
  top = max(tree, geoms, M)
  setter = "tree" if top == tree else ("geoms" if top == geoms else "M")
  return dict(words=top + _pad(10 * nb) + _pad(6 * nv), setter=setter, arena_qpos=_pad(nq) > _pad(9 * nb))


def vel_words(mjm):
  """k_velocity's words per world; "cfrc_by_nbody": the cdof_dot / cfrc_int slot is sized by nbody; "own_act": the actuation fields
  have slots of their own (not cinert's); "qld_sets": the dense per-tree factor sets the footprint."""
  nb, nv, nu = mjm.nbody, mjm.nv, mjm.nu
  head = 2 * _pad(nv)
  fields = _pad(6 * nv) + _pad(10 * nb) + _pad(nv) + _pad(6 * nb) + _pad(6 * max(nv, nb)) + _pad(6 * nb)
  own_act = _pad(nv) + _pad(nu) > _pad(10 * nb) + _pad(nv)
  if own_act:
    fields += _pad(nv) + _pad(nu)
  qld = _pad(qld_total(mjm))
  return dict(words=head + max(fields, qld), cfrc_by_nbody=nb > nv, own_act=own_act, qld_sets=qld > fields)


def lanes(words):
  """team_shape's lanes per world for an unbatched model of `words` words per world."""
  lpw = 8
  while lpw < 32 and (words * (32 // lpw) + 4) * 4 > BLOCK_MAX // 2:
    lpw *= 2
  return lpw


def vel_instance(mjm):
  """The k_velocity instance the model runs: "fluid", "pext" (gravity compensation, ball / free joint springs or tendons) or "plain"."""
  o = mjm.opt
  if float(o.density) > 0 or float(o.viscosity) > 0 or any(float(w) != 0 for w in o.wind):
    return "fluid"
  free_ball = [t in (C.JNT_FREE, C.JNT_BALL) for t in mjm.jnt_type]
  springs = any(f and float(k) != 0 for f, k in zip(free_ball, mjm.jnt_stiffness))
  return "pext" if any(float(g) != 0 for g in mjm.body_gravcomp) or springs or int(getattr(mjm, "ntendon", 0)) > 0 else "plain"


# ------------------------------------------------------------------------------------------------------------------------- scenes

_AXES = ("0 1 0", "0 0 1", "1 0 0")


def _chain(prefix, n, kinds, armature, pos, length=0.05):
  """n nested links along x, joint i of kind kinds[i % len(kinds)], hinge / slide axes cycling through _AXES."""
  out = []
  for i in range(n):
    kind, axis = kinds[i % len(kinds)], _AXES[i % 3]
    arm = f' armature="{armature * (1 + 0.25 * (i % 3)):g}"' if armature else ""
    out.append(f'<body name="{prefix}{i}" pos="{pos if i == 0 else f"{length} 0 0"}">'
               f'<joint name="{prefix}j{i}" type="{kind}" axis="{axis}" damping="0.01"{arm}/>'
               f'<geom type="capsule" fromto="0 0 0 {length} 0 0" size="0.01" mass="{0.05 + 0.01 * (i % 4):g}"/>')
  return "".join(out) + "</body>" * n


def _model(name, body, extra="", option=""):
  return f"""
<mujoco model="{name}">
  <option timestep="0.002"{option}/>
  <default><geom contype="0" conaffinity="0"/></default>
  <worldbody>
{body}
  </worldbody>
{extra}
</mujoco>"""


def deep_xml():
  """Two 64-dof chains (hinges; hinges alternating with slides): nv = 128.  The per-tree dense factor (2 x 64 x 64 words) sets
  k_velocity's footprint, and M (2 x 2080 entries) runs far past the MREG * LPW entries k_velocity prefetches.  Fixed tendons with
  springs, dampers and a dead band, one spanning both trees; joint and tendon actuators."""
  # armature 0.1 (not 0.01): with 0.01 an fp32 restatement's qacc_smooth is 2-4x outside the oracle band on these chains
  body = _chain("a", 64, ("hinge",), 0.1, "0 0 1") + _chain("b", 64, ("hinge", "slide"), 0.1, "0 0.5 1")
  extra = """
  <tendon>
    <fixed name="t_ab" stiffness="2" damping="0.1" springlength="-0.05 0.05"><joint joint="aj0" coef="1"/><joint joint="aj1" coef="-0.5"/></fixed>
    <fixed name="t_mid" damping="0.2"><joint joint="bj5" coef="1"/><joint joint="bj6" coef="0.7"/><joint joint="aj20" coef="-0.3"/></fixed>
    <fixed name="t_tip" stiffness="1"><joint joint="aj63" coef="1"/><joint joint="bj63" coef="1"/></fixed>
  </tendon>
  <actuator>
    <motor joint="aj0" gear="2"/> <motor joint="aj31" gear="1"/> <motor joint="bj1" gear="3" ctrlrange="-1 1" ctrllimited="true"/>
    <position joint="bj3" kp="10"/> <velocity joint="aj40" kv="0.2"/>
    <motor tendon="t_tip" gear="2"/> <general tendon="t_ab" gainprm="1.5" biastype="affine" biasprm="0 -1 -0.1"/>
  </actuator>"""
  return _model("deep", body, extra)


def _cams_lights(prefix, b_target):
  """A camera and a light in every mode, in the enclosing body's frame."""
  cams = "".join(f'<camera name="{prefix}c_{m}" pos="0.3 0.2 0.5" mode="{m}"{t}/>'
                 for m, t in (("fixed", ""), ("track", ""), ("trackcom", ""), ("targetbody", f' target="{b_target}"'), ("targetbodycom", f' target="{b_target}"')))
  lights = "".join(f'<light name="{prefix}l_{m}" pos="0.1 0.4 0.9" dir="0 -0.3 -1" mode="{m}"{t}/>'
                   for m, t in (("fixed", ""), ("track", ""), ("trackcom", ""), ("targetbody", f' target="{b_target}"'), ("targetbodycom", f' target="{b_target}"')))
  return cams + lights


def wide_xml(gravcomp=False, nbody=531):
  """A few hundred bodies on few dofs (nbody >> nv): moving trees carrying welded bodies, mocap bodies with welded children, static
  bodies and static world geoms.  Sites, cameras and lights in every mode.  gravcomp=True adds gravity compensation and a ball joint
  spring (the PEXT instance of k_velocity)."""
  gc = lambda v: f' gravcomp="{v}"' if gravcomp else ""
  spring = ' stiffness="2"' if gravcomp else ""
  star = "".join(f'<body name="hs{i}" pos="{0.05 * (i % 8) - 0.2:g} {0.05 * (i // 8) - 0.1:g} 0.1"><geom type="sphere" size="0.02" mass="0.01"/>'
                 f'{"<site/>" if i % 10 == 0 else ""}</body>' for i in range(40))
  def welded_chain(p, n):
    return "".join(f'<body name="{p}{i}" pos="0.04 0 0.01"><geom type="box" size="0.02 0.01 0.01" mass="0.02"/>' for i in range(n)) + "</body>" * n
  moving = f"""
    <body name="hub" pos="0 0 1"{gc(0.5)}>
      <freejoint/><geom type="box" size="0.1 0.1 0.05" mass="1"/><site name="s_hub" pos="0 0 0.1"/>
      {_cams_lights("hub", "arm")}
      {star}
    </body>
    <body name="arm" pos="1 0 1"{gc(1)}>
      <joint type="hinge" axis="0 1 0" armature="0.01" damping="0.1"/><geom type="capsule" fromto="0 0 0 0.2 0 0" size="0.02" mass="0.3"/>
      {welded_chain("aw", 40)}
    </body>
    <body name="pend" pos="-1 0 1">
      <joint type="ball" armature="0.01" damping="0.05"{spring}/><geom type="capsule" fromto="0 0 0 0 0 -0.2" size="0.02" mass="0.2"/>
      {welded_chain("pw", 20)}
      <body name="pend2" pos="0 0 -0.2"{gc(0.3)}>
        <joint type="hinge" axis="1 0 0" armature="0.01"/><geom type="sphere" size="0.03" mass="0.1"/><site name="s_pend2"/>
        {welded_chain("qw", 20)}
      </body>
    </body>
    <body name="mc0" mocap="true" pos="0.5 0.5 0.5" quat="0.92388 0 0.38268 0"><geom type="box" size="0.05 0.05 0.01"/>{welded_chain("m0w", 5)}</body>
    <body name="mc1" mocap="true" pos="-0.5 0.5 0.5"><geom type="sphere" size="0.04"/><site name="s_mc1"/>{welded_chain("m1w", 5)}</body>"""
  fixed = 1 + 1 + 40 + 1 + 40 + 1 + 20 + 1 + 20 + 2 + 10
  nstatic = nbody - fixed
  assert nstatic > 0
  static = "".join(f'<body name="st{i}" pos="{0.1 * (i % 20):g} {0.1 * (i // 20) + 2:g} {0.05 * (i % 3):g}" euler="0 {3 * i % 90} 0">'
                   f'<geom type="{("box", "sphere", "capsule")[i % 3]}" size="0.03 0.02 0.01"/>{"<site/>" if i % 50 == 0 else ""}</body>' for i in range(nstatic))
  world = ('<geom name="floor" type="plane" size="5 5 0.1" pos="0 0 -1"/><geom type="box" size="0.1 0.1 0.1" pos="2 2 0" euler="0 0 30"/>'
           '<site name="s_world" pos="0 0 2"/>' + _cams_lights("world", "hub"))
  return _model("wide_gravcomp" if gravcomp else "wide", world + moving + static)


def geoms_xml():
  """Many more geoms than bodies: a 12-hinge chain whose links carry 36 geoms each and 20 welded bodies of 2 geoms each, plus static
  world geoms -- 928 geoms on 253 bodies.  The geom poses (12 ngeom words from xipos on) set k_position's footprint."""
  shapes = ("sphere", "box", "capsule", "ellipsoid", "cylinder")
  out, n = [], 12
  for i in range(n):
    geoms = "".join(f'<geom type="{shapes[k % 5]}" size="0.01 0.008 0.006" pos="{0.01 * (k % 6):g} {0.01 * (k // 6) - 0.03:g} 0" euler="{5 * k} 0 0" mass="0.002"/>'
                    for k in range(36))
    welded = "".join(f'<body pos="0.02 {0.02 * (k - 10):g} 0.03" euler="0 0 {9 * k}"><geom type="sphere" size="0.005" mass="0.001"/>'
                     f'<geom type="box" size="0.004 0.004 0.004" pos="0 0 0.01" mass="0.001"/></body>' for k in range(20))
    out.append(f'<body name="g{i}" pos="{"0 0 1" if i == 0 else "0.06 0 0"}"><joint type="hinge" axis="{_AXES[i % 2]}" armature="0.01" damping="0.01"/>{geoms}{welded}')
  world = "".join(f'<geom type="box" size="0.05 0.05 0.05" pos="{0.2 * k:g} -1 0"/>' for k in range(16))
  return _model("geoms", world + "".join(out) + "</body>" * n)


def qpos_xml():
  """One body with six ball joints (armature) and one free-jointed body: nq = 31 > 9 nbody = 27, so qpos sizes k_position's arena."""
  balls = "".join(f'<joint name="b{i}" type="ball" pos="{0.02 * i:g} 0 0" armature="{0.01 + 0.005 * i:g}" damping="0.02"/>' for i in range(6))
  body = f"""
    <body name="knot" pos="0 0 1">{balls}<geom type="capsule" fromto="0 0 0 0.3 0 0" size="0.03" mass="0.5"/><site name="s_knot" pos="0.3 0 0"/></body>
    <body name="puck" pos="1 0 1"><freejoint/><geom type="box" size="0.1 0.06 0.03" mass="0.7"/></body>"""
  return _model("qpos", body)


def actuators_xml(nper=14):
  """Many actuators on four dofs (nu = 56): pad(nv) + pad(nu) exceeds cinert's slot, so k_velocity gives the actuation fields slots of
  their own.  Motors, position and velocity servos and affine general actuators, with control and force limits."""
  body = """
    <body name="cart" pos="0 0 1">
      <joint name="cx" type="slide" axis="1 0 0" armature="0.01" damping="0.5"/><joint name="cz" type="slide" axis="0 0 1" armature="0.01"/>
      <geom type="box" size="0.1 0.05 0.05" mass="1"/>
      <body name="pole" pos="0 0 0.05">
        <joint name="cp" type="hinge" axis="0 1 0" armature="0.01" damping="0.02"/><geom type="capsule" fromto="0 0 0 0 0 0.4" size="0.02" mass="0.3"/>
        <body name="tip" pos="0 0 0.4"><joint name="ct" type="hinge" axis="1 0 0" armature="0.01"/><geom type="sphere" size="0.04" mass="0.1"/></body>
      </body>
    </body>"""
  acts = []
  for j in ("cx", "cz", "cp", "ct"):
    for k in range(nper):
      kind = k % 5
      if kind == 0:
        acts.append(f'<motor joint="{j}" gear="{1 + 0.5 * k:g}" ctrlrange="-1 1" ctrllimited="true"/>')
      elif kind == 1:
        acts.append(f'<position joint="{j}" kp="{2 + k:g}" forcerange="-3 3" forcelimited="true"/>')
      elif kind == 2:
        acts.append(f'<velocity joint="{j}" kv="{0.1 * k:g}"/>')
      elif kind == 3:
        acts.append(f'<general joint="{j}" gaintype="affine" gainprm="1 0.2 -0.1" biastype="affine" biasprm="0.05 -0.5 -0.05"/>')
      else:
        acts.append(f'<motor joint="{j}" gear="{-0.3 * k:g}"/>')
  return _model("actuators", body, "<actuator>" + "".join(acts) + "</actuator>")


def pext_xml():
  """Gravity compensation (one joint routing it through the actuators) and ball and free joint springs: k_velocity's PEXT instance."""
  body = """
    <body name="ball0" pos="0 0 1" gravcomp="0.3">
      <joint type="free" stiffness="3" damping="0.2" armature="0.01"/><geom type="sphere" size="0.1" mass="1"/>
    </body>
    <body name="arm" pos="-0.6 0 0.6" gravcomp="1">
      <joint name="slide" type="slide" axis="0 0 1" actuatorgravcomp="true" armature="0.01" damping="2" stiffness="5" springref="0.02"/>
      <geom type="capsule" fromto="0 0 0 0.2 0 0" size="0.03" mass="0.8"/>
      <body name="fore" pos="0.2 0 0">
        <joint name="hinge" type="hinge" axis="0 1 0" armature="0.01" damping="0.1"/><geom type="capsule" fromto="0 0 0 0.25 0 0" size="0.025" mass="0.4"/>
        <body name="pend" pos="0.25 0 0" gravcomp="0.7">
          <joint name="ball" type="ball" armature="0.01" damping="0.05" stiffness="2"/>
          <geom type="capsule" fromto="0 0 0 0 0 -0.2" size="0.02" mass="0.3"/><site name="s_pend" pos="0 0 -0.2"/>
        </body>
      </body>
    </body>"""
  return _model("pext", body, '<actuator><motor joint="slide" gear="10"/><position joint="hinge" kp="20"/></actuator>')


def ill_xml():
  """One 64-hinge chain without armature: M is ill-conditioned, so only backward errors can be held to a tolerance."""
  return _model("ill", _chain("c", 64, ("hinge",), 0.0, "0 0 1"))


def padded_fluid_xml(xml, nstatic):
  """A fluid scene with `nstatic` static, non-colliding bodies appended after its own bodies: the original body and dof indices stay
  the same, and the static bodies carry no dof, so the fluid force they feel reaches no original output."""
  pads = "".join(f'<body name="pad{i}" pos="{0.05 * (i % 30):g} {0.05 * (i // 30) + 3:g} 0"><geom type="sphere" size="0.01" mass="0.001"/></body>'
                 for i in range(nstatic))
  assert xml.count("</worldbody>") == 1
  return xml.replace("</worldbody>", pads + "</worldbody>")


# scene -> (xml, regime check on the compiled model, k_position lanes, k_velocity lanes, k_velocity instance)
def _deep(mjm):
  v = vel_words(mjm)
  assert mjm.nv == 128 and list(mjm.tree_dofnum) == [64, 64], (mjm.nv, list(mjm.tree_dofnum))
  assert v["qld_sets"], v
  assert int(mjm.nC) > MREG * lanes(v["words"]), (mjm.nC, lanes(v["words"]))  # the M tail read in place is reached
  assert mjm.ntendon > 0 and (mjm.actuator_trntype == C.TRN_TENDON).any() and (mjm.actuator_trntype == C.TRN_JOINT).any()


def _wide(mjm):
  assert mjm.nbody >= 20 * mjm.nv and vel_words(mjm)["cfrc_by_nbody"], (mjm.nbody, mjm.nv)
  assert mjm.nsite > 0 and mjm.nmocap == 2
  assert sorted(set(mjm.cam_mode)) == sorted(set(mjm.light_mode)) == list(range(5)), (mjm.cam_mode, mjm.light_mode)
  assert (mjm.geom_bodyid == 0).sum() >= 2 and (mjm.body_weldid[1:] == 0).sum() > 100  # static world geoms and static bodies


def _geoms(mjm):
  assert mjm.ngeom >= 3 * mjm.nbody and pos_words(mjm)["setter"] == "geoms", pos_words(mjm)


def _qpos(mjm):
  p = pos_words(mjm)
  assert p["arena_qpos"] and mjm.nq > 9 * mjm.nbody, (mjm.nq, mjm.nbody)
  assert (mjm.jnt_type == C.JNT_BALL).sum() >= 3 and (mjm.jnt_type == C.JNT_FREE).sum() == 1


def _actuators(mjm):
  assert vel_words(mjm)["own_act"], (mjm.nv, mjm.nu, mjm.nbody)


def _pext(mjm):
  assert (mjm.body_gravcomp != 0).any() and (mjm.jnt_actgravcomp != 0).any()
  for t in (C.JNT_BALL, C.JNT_FREE):
    assert ((mjm.jnt_type == t) & (mjm.jnt_stiffness != 0)).any(), t


def _ill(mjm):
  assert mjm.nv == 64 and not (mjm.dof_armature != 0).any()


SCENES = {
  "deep": (deep_xml(), _deep, 16, 16, "pext"),
  "wide": (wide_xml(), _wide, 32, 32, "plain"),
  "wide_gravcomp": (wide_xml(gravcomp=True), _wide, 32, 32, "pext"),
  "geoms": (geoms_xml(), _geoms, 32, 16, "plain"),
  "qpos": (qpos_xml(), _qpos, 8, 8, "plain"),
  "actuators": (actuators_xml(), _actuators, 8, 8, "plain"),
  "pext": (pext_xml(), _pext, 8, 8, "pext"),
  "ill": (ill_xml(), _ill, 8, 8, "plain"),
}
ILL_CONDITIONED = {"ill"}


def _fluid(nbody0):
  def check(mjm):
    assert (mjm.body_weldid[nbody0:] == 0).all() and (mjm.body_dofnum[nbody0:] == 0).all()
  return check


# fluid scene of tests/fluid_scenes.py padded to reach k_velocity_fluid's 16- and 32-lane instances (the unpadded one runs 8 lanes)
FLUID = {}
for _name, _n, _nb, _lpw in (("chain", 0, 5, 8), ("chain", 240, 5, 16), ("chain", 470, 5, 32), ("ellipsoid", 240, 7, 16), ("ellipsoid", 470, 7, 32)):
  FLUID[f"{_name}_{_lpw}"] = (_name, padded_fluid_xml(fluid_scenes.SCENES[_name][0], _n) if _n else fluid_scenes.SCENES[_name][0], _fluid(_nb), _lpw, _nb)


def check(mjm, regime, pos_lanes, vel_lanes, instance):
  """The scene's regime, lanes per world of both kernels and k_velocity instance, from the compiled model's sizes."""
  regime(mjm)
  p, v = pos_words(mjm), vel_words(mjm)
  if pos_lanes is not None:
    assert lanes(p["words"]) == pos_lanes, (p, pos_lanes)
  assert lanes(v["words"]) == vel_lanes, (v, vel_lanes)
  assert vel_instance(mjm) == instance, vel_instance(mjm)
  if instance == "fluid":  # the fluid scenes are tests/fluid_scenes.py's own, limits included
    return
  assert (mjm.geom_contype == 0).all() and (mjm.geom_conaffinity == 0).all()
  assert not (mjm.jnt_limited != 0).any() and int(getattr(mjm, "neq", 0)) == 0
  if int(getattr(mjm, "ntendon", 0)):
    assert not (mjm.tendon_limited != 0).any()
