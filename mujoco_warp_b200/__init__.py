"""mujoco_warp_b200 -- H100-native (sm_90a) batched MuJoCo physics step behind the mujoco_warp API.

Public surface mirrors /root/reference/mujoco_warp/__init__.py for the step path: put_model, put_data, make_data,
reset_data, step, forward and the individually callable stages; `mjcf.load` stands in for mujoco's MJCF compiler.
"""

from . import scenes
from ._src import mjcf
from ._src._lib import build
from ._src.forward import camlight, collision, com_pos, crb, ctrl_noise, euler, factor_m, forward, fwd_acceleration, fwd_actuation
from ._src.forward import fwd_position, fwd_velocity, kinematics, last_launch_count, make_constraint, solve, step, step_profile, transmission
from ._src.forward import com_vel, contact_force, fwd_kinematics, get_state, implicit, mul_m, passive, rne, rungekutta4, sensor_acc, sensor_pos, sensor_vel, set_state, solve_m, step1, step2
from ._src.io import get_data_into, load_trajectory, make_data, override_model, put_data, put_model, reset_data, reset_data_keyframe
from ._src.trace import event_trace_step, flatten_trace
from ._src.types import BroadphaseFilter, BroadphaseType, ConeType, Constraint, ConstraintState, ConstraintType, Contact, Data
from ._src.types import BiasType, DynType, GainType, State, Statistic, TrnType
from ._src.types import DisableBit, EnableBit, GeomType, IntegratorType, JointType, Model, Option, OverflowType, SolverType

__all__ = [n for n in dir() if not n.startswith("_")]
