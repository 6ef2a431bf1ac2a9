"""newton_b200 - H100-native batched rigid-body stepper behind Newton's solver API."""

use_coord_layout_targets: bool = False
"""Default layout of the position targets an :class:`~newton_b200.actuators.Actuator` built without ``target_pos_indices``
reads (the reference's ``newton.use_coord_layout_targets``): ``True`` -> its ``pos_indices`` (coordinate layout), ``False``
-> its dof ``indices``.  Read once, when the actuator is built."""

from .sim import (  # noqa: F401
    MAXVAL, BodyFlags, Contacts, Control, GeoType, JointDofConfig, JointType, Model, ModelBuilder,
    ModelFlags, ShapeConfig, ShapeFlags, State, StateFlags, eval_fk, eval_ik, eval_inverse_dynamics_force,
    eval_inverse_dynamics_passive, eval_jacobian, eval_mass_matrix,
)
from .sim.collide import CollisionPipeline, SpeculativeContactConfig  # noqa: F401,E402
from . import solvers  # noqa: F401,E402
from . import selection  # noqa: F401,E402
from . import sensors  # noqa: F401,E402
from . import actuators  # noqa: F401,E402
from . import controllers  # noqa: F401,E402
from . import ik  # noqa: F401,E402
from .geometry import intersect_ray  # noqa: F401,E402
