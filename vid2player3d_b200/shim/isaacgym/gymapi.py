"""`isaacgym.gymapi` shim: constants and plain-data parameter classes only.

Only what the reference's config / task modules touch at import or config-parse time
(SURVEY.md §8b Level B).  `acquire_gym()` returns an object whose every method raises:
with the Level-A boundary the task classes never call gym.* (create_sim is stubbed).
"""

SIM_PHYSX = 1
SIM_FLEX = 0
UP_AXIS_Y = 0
UP_AXIS_Z = 1
DOF_MODE_NONE = 0
DOF_MODE_POS = 1
DOF_MODE_VEL = 2
DOF_MODE_EFFORT = 3
ENV_SPACE = 0
LOCAL_SPACE = 1
GLOBAL_SPACE = 2
MESH_VISUAL = 1
MESH_COLLISION = 2
MESH_VISUAL_AND_COLLISION = 3
STATE_ALL = 3
for _i, _k in enumerate(["ESCAPE", "V", "R", "L", "Q", "W", "A", "S", "D", "E", "F", "T", "Y", "J", "K",
                         "M", "N", "P", "B", "C", "G", "H", "X", "Z", "LEFT", "RIGHT", "UP", "DOWN", "SPACE",
                         "1", "2", "3", "4", "5", "6", "7", "8", "9", "0"]):
    globals()["KEY_" + _k] = _i


class Vec3:
    def __init__(self, x=0.0, y=0.0, z=0.0):
        self.x, self.y, self.z = float(x), float(y), float(z)

    def __iter__(self):
        return iter((self.x, self.y, self.z))

    def __repr__(self):
        return f"Vec3({self.x}, {self.y}, {self.z})"


class Quat:
    def __init__(self, x=0.0, y=0.0, z=0.0, w=1.0):
        self.x, self.y, self.z, self.w = float(x), float(y), float(z), float(w)


class Transform:
    def __init__(self, p=None, r=None):
        self.p = p if p is not None else Vec3()
        self.r = r if r is not None else Quat()


class PlaneParams:
    def __init__(self):
        self.normal = Vec3(0, 0, 1)
        self.distance = 0.0
        self.static_friction = 1.0
        self.dynamic_friction = 1.0
        self.restitution = 0.0


class AssetOptions:
    def __init__(self):
        self.angular_damping = 0.5
        self.linear_damping = 0.0
        self.max_angular_velocity = 64.0
        self.max_linear_velocity = 1000.0
        self.default_dof_drive_mode = DOF_MODE_NONE
        self.fix_base_link = False
        self.collapse_fixed_joints = False
        self.density = 1000.0
        self.armature = 0.0
        self.thickness = 0.02


class CameraProperties:
    def __init__(self):
        self.width = 1600
        self.height = 900
        self.horizontal_fov = 90.0


class PhysXParams:
    def __init__(self):
        self.solver_type = 1
        self.num_position_iterations = 4
        self.num_velocity_iterations = 1
        self.num_threads = 0
        self.use_gpu = False
        self.num_subscenes = 0
        self.contact_offset = 0.02
        self.rest_offset = 0.001
        self.bounce_threshold_velocity = 0.2
        self.max_depenetration_velocity = 100.0
        self.default_buffer_size_multiplier = 2.0
        self.max_gpu_contact_pairs = 1024 * 1024
        self.friction_offset_threshold = 0.04
        self.friction_correlation_distance = 0.025
        self.always_use_articulations = False
        self.contact_collection = 2


class FlexParams:
    def __init__(self):
        self.solver_type = 5
        self.num_outer_iterations = 4
        self.num_inner_iterations = 20
        self.relaxation = 0.75
        self.warm_start = 0.4
        self.shape_collision_margin = 0.01
        self.deterministic_mode = False


class SimParams:
    def __init__(self):
        self.dt = 1.0 / 60.0
        self.substeps = 2
        self.up_axis = UP_AXIS_Y
        self.gravity = Vec3(0.0, -9.8, 0.0)
        self.use_gpu_pipeline = False
        self.num_client_threads = 0
        self.physx = PhysXParams()
        self.flex = FlexParams()


class _NoGym:
    def __getattr__(self, name):
        def _raise(*a, **k):
            raise RuntimeError(
                f"isaacgym shim: gym.{name}() is not available - physics runs in the CUDA "
                "extension behind the Task surface (include/b200env.h), not through gymapi")
        return _raise


def acquire_gym():
    return _NoGym()
