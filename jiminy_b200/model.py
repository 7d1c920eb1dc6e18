"""Host-side model compiler: URDF + hardware TOML + options TOML -> flat `RobotTable`.

This is set-up code (runs once per robot), written in Python like the reference's own loader
(`python/jiminy_py/src/jiminy_py/robot.py:518-847`).  It reproduces what `jiminy::Model` /
`jiminy::Robot` hand to the engine:

* the Pinocchio 2.7 model built by `pinocchio::urdf::buildModel` (reference call site
  `core/src/utilities/pinocchio.cc:828-934`): joints visited depth-first with children sorted by
  **joint name** (urdfdom keeps joints in a `std::map`), fixed joints merged into their parent
  joint's body, `root_joint` free-flyer when `has_freeflyer` (SURVEY.md App. B/C);
* joint position limits (`core/src/robot/model.cc:1371-1440`);
* `SimpleMotor` proxies (`core/src/hardware/abstract_motor.cc:246-345`) and the rotor-inertia
  accumulation (`core/src/robot/robot.cc:243-246`);
* contact frames sorted by name (`robot.py:717`), sensors in attach order per type.

Nothing here touches the GPU; the resulting tables are handed to the C ABI (`include/jiminy_b200.h`).
"""
from __future__ import annotations

import math
import os
import tomllib
import xml.etree.ElementTree as ET
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

# Joint model codes, must match include/jiminy_b200.h
JB_JOINT_UNIVERSE = 0
JB_JOINT_RX, JB_JOINT_RY, JB_JOINT_RZ, JB_JOINT_RU = 1, 2, 3, 4
JB_JOINT_RUBX, JB_JOINT_RUBY, JB_JOINT_RUBZ, JB_JOINT_RUBU = 5, 6, 7, 8
JB_JOINT_PX, JB_JOINT_PY, JB_JOINT_PZ, JB_JOINT_PU = 9, 10, 11, 12
JB_JOINT_FREEFLYER = 13
JB_JOINT_SPHERICAL = 14

JOINT_NQ = {JB_JOINT_UNIVERSE: 0, JB_JOINT_FREEFLYER: 7, JB_JOINT_SPHERICAL: 4}
JOINT_NV = {JB_JOINT_UNIVERSE: 0, JB_JOINT_FREEFLYER: 6, JB_JOINT_SPHERICAL: 3}
for _t in (JB_JOINT_RX, JB_JOINT_RY, JB_JOINT_RZ, JB_JOINT_RU,
           JB_JOINT_PX, JB_JOINT_PY, JB_JOINT_PZ, JB_JOINT_PU):
    JOINT_NQ[_t] = 1
    JOINT_NV[_t] = 1
for _t in (JB_JOINT_RUBX, JB_JOINT_RUBY, JB_JOINT_RUBZ, JB_JOINT_RUBU):
    JOINT_NQ[_t] = 2
    JOINT_NV[_t] = 1

EPS = np.finfo(np.float64).eps
INF = float("inf")


# --------------------------------------------------------------------------- SE3 / inertia
def rpy_to_matrix(rpy: Sequence[float]) -> np.ndarray:
    """URDF fixed-axis roll/pitch/yaw -> rotation matrix, R = Rz(yaw) Ry(pitch) Rx(roll)."""
    r, p, y = (float(x) for x in rpy)
    cr, sr, cp, sp, cy, sy = math.cos(r), math.sin(r), math.cos(p), math.sin(p), math.cos(y), math.sin(y)
    return np.array([
        [cy * cp, cy * sp * sr - sy * cr, cy * sp * cr + sy * sr],
        [sy * cp, sy * sp * sr + cy * cr, sy * sp * cr - cy * sr],
        [-sp, cp * sr, cp * cr]])


@dataclass
class SE3:
    R: np.ndarray = field(default_factory=lambda: np.eye(3))
    p: np.ndarray = field(default_factory=lambda: np.zeros(3))

    def __mul__(self, other: "SE3") -> "SE3":
        return SE3(self.R @ other.R, self.R @ other.p + self.p)

    def inverse(self) -> "SE3":
        return SE3(self.R.T.copy(), -self.R.T @ self.p)

    def flat(self) -> np.ndarray:
        return np.concatenate([self.R.reshape(9), self.p])


@dataclass
class Inertia:
    """Spatial inertia as Pinocchio stores it: mass, lever (CoM), rotational inertia about the CoM."""
    mass: float = 0.0
    lever: np.ndarray = field(default_factory=lambda: np.zeros(3))
    I: np.ndarray = field(default_factory=lambda: np.zeros((3, 3)))

    def transformed(self, M: SE3) -> "Inertia":
        """`M.act(Y)`: express the inertia in the parent frame."""
        return Inertia(self.mass, M.R @ self.lever + M.p, M.R @ self.I @ M.R.T)

    def __add__(self, other: "Inertia") -> "Inertia":
        mab = self.mass + other.mass
        mab_inv = 1.0 / max(mab, EPS)
        ab = self.lever - other.lever
        skew_sq = np.outer(ab, ab) - np.dot(ab, ab) * np.eye(3)  # [ab]x [ab]x
        lever = (self.mass * self.lever + other.mass * other.lever) * mab_inv
        I = self.I + other.I - (self.mass * other.mass * mab_inv) * skew_sq
        return Inertia(mab, lever, I)

    def flat(self) -> np.ndarray:
        I = self.I
        return np.array([self.mass, *self.lever, I[0, 0], I[0, 1], I[1, 1], I[0, 2], I[1, 2], I[2, 2]])


# --------------------------------------------------------------------------- URDF parsing
@dataclass
class UrdfJoint:
    name: str
    type: str
    parent: str
    child: str
    origin: SE3
    axis: np.ndarray
    lower: float
    upper: float
    effort: float
    velocity: float


@dataclass
class UrdfBox:
    size: np.ndarray
    origin: SE3


@dataclass
class UrdfLink:
    name: str
    inertia: Inertia
    collision_boxes: List[UrdfBox]
    has_collision_mesh: bool


def _floats(text: Optional[str], default: Sequence[float]) -> np.ndarray:
    if text is None:
        return np.array(default, dtype=np.float64)
    return np.array([float(x) for x in text.split()], dtype=np.float64)


def _origin(elem: Optional[ET.Element]) -> SE3:
    if elem is None:
        return SE3()
    xyz = _floats(elem.get("xyz"), (0.0, 0.0, 0.0))
    rpy = _floats(elem.get("rpy"), (0.0, 0.0, 0.0))
    return SE3(rpy_to_matrix(rpy), xyz)


def parse_urdf(path: str) -> Tuple[str, Dict[str, UrdfLink], Dict[str, UrdfJoint]]:
    root = ET.parse(path).getroot()
    links: Dict[str, UrdfLink] = {}
    joints: Dict[str, UrdfJoint] = {}
    for le in root.findall("link"):
        ie = le.find("inertial")
        if ie is not None:
            M = _origin(ie.find("origin"))
            mass = float(ie.find("mass").get("value")) if ie.find("mass") is not None else 0.0
            it = ie.find("inertia")
            if it is not None:
                ixx, ixy, ixz = (float(it.get(k, 0.0)) for k in ("ixx", "ixy", "ixz"))
                iyy, iyz, izz = (float(it.get(k, 0.0)) for k in ("iyy", "iyz", "izz"))
            else:
                ixx = ixy = ixz = iyy = iyz = izz = 0.0
            I = np.array([[ixx, ixy, ixz], [ixy, iyy, iyz], [ixz, iyz, izz]])
            Y = Inertia(mass, M.p.copy(), M.R @ I @ M.R.T)
        else:
            Y = Inertia()
        boxes, has_mesh = [], False
        for ce in le.findall("collision"):
            ge = ce.find("geometry")
            if ge is None:
                continue
            be = ge.find("box")
            if be is not None:
                boxes.append(UrdfBox(_floats(be.get("size"), (0, 0, 0)), _origin(ce.find("origin"))))
            elif ge.find("mesh") is not None:
                has_mesh = True
        links[le.get("name")] = UrdfLink(le.get("name"), Y, boxes, has_mesh)
    for je in root.findall("joint"):
        lim = je.find("limit")
        jtype = je.get("type")
        axis_e = je.find("axis")
        axis = _floats(axis_e.get("xyz") if axis_e is not None else None, (1.0, 0.0, 0.0))
        lower = float(lim.get("lower", 0.0)) if lim is not None else 0.0
        upper = float(lim.get("upper", 0.0)) if lim is not None else 0.0
        effort = float(lim.get("effort", 0.0)) if lim is not None else INF
        velocity = float(lim.get("velocity", 0.0)) if lim is not None else INF
        joints[je.get("name")] = UrdfJoint(
            je.get("name"), jtype, je.find("parent").get("link"), je.find("child").get("link"),
            _origin(je.find("origin")), axis, lower, upper, effort, velocity)
    return root.get("name", "robot"), links, joints


# --------------------------------------------------------------------------- tables
@dataclass
class Frame:
    name: str
    joint: int      # parent joint index
    placement: SE3  # placement in the parent joint frame
    kind: str       # 'joint' | 'fixed_joint' | 'body' | 'op'
    base: str = ""  # 'op' frames: the frame it was attached to (`previousFrame`)


@dataclass
class Motor:
    name: str
    joint_name: str
    joint: int
    reduction: float = 1.0
    effort_limit: float = INF
    velocity_limit: float = INF
    velocity_effort_inv_slope: float = 0.0
    enable_effort_limit: bool = True
    enable_velocity_limit: bool = False
    enable_friction: bool = False
    friction_viscous_positive: float = 0.0
    friction_viscous_negative: float = 0.0
    friction_dry_positive: float = 0.0
    friction_dry_negative: float = 0.0
    friction_dry_slope: float = 0.0
    armature: float = 0.0  # joint side (option * reduction^2)
    backlash: float = 0.0  # transmission backlash (0 unless enableBacklash), abstract_motor.cc:347-355


@dataclass
class RobotTable:
    """Flat description of one robot, Pinocchio joint/q/v indexing (what the C ABI consumes)."""
    name: str
    has_freeflyer: bool
    joint_names: List[str]
    joint_type: np.ndarray
    parent: np.ndarray
    idx_q: np.ndarray
    idx_v: np.ndarray
    placement: np.ndarray      # [njoints, 12]
    axis: np.ndarray           # [njoints, 3]
    inertia: np.ndarray        # [njoints, 10]
    rotor_inertia: np.ndarray  # [nv]
    q_lower: np.ndarray        # [nq]
    q_upper: np.ndarray
    effort_limit: np.ndarray   # [nv] URDF (theoretical model) effort limits
    velocity_limit: np.ndarray  # [nv] URDF velocity limits
    frames: Dict[str, Frame]
    motors: List[Motor] = field(default_factory=list)
    contact_frame_names: List[str] = field(default_factory=list)
    imu_names: List[str] = field(default_factory=list)
    imu_frames: List[str] = field(default_factory=list)
    force_names: List[str] = field(default_factory=list)
    force_frames: List[str] = field(default_factory=list)
    encoder_names: List[str] = field(default_factory=list)
    encoder_joints: List[int] = field(default_factory=list)
    encoder_reduction: List[float] = field(default_factory=list)
    effort_names: List[str] = field(default_factory=list)
    effort_motors: List[int] = field(default_factory=list)
    contact_sensor_names: List[str] = field(default_factory=list)
    contact_sensor_index: List[int] = field(default_factory=list)
    links: Dict[str, UrdfLink] = field(default_factory=dict, repr=False)
    urdf_path: str = ""
    # flexibility joints (`add_flexibility_joints`): [njoints, 6] stiffness | damping, rows of the other joints zero
    flexibility: Optional[np.ndarray] = None
    flexibility_joint_names: List[str] = field(default_factory=list)

    # ---- Pinocchio-model-like accessors (what BaseJiminyEnv touches, SURVEY.md 8b)
    @property
    def njoints(self) -> int:
        return len(self.joint_names)

    @property
    def nq(self) -> int:
        return int(self.idx_q[-1] + JOINT_NQ[int(self.joint_type[-1])]) if self.njoints > 1 else 0

    @property
    def nv(self) -> int:
        return int(self.idx_v[-1] + JOINT_NV[int(self.joint_type[-1])]) if self.njoints > 1 else 0

    @property
    def nmotors(self) -> int:
        return len(self.motors)

    @property
    def mass(self) -> float:
        return float(self.inertia[1:, 0].sum())

    def joint_index(self, name: str) -> int:
        return self.joint_names.index(name)

    # ---- `robot.is_flexibility_enabled` / `robot.flexibility_joint_indices` (python/jiminy_pywrap/src/robot.cc)
    @property
    def is_flexibility_enabled(self) -> bool:
        return bool(self.flexibility_joint_names)

    @property
    def flexibility_joint_indices(self) -> List[int]:
        return [self.joint_index(n) for n in self.flexibility_joint_names]

    def neutral(self) -> np.ndarray:
        """`pinocchio::neutral`: zeros, (1, 0) for unbounded revolute, unit quaternion for free-flyer."""
        q = np.zeros(self.nq)
        for j in range(1, self.njoints):
            t, iq = int(self.joint_type[j]), int(self.idx_q[j])
            if t == JB_JOINT_FREEFLYER:
                q[iq + 6] = 1.0
            elif t == JB_JOINT_SPHERICAL:
                q[iq + 3] = 1.0
            elif t in (JB_JOINT_RUBX, JB_JOINT_RUBY, JB_JOINT_RUBZ, JB_JOINT_RUBU):
                q[iq] = 1.0
        return q

    # ---- mutation helpers mirroring robot.add_frame / add_contact_points
    def add_frame(self, name: str, body_name: str, placement: SE3) -> None:
        """`Model::addFrame` (model.cc): new OP frame rigidly attached to an existing frame."""
        if name in self.frames:
            raise ValueError(f"A frame with name '{name}' already exists.")
        base = self.frames[body_name]
        self.frames[name] = Frame(name, base.joint, base.placement * placement, "op", body_name)

    def add_contact_points(self, names: Sequence[str]) -> None:
        for n in names:
            if n not in self.frames:
                raise ValueError(f"Frame '{n}' does not exist.")
            if n in self.contact_frame_names:
                raise ValueError(f"Contact frame '{n}' already registered.")
            self.contact_frame_names.append(n)

    def remove_contact_points(self, names: Sequence[str]) -> None:
        for n in names:
            self.contact_frame_names.remove(n)

    def sensor_layout(self) -> Dict[str, Tuple[int, int, int]]:
        """type -> (offset, n_fields, n_sensors) in the flattened sensor row (field-major per type)."""
        out, off = {}, 0
        for key, nf, ns in (("ImuSensor", 6, len(self.imu_names)), ("ForceSensor", 6, len(self.force_names)),
                            ("EncoderSensor", 2, len(self.encoder_names)), ("EffortSensor", 1, len(self.effort_names)),
                            ("ContactSensor", 3, len(self.contact_sensor_names))):
            out[key] = (off, nf, ns)
            off += nf * ns
        out["width"] = (off, 0, 0)
        return out


def _cartesian_axis(axis: np.ndarray) -> Optional[int]:
    for k in range(3):
        e = np.zeros(3)
        e[k] = 1.0
        if np.array_equal(axis, e):
            return k
    return None


def build_robot_table(urdf_path: str, has_freeflyer: bool, joint_order: str = "alphabetical") -> RobotTable:
    """Restates `pinocchio::urdf::buildModel(+JointModelFreeFlyer)` as Jiminy calls it
    (`core/src/utilities/pinocchio.cc:828-934`).

    `joint_order`: 'alphabetical' (urdfdom `std::map` iteration order, SURVEY.md App. C) or
    'file' (document order) -- kept switchable because the ordering policy comes from library
    knowledge, not from a file of the reference.
    """
    name, links, joints = parse_urdf(urdf_path)
    children = {c.child for c in joints.values()}
    roots = [l for l in links if l not in children]
    if len(roots) != 1:
        raise ValueError(f"URDF must have exactly one root link, found {roots}.")
    root = roots[0]

    jlist = list(joints.values())
    if joint_order == "alphabetical":
        jlist = sorted(jlist, key=lambda j: j.name)
    elif joint_order != "file":
        raise ValueError("joint_order must be 'alphabetical' or 'file'.")
    child_joints: Dict[str, List[UrdfJoint]] = {l: [] for l in links}
    for j in jlist:
        child_joints[j.parent].append(j)

    names = ["universe"]
    jtype = [JB_JOINT_UNIVERSE]
    parent = [0]
    placement = [SE3()]
    axis = [np.zeros(3)]
    inertia = [Inertia()]
    lower: List[List[float]] = [[]]
    upper: List[List[float]] = [[]]
    eff: List[float] = []
    vel: List[float] = []
    frames: Dict[str, Frame] = {"universe": Frame("universe", 0, SE3(), "joint")}

    def add_body(joint: int, link: UrdfLink, M: SE3) -> None:
        inertia[joint] = inertia[joint] + link.inertia.transformed(M)
        frames.setdefault(link.name, Frame(link.name, joint, M, "body"))

    if has_freeflyer:
        names.append("root_joint")
        jtype.append(JB_JOINT_FREEFLYER)
        parent.append(0)
        placement.append(SE3())
        axis.append(np.zeros(3))
        inertia.append(Inertia())
        lower.append([-INF] * 3 + [-1.0 - EPS] * 4)
        upper.append([INF] * 3 + [1.0 + EPS] * 4)
        eff.extend([INF] * 6)
        vel.extend([INF] * 6)
        frames["root_joint"] = Frame("root_joint", 1, SE3(), "joint")
        add_body(1, links[root], SE3())
        root_joint = 1
    else:
        add_body(0, links[root], SE3())
        root_joint = 0

    def visit(link_name: str, joint: int, M_link: SE3) -> None:
        for j in child_joints[link_name]:
            M_joint = M_link * j.origin  # joint frame expressed in the parent *joint* frame
            child = links[j.child]
            if j.type == "fixed":
                frames.setdefault(j.name, Frame(j.name, joint, M_joint, "fixed_joint"))
                add_body(joint, child, M_joint)
                visit(j.child, joint, M_joint)
                continue
            if j.type in ("revolute", "continuous", "prismatic"):
                k = _cartesian_axis(j.axis)
                ax = j.axis if k is not None else j.axis / np.linalg.norm(j.axis)
                if j.type == "revolute":
                    t = (JB_JOINT_RX, JB_JOINT_RY, JB_JOINT_RZ)[k] if k is not None else JB_JOINT_RU
                    lo, hi = [j.lower], [j.upper]
                elif j.type == "continuous":
                    t = (JB_JOINT_RUBX, JB_JOINT_RUBY, JB_JOINT_RUBZ)[k] if k is not None else JB_JOINT_RUBU
                    lo, hi = [-1.0 - EPS] * 2, [1.0 + EPS] * 2  # model.cc:1380-1396
                else:
                    t = (JB_JOINT_PX, JB_JOINT_PY, JB_JOINT_PZ)[k] if k is not None else JB_JOINT_PU
                    lo, hi = [j.lower], [j.upper]
            else:
                raise NotImplementedError(f"URDF joint type '{j.type}' (joint '{j.name}') is not supported.")
            idx = len(names)
            names.append(j.name)
            jtype.append(t)
            parent.append(joint)
            placement.append(M_joint)
            axis.append(np.asarray(ax, dtype=np.float64))
            inertia.append(Inertia())
            lower.append(lo)
            upper.append(hi)
            eff.append(j.effort)
            vel.append(j.velocity)
            frames.setdefault(j.name, Frame(j.name, idx, SE3(), "joint"))
            add_body(idx, child, SE3())
            visit(j.child, idx, SE3())

    visit(root, root_joint, SE3())

    idx_q, idx_v, nq, nv = [], [], 0, 0
    for t in jtype:
        idx_q.append(nq)
        idx_v.append(nv)
        nq += JOINT_NQ[t]
        nv += JOINT_NV[t]
    return RobotTable(
        name=name, has_freeflyer=has_freeflyer, joint_names=names,
        joint_type=np.array(jtype, dtype=np.int32), parent=np.array(parent, dtype=np.int32),
        idx_q=np.array(idx_q, dtype=np.int32), idx_v=np.array(idx_v, dtype=np.int32),
        placement=np.stack([p.flat() for p in placement]), axis=np.stack(axis),
        inertia=np.stack([y.flat() for y in inertia]), rotor_inertia=np.zeros(nv),
        q_lower=np.array([x for l in lower for x in l], dtype=np.float64),
        q_upper=np.array([x for u in upper for x in u], dtype=np.float64),
        effort_limit=np.array(eff, dtype=np.float64), velocity_limit=np.array(vel, dtype=np.float64),
        frames=frames, links=links, urdf_path=os.path.abspath(urdf_path))


# --------------------------------------------------------------------------- hardware description
def attach_motor(robot: RobotTable, name: str, joint_name: str, **options) -> Motor:
    """`Robot::attachMotor` + `SimpleMotor::initialize` + `set_options` (robot.cc:190-258,
    abstract_motor.cc:246-345, basic_motors.h:20-28).  Option names are the reference's."""
    if any(m.name == name for m in robot.motors):
        raise ValueError(f"Another motor with name '{name}' is already attached.")
    j = robot.joint_index(joint_name)
    t = int(robot.joint_type[j])
    if JOINT_NV[t] != 1:
        raise ValueError("A motor can only be associated with a 1-dof linear or rotary joint.")
    iv = int(robot.idx_v[j])
    red = float(options.get("mechanicalReduction", 1.0))
    m = Motor(name=name, joint_name=joint_name, joint=j, reduction=red)
    m.enable_effort_limit = bool(options.get("enableEffortLimit", True))
    m.enable_velocity_limit = bool(options.get("enableVelocityLimit", False))
    if m.enable_velocity_limit and not m.enable_effort_limit:
        raise ValueError("'enableVelocityLimit' cannot be enabled without 'enableEffortLimit'.")
    m.velocity_effort_inv_slope = float(options.get("velocityEffortInvSlope", 0.0))
    m.effort_limit = (robot.effort_limit[iv] / red if options.get("effortLimitFromUrdf", True)
                      else float(options.get("effortLimit", 0.0)))
    m.velocity_limit = (robot.velocity_limit[iv] * red if options.get("velocityLimitFromUrdf", True)
                        else float(options.get("velocityLimit", 0.0)))
    m.enable_friction = bool(options.get("enableFriction", False))
    m.friction_viscous_positive = float(options.get("frictionViscousPositive", 0.0))
    m.friction_viscous_negative = float(options.get("frictionViscousNegative", 0.0))
    m.friction_dry_positive = float(options.get("frictionDryPositive", 0.0))
    m.friction_dry_negative = float(options.get("frictionDryNegative", 0.0))
    m.friction_dry_slope = float(options.get("frictionDrySlope", 0.0))
    for key, val in (("frictionViscousPositive", m.friction_viscous_positive),
                     ("frictionDryPositive", m.friction_dry_positive)):
        if val > 0.0:
            raise ValueError(f"'{key}' must be negative.")
    if options.get("enableBacklash", False):
        m.backlash = float(options.get("backlash", 0.0))
    if options.get("enableArmature", False):
        m.armature = float(options.get("armature", 0.0)) * red ** 2
    robot.rotor_inertia[iv] += m.armature
    robot.motors.append(m)
    return m


def attach_sensor(robot: RobotTable, sensor_type: str, name: str, **kw) -> None:
    """`Robot::attachSensor` + `<Sensor>::initialize` (basic_sensors.cc)."""
    if sensor_type == "ImuSensor":
        robot.imu_names.append(name)
        robot.imu_frames.append(kw["frame_name"])
    elif sensor_type == "ForceSensor":
        robot.force_names.append(name)
        robot.force_frames.append(kw["frame_name"])
    elif sensor_type == "EncoderSensor":
        if "motor_name" in kw:
            mi = [m.name for m in robot.motors].index(kw["motor_name"])
            robot.encoder_joints.append(robot.motors[mi].joint)
            robot.encoder_reduction.append(robot.motors[mi].reduction)
        else:
            robot.encoder_joints.append(robot.joint_index(kw["joint_name"]))
            robot.encoder_reduction.append(1.0)
        robot.encoder_names.append(name)
    elif sensor_type == "EffortSensor":
        robot.effort_names.append(name)
        robot.effort_motors.append([m.name for m in robot.motors].index(kw["motor_name"]))
    elif sensor_type == "ContactSensor":
        robot.contact_sensor_names.append(name)
        robot.contact_sensor_index.append(robot.contact_frame_names.index(kw["frame_name"]))
    else:
        raise NotImplementedError(f"Sensor type '{sensor_type}' is not supported.")
    for f in ("frame_name",):
        if f in kw and kw[f] not in robot.frames:
            raise ValueError(f"Frame '{kw[f]}' does not exist.")


def load_hardware_description_file(robot: RobotTable, hardware_path: str,
                                   avoid_instable_collisions: bool = True) -> dict:
    """Restates `jiminy_py.robot.load_hardware_description_file` (robot.py:518-847) for the
    features the BASELINE robots use: contact frames, collision bodies replaced by the vertices of
    their primitive collision boxes (robot.py:600-650), SimpleMotor and the five sensor types."""
    with open(hardware_path, "rb") as fh:
        hw = tomllib.load(fh)
    extra = dict(hw.get("Global", {}))
    collision_body_names = list(extra.pop("collisionBodyNames", []))
    contact_frame_names = list(extra.pop("contactFrameNames", []))

    if avoid_instable_collisions:
        # Replace the collision boxes by contact points at their vertices (robot.py:606-650)
        for body_name in list(collision_body_names):
            link = robot.links[body_name]
            for box_index, box in enumerate(link.collision_boxes):
                grids = [e.flatten() for e in np.meshgrid(
                    *[0.5 * v * np.array([-1.0, 1.0]) for v in box.size])]
                for i, xyz in enumerate(np.stack(grids, axis=1)):
                    frame_name = "_".join((body_name, "CollisionBox", str(box_index), str(i)))
                    robot.add_frame(frame_name, body_name, box.origin * SE3(np.eye(3), xyz))
                    contact_frame_names.append(frame_name)
            if link.collision_boxes or link.has_collision_mesh:
                collision_body_names.remove(body_name)
    if collision_body_names:
        raise NotImplementedError(
            "Collision bodies (hpp-fcl geometry pairs) are outside the accelerated path; only contact "
            f"frames are supported (bodies: {collision_body_names}).")
    robot.add_contact_points(sorted(set(contact_frame_names)))

    for motor_type, descr in hw.get("Motor", {}).items():
        if motor_type != "SimpleMotor":
            raise NotImplementedError(f"Motor type '{motor_type}' is not supported.")
        for motor_name, opts in descr.items():
            opts = dict(opts)
            joint_name = opts.pop("joint_name")
            if joint_name not in robot.joint_names:
                continue
            opts["enableArmature"] = True  # robot.py:753
            attach_motor(robot, motor_name, joint_name, **opts)

    for sensor_type, descr in hw.get("Sensor", {}).items():
        for sensor_name, opts in descr.items():
            opts = dict(opts)
            init = {k: opts.pop(k) for k in ("joint_name", "motor_name", "frame_name", "body_name", "frame_pose")
                    if k in opts}
            fname = init.get("frame_name")
            if fname is not None and fname not in robot.frames:
                pose = np.asarray(init.pop("frame_pose"), dtype=np.float64)
                robot.add_frame(fname, init.pop("body_name"), SE3(rpy_to_matrix(pose[3:]), pose[:3]))
            init.pop("frame_pose", None)
            init.pop("body_name", None)
            attach_sensor(robot, sensor_type, sensor_name, **init)
    return extra


def generate_default_hardware(robot: RobotTable) -> None:
    """What `BaseJiminyRobot.initialize` does when no hardware file exists (robot.py:872-958 via
    `generate_default_hardware_description_file`): one SimpleMotor + encoder + effort sensor per
    actuated 1-dof joint, in model order."""
    for j in range(1, robot.njoints):
        if JOINT_NV[int(robot.joint_type[j])] == 1 and np.isfinite(robot.effort_limit[robot.idx_v[j]]):
            attach_motor(robot, robot.joint_names[j], robot.joint_names[j])
    for m in list(robot.motors):
        attach_sensor(robot, "EncoderSensor", m.name, motor_name=m.name)
        attach_sensor(robot, "EffortSensor", m.name, motor_name=m.name)


# --------------------------------------------------------------------------- engine options
def default_engine_options() -> dict:
    """`Engine::getDefaultEngineOptions` (engine.h:260-341) -- the groups the step path reads."""
    return {
        "constraints": {"solver": "PGS", "regularization": 1e-3, "successiveSolveFailedMax": 100},
        "contacts": {"model": "constraint", "stiffness": 1e6, "damping": 2e3, "friction": 1.0,
                     "torsion": 0.0, "transitionEps": 1e-3, "transitionVelocity": 1e-2,
                     "stabilizationFreq": 20.0},
        "world": {"gravity": [0.0, 0.0, -9.81, 0.0, 0.0, 0.0]},
        "stepper": {"verbose": False, "randomSeedSeq": [0], "odeSolver": "runge_kutta_dopri",
                    "tolAbs": 1e-5, "tolRel": 1e-4, "dtMax": 0.02, "dtRestoreThresholdRel": 0.2,
                    "successiveIterFailedMax": 1000, "iterMax": 0, "timeout": 0.0,
                    "sensorsUpdatePeriod": 0.0, "controllerUpdatePeriod": 0.0,
                    "logInternalStepperSteps": False},
        "telemetry": {"enableConfiguration": True, "enableVelocity": True, "enableAcceleration": True},
    }


def load_options_file(options: dict, path: str) -> dict:
    """`Simulator.import_options` (simulator.py:1026-1064): merge `[engine.*]` TOML groups."""
    with open(path, "rb") as fh:
        data = tomllib.load(fh)
    for group, values in data.get("engine", {}).items():
        options.setdefault(group, {}).update(values)
    return options


SIMULATION_MIN_TIMESTEP = 1e-6
SIMULATION_MAX_TIMESTEP = 0.02
STEPPER_MIN_TIMESTEP = 1e-10


def is_gcd_included(*values: float) -> Tuple[bool, float]:
    """`isGcdIncluded` (helpers.hxx:97-178): is the smallest strictly positive period a divisor of
    all the others?  Returns (ok, min positive value or INF)."""
    pos = [v for v in values if v > EPS]
    if not pos:
        return True, INF
    vmin = min(pos)
    ok = all(abs(round(v / vmin) * vmin - v) < EPS * max(1.0, v / vmin) * 4 or
             math.fmod(v, vmin) < EPS or vmin - math.fmod(v, vmin) < EPS for v in pos)
    return ok, vmin


def validate_options(opt: dict) -> None:
    """The checks of `Engine::setOptions` (engine.cc:2654-2795) that concern this path."""
    st, ct = opt["stepper"], opt["contacts"]
    if st["dtMax"] < SIMULATION_MIN_TIMESTEP - EPS or st["dtMax"] > SIMULATION_MAX_TIMESTEP + EPS:
        raise ValueError("'dtMax' option is out of range.")
    if st["successiveIterFailedMax"] < 1:
        raise ValueError("'successiveIterFailedMax' must be strictly positive.")
    if st["odeSolver"] not in ("runge_kutta_dopri", "runge_kutta_4", "euler_explicit"):
        raise ValueError(f"Requested ODE solver '{st['odeSolver']}' not available.")
    for key in ("sensorsUpdatePeriod", "controllerUpdatePeriod"):
        p = st[key]
        if (EPS < p < SIMULATION_MIN_TIMESTEP) or p > SIMULATION_MAX_TIMESTEP:
            raise ValueError("Cannot simulate a discrete system with update period smaller than "
                             f"{SIMULATION_MIN_TIMESTEP}s or larger than {SIMULATION_MAX_TIMESTEP}s.")
    ok, _ = is_gcd_included(st["sensorsUpdatePeriod"], st["controllerUpdatePeriod"])
    if not ok:
        raise ValueError("In discrete mode, the controller and sensor update periods must be multiple of each other.")
    if ct["model"] not in ("spring_damper", "constraint"):
        raise ValueError(f"Requested contact model '{ct['model']}' not available.")
    if ct["transitionEps"] < 0.0:
        raise ValueError("Contact option 'transitionEps' must be positive.")
    if ct["transitionVelocity"] < EPS:
        raise ValueError("Contact option 'transitionVelocity' must be strictly positive.")
    if len(opt["world"]["gravity"]) != 6:
        raise ValueError("The size of the gravity force vector must be 6.")


# --------------------------------------------------------------------------- (de)serialisation
def robot_table_to_dict(robot: RobotTable) -> dict:
    """Compiled-table form of a robot (what ships in `jiminy_b200/robots/*.json`): everything the
    engine needs, nothing URDF-specific (no geometry)."""
    d = {
        "name": robot.name, "has_freeflyer": robot.has_freeflyer, "joint_names": robot.joint_names,
        "joint_type": robot.joint_type.tolist(), "parent": robot.parent.tolist(),
        "idx_q": robot.idx_q.tolist(), "idx_v": robot.idx_v.tolist(),
        "placement": robot.placement.tolist(), "axis": robot.axis.tolist(),
        "inertia": robot.inertia.tolist(), "rotor_inertia": robot.rotor_inertia.tolist(),
        "q_lower": robot.q_lower.tolist(), "q_upper": robot.q_upper.tolist(),
        "effort_limit": robot.effort_limit.tolist(), "velocity_limit": robot.velocity_limit.tolist(),
        "frames": {n: {"joint": f.joint, "placement": f.placement.flat().tolist(), "kind": f.kind, "base": f.base}
                   for n, f in robot.frames.items()},
        "flexibility": None if robot.flexibility is None else np.asarray(robot.flexibility).tolist(),
        "flexibility_joint_names": list(robot.flexibility_joint_names),
        "motors": [vars(m) for m in robot.motors],
        "contact_frame_names": robot.contact_frame_names,
        "imu_names": robot.imu_names, "imu_frames": robot.imu_frames,
        "force_names": robot.force_names, "force_frames": robot.force_frames,
        "encoder_names": robot.encoder_names, "encoder_joints": robot.encoder_joints,
        "encoder_reduction": robot.encoder_reduction,
        "effort_names": robot.effort_names, "effort_motors": robot.effort_motors,
        "contact_sensor_names": robot.contact_sensor_names,
        "contact_sensor_index": robot.contact_sensor_index,
    }

    def clean(x):
        if isinstance(x, dict):
            return {k: clean(v) for k, v in x.items()}
        if isinstance(x, (list, tuple)):
            return [clean(v) for v in x]
        if isinstance(x, (np.floating, float)):
            x = float(x)
            return x if math.isfinite(x) else ("inf" if x > 0 else "-inf")
        if isinstance(x, np.integer):
            return int(x)
        if isinstance(x, np.bool_):
            return bool(x)
        return x
    return clean(d)


def robot_table_from_dict(d: dict) -> RobotTable:
    def unclean(x):
        if isinstance(x, dict):
            return {k: unclean(v) for k, v in x.items()}
        if isinstance(x, list):
            return [unclean(v) for v in x]
        if x == "inf":
            return INF
        if x == "-inf":
            return -INF
        return x
    d = unclean(d)
    frames = {}
    for n, f in d["frames"].items():
        p = np.array(f["placement"], dtype=np.float64)
        frames[n] = Frame(n, int(f["joint"]), SE3(p[:9].reshape(3, 3).copy(), p[9:].copy()), f["kind"], f.get("base", ""))
    r = RobotTable(
        name=d["name"], has_freeflyer=bool(d["has_freeflyer"]), joint_names=list(d["joint_names"]),
        joint_type=np.array(d["joint_type"], dtype=np.int32), parent=np.array(d["parent"], dtype=np.int32),
        idx_q=np.array(d["idx_q"], dtype=np.int32), idx_v=np.array(d["idx_v"], dtype=np.int32),
        placement=np.array(d["placement"], dtype=np.float64), axis=np.array(d["axis"], dtype=np.float64),
        inertia=np.array(d["inertia"], dtype=np.float64),
        rotor_inertia=np.array(d["rotor_inertia"], dtype=np.float64),
        q_lower=np.array(d["q_lower"], dtype=np.float64), q_upper=np.array(d["q_upper"], dtype=np.float64),
        effort_limit=np.array(d["effort_limit"], dtype=np.float64),
        velocity_limit=np.array(d["velocity_limit"], dtype=np.float64), frames=frames)
    r.motors = [Motor(**m) for m in d["motors"]]
    for key in ("contact_frame_names", "imu_names", "imu_frames", "force_names", "force_frames",
                "encoder_names", "encoder_joints", "encoder_reduction", "effort_names", "effort_motors",
                "contact_sensor_names", "contact_sensor_index"):
        setattr(r, key, list(d[key]))
    if d.get("flexibility") is not None:
        r.flexibility = np.array(d["flexibility"], dtype=np.float64)
    r.flexibility_joint_names = list(d.get("flexibility_joint_names", []))
    return r


# --------------------------------------------------------------------------- model randomisation
# --------------------------------------------------------------------------- flexibility joints
FLEXIBLE_JOINT_SUFFIX = "Flexibility"   # core/include/jiminy/core/robot/model.h:19


def _inertia_from_flat(y: np.ndarray) -> Inertia:
    I = np.array([[y[4], y[5], y[7]], [y[5], y[6], y[8]], [y[7], y[8], y[9]]])
    return Inertia(float(y[0]), np.array(y[1:4], dtype=np.float64), I)


def _se3_from_flat(x: np.ndarray) -> SE3:
    return SE3(np.array(x[:9], dtype=np.float64).reshape(3, 3), np.array(x[9:12], dtype=np.float64))


def _insert_joint(robot: RobotTable, k: int, name: str, jtype: int, parent: int, placement: SE3, inertia: Inertia,
                  axis: Optional[np.ndarray] = None, lower: Optional[Sequence[float]] = None,
                  upper: Optional[Sequence[float]] = None) -> None:
    """Insert a joint at joint index `k` (every joint >= k moves up by one: the succession of `swapJointIndices` at the
    end of the reference's insertion routines, utilities/pinocchio.cc:404-458), in place."""
    shift = lambda j: j + 1 if j >= k else j   # noqa: E731
    iq, iv = (int(robot.idx_q[k]), int(robot.idx_v[k])) if k < robot.njoints else (robot.nq, robot.nv)
    nq, nv = JOINT_NQ[jtype], JOINT_NV[jtype]
    robot.joint_names.insert(k, name)
    robot.joint_type = np.insert(robot.joint_type, k, jtype).astype(np.int32)
    par = [shift(int(p)) for p in robot.parent]
    par.insert(k, parent)
    robot.parent = np.array(par, dtype=np.int32)
    robot.placement = np.insert(robot.placement, k, placement.flat(), axis=0)
    robot.axis = np.insert(robot.axis, k, np.zeros(3) if axis is None else np.asarray(axis, dtype=np.float64), axis=0)
    robot.inertia = np.insert(robot.inertia, k, inertia.flat(), axis=0)
    robot.rotor_inertia = np.insert(robot.rotor_inertia, iv, np.zeros(nv))
    robot.q_lower = np.insert(robot.q_lower, iq, np.full(nq, -1.0 - EPS) if lower is None else np.asarray(lower, dtype=np.float64))
    robot.q_upper = np.insert(robot.q_upper, iq, np.full(nq, 1.0 + EPS) if upper is None else np.asarray(upper, dtype=np.float64))
    robot.effort_limit = np.insert(robot.effort_limit, iv, np.full(nv, INF))
    robot.velocity_limit = np.insert(robot.velocity_limit, iv, np.full(nv, INF))
    if robot.flexibility is not None:
        robot.flexibility = np.insert(robot.flexibility, k, np.zeros(6), axis=0)
    idx_q, idx_v, nq_, nv_ = [], [], 0, 0
    for t in robot.joint_type:
        idx_q.append(nq_)
        idx_v.append(nv_)
        nq_ += JOINT_NQ[int(t)]
        nv_ += JOINT_NV[int(t)]
    robot.idx_q, robot.idx_v = np.array(idx_q, dtype=np.int32), np.array(idx_v, dtype=np.int32)
    for f in robot.frames.values():
        f.joint = shift(f.joint)
    for m in robot.motors:
        m.joint = shift(m.joint)
    robot.encoder_joints = [shift(j) for j in robot.encoder_joints]


def _insert_spherical_joint(robot: RobotTable, k: int, name: str, parent: int, placement: SE3, inertia: Inertia) -> None:
    _insert_joint(robot, k, name, JB_JOINT_SPHERICAL, parent, placement, inertia)   # quaternion limits: model.cc:1379-1398


BACKLASH_JOINT_SUFFIX = "Backlash"      # core/include/jiminy/core/robot/model.h:20


def add_backlash_joints(robot: RobotTable) -> RobotTable:
    """`Robot::initializeExtendedModel` (core/src/robot/robot.cc:582-629): for every motor with a transmission backlash
    (`enableBacklash`, `backlash` motor options) a joint `<joint>Backlash` of the same model is inserted right after the
    motorised joint (`addBacklashJointAfterMechanicalJoint`, utilities/pinocchio.cc:505-576): it takes over the body,
    the children and the frames of the joint, which keeps the motor and its rotor inertia, and its position is bounded by
    +- backlash / 2 -- a bound the engine enforces like any other (JointConstraint of the `boundJoints` registry).
    Returns a new table; the argument is left alone."""
    import copy
    out = copy.deepcopy(robot)
    for mi in range(len(out.motors)):
        m = out.motors[mi]
        if m.backlash < EPS:
            continue
        j = m.joint
        t = int(out.joint_type[j])
        if JOINT_NV[t] != 1:
            raise ValueError("Backlash can only be associated with a 1-dof linear or rotary joint.")
        name = out.joint_names[j] + BACKLASH_JOINT_SUFFIX
        if name in out.joint_names:
            raise ValueError(f"A joint with name '{name}' already exists.")
        k = j + 1
        body = _inertia_from_flat(out.inertia[j])
        lo, hi = ([-m.backlash / 2.0], [m.backlash / 2.0]) if JOINT_NQ[t] == 1 else (None, None)
        _insert_joint(out, k, name, t, j, SE3(), body, axis=out.axis[j].copy(), lower=lo, upper=hi)
        out.inertia[j] = Inertia().flat()
        for c in range(k + 1, out.njoints):
            if int(out.parent[c]) == j:
                out.parent[c] = k
        for f in out.frames.values():
            if f.joint == j and f.kind != "joint":
                f.joint = k
        out.frames[name] = Frame(name, k, SE3(), "joint")
    return out


def add_flexibility_joints(robot: RobotTable, flexibility_config: Sequence[dict]) -> RobotTable:
    """`Model::addFlexibilityJointsToExtendedModel` (core/src/robot/model.cc:1087-1165): one spherical joint per entry
    of `modelOptions["dynamics"]["flexibilityConfig"]` (`frameName`, `stiffness`, `damping`, `inertia`, 3 numbers each).

    * frame of a mechanical joint: `addFlexibilityJointBeforeMechanicalJoint` (utilities/pinocchio.cc:460-503) -- a
      weightless spherical joint named `<joint>Flexibility` at the joint's placement, the joint itself re-attached to it
      at the origin;
    * fixed frame: `addFlexibilityJointAtFixedFrame` (utilities/pinocchio.cc:578-727) -- the composite body is split at
      the frame: everything rigidly attached downstream of it (and the joints hanging from that) moves onto a spherical
      joint named like the frame.
    `inertia` is the armature-like rotor inertia of the three flexibility dofs (model.cc:1136-1144).  Returns a new
    table (the extended model); the argument (the theoretical model) is left alone.  Engine side:
    `Engine::computeInternalDynamics` (engine.cc:3367-3391)."""
    import copy
    out = copy.deepcopy(robot)
    if out.flexibility is None:
        out.flexibility = np.zeros((out.njoints, 6))
    for cfg in flexibility_config:
        if cfg["frameName"] not in robot.frames and cfg["frameName"] not in robot.joint_names:
            raise ValueError(f"Frame '{cfg['frameName']}' does not exists. Impossible to insert flexibility joint on it.")
    flex_names: List[str] = []
    for cfg in flexibility_config:
        frame_name = cfg["frameName"]
        # a joint and a link may share a name (ANYmal's URDF): the joint frame is the one meant
        is_joint = frame_name in out.joint_names[1:]
        fr = out.frames.get(frame_name)
        if is_joint:
            k = out.joint_index(frame_name)
            if int(out.joint_type[k]) in (JB_JOINT_FREEFLYER, JB_JOINT_SPHERICAL):
                raise ValueError("Flexible joint can only be inserted at fixed or joint frames.")
            flex_name = frame_name + FLEXIBLE_JOINT_SUFFIX
            parent, M = int(out.parent[k]), _se3_from_flat(out.placement[k])
            _insert_spherical_joint(out, k, flex_name, parent, M, Inertia())
            out.parent[k + 1] = k
            out.placement[k + 1] = SE3().flat()
            out.frames[flex_name] = Frame(flex_name, k, SE3(), "joint")
        elif fr is not None and fr.kind == "fixed_joint":
            flex_name = frame_name
            if not out.urdf_path or not os.path.exists(out.urdf_path) or not out.links:
                raise NotImplementedError("A flexibility at a fixed frame splits a composite body: it needs the URDF the table "
                                          "was built from (`build_robot_table`), which a compiled table does not keep.")
            _, _, ujoints = parse_urdf(out.urdf_path)
            if frame_name not in ujoints or ujoints[frame_name].type != "fixed":
                raise ValueError("Frame must be associated with fixed joint.")
            P, M_F = fr.joint, fr.placement
            # links rigidly attached downstream of the frame, and the moving joints hanging from them
            child_links, child_joints, stack = [], [], [ujoints[frame_name].child]
            while stack:
                link = stack.pop()
                child_links.append(link)
                for uj in ujoints.values():
                    if uj.parent != link:
                        continue
                    if uj.name in out.joint_names:      # a moving joint, or a fixed frame that already became a flexibility joint
                        child_joints.append(out.joint_index(uj.name))
                    elif uj.type == "fixed":
                        stack.append(uj.child)
            child_inertia = Inertia()
            for link in child_links:
                child_inertia = child_inertia + out.links[link].inertia.transformed(out.frames[link].placement)
            YP = _inertia_from_flat(out.inertia[P])
            if YP.mass - child_inertia.mass < 0.0:
                raise ValueError("Child body mass too large to be subtracted to joint mass.")
            out.inertia[P] = (YP + Inertia(-child_inertia.mass, child_inertia.lever, -child_inertia.I)).flat()
            k = min(child_joints) if child_joints else out.njoints
            M_inv = M_F.inverse()
            _insert_spherical_joint(out, k, flex_name, P, M_F, child_inertia.transformed(M_inv))
            for c in child_joints:
                out.parent[c + 1] = k
                out.placement[c + 1] = (M_inv * _se3_from_flat(out.placement[c + 1])).flat()
            moved = set(child_links) | {uj.name for uj in ujoints.values()
                                        if uj.type == "fixed" and uj.parent in child_links and uj.name not in out.joint_names}
            for f in out.frames.values():
                if f.joint == P and f.name != frame_name and (f.name in moved or (f.kind == "op" and _op_base(out, f, moved))) \
                        and f.kind != "joint":
                    f.joint, f.placement = k, M_inv * f.placement
            out.frames[frame_name] = Frame(frame_name, k, SE3(), "joint")
        else:
            raise ValueError("Flexible joint can only be inserted at fixed or joint frames.")
        flex_names.append(flex_name)
    for cfg, name in zip(flexibility_config, flex_names):
        j = out.joint_index(name)
        iv = int(out.idx_v[j])
        out.rotor_inertia[iv:iv + 3] = np.asarray(cfg["inertia"], dtype=np.float64)
        out.flexibility[j, :3] = np.asarray(cfg["stiffness"], dtype=np.float64)
        out.flexibility[j, 3:] = np.asarray(cfg["damping"], dtype=np.float64)
    for name in flex_names:   # model.cc:1146-1164
        j = out.joint_index(name)
        iv = int(out.idx_v[j])
        diag = out.rotor_inertia[iv:iv + 3] + out.inertia[j, [4, 6, 9]]
        if (diag < 1e-5).any():
            raise ValueError(f"The subtree diagonal inertia for flexibility joint {j} must be larger than 1e-5 "
                             f"for numerical stability: {diag}")
    out.flexibility_joint_names = list(out.flexibility_joint_names) + flex_names
    return out


def extended_state_from_theoretical(flex: RobotTable, rigid: RobotTable, q: np.ndarray, v: Optional[np.ndarray] = None):
    """`Model::getExtendedPositionFromTheoretical` / `getExtendedVelocityFromTheoretical` (model.cc): the state of the
    rigid (theoretical) model laid over the model with flexibility joints -- undeformed flexibilities (unit quaternion,
    no velocity), every other joint copied by name.  `q` [.., rigid.nq] -> [.., flex.nq] (and `v` likewise)."""
    q = np.asarray(q, dtype=np.float64)
    qe = np.broadcast_to(flex.neutral(), q.shape[:-1] + (flex.nq,)).copy()
    ve = None if v is None else np.zeros(np.asarray(v).shape[:-1] + (flex.nv,))
    for j in range(1, rigid.njoints):
        k = flex.joint_index(rigid.joint_names[j])
        t = int(rigid.joint_type[j])
        qe[..., flex.idx_q[k]:flex.idx_q[k] + JOINT_NQ[t]] = q[..., rigid.idx_q[j]:rigid.idx_q[j] + JOINT_NQ[t]]
        if ve is not None:
            ve[..., flex.idx_v[k]:flex.idx_v[k] + JOINT_NV[t]] = np.asarray(v)[..., rigid.idx_v[j]:rigid.idx_v[j] + JOINT_NV[t]]
    return qe if v is None else (qe, ve)


def default_model_options() -> dict:
    """`Model::getDefaultModelOptions` (core/include/jiminy/core/robot/model.h:136-178)."""
    return {"dynamics": {"inertiaBodiesBiasStd": 0.0, "massBodiesBiasStd": 0.0, "centerOfMassPositionBodiesBiasStd": 0.0,
                         "relativePositionBodiesBiasStd": 0.0, "enableFlexibility": True, "flexibilityConfig": []},
            "joints": {"positionLimitFromUrdf": True, "positionLimitLower": np.zeros(0), "positionLimitUpper": np.zeros(0)},
            "collisions": {"contactPointsPerBodyMax": 5}}


class Robot:
    """The model-option surface of `jiminy.Robot` (`get_model_options` / `set_model_options`, the theoretical and the
    extended model) over `RobotTable`s: `theoretical` is what the URDF and the hardware description gave,
    `extended` what the engine simulates -- rebuilt at every `set_model_options` in the reference's order
    (`Model::initializeExtendedModel`, model.cc:1047-1085, then `Robot::initializeExtendedModel`, robot.cc:582-629):
    flexibility joints, biases of the body inertias and joint placements, position limits of the mechanical joints,
    backlash joints.  Pass `robot.extended` (or the `Robot` itself) to `Engine.add_robot` / `BatchedEngine`."""

    def __init__(self, theoretical: RobotTable, seed: int = 0):
        self.theoretical = theoretical
        self._options = default_model_options()
        self._seed = seed
        self.extended = self._build()

    # ---- options
    def get_model_options(self) -> dict:
        import copy
        return copy.deepcopy(self._options)

    def set_model_options(self, options: dict) -> None:
        import copy
        opts = copy.deepcopy(options)
        dyn, joints = opts["dynamics"], opts["joints"]
        if not joints["positionLimitFromUrdf"]:
            n_mech = sum(1 for j in range(1, self.theoretical.njoints) if int(self.theoretical.joint_type[j]) != JB_JOINT_FREEFLYER
                         for _ in range(JOINT_NQ[int(self.theoretical.joint_type[j])]))
            for key in ("positionLimitLower", "positionLimitUpper"):
                if len(np.atleast_1d(joints[key])) != n_mech:       # model.cc:1557-1570
                    raise ValueError(f"Wrong vector size for '{key}'.")
        names = [c["frameName"] for c in dyn["flexibilityConfig"]]
        if len(set(names)) != len(names):                            # model.cc:1596-1611
            raise ValueError("Each flexibility frame name must be unique.")
        for key in ("inertiaBodiesBiasStd", "massBodiesBiasStd", "centerOfMassPositionBodiesBiasStd", "relativePositionBodiesBiasStd"):
            if dyn[key] < 0.0:
                raise ValueError(f"'{key}' must be positive.")
        previous, self._options = self._options, opts
        try:
            self.extended = self._build()
        except Exception:
            self._options = previous
            raise

    def _build(self) -> RobotTable:
        import copy
        dyn, joints = self._options["dynamics"], self._options["joints"]
        out = copy.deepcopy(self.theoretical)
        if dyn["enableFlexibility"] and len(dyn["flexibilityConfig"]):
            out = add_flexibility_joints(out, dyn["flexibilityConfig"])
        if any(dyn[k] > EPS for k in ("inertiaBodiesBiasStd", "massBodiesBiasStd", "centerOfMassPositionBodiesBiasStd",
                                      "relativePositionBodiesBiasStd")):
            out = biased_robot(out, np.random.default_rng(self._seed), mass_std=dyn["massBodiesBiasStd"],
                               com_std=dyn["centerOfMassPositionBodiesBiasStd"], inertia_std=dyn["inertiaBodiesBiasStd"],
                               relative_position_std=dyn["relativePositionBodiesBiasStd"])
        if not joints["positionLimitFromUrdf"]:
            # model.cc:1426-1434: one entry per position coordinate of the mechanical joints, in the theoretical model's order
            lo, hi, k = np.atleast_1d(joints["positionLimitLower"]), np.atleast_1d(joints["positionLimitUpper"]), 0
            out.q_lower, out.q_upper = out.q_lower.copy(), out.q_upper.copy()
            for j in range(1, self.theoretical.njoints):
                t = int(self.theoretical.joint_type[j])
                if t == JB_JOINT_FREEFLYER:
                    continue
                iq = int(out.idx_q[out.joint_index(self.theoretical.joint_names[j])])
                for c in range(JOINT_NQ[t]):
                    out.q_lower[iq + c], out.q_upper[iq + c] = lo[k], hi[k]
                    k += 1
        return add_backlash_joints(out)

    # ---- what the envs and the tests of the reference read
    @property
    def is_flexibility_enabled(self) -> bool:
        return self.extended.is_flexibility_enabled

    @property
    def flexibility_joint_names(self) -> List[str]:
        return list(self.extended.flexibility_joint_names)

    @property
    def flexibility_joint_indices(self) -> List[int]:
        return self.extended.flexibility_joint_indices

    @property
    def backlash_joint_names(self) -> List[str]:
        return [n for n in self.extended.joint_names if n.endswith(BACKLASH_JOINT_SUFFIX)]

    def get_extended_position_from_theoretical(self, q: np.ndarray) -> np.ndarray:
        return extended_state_from_theoretical(self.extended, self.theoretical, q)

    def get_extended_velocity_from_theoretical(self, v: np.ndarray) -> np.ndarray:
        q = np.broadcast_to(self.theoretical.neutral(), np.asarray(v).shape[:-1] + (self.theoretical.nq,))
        return extended_state_from_theoretical(self.extended, self.theoretical, q, v)[1]

    def get_theoretical_position_from_extended(self, q: np.ndarray) -> np.ndarray:
        q = np.asarray(q, dtype=np.float64)
        out = np.zeros(q.shape[:-1] + (self.theoretical.nq,))
        for j in range(1, self.theoretical.njoints):
            k = self.extended.joint_index(self.theoretical.joint_names[j])
            n = JOINT_NQ[int(self.theoretical.joint_type[j])]
            out[..., self.theoretical.idx_q[j]:self.theoretical.idx_q[j] + n] = q[..., self.extended.idx_q[k]:self.extended.idx_q[k] + n]
        return out


def _op_base(robot: RobotTable, frame: Frame, moved: set) -> bool:
    """An operational frame added with `add_frame` follows the frame it was attached to."""
    seen = set()
    while frame.kind == "op" and frame.base and frame.base not in seen:
        seen.add(frame.base)
        if frame.base in moved:
            return True
        frame = robot.frames[frame.base]
    return False


def _exp3(w: np.ndarray) -> np.ndarray:
    """Rotation matrix of a rotation vector (pinocchio::exp3)."""
    th = float(np.linalg.norm(w))
    K = np.array([[0.0, -w[2], w[1]], [w[2], 0.0, -w[0]], [-w[1], w[0], 0.0]])
    if th < 1e-12:
        return np.eye(3) + K
    return np.eye(3) + math.sin(th) / th * K + (1.0 - math.cos(th)) / (th * th) * (K @ K)


BIAS_EPS = 2.220446049250313e-16


def bias_normals(mass_std: float = 0.0, com_std: float = 0.0, inertia_std: float = 0.0,
                 relative_position_std: float = 0.0) -> int:
    """Standard normals one mechanical joint of `bias_bodies` consumes: centre of mass 3, mass 1, inertia axes 3 and
    moments 3, translation 3, for the standard deviations above machine epsilon."""
    return (3 * (com_std > BIAS_EPS) + (mass_std > BIAS_EPS) + 6 * (inertia_std > BIAS_EPS) +
            3 * (relative_position_std > BIAS_EPS))


def bias_bodies(inertia: np.ndarray, translation: np.ndarray, z: np.ndarray, eig, *, mass_std: float = 0.0,
                com_std: float = 0.0, inertia_std: float = 0.0, relative_position_std: float = 0.0):
    """Mechanical joints of `Model::addBiasedToExtendedModel` (core/src/robot/model.cc:1166-1236), batched over leading
    axes: returns new arrays of the joints' inertias [..., 10] (mass, lever, inertia about the centre of mass xx xy yy xz
    yz zz) and joint-placement translations [..., 3].  `z` [..., bias_normals]: each joint's single-precision standard
    normals, in the reference's order; `eig`: (moments [..., 3], axes [..., 3, 3]) of `np.linalg.eigh` of each joint's
    rotational inertia (broadcast against the leading axes).
    - the lever is scaled component-wise by N(1, com_std);
    - the mass by N(1, mass_std), never below min(mass, 1 g);
    - the principal axes are turned by the rotation vector N(0, inertia_std) (pinocchio::exp3) and the principal moments
      scaled by N(1, inertia_std);
    - the translation is scaled component-wise by N(1, relative_position_std).
    Each normal is formed in single precision (mean + std z), like the reference's draws.  Every operation is the one a
    single joint would take (elementwise ops, `dot` for the norm of the rotation vector, `math.sin` / `math.cos`,
    stacked `matmul`), so that a batch gives the bits of its joints drawn one at a time."""
    lead = np.broadcast_shapes(np.shape(inertia)[:-1], np.shape(z)[:-1])
    inertia = np.array(np.broadcast_to(inertia, lead + (10,)), dtype=np.float64, copy=True)
    translation = np.array(np.broadcast_to(translation, lead + (3,)), dtype=np.float64, copy=True)
    k = 0

    def normal(n, mean, std):
        nonlocal k
        x = (np.float32(mean) + np.float32(std) * z[..., k:k + n]).astype(np.float64)
        k += n
        return x
    if com_std > BIAS_EPS:
        inertia[..., 1:4] *= normal(3, 1.0, com_std)
    if mass_std > BIAS_EPS:
        m = inertia[..., 0]
        inertia[..., 0] = np.maximum(m * normal(1, 1.0, mass_std)[..., 0], np.minimum(m, 1.0e-3))
    if inertia_std > BIAS_EPS:
        moments, axes = eig
        w = normal(3, 0.0, inertia_std)
        flat = w.reshape(-1, 3)
        th = np.sqrt(np.array([r.dot(r) for r in flat])).reshape(lead)     # np.linalg.norm of each rotation vector
        sin = np.array([math.sin(t) for t in th.ravel()]).reshape(lead)
        cos = np.array([math.cos(t) for t in th.ravel()]).reshape(lead)
        zero = np.zeros(lead)
        K = np.stack([zero, -w[..., 2], w[..., 1], w[..., 2], zero, -w[..., 0], -w[..., 1], w[..., 0], zero], -1).reshape(lead + (3, 3))
        small = (th < 1e-12)[..., None, None]
        with np.errstate(divide="ignore", invalid="ignore"):
            big = np.eye(3) + (sin / th)[..., None, None] * K + ((1.0 - cos) / (th * th))[..., None, None] * (K @ K)
        R = np.where(small, np.eye(3) + K, big)
        ax = np.broadcast_to(axes, lead + (3, 3)) @ R
        mo = moments * normal(3, 1.0, inertia_std)
        D = np.zeros(lead + (3, 3))
        for a in range(3):
            D[..., a, a] = mo[..., a]
        I = ax @ D @ np.swapaxes(ax, -1, -2)
        inertia[..., 4:10] = np.stack([I[..., 0, 0], I[..., 0, 1], I[..., 1, 1], I[..., 0, 2], I[..., 1, 2], I[..., 2, 2]], -1)
    if relative_position_std > BIAS_EPS:
        translation *= normal(3, 1.0, relative_position_std)
    return inertia, translation


def inertia_eig(inertia: np.ndarray):
    """`np.linalg.eigh` of each rotational inertia of inertia rows [J, 10], one joint at a time: (moments [J, 3],
    axes [J, 3, 3])."""
    out = []
    for row in np.asarray(inertia, dtype=np.float64).reshape(-1, 10):
        xx, xy, yy, xz, yz, zz = row[4:10]
        out.append(np.linalg.eigh(np.array([[xx, xy, xz], [xy, yy, yz], [xz, yz, zz]])))
    return np.array([m for m, _ in out]).reshape(-1, 3), np.array([a for _, a in out]).reshape(-1, 3, 3)


def bias_joints(robot: RobotTable) -> List[int]:
    """The joints `addBiasedToExtendedModel` biases: the mechanical joints (`mechanicalJointNames_`), in the reference's
    order -- neither the root free-flyer nor the flexibility joints inserted into the extended model."""
    return [j for j in range(1, robot.njoints) if int(robot.joint_type[j]) != JB_JOINT_FREEFLYER and
            robot.joint_names[j] not in robot.flexibility_joint_names]


def body_rows(robot: RobotTable) -> np.ndarray:
    """Per joint [njoints, 13]: mass, lever xyz, inertia about the centre of mass (xx xy yy xz yz zz), joint-placement
    translation xyz -- the layout of `BatchedEngine.set_model_env`.  Row 0 (the universe) is zero."""
    rows = np.concatenate([np.asarray(robot.inertia, dtype=np.float64), np.asarray(robot.placement, dtype=np.float64)[:, 9:12]], 1)
    rows[0] = 0.0
    return rows


def with_body_rows(robot: RobotTable, rows: np.ndarray) -> RobotTable:
    """`robot` with the inertias and joint-placement translations of `rows` [njoints, 13] (`body_rows`' layout, row 0
    ignored); everything else is shared with `robot`."""
    import copy
    out = copy.copy(robot)
    out.inertia = np.array(robot.inertia, dtype=np.float64, copy=True)
    out.placement = np.array(robot.placement, dtype=np.float64, copy=True)
    out.inertia[1:] = rows[1:, :10]
    out.placement[1:, 9:12] = rows[1:, 10:13]
    return out


def biased_robot(robot: RobotTable, rng: np.random.Generator, *, mass_std: float = 0.0, com_std: float = 0.0,
                 inertia_std: float = 0.0, relative_position_std: float = 0.0) -> RobotTable:
    """One draw of `Model::addBiasedToExtendedModel` (core/src/robot/model.cc:1166-1236) with the model options
    `massBodiesBiasStd`, `centerOfMassPositionBodiesBiasStd`, `inertiaBodiesBiasStd`, `relativePositionBodiesBiasStd`:
    `bias_bodies` on every mechanical joint (`bias_joints`), in the reference's order.  Draws are single precision like
    the reference's; the stream is numpy's, not the engine's PCG32 (and Eigen's eigenvector signs are not reproduced):
    equal in distribution, not draw by draw.  Order of the reference (Model / Robot::initializeExtendedModel):
    flexibilities, then the biases, then the backlash joints -- call `add_backlash_joints` on the biased table, not
    before.  Returns a new table; everything but `inertia` and `placement` is shared with `robot`."""
    import copy
    out = copy.copy(robot)
    out.inertia = np.array(robot.inertia, dtype=np.float64, copy=True)
    out.placement = np.array(robot.placement, dtype=np.float64, copy=True)
    stds = dict(mass_std=mass_std, com_std=com_std, inertia_std=inertia_std, relative_position_std=relative_position_std)
    joints = bias_joints(robot)
    z = rng.standard_normal((len(joints), bias_normals(**stds)), dtype=np.float32)
    out.inertia[joints], out.placement[joints, 9:12] = bias_bodies(out.inertia[joints], out.placement[joints, 9:12], z,
                                                                    inertia_eig(out.inertia[joints]), **stds)
    return out
