"""
MJCF -> ModelPack compiler (host side, cold path).

Parses the reference's MJCF model files *as data* (xml.etree, no MuJoCo, no dm_control) and emits the
flat structure-of-arrays `ModelPack` consumed by the CUDA engine (csrc/locosim.cu) and by the CPU
oracle (oracle/locosim_ref.c).  It restates the subset of MuJoCo 2.3.7's model compiler that the
in-scope robots use (SURVEY.md §8a "model facts"):

  * <compiler> angle / autolimits / eulerseq / inertiafromgeom / balanceinertia / boundmass / boundinertia
  * <default> classes incl. nested classes and body `childclass`
  * <option> timestep / integrator / cone / impratio / iterations / tolerance / gravity
  * bodies, hinge+slide joints, inertial (diaginertia | fullinertia), primitive + mesh geoms, motors
  * derived constants MuJoCo computes at compile time (dof_invweight0, body_invweight0, stat.meaninertia,
    geom_rbound, collision pair filter)

XML surgery helpers mirror what the reference envs do through dm_control.mjcf
(/root/reference/loco_mujoco/environments/base.py:896-921).
"""
import copy
import os
import xml.etree.ElementTree as ET

import numpy as np

mjMINVAL = 1e-15

GEOM_PLANE, GEOM_HFIELD, GEOM_SPHERE, GEOM_CAPSULE, GEOM_ELLIPSOID, GEOM_CYLINDER, GEOM_BOX, GEOM_MESH = range(8)
GEOM_TYPES = dict(plane=GEOM_PLANE, hfield=GEOM_HFIELD, sphere=GEOM_SPHERE, capsule=GEOM_CAPSULE,
                  ellipsoid=GEOM_ELLIPSOID, cylinder=GEOM_CYLINDER, box=GEOM_BOX, mesh=GEOM_MESH)
JNT_SLIDE, JNT_HINGE = 2, 3          # MuJoCo's mjtJoint numbering (free=0, ball=1 unsupported here)
INT_EULER, INT_RK4 = 0, 1
CONE_PYRAMIDAL, CONE_ELLIPTIC = 0, 1

ACTUATOR_TAGS = ("general", "motor", "position", "velocity", "intvelocity", "damper", "cylinder", "muscle",
                 "adhesion")


# ----------------------------------------------------------------------------------------------------------
# small math helpers (quaternions are (w, x, y, z) like MuJoCo)
# ----------------------------------------------------------------------------------------------------------
def _floats(s):
    return np.array([float(x) for x in s.split()], dtype=np.float64)


def quat_mul(a, b):
    return np.array([a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3],
                     a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2],
                     a[0] * b[2] - a[1] * b[3] + a[2] * b[0] + a[3] * b[1],
                     a[0] * b[3] + a[1] * b[2] - a[2] * b[1] + a[3] * b[0]])


def quat_to_mat(q):
    w, x, y, z = q
    return np.array([[w * w + x * x - y * y - z * z, 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), w * w - x * x + y * y - z * z, 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), w * w - x * x - y * y + z * z]])


def mat_to_quat(R):
    """Rotation matrix -> unit quaternion (robust branch selection)."""
    t = np.trace(R)
    if t > 0:
        s = np.sqrt(t + 1.0) * 2
        q = np.array([0.25 * s, (R[2, 1] - R[1, 2]) / s, (R[0, 2] - R[2, 0]) / s, (R[1, 0] - R[0, 1]) / s])
    elif R[0, 0] > R[1, 1] and R[0, 0] > R[2, 2]:
        s = np.sqrt(1.0 + R[0, 0] - R[1, 1] - R[2, 2]) * 2
        q = np.array([(R[2, 1] - R[1, 2]) / s, 0.25 * s, (R[0, 1] + R[1, 0]) / s, (R[0, 2] + R[2, 0]) / s])
    elif R[1, 1] > R[2, 2]:
        s = np.sqrt(1.0 + R[1, 1] - R[0, 0] - R[2, 2]) * 2
        q = np.array([(R[0, 2] - R[2, 0]) / s, (R[0, 1] + R[1, 0]) / s, 0.25 * s, (R[1, 2] + R[2, 1]) / s])
    else:
        s = np.sqrt(1.0 + R[2, 2] - R[0, 0] - R[1, 1]) * 2
        q = np.array([(R[1, 0] - R[0, 1]) / s, (R[0, 2] + R[2, 0]) / s, (R[1, 2] + R[2, 1]) / s, 0.25 * s])
    return q / np.linalg.norm(q)


def axisangle_to_quat(axis, angle):
    n = np.linalg.norm(axis)
    if n < mjMINVAL:
        return np.array([1.0, 0, 0, 0])
    axis = axis / n
    return np.concatenate([[np.cos(angle / 2)], np.sin(angle / 2) * axis])


def z_to_quat(vec):
    """Quaternion rotating the z axis onto `vec` (MuJoCo's mjuu_z2quat, used for `fromto` and `zaxis`)."""
    vec = vec / np.linalg.norm(vec)
    z = np.array([0.0, 0, 1])
    axis = np.cross(z, vec)
    s = np.linalg.norm(axis)
    if s < 1e-10:
        axis = np.array([1.0, 0, 0])
    else:
        axis = axis / s
    ang = np.arctan2(s, vec[2])
    return np.concatenate([[np.cos(ang / 2)], np.sin(ang / 2) * axis])


# ----------------------------------------------------------------------------------------------------------
# XML surgery (what the reference does with dm_control.mjcf handles)
# ----------------------------------------------------------------------------------------------------------
class XmlHandle:
    """A mutable MJCF document. Mirrors the tiny part of dm_control.mjcf's API the reference envs use."""

    def __init__(self, path):
        self.path = os.path.abspath(path)
        self.dir = os.path.dirname(self.path)
        self.tree = ET.parse(path)
        self.root = self.tree.getroot()
        self._expand_includes(self.root, self.dir)

    def _expand_includes(self, elem, base):
        for i, ch in enumerate(list(elem)):
            if ch.tag == "include":
                sub = ET.parse(os.path.join(base, ch.get("file"))).getroot()
                idx = list(elem).index(ch)
                elem.remove(ch)
                for k, sc in enumerate(list(sub)):
                    elem.insert(idx + k, sc)
            else:
                self._expand_includes(ch, base)

    def copy(self):
        return copy.deepcopy(self)

    # -- lookup ------------------------------------------------------------------------------------------
    def _parent_map(self):
        return {c: p for p in self.root.iter() for c in p}

    def find(self, kind, name):
        """kind in {body, joint, geom, site, actuator, equality, mesh, default}"""
        if kind == "actuator":
            sec = self.root.find("actuator")
            if sec is not None:
                for e in sec:
                    if e.get("name") == name:
                        return e
            return None
        if kind == "equality":
            sec = self.root.find("equality")
            if sec is not None:
                for e in sec:
                    if e.get("name") == name:
                        return e
            return None
        if kind == "default":
            for e in self.root.iter("default"):
                if e.get("class") == name:
                    return e
            return None
        wb = self.root.find("worldbody")
        for e in wb.iter(kind):
            if e.get("name") == name:
                return e
        if kind == "mesh":
            for e in self.root.iter("mesh"):
                if e.get("name") == name:
                    return e
        return None

    def remove(self, elem):
        pm = self._parent_map()
        pm[elem].remove(elem)

    def delete(self, joints_to_remove=(), motors_to_remove=(), equ_constraints=()):
        """LocoEnv._delete_from_xml_handle (base.py:896-921)."""
        for j in joints_to_remove:
            self.remove(self.find("joint", j))
        for m in motors_to_remove:
            self.remove(self.find("actuator", m))
        for e in equ_constraints:
            self.remove(self.find("equality", e))
        return self

    def add(self, parent, tag, **attrs):
        e = ET.SubElement(parent, tag)
        for k, v in attrs.items():
            if k == "dclass":
                k = "class"
            e.set(k, v if isinstance(v, str) else " ".join(repr(float(x)) for x in np.atleast_1d(v)))
        return e


# ----------------------------------------------------------------------------------------------------------
# defaults
# ----------------------------------------------------------------------------------------------------------
class _Defaults:
    def __init__(self, root):
        self.classes = {"main": {}}
        top = [d for d in root.findall("default")]
        for d in top:
            self._parse(d, "main", is_top=True)

    def _parse(self, elem, parent_name, is_top=False):
        name = elem.get("class")
        if is_top and name is None:
            name = "main"
        if name == "main" or name is None:
            cur = self.classes["main"]
            name = "main"
        else:
            cur = copy.deepcopy(self.classes[parent_name])
            self.classes[name] = cur
        for ch in elem:
            if ch.tag == "default":
                continue
            tag = "actuator" if ch.tag in ACTUATOR_TAGS else ch.tag
            cur.setdefault(tag, {})
            cur[tag].update(ch.attrib)
        for ch in elem:
            if ch.tag == "default":
                self._parse(ch, name)

    def resolve(self, elem, childclass):
        tag = "actuator" if elem.tag in ACTUATOR_TAGS else elem.tag
        cls = elem.get("class") or childclass or "main"
        if cls not in self.classes:
            raise ValueError("unknown default class %r" % cls)
        out = dict(self.classes[cls].get(tag, {}))
        out.update({k: v for k, v in elem.attrib.items() if k != "class"})
        return out


# ----------------------------------------------------------------------------------------------------------
# mesh loading (binary/ascii STL, OBJ): vertices only; hull computed with scipy's Qhull
# ----------------------------------------------------------------------------------------------------------
def _load_mesh_vertices(path):
    ext = os.path.splitext(path)[1].lower()
    if ext == ".stl":
        with open(path, "rb") as f:
            data = f.read()
        ntri = int(np.frombuffer(data[80:84], dtype="<u4")[0]) if len(data) >= 84 else 0
        if len(data) == 84 + 50 * ntri:
            rec = np.frombuffer(data[84:], dtype=np.dtype([("n", "<f4", 3), ("v", "<f4", 9), ("a", "<u2")]))
            faces = rec["v"].reshape(-1, 3, 3).astype(np.float64)
        else:
            verts = []
            for line in data.decode("ascii", "ignore").splitlines():
                p = line.split()
                if len(p) == 4 and p[0] == "vertex":
                    verts.append([float(p[1]), float(p[2]), float(p[3])])
            faces = np.array(verts, dtype=np.float64).reshape(-1, 3, 3)
        return faces.reshape(-1, 3), np.arange(faces.shape[0] * 3).reshape(-1, 3)
    if ext == ".obj":
        v, f = [], []
        with open(path) as fh:
            for line in fh:
                p = line.split()
                if not p:
                    continue
                if p[0] == "v":
                    v.append([float(p[1]), float(p[2]), float(p[3])])
                elif p[0] == "f":
                    idx = [int(t.split("/")[0]) - 1 for t in p[1:]]
                    for k in range(1, len(idx) - 1):
                        f.append([idx[0], idx[k], idx[k + 1]])
        return np.array(v, dtype=np.float64), np.array(f, dtype=np.int64)
    raise ValueError("unsupported mesh format: " + path)


# ----------------------------------------------------------------------------------------------------------
# compiled model container
# ----------------------------------------------------------------------------------------------------------
class Model:
    """Flat compiled model ("ModelPack"). All reals float64, ints int32."""

    def names(self, kind):
        return getattr(self, kind + "_names")

    def joint_id(self, name):
        return self.jnt_names.index(name)

    def actuator_id(self, name):
        return self.actuator_names.index(name)

    def geom_id(self, name):
        return self.geom_names.index(name)

    def body_id(self, name):
        return self.body_names.index(name)

    def body_index(self, name):
        """Index of body `name` in the compiled model (the row of LocoEnv.xfrc_applied). ValueError for an unknown name and
        for a body that fuse_static merged into its parent (the message names the body it now belongs to)."""
        if name in self.body_names:
            return self.body_names.index(name)
        fused = getattr(self, "fused_bodies", {})
        if name in fused:
            raise ValueError("body %r has no joint and was fused into %r (fuse_static=True): apply the force to %r"
                             % (name, fused[name], fused[name]))
        raise ValueError("unknown body %r (bodies of the compiled model: %s)" % (name, ", ".join(self.body_names)))


def _orientation(attrs, comp):
    if "quat" in attrs:
        q = _floats(attrs["quat"])
        return q / np.linalg.norm(q)
    scale = 1.0 if comp["angle"] == "radian" else np.pi / 180.0
    if "axisangle" in attrs:
        a = _floats(attrs["axisangle"])
        return axisangle_to_quat(a[:3], a[3] * scale)
    if "euler" in attrs:
        e = _floats(attrs["euler"]) * scale
        q = np.array([1.0, 0, 0, 0])
        for ch, ang in zip(comp["eulerseq"], e):
            ax = dict(x=[1.0, 0, 0], y=[0, 1.0, 0], z=[0, 0, 1.0])[ch.lower()]
            qi = axisangle_to_quat(np.array(ax), ang)
            q = quat_mul(q, qi) if ch.islower() else quat_mul(qi, q)
        return q / np.linalg.norm(q)
    if "xyaxes" in attrs:
        a = _floats(attrs["xyaxes"])
        x = a[:3] / np.linalg.norm(a[:3])
        y = a[3:] - np.dot(a[3:], x) * x
        y /= np.linalg.norm(y)
        return mat_to_quat(np.stack([x, y, np.cross(x, y)], axis=1))
    if "zaxis" in attrs:
        return z_to_quat(_floats(attrs["zaxis"]))
    return np.array([1.0, 0, 0, 0])


def _eig_inertia(full):
    """fullinertia (ixx iyy izz ixy ixz iyz) -> (diag, iquat) with iquat rotating principal -> parent frame."""
    ixx, iyy, izz, ixy, ixz, iyz = full
    M = np.array([[ixx, ixy, ixz], [ixy, iyy, iyz], [ixz, iyz, izz]])
    w, V = np.linalg.eigh(M)
    order = np.argsort(-w)
    w, V = w[order], V[:, order]
    if np.linalg.det(V) < 0:
        V[:, 2] = -V[:, 2]
    return w, mat_to_quat(V)


def mesh_legacy_inertia(v, f):
    """
    Volume, centre of mass and inertia tensor (unit density, about the CoM, mesh frame) of a triangle mesh with
    MuJoCo 2.3.7's default `inertia="legacy"` rule: pyramids from the area-weighted face centroid to every face,
    each counted with the ABSOLUTE value of its volume.
    """
    tri = v[f]                                        # [nf, 3, 3]
    cen = tri.mean(axis=1)
    nrm = np.cross(tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0])
    area2 = np.linalg.norm(nrm, axis=1)
    ok = area2 > 1e-14
    tri, cen, nrm, area2 = tri[ok], cen[ok], nrm[ok], area2[ok]
    area = 0.5 * area2
    unit = nrm / area2[:, None]
    facecen = (cen * area[:, None]).sum(axis=0) / area.sum()
    vol = np.abs(np.einsum("ij,ij->i", unit, cen - facecen) * area / 3.0)
    volume = vol.sum()
    com = (vol[:, None] * (0.75 * cen + 0.25 * facecen)).sum(axis=0) / volume
    t = tri - com
    cen_c = t.mean(axis=1)
    vol2 = np.abs(np.einsum("ij,ij->i", unit, cen_c) * area / 3.0)
    P = np.zeros((3, 3))
    for k in range(len(t)):
        a, b, c = t[k]
        ssum = a + b + c
        P += vol2[k] / 20.0 * (np.outer(a, a) + np.outer(b, b) + np.outer(c, c) + np.outer(ssum, ssum))
    I = np.trace(P) * np.eye(3) - P
    return volume, com, I


def _geom_inertia(gtype, size, density, mass_attr, mesh=None):
    """mass and diagonal inertia (in geom frame) of a primitive geom."""
    if gtype == GEOM_SPHERE:
        vol = 4.0 / 3.0 * np.pi * size[0] ** 3
        unit = np.array([1, 1, 1]) * 2.0 / 5.0 * size[0] ** 2
    elif gtype == GEOM_CAPSULE:
        r, h = size[0], 2 * size[1]
        vc, vs = np.pi * r * r * h, 4.0 / 3.0 * np.pi * r ** 3
        vol = vc + vs
        mc, ms = vc / vol, vs / vol
        izz = mc * r * r / 2 + ms * 2 * r * r / 5
        ixx = mc * (h * h / 12 + r * r / 4) + ms * (2 * r * r / 5 + h * h / 4 + 3 * h * r / 8)
        unit = np.array([ixx, ixx, izz])
    elif gtype == GEOM_CYLINDER:
        r, h = size[0], 2 * size[1]
        vol = np.pi * r * r * h
        unit = np.array([(3 * r * r + h * h) / 12, (3 * r * r + h * h) / 12, r * r / 2])
    elif gtype == GEOM_BOX:
        vol = 8 * size[0] * size[1] * size[2]
        unit = np.array([size[1] ** 2 + size[2] ** 2, size[0] ** 2 + size[2] ** 2, size[0] ** 2 + size[1] ** 2]) / 3
    elif gtype == GEOM_ELLIPSOID:
        vol = 4.0 / 3.0 * np.pi * size[0] * size[1] * size[2]
        unit = np.array([size[1] ** 2 + size[2] ** 2, size[0] ** 2 + size[2] ** 2, size[0] ** 2 + size[1] ** 2]) / 5
    else:
        return 0.0, np.zeros(3)
    mass = mass_attr if mass_attr is not None else vol * density
    return mass, unit * mass


# ----------------------------------------------------------------------------------------------------------
# the compiler
# ----------------------------------------------------------------------------------------------------------
def compile_model(handle, timestep=None, collision_mesh_max_verts=64, fuse_static=True):
    """
    Compile an XmlHandle into a Model.

    timestep: override of <option timestep> (LocoEnv passes timestep=0.001, base.py:33; mushroom's MuJoCo
              ctor writes it into model.opt.timestep).
    """
    root = handle.root
    m = Model()

    # ---- compiler / option --------------------------------------------------------------------------------
    comp = dict(angle="degree", autolimits="false", eulerseq="xyz", inertiafromgeom="auto",
                balanceinertia="false", boundmass="0", boundinertia="0", meshdir="", settotalmass="-1",
                coordinate="local")
    for c in root.findall("compiler"):
        comp.update(c.attrib)
    assert comp["coordinate"] == "local"
    opt = dict(timestep="0.002", gravity="0 0 -9.81", integrator="Euler", cone="pyramidal", impratio="1",
               solver="Newton", iterations="100", tolerance="1e-8", noslip_iterations="0")
    for o in root.findall("option"):
        opt.update({k: v for k, v in o.attrib.items()})
    if opt["solver"].lower() != "newton":
        raise NotImplementedError("only the Newton solver is implemented (all in-scope models use it)")
    m.opt_timestep = float(opt["timestep"]) if timestep is None else float(timestep)
    m.opt_gravity = _floats(opt["gravity"])
    m.opt_integrator = dict(euler=INT_EULER, rk4=INT_RK4)[opt["integrator"].lower()]
    m.opt_cone = dict(pyramidal=CONE_PYRAMIDAL, elliptic=CONE_ELLIPTIC)[opt["cone"].lower()]
    m.opt_impratio = float(opt["impratio"])
    m.opt_iterations = int(opt["iterations"])
    m.opt_tolerance = float(opt["tolerance"])
    angle_scale = 1.0 if comp["angle"] == "radian" else np.pi / 180.0
    autolimits = comp["autolimits"] == "true"

    defaults = _Defaults(root)

    # ---- meshes ----------------------------------------------------------------------------------------
    meshes = {}
    for asset in root.findall("asset"):
        for me in asset.findall("mesh"):
            a = defaults.resolve(me, None)
            fname = a.get("file")
            name = a.get("name") or os.path.splitext(os.path.basename(fname))[0]
            meshes[name] = dict(file=os.path.join(handle.dir, comp["meshdir"], fname),
                                scale=_floats(a.get("scale", "1 1 1")), verts=None)

    # ---- traverse bodies ---------------------------------------------------------------------------------
    B = dict(name=[], parent=[], pos=[], quat=[], ipos=[], iquat=[], mass=[], inertia=[], jntadr=[], jntnum=[],
             has_inertial=[])
    J = dict(name=[], type=[], body=[], pos=[], axis=[], limited=[], range=[], stiffness=[], armature=[],
             damping=[], frictionloss=[], ref=[], springref=[], margin=[], solreflimit=[], solimplimit=[],
             solreffriction=[], solimpfriction=[])
    G = dict(name=[], type=[], body=[], size=[], pos=[], quat=[], friction=[], margin=[], gap=[], solref=[],
             solimp=[], solmix=[], condim=[], priority=[], contype=[], conaffinity=[], mesh=[], mass=[],
             density=[], group=[])
    S = dict(name=[], body=[], pos=[], quat=[])

    def solimp5(s):
        v = _floats(s)
        full = np.array([0.9, 0.95, 0.001, 0.5, 2.0])
        full[:len(v)] = v
        return full

    def visit(belem, parent_id, childclass):
        bid = len(B["name"])
        is_world = belem.tag == "worldbody"
        cc = belem.get("childclass") or childclass
        B["name"].append("world" if is_world else belem.get("name", "body%d" % bid))
        B["parent"].append(parent_id if not is_world else 0)
        B["pos"].append(np.zeros(3) if is_world else _floats(belem.get("pos", "0 0 0")))
        B["quat"].append(np.array([1.0, 0, 0, 0]) if is_world else _orientation(belem.attrib, comp))
        inert = belem.find("inertial")
        if inert is not None:
            ia = inert.attrib
            B["ipos"].append(_floats(ia.get("pos", "0 0 0")))
            B["mass"].append(float(ia["mass"]))
            if "fullinertia" in ia:
                d, q = _eig_inertia(_floats(ia["fullinertia"]))
                B["inertia"].append(d)
                B["iquat"].append(q)
            else:
                B["inertia"].append(_floats(ia["diaginertia"]))
                B["iquat"].append(_orientation(ia, comp))
            B["has_inertial"].append(True)
        else:
            B["ipos"].append(np.zeros(3))
            B["iquat"].append(np.array([1.0, 0, 0, 0]))
            B["mass"].append(0.0)
            B["inertia"].append(np.zeros(3))
            B["has_inertial"].append(False)
        B["jntadr"].append(len(J["name"]))
        nj = 0
        for je in belem.findall("joint"):
            a = defaults.resolve(je, cc)
            jt = a.get("type", "hinge")
            if jt not in ("hinge", "slide"):
                raise NotImplementedError("joint type %s (in-scope models use hinge/slide only)" % jt)
            J["name"].append(a.get("name", "joint%d" % len(J["name"])))
            J["type"].append(JNT_HINGE if jt == "hinge" else JNT_SLIDE)
            J["body"].append(bid)
            J["pos"].append(_floats(a.get("pos", "0 0 0")))
            ax = _floats(a.get("axis", "0 0 1"))
            J["axis"].append(ax / np.linalg.norm(ax))
            rng = _floats(a.get("range", "0 0"))
            if jt == "hinge":
                rng = rng * angle_scale
            lim = a.get("limited", "auto")
            if lim == "auto":
                limited = autolimits and (rng[0] != 0 or rng[1] != 0) and rng[0] < rng[1]
                if not autolimits and (rng[0] != 0 or rng[1] != 0):
                    # MuJoCo 2.3.7 errors here; the in-scope models never hit this
                    raise ValueError("joint %s: range without limited and autolimits=false" % J["name"][-1])
            else:
                limited = lim == "true"
            J["limited"].append(int(limited))
            J["range"].append(rng)
            sc = angle_scale if jt == "hinge" else 1.0
            J["stiffness"].append(float(a.get("stiffness", 0)))
            J["armature"].append(float(a.get("armature", 0)))
            J["damping"].append(float(a.get("damping", 0)))
            J["frictionloss"].append(float(a.get("frictionloss", 0)))
            J["ref"].append(float(a.get("ref", 0)) * sc)
            J["springref"].append(float(a.get("springref", 0)) * sc)
            J["margin"].append(float(a.get("margin", 0)))
            J["solreflimit"].append(_floats(a.get("solreflimit", "0.02 1")))
            J["solimplimit"].append(solimp5(a.get("solimplimit", "0.9 0.95 0.001 0.5 2")))
            J["solreffriction"].append(_floats(a.get("solreffriction", "0.02 1")))
            J["solimpfriction"].append(solimp5(a.get("solimpfriction", "0.9 0.95 0.001 0.5 2")))
            nj += 1
        if belem.find("freejoint") is not None:
            raise NotImplementedError("freejoint")
        B["jntnum"].append(nj)
        for ge in belem.findall("geom"):
            a = defaults.resolve(ge, cc)
            gt = a.get("type", "sphere")
            if "mesh" in a and "type" not in a:
                gt = "mesh"
            gtype = GEOM_TYPES[gt]
            size = np.zeros(3)
            sv = _floats(a.get("size", "0 0 0"))
            size[:len(sv)] = sv
            pos = _floats(a.get("pos", "0 0 0"))
            quat = _orientation(a, comp)
            if "fromto" in a:
                ft = _floats(a["fromto"])
                vec = ft[3:] - ft[:3]       # MuJoCo: from - to is used for the z axis direction (to -> from)
                pos = 0.5 * (ft[:3] + ft[3:])
                quat = z_to_quat(ft[:3] - ft[3:])
                half = 0.5 * np.linalg.norm(vec)
                if gtype in (GEOM_CAPSULE, GEOM_CYLINDER):
                    size[1] = half
                elif gtype in (GEOM_BOX, GEOM_ELLIPSOID):
                    size[2] = half
            G["name"].append(a.get("name", ""))
            G["type"].append(gtype)
            G["body"].append(bid)
            G["size"].append(size)
            G["pos"].append(pos)
            G["quat"].append(quat)
            fr = np.array([1.0, 0.005, 0.0001])
            fv = _floats(a.get("friction", "1 0.005 0.0001"))
            fr[:len(fv)] = fv
            G["friction"].append(fr)
            G["margin"].append(float(a.get("margin", 0)))
            G["gap"].append(float(a.get("gap", 0)))
            G["solref"].append(_floats(a.get("solref", "0.02 1")))
            G["solimp"].append(solimp5(a.get("solimp", "0.9 0.95 0.001 0.5 2")))
            G["solmix"].append(float(a.get("solmix", 1)))
            G["condim"].append(int(a.get("condim", 3)))
            G["priority"].append(int(a.get("priority", 0)))
            G["contype"].append(int(a.get("contype", 1)))
            G["conaffinity"].append(int(a.get("conaffinity", 1)))
            G["mesh"].append(a.get("mesh"))
            G["mass"].append(float(a["mass"]) if "mass" in a else None)
            G["density"].append(float(a.get("density", 1000)))
            G["group"].append(int(a.get("group", 0)))
        for se in belem.findall("site"):
            a = defaults.resolve(se, cc)
            S["name"].append(a.get("name", ""))
            S["body"].append(bid)
            pos = _floats(a.get("pos", "0 0 0"))
            quat = _orientation(a, comp)
            if "fromto" in a:
                ft = _floats(a["fromto"])
                pos = 0.5 * (ft[:3] + ft[3:])
                quat = z_to_quat(ft[:3] - ft[3:])
            S["pos"].append(pos)
            S["quat"].append(quat)
        for ce in belem.findall("body"):
            visit(ce, bid, cc)

    visit(root.find("worldbody"), 0, None)

    nbody, njnt, ngeom_all = len(B["name"]), len(J["name"]), len(G["name"])
    m.nbody, m.njnt, m.nq, m.nv = nbody, njnt, njnt, njnt
    m.body_names, m.jnt_names = B["name"], J["name"]
    m.site_names = S["name"]
    m.site_bodyid = np.array(S["body"], dtype=np.int32)
    m.site_pos = np.array(S["pos"], dtype=np.float64).reshape(-1, 3)
    m.site_quat = np.array(S["quat"], dtype=np.float64).reshape(-1, 4)
    m.body_parentid = np.array(B["parent"], dtype=np.int32)
    m.body_pos = np.array(B["pos"])
    m.body_quat = np.array(B["quat"])
    m.body_jntadr = np.array(B["jntadr"], dtype=np.int32)
    m.body_jntnum = np.array(B["jntnum"], dtype=np.int32)
    m.body_dofadr, m.body_dofnum = m.body_jntadr.copy(), m.body_jntnum.copy()

    # ---- body inertia: explicit <inertial>, else from geoms (inertiafromgeom=auto) -----------------------
    body_mass = np.array(B["mass"], dtype=np.float64)
    body_inertia = np.array(B["inertia"], dtype=np.float64)
    body_ipos = np.array(B["ipos"], dtype=np.float64)
    body_iquat = np.array(B["iquat"], dtype=np.float64)
    ifg = comp["inertiafromgeom"]
    for b in range(1, nbody):
        use_geoms = (ifg == "true") or (ifg == "auto" and not B["has_inertial"][b])
        if not use_geoms:
            continue
        gids = [g for g in range(ngeom_all) if G["body"][g] == b and G["type"][g] != GEOM_PLANE]
        if not gids:
            continue
        masses, coms, Is = [], [], []
        for g in gids:
            R = quat_to_mat(G["quat"][g])
            if G["type"][g] == GEOM_MESH:
                if G["density"][g] == 0 and G["mass"][g] is None:
                    continue
                me = meshes[G["mesh"][g]]
                if "legacy" not in me:
                    v, f = _load_mesh_vertices(me["file"])
                    me["legacy"] = mesh_legacy_inertia(v * me["scale"], f)
                vol, mcom, mI = me["legacy"]
                # MuJoCo 2.3.7 treats a mesh geom as its *equivalent inertia box* (the box with the mesh's
                # principal moments at unit density): mass = density * box volume, inertia = that box's.
                # (Pinned by the Talos.walk golden: pelvis mass/inertia = 0.93377 x the exact mesh values.)
                w, pq = _eig_inertia([mI[0, 0], mI[1, 1], mI[2, 2], mI[0, 1], mI[0, 2], mI[1, 2]])
                bs = np.array([np.sqrt(6 * (w[1] + w[2] - w[0]) / vol), np.sqrt(6 * (w[0] + w[2] - w[1]) / vol),
                               np.sqrt(6 * (w[0] + w[1] - w[2]) / vol)]) / 2
                mass = G["mass"][g] if G["mass"][g] is not None else 8 * bs.prod() * G["density"][g]
                diag = mass / 3.0 * np.array([bs[1] ** 2 + bs[2] ** 2, bs[0] ** 2 + bs[2] ** 2, bs[0] ** 2 + bs[1] ** 2])
                Rp = R @ quat_to_mat(pq)
                masses.append(mass)
                coms.append(G["pos"][g] + R @ mcom)
                Is.append(Rp @ np.diag(diag) @ Rp.T)
                continue
            mass, diag = _geom_inertia(G["type"][g], G["size"][g], G["density"][g], G["mass"][g])
            masses.append(mass)
            coms.append(G["pos"][g])
            Is.append(R @ np.diag(diag) @ R.T)
        if not masses:
            continue
        mt = sum(masses)
        if mt <= 0:
            continue
        com = sum(mi * ci for mi, ci in zip(masses, coms)) / mt
        I = np.zeros((3, 3))
        for mi, ci, Ii in zip(masses, coms, Is):
            d = ci - com
            I += Ii + mi * (np.dot(d, d) * np.eye(3) - np.outer(d, d))
        w, q = _eig_inertia([I[0, 0], I[1, 1], I[2, 2], I[0, 1], I[0, 2], I[1, 2]])
        body_mass[b], body_inertia[b], body_ipos[b], body_iquat[b] = mt, w, com, q
    # mjCBody::Compile order: enforce the minimum mass / inertia first, then balance the triangle inequality
    bm, bi = float(comp["boundmass"]), float(comp["boundinertia"])
    for b in range(1, nbody):
        body_mass[b] = max(body_mass[b], bm)
        body_inertia[b] = np.maximum(body_inertia[b], bi)
    if comp["balanceinertia"] == "true":
        for b in range(1, nbody):
            A, Bi, C = body_inertia[b]
            if A + Bi < C or A + C < Bi or Bi + C < A:
                body_inertia[b] = (A + Bi + C) / 3.0
    m.body_mass, m.body_inertia, m.body_ipos, m.body_iquat = body_mass, body_inertia, body_ipos, body_iquat

    # weld ids / root ids
    weld = np.zeros(nbody, dtype=np.int32)
    rootid = np.zeros(nbody, dtype=np.int32)
    for b in range(1, nbody):
        p = m.body_parentid[b]
        weld[b] = b if m.body_jntnum[b] > 0 else weld[p]
        rootid[b] = b if p == 0 else rootid[p]
    m.body_weldid, m.body_rootid = weld, rootid

    # ---- joints / dofs -----------------------------------------------------------------------------------
    m.jnt_type = np.array(J["type"], dtype=np.int32)
    m.jnt_bodyid = np.array(J["body"], dtype=np.int32)
    m.jnt_pos = np.array(J["pos"]).reshape(-1, 3)
    m.jnt_axis = np.array(J["axis"]).reshape(-1, 3)
    m.jnt_limited = np.array(J["limited"], dtype=np.int32)
    m.jnt_range = np.array(J["range"]).reshape(-1, 2)
    m.jnt_stiffness = np.array(J["stiffness"])
    m.jnt_margin = np.array(J["margin"])
    m.jnt_solref = np.array(J["solreflimit"]).reshape(-1, 2)
    m.jnt_solimp = np.array(J["solimplimit"]).reshape(-1, 5)
    m.qpos0 = np.array(J["ref"])
    m.qpos_spring = np.array(J["springref"])
    m.dof_bodyid = m.jnt_bodyid.copy()
    m.dof_armature = np.array(J["armature"])
    m.dof_damping = np.array(J["damping"])
    m.dof_frictionloss = np.array(J["frictionloss"])
    m.dof_solref = np.array(J["solreffriction"]).reshape(-1, 2)
    m.dof_solimp = np.array(J["solimpfriction"]).reshape(-1, 5)
    dof_parent = -np.ones(njnt, dtype=np.int32)
    last_dof_of_body = -np.ones(nbody, dtype=np.int32)   # last dof on the path root..body (inclusive)
    for b in range(1, nbody):
        prev = last_dof_of_body[m.body_parentid[b]]
        for k in range(m.body_jntnum[b]):
            d = m.body_jntadr[b] + k
            dof_parent[d] = prev
            prev = d
        last_dof_of_body[b] = prev
    m.dof_parentid = dof_parent
    m.body_lastdof = last_dof_of_body

    # ---- geoms: keep only geoms that can collide (contype|conaffinity != 0); others are visual only ----------
    keep = [g for g in range(ngeom_all) if (G["contype"][g] != 0 or G["conaffinity"][g] != 0)]
    mesh_vert_adr, mesh_vert_num, mesh_verts = [], [], []
    g_size = []
    g_pos, g_quat = [], []
    for g in keep:
        size = G["size"][g].copy()
        pos, quat = G["pos"][g].copy(), G["quat"][g].copy()
        if G["type"][g] == GEOM_MESH:
            me = meshes[G["mesh"][g]]
            if me["verts"] is None:
                v, f = _load_mesh_vertices(me["file"])
                v = v * me["scale"]
                me["raw"] = (v, f)
                me["verts"] = _mesh_prepare(v, f)
            hull, center, mquat, aabb = me["verts"]
            # MuJoCo recentres the mesh at its own CoM/principal frame and composes that into geom pos/quat
            pos = pos + quat_to_mat(quat) @ center
            quat = quat_mul(quat, mquat)
            mesh_vert_adr.append(len(mesh_verts))
            mesh_vert_num.append(len(hull))
            mesh_verts.extend(list(hull))
            size = aabb
        else:
            mesh_vert_adr.append(-1)
            mesh_vert_num.append(0)
        g_size.append(size)
        g_pos.append(pos)
        g_quat.append(quat)
    m.ngeom = len(keep)
    m.geom_names = [G["name"][g] for g in keep]
    m.geom_type = np.array([G["type"][g] for g in keep], dtype=np.int32)
    m.geom_bodyid = np.array([G["body"][g] for g in keep], dtype=np.int32)
    m.geom_size = np.array(g_size).reshape(-1, 3)
    m.geom_pos = np.array(g_pos).reshape(-1, 3)
    m.geom_quat = np.array(g_quat).reshape(-1, 4)
    m.geom_friction = np.array([G["friction"][g] for g in keep]).reshape(-1, 3)
    m.geom_margin = np.array([G["margin"][g] for g in keep])
    m.geom_gap = np.array([G["gap"][g] for g in keep])
    m.geom_solref = np.array([G["solref"][g] for g in keep]).reshape(-1, 2)
    m.geom_solimp = np.array([G["solimp"][g] for g in keep]).reshape(-1, 5)
    m.geom_solmix = np.array([G["solmix"][g] for g in keep])
    m.geom_condim = np.array([G["condim"][g] for g in keep], dtype=np.int32)
    m.geom_priority = np.array([G["priority"][g] for g in keep], dtype=np.int32)
    m.geom_contype = np.array([G["contype"][g] for g in keep], dtype=np.int32)
    m.geom_conaffinity = np.array([G["conaffinity"][g] for g in keep], dtype=np.int32)
    m.geom_meshadr = np.array(mesh_vert_adr, dtype=np.int32)
    m.geom_meshnum = np.array(mesh_vert_num, dtype=np.int32)
    m.mesh_vert = np.array(mesh_verts, dtype=np.float64).reshape(-1, 3)
    rb = np.zeros(m.ngeom)
    for i in range(m.ngeom):
        t, s = m.geom_type[i], m.geom_size[i]
        if t == GEOM_SPHERE:
            rb[i] = s[0]
        elif t == GEOM_CAPSULE:
            rb[i] = s[0] + s[1]
        elif t == GEOM_CYLINDER:
            rb[i] = np.sqrt(s[0] ** 2 + s[1] ** 2)
        elif t in (GEOM_BOX, GEOM_ELLIPSOID):
            rb[i] = np.linalg.norm(s) if t == GEOM_BOX else max(s)
        elif t == GEOM_MESH:
            rb[i] = np.linalg.norm(s)
        else:
            rb[i] = 0.0
    m.geom_rbound = rb

    # ---- collision pair filter (static part of mj_collision's broadphase) --------------------------------
    pairs, dropped, approx = [], [], []
    for g1 in range(m.ngeom):
        for g2 in range(g1 + 1, m.ngeom):
            b1, b2 = m.geom_bodyid[g1], m.geom_bodyid[g2]
            if not ((m.geom_contype[g1] & m.geom_conaffinity[g2]) or (m.geom_contype[g2] & m.geom_conaffinity[g1])):
                continue
            w1, w2 = weld[b1], weld[b2]
            if w1 == w2:
                continue
            wp1, wp2 = weld[m.body_parentid[w1]], weld[m.body_parentid[w2]]
            if w1 != 0 and w2 != 0 and (w1 == wp2 or w2 == wp1):
                continue
            # order so that type(g1) <= type(g2) (MuJoCo's collision table is upper triangular)
            a, b = (g1, g2) if m.geom_type[g1] <= m.geom_type[g2] else (g2, g1)
            if m.geom_type[a] == GEOM_PLANE and m.geom_type[b] == GEOM_PLANE:
                continue
            ta, tb = m.geom_type[a], m.geom_type[b]
            # MuJoCo 2.3.7 collision table (type(a) <= type(b)): dedicated routines for plane-X, sphere-sphere, sphere-capsule,
            # capsule-capsule, sphere-box (all restated); capsule-box / box-box have dedicated MULTI-contact routines that are
            # not restated: they run through the general convex routine (one contact, counted in n_approx_pairs);
            # every other pair of sphere | capsule | cylinder | box | mesh is mjc_Convex (MPR) in MuJoCo too.
            convexable = (GEOM_SPHERE, GEOM_CAPSULE, GEOM_CYLINDER, GEOM_BOX, GEOM_MESH)
            if ta == GEOM_PLANE:
                supported = tb in convexable
            else:
                supported = ta in convexable and tb in convexable
            if not supported:
                dropped.append((a, b))          # ellipsoids, height fields: no in-scope model has them
                continue
            if (ta, tb) in ((GEOM_CAPSULE, GEOM_BOX), (GEOM_BOX, GEOM_BOX)):
                approx.append((a, b))
            pairs.append((a, b))
    m.npair = len(pairs)
    m.n_dropped_pairs = len(dropped)
    m.n_approx_pairs = len(approx)
    m.pair_geom = np.array(pairs, dtype=np.int32).reshape(-1, 2)

    # ---- actuators ------------------------------------------------------------------------------------------
    A = dict(name=[], dof=[], gear=[], ctrllimited=[], ctrlrange=[], forcelimited=[], forcerange=[], gain=[],
             bias=[])
    for sec in root.findall("actuator"):
        for ae in sec:
            a = defaults.resolve(ae, None)
            if ae.tag not in ("motor", "general", "position"):
                raise NotImplementedError("actuator <%s> (in-scope models use <motor>, <general> and <position>)" % ae.tag)
            if "joint" not in a:
                raise NotImplementedError("only joint transmissions")
            A["name"].append(a.get("name", ""))
            A["dof"].append(J["name"].index(a["joint"]))
            A["gear"].append(_floats(a.get("gear", "1"))[0])
            cr = _floats(a.get("ctrlrange", "0 0"))
            cl = a.get("ctrllimited", "auto")
            A["ctrllimited"].append(int(cl == "true" or (cl == "auto" and autolimits and cr[0] < cr[1])))
            A["ctrlrange"].append(cr)
            fr = _floats(a.get("forcerange", "0 0"))
            fl = a.get("forcelimited", "auto")
            A["forcelimited"].append(int(fl == "true" or (fl == "auto" and autolimits and fr[0] < fr[1])))
            A["forcerange"].append(fr)
            gp = _floats(a.get("gainprm", "1"))[0] if ae.tag == "general" else 1.0
            bp = np.zeros(3)
            if ae.tag == "general" and "biasprm" in a:
                v = _floats(a["biasprm"])
                bp[:min(3, len(v))] = v[:3]
            if ae.tag == "position":
                # MuJoCo 2.3.7 <position>: gainprm[0] = kp, biasprm = (0, -kp, 0), i.e. force = kp (ctrl - length)
                gp = _floats(a.get("kp", "1"))[0]
                bp = np.array([0.0, -gp, 0.0])
            A["gain"].append(gp)
            A["bias"].append(bp)
            # the engine and the oracle evaluate the bias at qpos[dof] / qvel[dof], where MuJoCo uses the actuator length
            # gear * qpos and velocity gear * qvel of a hinge or slide joint: other cases would be computed wrongly
            if np.any(bp[1:] != 0):
                if J["type"][A["dof"][-1]] not in (JNT_HINGE, JNT_SLIDE):
                    raise NotImplementedError("actuator %r: a length-dependent bias needs a hinge or slide joint"
                                              % A["name"][-1])
                if A["gear"][-1] != 1.0:
                    raise NotImplementedError("actuator %r: a length-dependent bias needs gear 1, not %g"
                                              % (A["name"][-1], A["gear"][-1]))
    m.nu = len(A["name"])
    m.actuator_names = A["name"]
    m.actuator_dof = np.array(A["dof"], dtype=np.int32)
    m.actuator_gear = np.array(A["gear"], dtype=np.float64)
    m.actuator_ctrllimited = np.array(A["ctrllimited"], dtype=np.int32)
    m.actuator_ctrlrange = np.array(A["ctrlrange"], dtype=np.float64).reshape(-1, 2)
    m.actuator_forcelimited = np.array(A["forcelimited"], dtype=np.int32)
    m.actuator_forcerange = np.array(A["forcerange"], dtype=np.float64).reshape(-1, 2)
    m.actuator_gain = np.array(A["gain"], dtype=np.float64)
    m.actuator_bias = np.array(A["bias"], dtype=np.float64).reshape(-1, 3)

    for sec in root.findall("equality"):
        for eq in sec:
            if eq.get("active", "true") == "true":
                raise NotImplementedError("active equality constraint %r (the in-scope task configurations remove "
                                          "them all or leave them inactive)" % eq.get("name"))

    set_constants(m)
    if fuse_static:
        fuse_static_bodies(m)
    return m


def _mesh_prepare(v, f, max_verts=None):
    """
    Convex hull + recentring of a mesh, like MuJoCo's mesh compile step (user_mesh.cc, 2.3.7 default
    inertia="legacy"): the mesh is expressed in the frame of the centre of mass / principal axes of the ORIGINAL
    triangle mesh under the legacy volume rule (`mesh_legacy_inertia`), and geoms referencing it get that transform
    composed in. The frame origin is the geom centre libccd's MPR starts from (mjccd_center), so it has to be
    MuJoCo's; the collision vertices are those of the convex hull. Returns (hull_vertices_local, center, quat,
    aabb_halfsizes).
    """
    from scipy.spatial import ConvexHull
    hull = ConvexHull(v)
    hv = v[hull.vertices]
    _, center, I = mesh_legacy_inertia(v, f)
    w, q = _eig_inertia([I[0, 0], I[1, 1], I[2, 2], I[0, 1], I[0, 2], I[1, 2]])
    R = quat_to_mat(q)
    # MuJoCo stores mesh vertices as float32 AFTER the transformation into this frame (mjModel.mesh_vert is float*);
    # rounding here the same way reproduces its vertex positions (the rounding is indifferent to the sign / order
    # conventions of the principal axes)
    local = ((hv - center) @ R).astype(np.float32).astype(np.float64)
    aabb = np.abs(((v - center) @ R).astype(np.float32).astype(np.float64)).max(axis=0)
    return local, center, q, aabb


# ----------------------------------------------------------------------------------------------------------
# constants MuJoCo derives at compile time (mj_setConst): need kinematics + mass matrix at qpos0
# ----------------------------------------------------------------------------------------------------------
def _kinematics(m, qpos):
    xpos = np.zeros((m.nbody, 3))
    xquat = np.zeros((m.nbody, 4))
    xquat[0, 0] = 1
    xanchor = np.zeros((m.njnt, 3))
    xaxis = np.zeros((m.njnt, 3))
    for b in range(1, m.nbody):
        p = m.body_parentid[b]
        Rp = quat_to_mat(xquat[p])
        pos = xpos[p] + Rp @ m.body_pos[b]
        quat = quat_mul(xquat[p], m.body_quat[b])
        for k in range(m.body_jntnum[b]):
            j = m.body_jntadr[b] + k
            R = quat_to_mat(quat)
            xanchor[j] = pos + R @ m.jnt_pos[j]
            xaxis[j] = R @ m.jnt_axis[j]
            if m.jnt_type[j] == JNT_SLIDE:
                pos = pos + xaxis[j] * (qpos[j] - m.qpos0[j])
            else:
                quat = quat_mul(quat, axisangle_to_quat(m.jnt_axis[j], qpos[j] - m.qpos0[j]))
                pos = xanchor[j] - quat_to_mat(quat) @ m.jnt_pos[j]
        xpos[b], xquat[b] = pos, quat / np.linalg.norm(quat)
    return xpos, xquat, xanchor, xaxis


def mass_matrix(m, qpos):
    """Dense joint-space inertia M(q) (+armature) and per-body 6 x nv CoM Jacobians [trans; rot]."""
    xpos, xquat, xanchor, xaxis = _kinematics(m, qpos)
    nv = m.nv
    M = np.diag(m.dof_armature.astype(np.float64))
    jacs = np.zeros((m.nbody, 6, nv))
    for b in range(1, m.nbody):
        R = quat_to_mat(xquat[b])
        xipos = xpos[b] + R @ m.body_ipos[b]
        Ri = R @ quat_to_mat(m.body_iquat[b])
        d = m.body_lastdof[b]
        Jp, Jr = np.zeros((3, nv)), np.zeros((3, nv))
        while d >= 0:
            if m.jnt_type[d] == JNT_SLIDE:
                Jp[:, d] = xaxis[d]
            else:
                Jr[:, d] = xaxis[d]
                Jp[:, d] = np.cross(xaxis[d], xipos - xanchor[d])
            d = m.dof_parentid[d]
        jacs[b, :3], jacs[b, 3:] = Jp, Jr
        Iw = Ri @ np.diag(m.body_inertia[b]) @ Ri.T
        M += m.body_mass[b] * Jp.T @ Jp + Jr.T @ Iw @ Jr
    return M, jacs


def set_constants(m):
    M, jacs = mass_matrix(m, m.qpos0)
    Minv = np.linalg.inv(M)
    m.dof_invweight0 = np.diag(Minv).copy()
    biw = np.zeros((m.nbody, 2))
    for b in range(1, m.nbody):
        A = jacs[b] @ Minv @ jacs[b].T
        biw[b, 0] = max(mjMINVAL, (A[0, 0] + A[1, 1] + A[2, 2]) / 3)
        biw[b, 1] = max(mjMINVAL, (A[3, 3] + A[4, 4] + A[5, 5]) / 3)
        if m.body_weldid[b] == 0:
            biw[b] = 0
    m.body_invweight0 = biw
    # contacts look invweight up through the geom's body; keeping it per geom makes static-body fusion exact
    m.geom_invweight0 = biw[m.geom_bodyid].copy() if m.ngeom else np.zeros((0, 2))
    m.stat_meaninertia = float(np.mean(np.diag(M))) if m.nv else 1.0


def fuse_static_bodies(m):
    """
    Merge every joint-less body into its parent (inertia composed, geoms / sites / child bodies re-expressed in the
    parent frame). Dynamically identical to the unfused tree (MuJoCo's own `fusestatic`), but the engine then walks
    9-14 bodies instead of 33-46. Compile-time constants that MuJoCo evaluates per *original* body (body_invweight0
    used by contacts) were already baked per geom (geom_invweight0) before fusing.
    """
    nb = m.nbody
    parent = m.body_parentid.copy()
    pos, quat = m.body_pos.copy(), m.body_quat.copy()
    mass = m.body_mass.copy()
    ipos = m.body_ipos.copy()
    # full inertia tensors about the body CoM, in the body frame
    Ifull = np.zeros((nb, 3, 3))
    for b in range(nb):
        R = quat_to_mat(m.body_iquat[b])
        Ifull[b] = R @ np.diag(m.body_inertia[b]) @ R.T
    gpos, gquat, gbody = m.geom_pos.copy(), m.geom_quat.copy(), m.geom_bodyid.copy()
    spos, squat, sbody = m.site_pos.copy(), m.site_quat.copy(), m.site_bodyid.copy()
    alive = np.ones(nb, dtype=bool)
    for b in range(nb - 1, 0, -1):
        p = parent[b]
        if m.body_jntnum[b] != 0 or p == 0:
            continue
        Rb = quat_to_mat(quat[b])
        # inertia of b expressed in p's frame
        cb = pos[b] + Rb @ ipos[b]
        Ib = Rb @ Ifull[b] @ Rb.T
        mt = mass[p] + mass[b]
        if mt > 0:
            c = (mass[p] * ipos[p] + mass[b] * cb) / mt
            def shift(I, ms, d):
                return I + ms * (np.dot(d, d) * np.eye(3) - np.outer(d, d))
            Ifull[p] = shift(Ifull[p], mass[p], ipos[p] - c) + shift(Ib, mass[b], cb - c)
            ipos[p], mass[p] = c, mt
        for g in range(m.ngeom):
            if gbody[g] == b:
                gpos[g] = pos[b] + Rb @ gpos[g]
                gquat[g] = quat_mul(quat[b], gquat[g])
                gbody[g] = p
        for k in range(len(sbody)):
            if sbody[k] == b:
                spos[k] = pos[b] + Rb @ spos[k]
                squat[k] = quat_mul(quat[b], squat[k])
                sbody[k] = p
        for c2 in range(b + 1, nb):
            if alive[c2] and parent[c2] == b:
                pos[c2] = pos[b] + Rb @ pos[c2]
                quat[c2] = quat_mul(quat[b], quat[c2])
                parent[c2] = p
        alive[b] = False
    keep = np.nonzero(alive)[0]
    # name of every fused body -> name of the body it now belongs to (parent[b] is b's parent when b was fused)
    fused = {}
    for b in range(1, nb):
        if not alive[b]:
            p = parent[b]
            while not alive[p]:
                p = parent[p]
            fused[m.body_names[b]] = m.body_names[p]
    m.fused_bodies = fused
    remap = -np.ones(nb, dtype=np.int64)
    remap[keep] = np.arange(len(keep))
    inertia, iquat = np.zeros((len(keep), 3)), np.zeros((len(keep), 4))
    for k, b in enumerate(keep):
        I = Ifull[b]
        if mass[b] > 0 or np.any(I != 0):
            w, q = _eig_inertia([I[0, 0], I[1, 1], I[2, 2], I[0, 1], I[0, 2], I[1, 2]])
        else:
            w, q = np.zeros(3), np.array([1.0, 0, 0, 0])
        inertia[k], iquat[k] = w, q
    m.nbody = len(keep)
    m.body_names = [m.body_names[b] for b in keep]
    m.body_parentid = remap[parent[keep]].astype(np.int32)
    m.body_parentid[0] = 0
    m.body_pos, m.body_quat = pos[keep], quat[keep]
    m.body_ipos, m.body_iquat, m.body_mass, m.body_inertia = ipos[keep], iquat, mass[keep], inertia
    for name in ("body_jntadr", "body_jntnum", "body_dofadr", "body_dofnum", "body_lastdof"):
        setattr(m, name, getattr(m, name)[keep])
    m.body_invweight0 = m.body_invweight0[keep]
    m.body_weldid = np.arange(m.nbody, dtype=np.int32)
    m.body_rootid = np.array([0] + [1] * (m.nbody - 1), dtype=np.int32)
    m.jnt_bodyid = remap[m.jnt_bodyid].astype(np.int32)
    m.dof_bodyid = m.jnt_bodyid.copy()
    m.geom_bodyid, m.geom_pos, m.geom_quat = remap[gbody].astype(np.int32), gpos, gquat
    m.site_bodyid, m.site_pos, m.site_quat = remap[sbody].astype(np.int32), spos, squat
