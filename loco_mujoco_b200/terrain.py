"""
Height-field terrain (MuJoCo's hfield geom) for UnitreeA1: the field itself, its attachment to a compiled model, and a seeded
generator of tiled training terrains. numpy only; the engine's semantics are stated in include/locosim.h
(locosim_set_terrain_origin).

    hf = terrain.tiled_terrain(n_rows=4, n_cols=4, seed=0)
    env = LocoEnv.make("UnitreeA1.simple", num_envs=4096, terrain=hf)
    origins = hf.tile_origins()                       # [n_rows * n_cols, 2] tile centres, each a flat platform at z = 0
    env.terrain_origin[:] = torch.as_tensor(origins[np.arange(4096) % len(origins)], device=env.terrain_origin.device)
"""
import copy

import numpy as np

from .modelpack import GEOM_HFIELD, GEOM_PLANE


class HeightField:
    """A grid of terrain heights in metres: heights_m[r, c] is the surface height at x = c * 2 rx / (ncol - 1) - rx + pos[0],
    y = r * 2 ry / (nrow - 1) - ry + pos[1] (rows along y, columns along x). `base` > 0 is the depth of the solid below its
    lowest sample. Stored as MuJoCo's compiler stores an hfield: `data` normalised to [0, 1], `elevation` = max - min, and
    the minimum moved into the geom's z position (`geom_pos`)."""

    def __init__(self, heights_m, size, base=1.0, pos=(0.0, 0.0, 0.0)):
        h = np.asarray(heights_m, dtype=np.float64)
        if h.ndim != 2 or h.shape[0] < 2 or h.shape[1] < 2:
            raise ValueError("heights_m must be a [nrow, ncol] array with nrow, ncol >= 2, got shape %s" % (h.shape,))
        if not np.all(np.isfinite(h)):
            raise ValueError("heights_m must be finite")
        size = tuple(float(v) for v in size)
        if len(size) != 2 or not (size[0] > 0 and size[1] > 0):
            raise ValueError("size must be (rx, ry) with rx, ry > 0 (half extents in metres), got %r" % (size,))
        if not float(base) > 0:
            raise ValueError("base must be positive, got %r" % (base,))
        pos = np.asarray(pos, dtype=np.float64)
        if pos.shape != (3,) or not np.all(np.isfinite(pos)):
            raise ValueError("pos must be 3 finite numbers")
        lo, hi = float(h.min()), float(h.max())
        self.elevation = hi - lo
        self.data = (h - lo) / self.elevation if self.elevation > 0 else np.zeros_like(h)
        self.rx, self.ry = size
        self.base = float(base)
        self.geom_pos = np.array([pos[0], pos[1], pos[2] + lo])
        self.tiles = None           # (n_rows, n_cols, tile_size) of a tiled_terrain field

    def tile_origins(self):
        """[n_rows * n_cols, 2] centres (x, y) of the tiles of a tiled_terrain field, row major: the terrain origins that put
        an env on each tile's platform"""
        if self.tiles is None:
            raise ValueError("not a tiled_terrain field")
        n_rows, n_cols, t = self.tiles
        x = self.geom_pos[0] - self.rx + (np.arange(n_cols) + 0.5) * t
        y = self.geom_pos[1] - self.ry + (np.arange(n_rows) + 0.5) * t
        return np.stack(np.meshgrid(x, y), axis=-1).reshape(-1, 2)

    @property
    def shape(self):
        return self.data.shape

    @property
    def size4(self):
        """MuJoCo's hfield size: (rx, ry, elevation, base)"""
        return np.array([self.rx, self.ry, self.elevation, self.base])

    def heights(self):
        """[nrow, ncol] heights in metres (world z of the samples, before any env's origin shift)"""
        return self.data * self.elevation + self.geom_pos[2]

    def sample_xy(self):
        """x [ncol] and y [nrow] of the samples in the world (before any env's origin shift)"""
        nrow, ncol = self.data.shape
        x = np.arange(ncol) * (2 * self.rx / (ncol - 1)) - self.rx + self.geom_pos[0]
        y = np.arange(nrow) * (2 * self.ry / (nrow - 1)) - self.ry + self.geom_pos[1]
        return x, y


def attach(model, hf):
    """A copy of compiled `model` with height field `hf` as its last geom ("terrain", on the world body, unrotated). The terrain
    copies the floor plane's contact parameters and is paired, as geom1, with exactly the geoms the floor is paired with; its
    pairs follow every other pair. The floor stays. Existing geom indices do not move."""
    if not isinstance(hf, HeightField):
        raise TypeError("terrain must be a loco_mujoco_b200.terrain.HeightField, got %s" % type(hf).__name__)
    if getattr(model, "hfield", None) is not None:
        raise ValueError("the model already has a terrain (one height field per model)")
    t = np.asarray(model.geom_type)
    floors = [g for g in range(model.ngeom) if t[g] == GEOM_PLANE and int(np.asarray(model.geom_bodyid)[g]) == 0]
    if not floors:
        raise ValueError("the model has no floor plane to take the terrain's contact parameters from")
    f = floors[0]
    m = copy.deepcopy(model)
    g = m.ngeom

    def grow(name, value, width):
        a = np.asarray(getattr(m, name))
        row = np.asarray(value, dtype=a.dtype).reshape(width)
        setattr(m, name, np.concatenate([a.reshape(-1), row]) if a.ndim == 1 else np.concatenate([a, row[None]]))

    def floor_row(name, width):
        a = np.asarray(getattr(model, name))
        return a.reshape(-1, width)[f] if width > 1 else a.reshape(-1)[f]

    for name in ("geom_bodyid", "geom_condim", "geom_priority", "geom_friction", "geom_margin", "geom_gap", "geom_solref",
                 "geom_solimp", "geom_solmix", "geom_invweight0", "geom_contype", "geom_conaffinity"):
        width = {"geom_friction": 3, "geom_solref": 2, "geom_solimp": 5, "geom_invweight0": 2}.get(name, 1)
        grow(name, floor_row(name, width), width)
    grow("geom_type", GEOM_HFIELD, 1)
    grow("geom_meshadr", -1, 1)
    grow("geom_meshnum", 0, 1)
    grow("geom_size", [hf.rx, hf.ry, hf.elevation], 3)
    grow("geom_pos", hf.geom_pos, 3)
    grow("geom_quat", [1.0, 0.0, 0.0, 0.0], 4)
    grow("geom_rbound", np.sqrt(hf.rx ** 2 + hf.ry ** 2 + max(hf.elevation, hf.base) ** 2), 1)
    pg = np.asarray(m.pair_geom).reshape(-1, 2)
    partners = sorted(int(b) for a, b in pg if a == f)
    m.pair_geom = np.concatenate([pg, np.array([[g, b] for b in partners], dtype=pg.dtype).reshape(-1, 2)]).astype(pg.dtype)
    if np.asarray(model.pair_geom).ndim == 1:
        m.pair_geom = m.pair_geom.reshape(-1)
    m.ngeom = g + 1
    m.npair = len(np.asarray(m.pair_geom).reshape(-1, 2))
    m.geom_names = list(m.geom_names) + ["terrain"]
    m.hfield = hf
    return m


def _tile(kind, difficulty, n, res, platform, rng, max_rough, max_slope, max_step, step_width):
    """heights [n + 1, n + 1] of one square tile of n cells (side n * res), its centre on the middle sample"""
    u = (np.arange(n + 1) - n / 2) * res
    d = np.maximum(np.abs(u)[None, :], np.abs(u)[:, None])           # Chebyshev distance from the centre
    out = np.maximum(d - platform / 2, 0.0)                           # distance outside the central platform
    if kind == "flat":
        z = np.zeros_like(d)
    elif kind == "rough":
        z = rng.uniform(-1.0, 1.0, size=d.shape) * max_rough * difficulty
    elif kind == "slope":
        z = -max_slope * difficulty * out                             # a pyramid sloping down from the platform
    elif kind == "stairs":
        z = -max_step * difficulty * np.ceil(out / step_width - 1e-9)    # steps down from the platform
    else:
        raise ValueError("unknown tile kind %r (flat, rough, slope, stairs)" % (kind,))
    z[d <= platform / 2 + 1e-9] = 0.0
    return z


def tiled_terrain(n_rows=4, n_cols=4, tile_size=8.0, resolution=0.1, kinds=("flat", "rough", "slope", "stairs"),
                  max_rough=0.05, max_slope=0.3, max_step=0.1, step_width=0.4, platform=1.0, base=1.0, seed=0):
    """A seeded curriculum field in the style of legged_gym: n_rows x n_cols square tiles of side `tile_size` metres; row i
    has difficulty (i + 1) / n_rows (roughness, slope and step height scale with it), column j is of kind
    kinds[j % len(kinds)]: flat, uniform rough, pyramid slope or pyramid stairs (both going down from the centre). Every
    tile has a flat square platform of side `platform` at z = 0 around its centre; `tile_origins()` of the result gives
    those centres. The field is centred on the world origin."""
    if n_rows < 1 or n_cols < 1:
        raise ValueError("n_rows and n_cols must be positive")
    n = tile_size / resolution
    if not (resolution > 0 and abs(n - round(n)) < 1e-9 and int(round(n)) % 2 == 0):
        raise ValueError("tile_size / resolution must be an even integer (a sample on every tile centre)")
    if not 0 < platform < tile_size:
        raise ValueError("platform must lie in (0, tile_size)")
    n = int(round(n))
    rng = np.random.RandomState(seed)
    H = np.zeros((n_rows * n + 1, n_cols * n + 1))
    for i in range(n_rows):
        for j in range(n_cols):
            z = _tile(kinds[j % len(kinds)], (i + 1) / n_rows, n, resolution, platform, rng, max_rough, max_slope,
                      max_step, step_width)
            # (a tile's border samples are shared with its neighbours: the later tile's values win)
            H[i * n:(i + 1) * n + 1, j * n:(j + 1) * n + 1] = z
    hf = HeightField(H, (n_cols * tile_size / 2, n_rows * tile_size / 2), base=base)
    hf.tiles = (n_rows, n_cols, float(tile_size))
    return hf

