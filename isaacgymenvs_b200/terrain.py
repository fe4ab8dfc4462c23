"""Height-field terrain generator for AnymalTerrain.

The reference builds its terrain with `isaacgym.terrain_utils` (`tasks/anymal_terrain.py:542-653`),
which ships inside the closed Isaac Gym package and is not under the reference checkout.  The generators
below are restated from what the call sites require (argument meaning, units, the SubTerrain
fields they touch) and the published behaviour of those helpers: integer height samples
(`vertical_scale` metres per unit) on a `horizontal_scale` grid.  Exact sample-for-sample equality
with the closed helpers is [unverifiable here]; the terrain is a synthetic INPUT of the path, and
`Terrain` reproduces the reference class's layout arithmetic (border, tile placement, env_origins,
curriculum / random selection: anymal_terrain.py:543-673) exactly.

The reference then triangulates the field (`convert_heightfield_to_trimesh`) for PhysX; this engine
collides against the height field directly (DESIGN.md), so no trimesh is produced.
"""
import numpy as np


class SubTerrain:
    def __init__(self, terrain_name="terrain", width=256, length=256, vertical_scale=1.0, horizontal_scale=1.0):
        self.terrain_name = terrain_name
        self.vertical_scale = vertical_scale
        self.horizontal_scale = horizontal_scale
        self.width = width
        self.length = length
        self.height_field_raw = np.zeros((self.width, self.length), dtype=np.int16)


def _bilinear_upsample(z, nx, ny):
    """z on a coarse regular grid spanning the tile -> (nx, ny) samples, linear in each axis."""
    x_src = np.linspace(0.0, 1.0, z.shape[0]); y_src = np.linspace(0.0, 1.0, z.shape[1])
    x_dst = np.linspace(0.0, 1.0, nx); y_dst = np.linspace(0.0, 1.0, ny)
    tmp = np.stack([np.interp(x_dst, x_src, z[:, j]) for j in range(z.shape[1])], axis=1)
    return np.stack([np.interp(y_dst, y_src, tmp[i, :]) for i in range(nx)], axis=0)


def random_uniform_terrain(terrain, min_height, max_height, step=1, downsampled_scale=None, rng=np.random):
    if downsampled_scale is None:
        downsampled_scale = terrain.horizontal_scale
    lo = int(min_height / terrain.vertical_scale); hi = int(max_height / terrain.vertical_scale)
    st = max(1, int(step / terrain.vertical_scale))
    heights_range = np.arange(lo, hi + st, st)
    shape = (int(terrain.width * terrain.horizontal_scale / downsampled_scale),
             int(terrain.length * terrain.horizontal_scale / downsampled_scale))
    coarse = rng.choice(heights_range, shape)
    z = np.rint(_bilinear_upsample(coarse.astype(np.float64), terrain.width, terrain.length))
    terrain.height_field_raw += z.astype(np.int16)
    return terrain


def pyramid_sloped_terrain(terrain, slope=1, platform_size=1.):
    x = np.arange(0, terrain.width); y = np.arange(0, terrain.length)
    cx, cy = int(terrain.width / 2), int(terrain.length / 2)
    xx = ((cx - np.abs(cx - x)) / cx).reshape(terrain.width, 1)
    yy = ((cy - np.abs(cy - y)) / cy).reshape(1, terrain.length)
    max_height = int(slope * (terrain.horizontal_scale / terrain.vertical_scale) * (terrain.width / 2))
    terrain.height_field_raw += (max_height * xx * yy).astype(terrain.height_field_raw.dtype)
    ps = int(platform_size / terrain.horizontal_scale / 2)
    x1, y1 = terrain.width // 2 - ps, terrain.length // 2 - ps
    min_h = min(terrain.height_field_raw[x1, y1], 0); max_h = max(terrain.height_field_raw[x1, y1], 0)
    terrain.height_field_raw = np.clip(terrain.height_field_raw, min_h, max_h)
    return terrain


def pyramid_stairs_terrain(terrain, step_width, step_height, platform_size=1.):
    sw = int(step_width / terrain.horizontal_scale); sh = int(step_height / terrain.vertical_scale)
    ps = int(platform_size / terrain.horizontal_scale)
    height = 0
    start_x, stop_x, start_y, stop_y = 0, terrain.width, 0, terrain.length
    while (stop_x - start_x) > ps and (stop_y - start_y) > ps:
        start_x += sw; stop_x -= sw; start_y += sw; stop_y -= sw
        height += sh
        terrain.height_field_raw[start_x:stop_x, start_y:stop_y] = height
    return terrain


def discrete_obstacles_terrain(terrain, max_height, min_size, max_size, num_rects, platform_size=1., rng=np.random):
    mh = int(max_height / terrain.vertical_scale)
    mn = int(min_size / terrain.horizontal_scale); mx = int(max_size / terrain.horizontal_scale)
    ps = int(platform_size / terrain.horizontal_scale)
    (i, j) = terrain.height_field_raw.shape
    height_range = [-mh, -mh // 2, mh // 2, mh]
    width_range = range(mn, mx, 4); length_range = range(mn, mx, 4)
    for _ in range(num_rects):
        w = rng.choice(width_range); l = rng.choice(length_range)
        si = rng.choice(range(0, i - w, 4)); sj = rng.choice(range(0, j - l, 4))
        terrain.height_field_raw[si:si + w, sj:sj + l] = rng.choice(height_range)
    x1, x2 = (terrain.width - ps) // 2, (terrain.width + ps) // 2
    y1, y2 = (terrain.length - ps) // 2, (terrain.length + ps) // 2
    terrain.height_field_raw[x1:x2, y1:y2] = 0
    return terrain


def stepping_stones_terrain(terrain, stone_size, stone_distance, max_height, platform_size=1., depth=-10, rng=np.random):
    ss = max(1, int(stone_size / terrain.horizontal_scale)); sd = int(stone_distance / terrain.horizontal_scale)
    mh = int(max_height / terrain.vertical_scale); ps = int(platform_size / terrain.horizontal_scale)
    height_range = np.arange(-mh - 1, mh, step=1)
    terrain.height_field_raw[:, :] = int(depth / terrain.vertical_scale)
    sx = 0
    while sx < terrain.width:
        sy = -rng.randint(0, ss) if ss > 1 else 0
        while sy < terrain.length:
            y0, y1 = max(0, sy), min(terrain.length, sy + ss)
            if y1 > y0:
                terrain.height_field_raw[sx:min(terrain.width, sx + ss), y0:y1] = rng.choice(height_range)
            sy += ss + sd
        sx += ss + sd
    x1, x2 = (terrain.width - ps) // 2, (terrain.width + ps) // 2
    y1, y2 = (terrain.length - ps) // 2, (terrain.length + ps) // 2
    terrain.height_field_raw[x1:x2, y1:y2] = 0
    return terrain


class Terrain:
    """Layout arithmetic of the reference class (anymal_terrain.py:543-673), generators above."""

    def __init__(self, cfg, num_robots, seed=42):
        self.type = cfg["terrainType"]
        if self.type in ["none", "plane"]:
            return
        self.rng = np.random.RandomState(seed)
        self.horizontal_scale = 0.1
        self.vertical_scale = 0.005
        self.border_size = 20
        self.env_length = cfg["mapLength"]
        self.env_width = cfg["mapWidth"]
        self.proportions = [np.sum(cfg["terrainProportions"][:i + 1]) for i in range(len(cfg["terrainProportions"]))]
        self.env_rows = cfg["numLevels"]
        self.env_cols = cfg["numTerrains"]
        self.num_maps = self.env_rows * self.env_cols
        self.num_per_env = int(num_robots / self.num_maps)
        self.env_origins = np.zeros((self.env_rows, self.env_cols, 3))
        self.width_per_env_pixels = int(self.env_width / self.horizontal_scale)
        self.length_per_env_pixels = int(self.env_length / self.horizontal_scale)
        self.border = int(self.border_size / self.horizontal_scale)
        self.tot_cols = int(self.env_cols * self.width_per_env_pixels) + 2 * self.border
        self.tot_rows = int(self.env_rows * self.length_per_env_pixels) + 2 * self.border
        self.height_field_raw = np.zeros((self.tot_rows, self.tot_cols), dtype=np.int16)
        if cfg.get("heightSamplesOverride") is not None:       # test hook: a given (tot_rows, tot_cols) int16 field
            self.height_field_raw[:] = np.asarray(cfg["heightSamplesOverride"], dtype=np.int16)
        elif cfg["curriculum"]:
            self.curiculum(num_robots, num_terrains=self.env_cols, num_levels=self.env_rows)
        else:
            self.randomized_terrain()
        self.heightsamples = self.height_field_raw

    def _new_tile(self):
        return SubTerrain("terrain", width=self.width_per_env_pixels, length=self.width_per_env_pixels,
                          vertical_scale=self.vertical_scale, horizontal_scale=self.horizontal_scale)

    def _place(self, terrain, i, j):
        sx = self.border + i * self.length_per_env_pixels; ex = self.border + (i + 1) * self.length_per_env_pixels
        sy = self.border + j * self.width_per_env_pixels; ey = self.border + (j + 1) * self.width_per_env_pixels
        self.height_field_raw[sx:ex, sy:ey] = terrain.height_field_raw
        x1 = int((self.env_length / 2. - 1) / self.horizontal_scale); x2 = int((self.env_length / 2. + 1) / self.horizontal_scale)
        y1 = int((self.env_width / 2. - 1) / self.horizontal_scale); y2 = int((self.env_width / 2. + 1) / self.horizontal_scale)
        z = np.max(terrain.height_field_raw[x1:x2, y1:y2]) * self.vertical_scale
        self.env_origins[i, j] = [(i + 0.5) * self.env_length, (j + 0.5) * self.env_width, z]

    def randomized_terrain(self):
        r = self.rng
        for k in range(self.num_maps):
            (i, j) = np.unravel_index(k, (self.env_rows, self.env_cols))
            t = self._new_tile()
            choice = r.uniform(0, 1)
            if choice < 0.1:
                if r.choice([0, 1]):
                    pyramid_sloped_terrain(t, r.choice([-0.3, -0.2, 0, 0.2, 0.3]))
                    random_uniform_terrain(t, min_height=-0.1, max_height=0.1, step=0.05, downsampled_scale=0.2, rng=r)
                else:
                    pyramid_sloped_terrain(t, r.choice([-0.3, -0.2, 0, 0.2, 0.3]))
            elif choice < 0.6:
                pyramid_stairs_terrain(t, step_width=0.31, step_height=r.choice([-0.15, 0.15]), platform_size=3.)
            elif choice < 1.:
                discrete_obstacles_terrain(t, 0.15, 1., 2., 40, platform_size=3., rng=r)
            self._place(t, i, j)

    def curiculum(self, num_robots, num_terrains, num_levels):
        r = self.rng
        for j in range(num_terrains):
            for i in range(num_levels):
                t = self._new_tile()
                difficulty = i / num_levels
                choice = j / num_terrains
                slope = difficulty * 0.4
                step_height = 0.05 + 0.175 * difficulty
                discrete_obstacles_height = 0.025 + difficulty * 0.15
                stepping_stones_size = 2 - 1.8 * difficulty
                if choice < self.proportions[0]:
                    if choice < 0.05:
                        slope *= -1
                    pyramid_sloped_terrain(t, slope=slope, platform_size=3.)
                elif choice < self.proportions[1]:
                    if choice < 0.15:
                        slope *= -1
                    pyramid_sloped_terrain(t, slope=slope, platform_size=3.)
                    random_uniform_terrain(t, min_height=-0.1, max_height=0.1, step=0.025, downsampled_scale=0.2, rng=r)
                elif choice < self.proportions[3]:
                    if choice < self.proportions[2]:
                        step_height *= -1
                    pyramid_stairs_terrain(t, step_width=0.31, step_height=step_height, platform_size=3.)
                elif choice < self.proportions[4]:
                    discrete_obstacles_terrain(t, discrete_obstacles_height, 1., 2., 40, platform_size=3., rng=r)
                else:
                    stepping_stones_terrain(t, stone_size=stepping_stones_size, stone_distance=0.1, max_height=0., platform_size=3., rng=r)
                self._place(t, i, j)


class HeightfieldMesh(np.ndarray):
    """Vertex / triangle array of a mesh built from a height field; remembers the samples and scales it came from, through
    `.flatten()` and slicing, so `gym.add_triangle_mesh` can hand the engine the height field itself."""

    def __new__(cls, arr, source=None):
        obj = np.asarray(arr).view(cls)
        obj.source = source
        return obj

    def __array_finalize__(self, obj):
        self.source = getattr(obj, "source", None)


def convert_heightfield_to_trimesh(height_field_raw, horizontal_scale, vertical_scale, slope_threshold=None):
    """isaacgym.terrain_utils.convert_heightfield_to_trimesh as its call site uses it (anymal_terrain.py:576): one vertex
    per sample at (i*hs, j*hs, h*vs), two triangles per cell; where the slope between neighbours exceeds `slope_threshold`
    the vertex on the low side is moved by one cell so that the step becomes a vertical wall.  Returns (vertices (n,3)
    float32, triangles (m,3) uint32), tagged with the source height field."""
    hf = np.asarray(height_field_raw)
    rows, cols = hf.shape
    y = np.linspace(0, (cols - 1) * horizontal_scale, cols)
    x = np.linspace(0, (rows - 1) * horizontal_scale, rows)
    yy, xx = np.meshgrid(y, x)
    if slope_threshold is not None:
        t = slope_threshold * horizontal_scale / vertical_scale
        move_x = np.zeros((rows, cols)); move_y = np.zeros((rows, cols)); move_c = np.zeros((rows, cols))
        move_x[:rows - 1, :] += (hf[1:, :] - hf[:rows - 1, :] > t)
        move_x[1:, :] -= (hf[:rows - 1, :] - hf[1:, :] > t)
        move_y[:, :cols - 1] += (hf[:, 1:] - hf[:, :cols - 1] > t)
        move_y[:, 1:] -= (hf[:, :cols - 1] - hf[:, 1:] > t)
        move_c[:rows - 1, :cols - 1] += (hf[1:, 1:] - hf[:rows - 1, :cols - 1] > t)
        move_c[1:, 1:] -= (hf[:rows - 1, :cols - 1] - hf[1:, 1:] > t)
        xx = xx + (move_x + move_c * (move_x == 0)) * horizontal_scale
        yy = yy + (move_y + move_c * (move_y == 0)) * horizontal_scale
    vertices = np.zeros((rows * cols, 3), dtype=np.float32)
    vertices[:, 0] = xx.flatten(); vertices[:, 1] = yy.flatten(); vertices[:, 2] = hf.flatten() * vertical_scale
    triangles = -np.ones((2 * (rows - 1) * (cols - 1), 3), dtype=np.uint32)
    for i in range(rows - 1):
        ind0 = np.arange(0, cols - 1) + i * cols
        ind1, ind2, ind3 = ind0 + 1, ind0 + cols, ind0 + cols + 1
        start, stop = 2 * i * (cols - 1), 2 * i * (cols - 1) + 2 * (cols - 1)
        triangles[start:stop:2, 0] = ind0; triangles[start:stop:2, 1] = ind3; triangles[start:stop:2, 2] = ind1
        triangles[start + 1:stop:2, 0] = ind0; triangles[start + 1:stop:2, 1] = ind2; triangles[start + 1:stop:2, 2] = ind3
    src = dict(height_field=np.ascontiguousarray(hf, dtype=np.int16), horizontal_scale=float(horizontal_scale),
               vertical_scale=float(vertical_scale))
    return HeightfieldMesh(vertices, src), HeightfieldMesh(triangles, src)


def trimesh_to_heightfield(vertices, triangles, horizontal_scale=None, vertical_scale=None, max_samples=8_000_000):
    """A general terrain mesh for `gym.add_triangle_mesh` (anymal_terrain.py:196-208 passes flat vertex / index arrays): the
    engine collides with height fields, so a mesh that is a terrain -- a surface z(x, y) over its bounding rectangle -- is
    sampled onto a regular grid (the highest surface point above each grid node; nodes no triangle covers get the lowest
    vertex).  Overhangs and caves are not representable and collapse to their upper surface.

    horizontal_scale: grid spacing; default = the 40th percentile of the mesh's horizontal edge lengths (a grid mesh has two
    axis-aligned edges for every diagonal; clipped to [0.02, 0.5] m), which
    reproduces a mesh made from a height field node for node.  vertical_scale: int16 quantum; default keeps the range within
    +-30000 quanta and is at most 1 mm.  Returns dict(height_field (nx, ny) int16, horizontal_scale, vertical_scale,
    offset (x0, y0) of sample (0, 0) in the mesh's own coordinates)."""
    v = np.asarray(vertices, dtype=np.float64).reshape(-1, 3)
    t = np.asarray(triangles).astype(np.int64).reshape(-1, 3)
    if len(t) == 0 or t.min() < 0 or t.max() >= len(v):
        raise ValueError("trimesh_to_heightfield: empty mesh or triangle index out of range")
    p = v[t]                                                       # (T, 3, 3)
    if horizontal_scale is None:
        e = np.concatenate([np.linalg.norm(p[:, a, :2] - p[:, b, :2], axis=1) for a, b in ((0, 1), (1, 2), (2, 0))])
        e = e[e > 1e-9]
        horizontal_scale = float(np.clip(np.round(np.percentile(e, 40), 6), 0.02, 0.5)) if len(e) else 0.1     # float32 vertices: 0.1 arrives as 0.10000001
    hs = float(horizontal_scale)
    x0, y0 = float(v[:, 0].min()), float(v[:, 1].min())
    nx = int(np.floor((v[:, 0].max() - x0) / hs + 1e-4)) + 1
    ny = int(np.floor((v[:, 1].max() - y0) / hs + 1e-4)) + 1
    if nx * ny > max_samples:
        raise ValueError(f"trimesh_to_heightfield: {nx} x {ny} samples at spacing {hs}; pass a coarser horizontal_scale")
    zlo = float(v[:, 2].min())
    H = np.full((nx, ny), -np.inf)
    # triangles in the order of their bounding-box size: the many small ones (a cell or two) are handled in bulk
    g = (p[:, :, :2] - np.array([x0, y0])) / hs                    # grid coordinates
    i0 = np.maximum(np.ceil(g[:, :, 0].min(1) - 1e-4).astype(np.int64), 0); i1 = np.minimum(np.floor(g[:, :, 0].max(1) + 1e-4).astype(np.int64), nx - 1)
    j0 = np.maximum(np.ceil(g[:, :, 1].min(1) - 1e-4).astype(np.int64), 0); j1 = np.minimum(np.floor(g[:, :, 1].max(1) + 1e-4).astype(np.int64), ny - 1)
    wi, wj = i1 - i0 + 1, j1 - j0 + 1
    ok = (wi > 0) & (wj > 0)
    a, b, c = g[:, 0], g[:, 1], g[:, 2]
    det = (b[:, 0] - a[:, 0]) * (c[:, 1] - a[:, 1]) - (c[:, 0] - a[:, 0]) * (b[:, 1] - a[:, 1])
    ok &= np.abs(det) > 1e-12                                      # vertical / degenerate triangles carry no height
    for di in range(int(wi[ok].max()) if ok.any() else 0):
        for dj in range(int(wj[ok].max())):
            sel = np.nonzero(ok & (wi > di) & (wj > dj))[0]
            if len(sel) == 0:
                continue
            gi, gj = i0[sel] + di, j0[sel] + dj
            px, py = gi - a[sel, 0], gj - a[sel, 1]
            l1 = (px * (c[sel, 1] - a[sel, 1]) - (c[sel, 0] - a[sel, 0]) * py) / det[sel]
            l2 = ((b[sel, 0] - a[sel, 0]) * py - px * (b[sel, 1] - a[sel, 1])) / det[sel]
            inside = (l1 >= -1e-4) & (l2 >= -1e-4) & (l1 + l2 <= 1 + 1e-4)         # nodes on an edge belong to both triangles
            z = p[sel, 0, 2] + l1 * (p[sel, 1, 2] - p[sel, 0, 2]) + l2 * (p[sel, 2, 2] - p[sel, 0, 2])
            np.maximum.at(H, (gi[inside], gj[inside]), z[inside])
    H[~np.isfinite(H)] = zlo
    zr = max(abs(float(H.max())), abs(float(H.min())), 1e-9)
    if vertical_scale is None:
        vertical_scale = min(1e-3, zr / 30000.0) if zr / 1e-3 <= 30000 else zr / 30000.0
    q = np.rint(H / vertical_scale)
    if np.abs(q).max() > 32767:
        raise ValueError("trimesh_to_heightfield: heights exceed the int16 range at this vertical_scale")
    return dict(height_field=np.ascontiguousarray(q.astype(np.int16)), horizontal_scale=hs, vertical_scale=float(vertical_scale),
                offset=(x0, y0))
