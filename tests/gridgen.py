"""Synthetic grids for the parity tests (numpy; small sizes).  All arrays are indexed [z, y, x]."""
import numpy as np


def _hash3(x, y, z, seed):
    h = (x.astype(np.uint64) * np.uint64(73856093)) ^ (y.astype(np.uint64) * np.uint64(19349663)) ^ \
        (z.astype(np.uint64) * np.uint64(83492791)) ^ np.uint64(seed * 2654435761 & 0xFFFFFFFF)
    h &= np.uint64(0xFFFFFFFF)
    h ^= h >> np.uint64(13); h = (h * np.uint64(0x5BD1E995)) & np.uint64(0xFFFFFFFF)
    h ^= h >> np.uint64(15); h = (h * np.uint64(0x27D4EB2F)) & np.uint64(0xFFFFFFFF)
    h ^= h >> np.uint64(16)
    return h


def sphere_floats(n, center=None, radius=None):
    c = (n / 2.0,) * 3 if center is None else center
    r = 0.3 * n if radius is None else radius
    z, y, x = np.meshgrid(np.arange(n, dtype=np.float32), np.arange(n, dtype=np.float32), np.arange(n, dtype=np.float32), indexing="ij")
    d = np.sqrt((x - c[0]) ** 2 + (y - c[1]) ** 2 + (z - c[2]) ** 2) - np.float32(r)
    return np.clip(d, -100, 100).astype(np.float32)


def hostile(n, seed=7, vmax=3, materials=3):
    """SURVEY.md Appendix C.3: wavy terrain + hash noise near the surface + forced zeros, hash materials/blends.
    Returns already-quantised int8 distances."""
    z, y, x = np.meshgrid(np.arange(n), np.arange(n), np.arange(n), indexing="ij")
    d = z - (n / 2.0 + 6 * np.sin(0.21 * x) * np.cos(0.17 * y) + 3 * np.sin(0.05 * (x + y)))
    return _hostile_band(x, y, z, d, seed, vmax, materials)


def _hostile_band(x, y, z, d, seed, vmax, materials):
    """hostile()'s content around the signed distance field d, at the voxel coordinates x, y, z."""
    q = (np.sign(d) * np.ceil(np.abs(d))).astype(np.int64)
    h = _hash3(x, y, z, seed)
    near = np.abs(d) < 6
    q = np.where(near, q + (h % np.uint64(2 * vmax + 1)).astype(np.int64) - vmax, q)
    q = np.where(near & ((h >> np.uint64(8)) % np.uint64(4) == 0), 0, q)
    lim = max(4, vmax + 1)
    q = np.clip(q, -lim, lim).astype(np.int8)
    hm = _hash3(x // 5, y // 5, z // 3, seed + 1)
    mat = (hm % np.uint64(materials)).astype(np.uint8)
    blend = ((h >> np.uint64(16)) & np.uint64(0xFF)).astype(np.uint8)
    return np.ascontiguousarray(q), np.ascontiguousarray(mat), np.ascontiguousarray(blend)


def noise_full(n, seed=3, lo=-5, hi=5):
    """Every voxel random in [lo, hi]: (almost) every cell non-trivial, worst case for counts."""
    z, y, x = np.meshgrid(np.arange(n), np.arange(n), np.arange(n), indexing="ij")
    h = _hash3(x, y, z, seed)
    q = (h % np.uint64(hi - lo + 1)).astype(np.int64) + lo
    mat = ((h >> np.uint64(10)) % np.uint64(4)).astype(np.uint8)
    blend = ((h >> np.uint64(20)) & np.uint64(0xFF)).astype(np.uint8)
    return np.ascontiguousarray(q.astype(np.int8)), np.ascontiguousarray(mat), np.ascontiguousarray(blend)


# ---- patchwork: every 16^3 block picks its own content, so a small grid mixes every kind of block ------------------
# NEG_RAW: inside (-4 / -3 per voxel), stored raw by the run-length coder, so never BF_Empty.  A uniform -4 block among
# uniform +4 ones would be skipped at level 0 (TransVoxelImpl.cpp:520) together with its neighbours, and the reference's
# coarse cells over it then read an uninitialised material (see skip_quirk): that configuration has its own grid.
UNI_POS, NEG_RAW, BAND, NOISE, VERTS, ZERO, BUBBLE, CHECKER = range(8)
KIND_NAMES = ("uniform+", "negative raw", "band", "noise", "vertex-heavy", "zero", "bubble", "checker")
_KIND_WEIGHTS = ((BAND, 28), (NOISE, 10), (VERTS, 12), (ZERO, 8), (BUBBLE, 14), (CHECKER, 14), (NEG_RAW, 14))
_BUBBLE_SPOTS = np.array([(0, 0, 0), (8, 8, 8), (0, 8, 4), (4, 12, 8), (2, 6, 10), (5, 9, 3), (15, 1, 7), (11, 13, 15)])  # (x, y, z)


def _noise_regions(nb):
    """(origin block (x, y, z), size in blocks) of the all-noise regions: one aligned to a level-1 / level-2 block, one not."""
    if nb == 4:
        return [((2, 0, 0), 2), ((1, 1, 2), 2)]
    nb2 = nb // 4
    return [((4 * (nb2 - 1), 0, 4 * (nb2 // 2)), 4), ((1, nb - 3, 1), 2)]


def patchwork_kinds(n, seed=1):
    """The kind of every 16^3 block, [bz, by, bx]: a seeded hash of the block coordinate, then the fixed placements
    (noise regions, non-uniform blocks on every face / edge / corner of the grid, a vertex-heavy block in the far corner)."""
    nb = n // 16
    assert nb >= 4 and n % 16 == 0
    bz, by, bx = np.meshgrid(np.arange(nb), np.arange(nb), np.arange(nb), indexing="ij")
    h = _hash3(bx, by, bz, seed)
    kinds = np.full((nb, nb, nb), UNI_POS, np.uint8)
    p = min(0.5, 120.0 / nb ** 2)  # bounded work at 1024^3: a few thousand non-uniform blocks
    nonuni = (h % np.uint64(10000)).astype(np.float64) < p * 10000
    w = ((h >> np.uint64(16)) % np.uint64(100)).astype(np.int64)
    lo = 0
    for kind, weight in _KIND_WEIGHTS:
        kinds[nonuni & (w >= lo) & (w < lo + weight)] = kind
        lo += weight
    fixed = np.zeros_like(nonuni)
    for (ox, oy, oz), size in _noise_regions(nb):
        kinds[oz:oz + size, oy:oy + size, ox:ox + size] = NOISE
        fixed[oz:oz + size, oy:oy + size, ox:ox + size] = True
    picks = (BAND, NOISE, CHECKER)
    for z in (0, nb // 2, nb - 1):
        for y in (0, nb // 2, nb - 1):
            for x in (0, nb // 2, nb - 1):
                if (x, y, z) == (nb // 2,) * 3 or fixed[z, y, x]:
                    continue
                kinds[z, y, x] = picks[int(h[z, y, x] >> np.uint64(24)) % 3]
                fixed[z, y, x] = True
    # a vertex-heavy block needs positive voxels on its 7 high neighbours' near faces (its cells stay <= 1024): the far
    # corner has no such neighbours; elsewhere the neighbours become uniform +4, or the block a band if one is fixed
    kinds[nb - 1, nb - 1, nb - 1] = VERTS
    fixed[nb - 1, nb - 1, nb - 1] = True
    verts = kinds == VERTS
    shifts = [(dz, dy, dx) for dz in (0, 1) for dy in (0, 1) for dx in (0, 1) if dz or dy or dx]

    def high_neighbours(mask):
        out = np.zeros_like(mask)
        for dz, dy, dx in shifts:
            out[dz:, dy:, dx:] |= mask[:nb - dz, :nb - dy, :nb - dx]
        return out

    def any_high_neighbour(mask):
        out = np.zeros_like(mask)
        for dz, dy, dx in shifts:
            out[:nb - dz, :nb - dy, :nb - dx] |= mask[dz:, dy:, dx:]
        return out

    blocked = verts & any_high_neighbour(fixed)
    kinds[blocked] = BAND
    verts &= ~blocked
    clear = high_neighbours(verts) & ~fixed
    kinds[clear] = UNI_POS
    return kinds


def _block_coords(bx, by, bz):
    l = np.arange(16)
    lz, ly, lx = np.meshgrid(l, l, l, indexing="ij")
    return (bx[:, None, None, None] * 16 + lx, by[:, None, None, None] * 16 + ly, bz[:, None, None, None] * 16 + lz, lx, ly, lz)


def _patch_content(kind, bx, by, bz, seed):
    """(dist, mat, blend) of a batch of blocks of one kind, each [B, 16, 16, 16] in [z, y, x] order."""
    x, y, z, lx, ly, lz = _block_coords(bx, by, bz)
    hb = _hash3(bx, by, bz, seed + 17)[:, None, None, None]
    shape = x.shape

    def const(v):
        return np.broadcast_to(np.asarray(v).astype(np.uint8), shape)

    if kind == NEG_RAW:  # 4096 runs: more than the 2048 run ends after which CompressBlock stores the block raw
        return (-4 + (x & 1)).astype(np.int8), const(1 + hb % np.uint64(3)), const((hb >> np.uint64(8)) & np.uint64(0xFF))
    if kind == ZERO:  # all zero: not BF_Empty, and every cell trivial
        return np.zeros(shape, np.int8), const(hb % np.uint64(4)), const((hb >> np.uint64(8)) & np.uint64(0xFF))
    if kind in (BAND, CHECKER):
        wave = 3 * np.sin(0.21 * x) * np.cos(0.17 * y) + 2 * np.sin(0.05 * (x + y))
        d = z - (bz[:, None, None, None] * 16 + 8 + wave)
        q, mat, blend = _hostile_band(x, y, z, d, seed + 3 * kind, 8 if kind == BAND else 2, 5)
        if kind == CHECKER:  # material checkerboards of 1- and 2-voxel cubes: the majority votes tie
            two = ((hb >> np.uint64(4)) & np.uint64(1)).astype(bool)
            parity = np.where(two, (x // 2 + y // 2 + z // 2) & 1, (x + y + z) & 1)
            mat = (1 + parity + 2 * (hb % np.uint64(2)).astype(np.int64)).astype(np.uint8)
        return q, mat, blend
    if kind == NOISE:  # (almost) every cell non-trivial: more than 1024 per block
        h = _hash3(x, y, z, seed + 5)
        q = ((h % np.uint64(11)).astype(np.int64) - 5).astype(np.int8)
        return q, ((h >> np.uint64(10)) % np.uint64(4)).astype(np.uint8), ((h >> np.uint64(20)) & np.uint64(0xFF)).astype(np.uint8)
    if kind == VERTS:  # sign checkerboard in the four low z layers: 1024 non-trivial cells, ~2900 new vertices
        h = _hash3(x, y, z, seed + 7)
        mag = 1 + (h % np.uint64(4)).astype(np.int64)
        q = np.where(lz < 4, np.where((x + y + z) & 1, mag, -mag), 4).astype(np.int8)
        return q, const(hb % np.uint64(3)), ((h >> np.uint64(8)) & np.uint64(0xFF)).astype(np.uint8)
    if kind == BUBBLE:  # +4 with one negative and one zero voxel, on and off the 2^L strides
        q = np.full(shape, 4, np.int8)
        k = np.arange(len(bx))
        a = _BUBBLE_SPOTS[(hb[:, 0, 0, 0] % np.uint64(8)).astype(np.int64)]
        b = _BUBBLE_SPOTS[((hb[:, 0, 0, 0] >> np.uint64(3)) % np.uint64(7) + np.uint64(1) + (hb[:, 0, 0, 0] % np.uint64(8))).astype(np.int64) % 8]
        q[k, a[:, 2], a[:, 1], a[:, 0]] = -(1 + ((hb[:, 0, 0, 0] >> np.uint64(6)) % np.uint64(4)).astype(np.int64))
        q[k, b[:, 2], b[:, 1], b[:, 0]] = 0
        return q, const(hb % np.uint64(5)), const((hb >> np.uint64(8)) & np.uint64(0xFF))
    raise ValueError(kind)


def patchwork(n, seed=1):
    """A hostile grid made of 16^3 patches (kinds: patchwork_kinds), deterministic.  Only the non-uniform blocks are
    generated, a batch of one kind at a time, straight into the three output arrays ([z, y, x])."""
    nb = n // 16
    kinds = patchwork_kinds(n, seed)
    dist = np.full((n, n, n), 4, np.int8)
    mat = np.zeros((n, n, n), np.uint8)
    blend = np.zeros((n, n, n), np.uint8)
    views = [a.reshape(nb, 16, nb, 16, nb, 16) for a in (dist, mat, blend)]
    for kind in range(1, len(KIND_NAMES)):
        where = np.argwhere(kinds == kind)
        for s in range(0, len(where), 256):
            bz, by, bx = (where[s:s + 256, i].astype(np.int64) for i in range(3))
            for view, part in zip(views, _patch_content(kind, bx, by, bz, seed)):
                view[bz, :, by, :, bx, :] = part
    return dist, mat, blend


def nontrivial_cells_per_block(dist, level):
    """Non-trivial cells (corner signs differ) of every level-`level` block, [bz, by, bx]: corners sampled at stride
    2^level, coordinates clamped to n - 1 as the kernels and the reference do at the far edge."""
    n = dist.shape[0]
    m = 1 << level
    k = n // m
    at = np.minimum(np.arange(k + 1) * m, n - 1)
    neg = dist[np.ix_(at, at, at)] < 0
    any_, all_ = np.zeros((k, k, k), bool), np.ones((k, k, k), bool)
    for dz in (0, 1):
        for dy in (0, 1):
            for dx in (0, 1):
                c = neg[dz:dz + k, dy:dy + k, dx:dx + k]
                any_ |= c
                all_ &= c
    nb = k // 16
    return (any_ & ~all_).reshape(nb, 16, nb, 16, nb, 16).sum(axis=(1, 3, 5))


def edge_edit_sequence(n, count, seed=5):
    """Sphere edits (integer centre, radius, extent = 2 r + 4, add?) whose boxes touch a face, an edge or a corner of the
    grid in turn and stay inside [0, n]: the clipped ranges of an incremental run at the grid's edge."""
    rng = np.random.RandomState(seed)
    out = []
    for i in range(count):
        r = int(rng.choice([4, 6, 8]))
        half = r + 2
        pos = [int(v) for v in rng.randint(half, n - half + 1, size=3)]
        for axis in rng.permutation(3)[:1 + i % 3]:   # 1, 2, 3 axes at the edge: face, edge, corner
            pos[axis] = half if rng.randint(2) else n - half
        out.append((pos, float(r), float(2 * half), i % 2 == 0))
    return out


def skip_quirk(n=64):
    """+4 everywhere but a few uniform -4 blocks whose 27-neighbourhoods hold only uniform (BF_Empty) blocks, and one
    band block elsewhere.  The reference skips those level-0 blocks although the surface runs along their faces
    (TransVoxelImpl.cpp:520); its coarse cells over them have no child with a material and read an uninitialised
    Cell::Material (:1052-1086), so only level 0 and the statistics are defined there."""
    assert n == 64
    dist = np.full((n, n, n), 4, np.int8)
    mat = np.zeros((n, n, n), np.uint8)
    blend = np.zeros((n, n, n), np.uint8)
    for bx, by, bz, m in ((1, 1, 1, 2), (2, 2, 2, 3), (3, 0, 3, 1)):
        dist[bz * 16:bz * 16 + 16, by * 16:by * 16 + 16, bx * 16:bx * 16 + 16] = -4
        mat[bz * 16:bz * 16 + 16, by * 16:by * 16 + 16, bx * 16:bx * 16 + 16] = m
    bx = np.array([0]); by = np.array([3]); bz = np.array([0])
    for a, part in zip((dist, mat, blend), _patch_content(BAND, bx, by, bz, 1)):
        a[0:16, 48:64, 0:16] = part[0]
    return dist, mat, blend
