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


def hostile_full_range(n, seed=13, materials=5):
    """hostile()'s wavy surface with distances over the whole int8 range: the field saturates at -128 / 127 a few voxels
    off the surface, the band adds noise of +-100 and forced zeros, and (-128, 127) / (127, -128) pairs sit on cell edges
    along x, y and z.  The values are clipped to [-128, 127] before the cast (no wrap of 128 to -128)."""
    z, y, x = np.meshgrid(np.arange(n), np.arange(n), np.arange(n), indexing="ij")
    d = z - (n / 2.0 + 6 * np.sin(0.21 * x) * np.cos(0.17 * y) + 3 * np.sin(0.05 * (x + y)))
    h = _hash3(x, y, z, seed)
    q = (np.sign(d) * np.ceil(np.abs(24 * d))).astype(np.int64)
    near = np.abs(d) < 6
    q = np.where(near, q + (h % np.uint64(201)).astype(np.int64) - 100, q)
    q = np.where(near & ((h >> np.uint64(8)) % np.uint64(4) == 0), 0, q)
    q = np.clip(q, -128, 127)
    for axis, bit in ((0, 12), (1, 16), (2, 20)):   # z, y, x pairs: voxel v and its +1 neighbour along the axis
        pick = near & ((h >> np.uint64(bit)) % np.uint64(8) == 0)
        pick &= (np.stack([z, y, x])[axis] % 2 == 0) & (np.stack([z, y, x])[axis] < n - 1)
        lo = np.where((h >> np.uint64(bit + 3)) & np.uint64(1), -128, 127)
        src = np.argwhere(pick)
        dst = src.copy(); dst[:, axis] += 1
        q[tuple(src.T)] = lo[pick]
        q[tuple(dst.T)] = np.where(lo[pick] == -128, 127, -128)
    hm = _hash3(x // 5, y // 5, z // 3, seed + 1)
    mat = (hm % np.uint64(materials)).astype(np.uint8)
    blend = ((h >> np.uint64(24)) & np.uint64(0xFF)).astype(np.uint8)
    return np.ascontiguousarray(q.astype(np.int8)), np.ascontiguousarray(mat), np.ascontiguousarray(blend)


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


# ---- rle_edges: the run-length thresholds of the grid store -------------------------------------------------------------
# CompressBlock (VoxelGrid.cpp:610-672) ends a run at a value change or after 255 bytes and stores a channel raw once 2048
# run ends were seen, i.e. at 2049 runs or more; BF_Empty = run-length coded and every voxel of one strict sign.  The
# kernels decide BF_Empty from the scan's count of value changes inside the 16-byte rows (x): with 2048 or more the block
# is raw, below 1777 it cannot reach 2049 runs (at most 255 row seams + 16 splits + 1 more), and in between
# vxb_block_info_kernel walks the block (vxb_kernels.cuh).  Block contents below are [z, y, x] = 4096 bytes in
# CompressBlock's order (x fastest).

def runs_of(flat):
    """CompressBlock's run count of 4096 bytes: maximal runs of one value, each cut every 255 bytes."""
    flat = np.asarray(flat)
    ends = np.flatnonzero(flat[1:] != flat[:-1]) + 1
    lengths = np.diff(np.concatenate([[0], ends, [flat.size]]))
    return int(((lengths + 254) // 255).sum())


def inrow_changes(flat):
    """The scan's count: adjacent bytes that differ inside the 16-byte rows (row seams not counted)."""
    rows = np.asarray(flat).reshape(-1, 16)
    return int((rows[:, 1:] != rows[:, :-1]).sum())


def _from_runs(values, lengths):
    out = np.repeat(np.asarray(values, np.int64), np.asarray(lengths, np.int64))
    assert out.size == 4096, out.size
    return out


def _pairs(a, b):
    """a a b b a a b b ...: 2048 runs of 2, 1792 in-row changes (7 per row) + 255 changes at the row seams."""
    return np.where((np.arange(4096) // 2) % 2 == 0, a, b).astype(np.int64)


def _with_split_runs(a, b, runs):
    """510 bytes of a (two runs: one 255-byte cut), then `runs` - 2 runs alternating b, a, ...: first runs of 1 byte,
    then of 2, as many of each as fill the other 3586 bytes."""
    k = runs - 2
    ones = 2 * k - 3586
    return _from_runs([a] + [b, a] * (k // 2) + [b] * (k % 2), [510] + [1] * ones + [2] * (k - ones))


def _threshold_block(kind, s):
    """One threshold block's distance bytes (int8), of sign s: values s, 2s and 3s, or a zero."""
    a, b, c = s, 2 * s, 3 * s
    v = _pairs(a, b)
    if kind == "runs2047":
        v[4092:] = a                                       # the last pair joins the one before: 2047 runs
    elif kind == "runs2048":
        pass
    elif kind == "runs2049":
        v[1] = c                                           # a c b b ...: one more run end
    elif kind in ("inrow1776", "inrow1777"):
        rows = v.reshape(256, 16)
        rows[:1792 - int(kind[5:]), 14:] = rows[:1792 - int(kind[5:]), 13:14]   # the row's last change goes
    elif kind in ("inrow2047", "inrow2048"):
        rows = v.reshape(256, 16)
        full = 32 if kind == "inrow2048" else 31
        rows[:full] = np.where(np.arange(16) % 2 == 0, a, b)   # 15 in-row changes instead of 7
        if kind == "inrow2047":
            rows[31] = np.where(np.arange(16) % 2 == 0, a, b); rows[31, 15] = rows[31, 14]   # 14
    elif kind in ("split2048", "split2049"):
        v = _with_split_runs(a, b, int(kind[5:]))
    elif kind == "zero_first":
        v[0] = 0
    elif kind == "zero_last":
        v[4095] = 0
    elif kind == "uniform":
        v[:] = -128 if s < 0 else 127
    else:
        raise ValueError(kind)
    return v.astype(np.int8)


# not BF_Empty (nothing of rle_edges_kept is skipped) / BF_Empty (rle_edges_skipped), each as a -1/-2 block among +4 ones
# and a +1/+2 block on the low x side of a uniform -4 block
KEPT_VARIANTS = ("runs2049", "inrow2047", "inrow2048", "split2049", "zero_first", "zero_last")
SKIPPED_VARIANTS = ("runs2047", "runs2048", "inrow1776", "inrow1777", "split2048")
_SKIPPED_EXTRA = [("uniform", -1), ("uniform", 1)]


def _channel_variant(kind, lo, hi):
    """A material / blend channel at a run-length threshold, values lo / hi (uint8)."""
    if kind in ("runs2047", "runs2048", "runs2049"):
        v = _threshold_block(kind, 1)
        return np.select([v == 1, v == 2], [lo, hi], lo ^ hi)
    if kind == "seams":   # runs of exactly 255, 256, 510 and 511 bytes, starting off the row seams (+ 1- and 3-byte fillers)
        lengths, values, total, i = [], [], 0, 0
        cycle = (7, 255, 256, 1, 510, 3, 511)
        while total < 4096:
            L = min(cycle[i % len(cycle)], 4096 - total)
            lengths.append(L); values.append((lo, hi, (lo + 1) & 0xFF)[i % 3]); total += L; i += 1
        return _from_runs(values, lengths)
    return np.full(4096, {"uniform0": 0, "uniform80": 0x80, "uniformFF": 0xFF}[kind])


CHANNEL_VARIANTS = ("runs2047", "runs2048", "runs2049", "seams", "uniform0", "uniform80", "uniformFF")


def _thresholds(variants, extra):
    slots = [(x, y, z) for z in (0, 3, 6) for y in (0, 3, 6) for x in (0, 3)]
    placed = [(kind, s) for kind in variants for s in (-1, 1)] + list(extra)
    assert len(placed) <= len(slots)
    return [(kind, s, slot) for (kind, s), slot in zip(placed, slots)]


def rle_edges_thresholds(name):
    """(variant, sign, (bx, by, bz)) of every threshold block of rle_edges_kept / rle_edges_skipped."""
    if name == "rle_edges_kept":
        return _thresholds(KEPT_VARIANTS, [])
    assert name == "rle_edges_skipped", name
    return _thresholds(SKIPPED_VARIANTS, _SKIPPED_EXTRA)


def _rle_edges(n, variants, extra):
    """Threshold blocks T on the slots x in {0, 3}, y and z in {0, 3, 6}: three blocks apart, so that the level-0 skip of T
    and its 26 neighbours depends on T's flag alone (a block with non-trivial cells is within one block of its T).  The
    material / blend threshold channels fill the blocks with x >= 6, more than a block away from every surface, so that no
    cell ever reads them (their materials include 255, EMPTY_MATERIAL) and they only meet the codec."""
    assert n == 128
    nb = n // 16
    dist = np.full((n, n, n), 4, np.int8)
    mat = np.zeros((n, n, n), np.uint8)
    blend = np.zeros((n, n, n), np.uint8)

    def put(a, bx, by, bz, flat):
        a[bz * 16:bz * 16 + 16, by * 16:by * 16 + 16, bx * 16:bx * 16 + 16] = np.asarray(flat).reshape(16, 16, 16)

    l = np.arange(16)
    lz, ly, lx = np.meshgrid(l, l, l, indexing="ij")
    for k, (kind, s, (bx, by, bz)) in enumerate(_thresholds(variants, extra)):
        put(dist, bx, by, bz, _threshold_block(kind, s))
        h = _hash3(lx + 16 * bx, ly + 16 * by, lz + 16 * bz, 29 + k)
        put(mat, bx, by, bz, (1 + (_hash3(lx // 4, ly // 4, lz // 4, k) % np.uint64(3))).astype(np.uint8))
        put(blend, bx, by, bz, (h & np.uint64(0xFF)).astype(np.uint8))
        if s > 0:   # the surface along T's high x face: a uniform -4 block there
            put(dist, bx + 1, by, bz, np.full(4096, -4))
            put(mat, bx + 1, by, bz, np.full(4096, 2))
    k = 0
    for bz in range(nb):
        for by in range(nb):
            for bx in (6, 7):
                if k < len(CHANNEL_VARIANTS) ** 2:
                    mv, bv = CHANNEL_VARIANTS[k % len(CHANNEL_VARIANTS)], CHANNEL_VARIANTS[k // len(CHANNEL_VARIANTS)]
                    put(mat, bx, by, bz, _channel_variant(mv, 1, 2))
                    put(blend, bx, by, bz, _channel_variant(bv, 0x7F, 0x80))
                k += 1
    return dist, mat, blend


def rle_edges_kept(n=128):
    """Threshold blocks that are not BF_Empty: 2049 runs found by the walk, 2047 in-row changes (walked) and 2048 (raw
    without a walk), 2049 runs with 255-byte cuts, a single 0 as the first / last byte.  Nothing is skipped at level 0,
    so every level is defined in the reference."""
    return _rle_edges(n, KEPT_VARIANTS, [])


def rle_edges_skipped(n=128):
    """Threshold blocks that are BF_Empty: 2047 / 2048 runs found by the walk, 1776 (not walked) / 1777 (walked) in-row
    changes, 2048 runs with 255-byte cuts, uniform -128 and uniform 127.  The reference skips them with their neighbours
    although the surface runs along their faces; like skip_quirk, its coarse levels are then undefined."""
    return _rle_edges(n, SKIPPED_VARIANTS, _SKIPPED_EXTRA)


# ---- thresholds256: the per-block capacities of the block kernels, rung by rung ------------------------------------------
# VxbBlockCaps (voxels_b200/csrc/vxb_emit.cuh): a block of vxb_block_kernel<0|1|2> holds at most CAP = 1024 non-trivial
# cells and, at level 0, VL = 2048 new vertices in shared memory; past either it goes to vxb_big_block_kernel.  Every
# ladder block below sits at an exact count on either side of those capacities (and of half of them).
#
# A +4 background; each ladder block is stamped on its level's lattice (stride 2^level, local coordinates 0..16):
#   - isolated negative samples at odd local coordinates, x in {11, 13, 15}: 8 cells each, disjoint;
#   - diagonal pairs u, u + (1, 1, 1) with u in {1, 5} x {12} x {1, 5, 9, 13}: 15 cells each (the shared cell counts once),
#     so that 8 k + 15 p reaches every count;
#   - (level 0) a +-2 checkerboard filled in raster order (z, y, x) over local [1, 9] x [1, 9] x [1, 15], negative where
#     x + y + z is odd: about 2.2 vertices per cell.
# All of it lies in local 1..15, so a block's content changes no other block's cells at its level, and every negative
# sample has an odd grid coordinate at the level below, so level-0 content is invisible to level 1 and level-1 content to
# level 2 (a level-l sample is a sample of every finer level, where it adds isolated-sample cells to the blocks under it).
# The one exception is the 4096-cell block: a checkerboard over all of local 0..15, whose low face adds cells to its low
# neighbours (plain background blocks).  Materials and blends are hashed over the whole grid as in hostile(), so vertex
# reuse across cells of different materials (TransVoxelImpl.cpp:1611-1619) shapes the vertex counts: the parameters below
# were found by a search with the reference's per-block vertex count as the judge, and are checked by
# tests/test_thresholds_cpu.py.

TH_N = 256
_TH_SEED = 41
_TH_BOX = (9, 9, 15)                            # checkerboard extents (x, y, z) from local (1, 1, 1)
_TH_ISO = [(x, y, z) for x in (11, 13, 15) for z in range(1, 16, 2) for y in range(1, 16, 2)]
_TH_PAIRS = [(x, 12, z) for z in (1, 5, 9, 13) for x in (1, 5)]

# name -> (level, block (bx, by, bz) at that level, (content, cells, vertices) of variant A, the same of variant B or None).
# Content = (m, k, o, p): the first m samples of the checkerboard, k isolated samples _TH_ISO[o:o + k] and p diagonal pairs
# _TH_PAIRS[:p]; "full" is the 4096-cell checkerboard.  Vertices = the reference's per-block vertex count, None where the
# rung is a cell count only (those blocks stay far below 2048 vertices).  Variant B of a flip pair differs from A only in
# local 1..15 of its block.
TH_BLOCKS = {
    # level 0 (vxb_block_kernel<0>), non-trivial cells
    "L0_cells255": (0, (12, 12, 12), ((0, 30, 0, 1), 255, None), None),
    "L0_cells256": (0, (13, 12, 12), ((0, 32, 0, 0), 256, None), None),
    "L0_cells257": (0, (14, 12, 12), ((0, 19, 0, 7), 257, None), None),
    "L0_cells511": (0, (15, 12, 12), ((0, 62, 0, 1), 511, None), None),
    "L0_cells512": (0, (12, 13, 12), ((0, 64, 0, 0), 512, None), None),
    "L0_cells513": (0, (13, 13, 12), ((0, 51, 0, 7), 513, None), None),
    "L0_cells1023": (0, (14, 13, 12), ((0, 126, 0, 1), 1023, None), None),
    "L0_cells1024": (0, (15, 13, 12), ((0, 128, 0, 0), 1024, None), ((0, 115, 0, 7), 1025, None)),
    "L0_cells1025": (0, (12, 14, 12), ((0, 115, 0, 7), 1025, None), None),
    "L0_cells4096": (0, (13, 1, 1), ("full", 4096, None), None),
    # level 0, new vertices with at most 1024 cells
    "L0_verts1023": (0, (14, 12, 13), ((199, 1, 0, 0), 357, 1023), None),
    "L0_verts1024": (0, (13, 13, 13), ((201, 0, 0, 0), 351, 1024), None),
    "L0_verts1025": (0, (15, 12, 13), ((187, 1, 0, 0), 343, 1025), None),
    "L0_verts2047": (0, (12, 12, 13), ((441, 5, 12, 0), 688, 2047), None),
    "L0_verts2048": (0, (14, 14, 13), ((381, 2, 16, 0), 587, 2048), ((375, 5, 8, 0), 604, 2049)),
    "L0_verts2049": (0, (13, 14, 13), ((373, 2, 0, 0), 578, 2049), None),
    # level 0, both capacities: both arrays full / one vertex past a full cell list / one cell past, vertices full
    "L0_cells1024_verts2048": (0, (14, 13, 14), ((133, 93, 4, 1), 1024, 2048), ((125, 96, 0, 0), 1024, 2049)),
    "L0_cells1024_verts2049": (0, (13, 12, 13), ((235, 68, 4, 6), 1024, 2049), None),
    "L0_cells1025_verts2048": (0, (14, 13, 13), ((151, 85, 0, 4), 1025, 2048), None),
    # level 1 (vxb_block_kernel<1>) and level 2, the first coarse level of 256^3 (vxb_block_kernel<2>): non-trivial cells
    "L1_cells511": (1, (2, 2, 2), ((0, 62, 0, 1), 511, None), None),
    "L1_cells512": (1, (3, 2, 2), ((0, 64, 0, 0), 512, None), None),
    "L1_cells513": (1, (2, 3, 2), ((0, 51, 0, 7), 513, None), None),
    "L1_cells1023": (1, (3, 3, 2), ((0, 126, 0, 1), 1023, None), None),
    "L1_cells1024": (1, (2, 2, 3), ((0, 128, 0, 0), 1024, None), ((0, 115, 0, 7), 1025, None)),
    "L1_cells1025": (1, (3, 2, 3), ((0, 115, 0, 7), 1025, None), None),
    "L2_cells511": (2, (0, 0, 0), ((0, 62, 0, 1), 511, None), None),
    "L2_cells512": (2, (2, 0, 0), ((0, 64, 0, 0), 512, None), None),
    "L2_cells513": (2, (0, 2, 0), ((0, 51, 0, 7), 513, None), None),
    "L2_cells1023": (2, (2, 2, 0), ((0, 126, 0, 1), 1023, None), None),
    "L2_cells1024": (2, (0, 0, 2), ((0, 128, 0, 0), 1024, None), ((0, 115, 0, 7), 1025, None)),
    "L2_cells1025": (2, (2, 0, 2), ((0, 115, 0, 7), 1025, None), None),
}
TH_FLIPS = tuple(name for name, spec in TH_BLOCKS.items() if spec[3] is not None)


def th_channels(x, y, z):
    """(material, blend) at grid coordinates, hashed as in hostile(): materials in 5 x 5 x 3 voxel patches."""
    hm = _hash3(x // 5, y // 5, z // 3, _TH_SEED + 1)
    h = _hash3(x, y, z, _TH_SEED)
    return (hm % np.uint64(4)).astype(np.uint8), ((h >> np.uint64(16)) & np.uint64(0xFF)).astype(np.uint8)


def th_content(level, content, origin):
    """The negative / checkerboard samples of one ladder block: [(x, y, z) grid coordinates], [values]."""
    s = 1 << level
    ox, oy, oz = origin
    pts, vals = [], []
    if content == "full":
        for z in range(16):
            for y in range(16):
                for x in range(16):
                    pts.append((x, y, z)); vals.append(-2 if (x + y + z) & 1 else 2)
    else:
        m, k, o, p = content
        bx, by, bz = _TH_BOX
        box = [(x, y, z) for z in range(1, bz + 1) for y in range(1, by + 1) for x in range(1, bx + 1)]
        for x, y, z in box[:m]:
            pts.append((x, y, z)); vals.append(-2 if (x + y + z) & 1 else 2)
        for x, y, z in _TH_ISO[o:o + k]:
            pts.append((x, y, z)); vals.append(None)
        for x, y, z in _TH_PAIRS[:p]:
            pts += [(x, y, z), (x + 1, y + 1, z + 1)]; vals += [None, None]
    g = np.array([(ox + s * x, oy + s * y, oz + s * z) for x, y, z in pts], np.int64).reshape(-1, 3)
    h = _hash3(g[:, 0], g[:, 1], g[:, 2], _TH_SEED + 2)
    v = np.array([-1 - int(hh % np.uint64(4)) if val is None else val for val, hh in zip(vals, h)], np.int64)
    return g, v


def th_stamp(dist, level, block, content):
    """Writes one ladder block's content into dist ([z, y, x]) over a +4 background."""
    m = 16 << level
    g, v = th_content(level, content, tuple(b * m for b in block))
    dist[g[:, 2], g[:, 1], g[:, 0]] = v


def th_restamp(dist, name, variant_b):
    """A copy of a thresholds256 distance array with block `name` (a flip pair) in variant B (or back in A)."""
    level, block, a, b = TH_BLOCKS[name]
    m = 16 << level
    out = dist.copy()
    out[tuple(slice(v * m + 1, v * m + m) for v in reversed(block))] = 4
    th_stamp(out, level, block, (b if variant_b else a)[0])
    return out


def thresholds256(variant=None):
    """The ladder grid, every block in variant A; `variant` = name of a flip pair whose block takes variant B."""
    n = TH_N
    dist = np.full((n, n, n), 4, np.int8)
    for name, (level, block, a, b) in TH_BLOCKS.items():
        th_stamp(dist, level, block, (b if name == variant else a)[0])
    z, y, x = np.meshgrid(np.arange(n), np.arange(n), np.arange(n), indexing="ij")
    mat, blend = th_channels(x, y, z)
    return dist, np.ascontiguousarray(mat), np.ascontiguousarray(blend)
