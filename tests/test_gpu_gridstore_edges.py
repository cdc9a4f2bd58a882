"""The grid store around the polygonizer at its exact integer thresholds, against the unmodified reference grid store:

  - the empty-block rule: vxb_block_info_kernel decides BF_Empty from the scan's in-row change count and walks a
    one-signed block whose count lies in [1777, 2047] (CompressBlock's "raw at 2049 runs"); the level-0 skip reads that
    flag, so an off-by-one adds or drops whole level-0 blocks (gridgen.rle_edges_kept / rle_edges_skipped; with virtual
    ranks: test_gpu_sharded.test_virtual_ranks_equal_single_run);
  - the run-length codec at 2048 / 2049 runs and with blobs that Grid::Load accepts but PackForSave never writes (zero-length
    runs, adjacent runs of one value, one value in 64 and 65 runs: either side of the decoder's single-value shortcut);
  - the full-size codec paths: more than 1024 blocks per prefix sum, the 4- and 8-slab (streamed) packed uploads, 1024^3;
  - edits that take distances to +-100 with plane and terrain surfaces, odd extents and boxes outside the grid, then the
    pack and the polygonizer on the edited grid.
The codec at the thresholds on the small grids is test_gpu_gridstore.test_pack_equals_reference_pack_for_save."""
import numpy as np
import pytest

import compare
import golden_hash
import gridgen
import grids
from parity import run_both, run_skipping_grid
from test_gpu_gridstore import assert_dense_equal
from test_gpu_paths import _context

pytestmark = pytest.mark.gpu

HEAD = 16   # version, w, d, h; then the size table (3 x u32 per block), then per block {flags, distance, material, blend}


def _blob_equal(got, want, what):
    assert len(got) == len(want), "%s: blob size %d vs %d" % (what, len(got), len(want))
    if not np.array_equal(got, want):
        bad = np.nonzero(got != want)[0]
        raise AssertionError("%s: blob differs at %d bytes, first offset %d" % (what, len(bad), bad[0]))


def _dense_equal(want, got, what):
    for a, b, ch in zip(want, got, ("distance", "material", "blend")):
        if not np.array_equal(a, b):
            bad = np.argwhere(a != b)
            raise AssertionError("%s: %s differs at %d voxels, first (z,y,x)=%s: want %d, got %d"
                                 % (what, ch, len(bad), bad[0], a[tuple(bad[0])], b[tuple(bad[0])]))


# ---- the empty-block rule ------------------------------------------------------------------------------------------

@pytest.mark.parametrize("limit", (0, 1, 2))
def test_rle_edges_kept_all_levels(reference, limit):
    """Threshold blocks that are not BF_Empty (2049 runs found by the walk, raw without a walk, a zero at either end):
    nothing is skipped, so every level and the statistics must equal the reference."""
    dist, mat, blend = gridgen.rle_edges_kept()
    ctx = _context(limit)
    try:
        problems, res = run_both(reference, ctx, dist, mat, blend)
        assert not problems, ("launch limit %d:\n" % limit) + "\n".join(problems[:10])
    finally:
        ctx.close()


@pytest.mark.parametrize("limit", (0, 2))
def test_rle_edges_skipped_against_reference_and_restatement(reference, restatement, limit):
    """BF_Empty threshold blocks (2047 / 2048 runs found by the walk, 1776 / 1777 in-row changes, uniform -128 / 127) are
    skipped at level 0 with their neighbours: parity.run_skipping_grid."""
    dist, mat, blend = gridgen.rle_edges_skipped()
    ctx = _context(limit)
    try:
        problems = run_skipping_grid(reference, restatement, ctx, dist, mat, blend)
        assert not problems, "\n".join(problems[:10])
    finally:
        ctx.close()


# ---- valid blobs that PackForSave never writes ---------------------------------------------------------------------

def _rle(values, lengths):
    out = np.empty(2 * len(values), np.uint8)
    out[0::2] = lengths
    out[1::2] = np.asarray(values).astype(np.int64) & 0xFF
    assert int(np.asarray(lengths).sum()) == 4096
    return out


def _noncanonical_channels():
    """(name, stored bytes, raw?) of channels Grid::Load accepts, whose bytes CompressBlock would code differently."""
    out = []
    # zero-length runs: first, in between (between equal and between different values) and last
    lengths, values = [0], [9]
    for i in range(40):
        lengths += [100, 0]; values += [(i % 3) + 1, 7 if i % 2 else (i % 3) + 1]
    lengths += [96, 0]; values += [2, 5]
    out.append(("zero-length runs", _rle(values, lengths), False))
    out.append(("adjacent runs of one value", _rle([3] * 16 + [1] * 16, [128] * 32), False))
    out.append(("one value in 64 runs", _rle([2] * 64, [64] * 64), False))                      # the single-value shortcut
    out.append(("one value in 65 runs", _rle([2] * 65, [63] * 64 + [64]), False))               # just past it: decoded
    out.append(("one value in 65 runs with zero-length ones", _rle([1] * 65, [0] + [64] * 64), False))
    out.append(("2048 runs of one value (4096 bytes, raw flag clear)", _rle([1] * 2048, [2] * 2048), False))
    alt = np.where(np.arange(2048) % 2 == 0, 1, 2)
    out.append(("2048 runs (4096 bytes, raw flag clear)", _rle(alt, [2] * 2048), False))
    out.append(("raw", (np.arange(4096) * 7 % 5 + 1).astype(np.uint8), True))
    return out


def _decode(stored, raw):
    if raw:
        return stored.copy()
    return np.repeat(stored[1::2], stored[0::2].astype(np.int64))


def _noncanonical_blob(n=32):
    """A blob of (n/16)^3 blocks whose three channels cycle through _noncanonical_channels (and a negated distance copy),
    with every flags word what CompressBlock gives for the decoded bytes; returns (blob, [dist, mat, blend])."""
    chans = _noncanonical_channels()
    nb = n // 16
    blocks = nb ** 3
    sizes, data = [], []
    dense = [np.zeros((n, n, n), np.int8), np.zeros((n, n, n), np.uint8), np.zeros((n, n, n), np.uint8)]
    for b in range(blocks):
        bx, by, bz = b % nb, (b // nb) % nb, b // (nb * nb)
        picks = [chans[(b + 3 * ch) % len(chans)] for ch in range(3)]
        if b % 2:   # negative distances: one-signed blocks of both signs
            name, stored, raw = picks[0]
            stored = stored.copy()
            if raw:
                stored = (-stored.astype(np.int8)).astype(np.uint8)
            else:
                stored[1::2] = (-stored[1::2].astype(np.int8)).astype(np.uint8)
            picks[0] = (name, stored, raw)
        flags = 0
        for ch, (name, stored, raw) in enumerate(picks):
            flat = _decode(stored, raw)
            dense[ch][bz * 16:bz * 16 + 16, by * 16:by * 16 + 16, bx * 16:bx * 16 + 16] = flat.view(dense[ch].dtype).reshape(16, 16, 16)
            runs = gridgen.runs_of(flat)
            assert raw == (runs > 2048), name   # stored raw exactly when CompressBlock stores it raw
            if raw:
                flags |= 2 << ch
            v = flat.view(np.int8)
            if ch == 0 and not raw and ((v > 0).all() or (v < 0).all()):
                flags |= 1
            sizes.append(stored.size)
        data.append(np.frombuffer(np.uint32(flags).tobytes(), np.uint8))
        data += [p[1] for p in picks]
    head = np.array([1, n, n, n], np.uint32).view(np.uint8)
    blob = np.concatenate([head, np.array(sizes, np.uint32).view(np.uint8)] + data)
    return blob, dense


def test_noncanonical_blobs_decode_like_grid_load(reference, gpu_context):
    blob, dense = _noncanonical_blob()
    g = reference.grid_load(blob)
    assert g is not None, "Grid::Load refused the blob"
    try:
        want = reference.grid_to_dense(g)
        _dense_equal(dense, want, "the test's own decode vs Grid::Load")
        gpu_context.upload_packed(blob)
        _dense_equal(want, gpu_context.download_dense(), "vxb_grid_upload_packed vs Grid::Load")
        # and the polygonizer on the decoded grid (the flags were set the way CompressBlock sets them)
        s, _ = reference.polygonize(g)
        gpu_context.set_materials(None, None)
        gpu_context.polygonize()
        res = gpu_context.download()
        problems = []
        for l in range(reference.surface_levels(s)):
            problems += compare.level_diff(reference.surface_level(s, l), res.level(l), "L%d" % l)
        reference.surface_destroy(s)
        assert not problems, "\n".join(problems[:10])
    finally:
        reference.grid_destroy(g)


# ---- full size ----------------------------------------------------------------------------------------------------

def _streamed(gpu_context, good, n):
    """upload_packed_streamed with a producer that writes each slab only when asked; returns the slabs asked for."""
    nb = n // 16
    head = HEAD + nb ** 3 * 12
    sizes = good[HEAD:head].view(np.uint32).reshape(-1, 3).astype(np.int64)
    offsets = head + np.concatenate([[0], np.cumsum(4 + sizes.sum(axis=1))])
    blob = np.zeros_like(good)
    blob[:head] = good[:head]
    asked = []

    def produce(l0, l1):
        asked.append((l0, l1))
        a, b = offsets[l0 * nb * nb], offsets[l1 * nb * nb]
        blob[a:b] = good[a:b]

    gpu_context.upload_packed_streamed(blob, produce)
    return asked


@pytest.mark.parametrize("name", ["patchwork256", "patchwork512"])
def test_full_size_pack_and_packed_uploads(reference, gpu_context, name):
    """More than 1024 blocks: every thread of vxb_pack_offsets_kernel sums several blocks; the packed upload decodes in 4
    z-slabs, the streamed one in 4 (256^3) or 8 (512^3)."""
    import voxels_b200
    dist, mat, blend = grids.by_name(name)
    n = dist.shape[0]
    nb = n // 16
    g = reference.grid_from_dense(dist, mat, blend)
    want = reference.grid_pack(g)
    reference.grid_destroy(g)
    gpu_context.upload_dense(dist, mat, blend)
    _blob_equal(gpu_context.pack(), want, "vxb_grid_pack")
    _blob_equal(voxels_b200.pack_dense(dist, mat, blend), want, "pack_dense")
    gpu_context.upload_packed(want)
    _dense_equal((dist, mat, blend), gpu_context.download_dense(), "upload_packed")
    asked = _streamed(gpu_context, want, n)
    slabs = 8 if nb >= 32 else 4
    assert asked == [(nb * c // slabs, nb * (c + 1) // slabs) for c in range(slabs)], asked
    _dense_equal((dist, mat, blend), gpu_context.download_dense(), "upload_packed_streamed")


def test_terrain_1024_pack_round_trip(gpu_context):
    """The benchmark's 1024^3 terrain: the device pack equals the host packer of the same voxels, and the packed upload
    of it gives back every voxel."""
    import voxels_b200
    from voxels_b200 import capi
    n = 1024
    gpu_context.fill(n, capi.Surface.terrain(n))
    dense = gpu_context.download_dense()
    blob = gpu_context.pack()
    _blob_equal(blob, voxels_b200.pack_dense(*dense), "vxb_grid_pack vs pack_dense")
    gpu_context.upload_packed(blob)
    _dense_equal(dense, gpu_context.download_dense(), "upload_packed(pack())")


# ---- edits beyond +-4, then the codec and the polygonizer ----------------------------------------------------------

def _edit_sequence():
    """(what, position, extents, surface or material, injection type or add?) at n = 128 on the 128 terrain."""
    from voxels_b200 import capi
    plane = capi.Surface.plane
    terrain = capi.Surface.terrain
    S, M = "surface", "material"
    return [
        (S, (64, 64, 64), (80, 80, 80), plane((2.5, 1.5, 3.0), 4.0), 0),                 # add: down to -100
        (S, (40.5, 90.25, 70), (70, 66, 90), plane((-2.0, 3.0, 2.5), -3.0), 2),          # subtract: up to +100
        (S, (100, 30, 50), (64, 64, 64), plane((1.0, -2.5, 4.0), 10.0), 1),              # subtract-add-inner
        (S, (64, 64, 40), (128, 128, 30), terrain(256, origin=(10, 20), seed=7), 0),      # the whole grid in x and y
        (S, (20, 100, 90), (64, 72, 64), terrain(64, origin=(5, 5), seed=3), 2),
        (S, (90, 90, 100), (66, 66, 66), terrain(128), 1),
        (S, (33.3, 47.7, 61.1), (0.5, 0.5, 0.5), plane((0.0, 0.0, 1.0), 50.0), 0),       # sub-voxel extents
        (S, (50, 50, 50), (0, 0, 0), plane((1.0, 1.0, 1.0), 0.0), 0),                     # zero extents
        (S, (70, 70, 70), (-20, 30, 30), plane((1.0, 1.0, 1.0), 0.0), 0),                 # a negative extent
        (S, (-10, 64, 64), (20, 20, 20), plane((1.0, 1.0, 1.0), 0.0), 0),                 # grazes the low x face
        (S, (-40, 64, 64), (20, 20, 20), plane((1.0, 1.0, 1.0), 0.0), 0),                 # wholly outside, low
        (S, (200, 64, 64), (30, 30, 30), plane((1.0, 1.0, 1.0), 0.0), 2),                 # wholly outside, high
        (S, (120, 5, 126), (40, 40, 40), plane((3.0, -1.0, 2.0), 1.0), 0),                # partly outside: a corner
        (S, (8, 120, 64), (70, 30, 200), terrain(128, origin=(3, 9)), 2),                 # partly outside: two faces
        (M, (64, 64, 64), (80, 80, 80), 3, True),
        (M, (64, 64, 64), (80, 80, 80), 3, True),                                         # blend saturates at 255
        (M, (66, 60, 62), (72, 72, 72), 3, False),
        (M, (66, 60, 62), (72, 72, 72), 3, False),                                        # ... and at 0
        (M, (10, 120, 64), (70, 70, 70), 5, True),                                        # partly outside
        (M, (60.5, 61.25, 59.75), (0.5, 0.5, 0.5), 1, True),
        (M, (60, 60, 60), (0, 0, 0), 1, True),
        (M, (60, 60, 60), (-30, -30, -30), 1, True),
        (M, (300, 64, 64), (40, 40, 40), 2, False),                                        # wholly outside
        (S, (64, 64, 64), (16, 16, 16), plane((0.0, 0.0, 1.0), 0.5), 1),                  # a last surface edit over the materials
    ]


def test_edits_beyond_four_then_pack_and_polygonize(reference, gpu_context):
    from voxels_b200 import capi
    n = 128
    ctx = gpu_context
    s = capi.Surface.terrain(n)
    g = reference.grid_create_builtin(n, s)
    try:
        ctx.fill(n, s)
        for i, (what, pos, ext, arg, kind) in enumerate(_edit_sequence()):
            label = "edit %d (%s at %s, extents %s)" % (i, what, pos, ext)
            if what == "surface":
                want_box = reference.grid_inject_builtin(g, pos, ext, arg, kind)
                got_box = ctx.inject_surface(pos, ext, arg, kind)
            else:
                want_box = reference.grid_inject_material(g, pos, ext, arg, kind)
                got_box = ctx.inject_material(pos, ext, arg, kind)
            assert np.array_equal(want_box, got_box), "%s: returned box %s vs %s" % (label, want_box, got_box)
            assert_dense_equal(reference, g, ctx, label)
        dist, mat, blend = reference.grid_to_dense(g)
        assert dist.min() <= -100 and dist.max() >= 100, (dist.min(), dist.max())
        assert mat.max() < 255 and (blend == 255).any() and (blend == 0).any()
        # the flags words are recomputed on the edited values (BF_Empty of blocks holding +-100)
        _blob_equal(ctx.pack(), reference.grid_pack(g), "vxb_grid_pack after the edits")
        digests = []
        for threads in (1, 4):
            sf, _ = reference.polygonize(g, threads=threads)
            digests.append([golden_hash.level_digests(reference.surface_level(sf, l)) for l in range(reference.surface_levels(sf))])
            reference.surface_destroy(sf)
        assert digests[0] == digests[1], "the edited grid reaches the reference's undefined material case: change the edits"
        sf, _ = reference.polygonize(g)
        ctx.set_materials(None, None)
        info = ctx.polygonize()
        res = ctx.download()
        problems = []
        assert info.levels_total == reference.surface_levels(sf)
        for l in range(info.levels_total):
            problems += compare.level_diff(reference.surface_level(sf, l), res.level(l), "L%d" % l)
        if not np.array_equal(reference.surface_stats(sf), res.stats):
            problems.append("stats differ: ref %s gpu %s" % (reference.surface_stats(sf), res.stats))
        reference.surface_destroy(sf)
        assert not problems, "\n".join(problems[:10])
    finally:
        reference.grid_destroy(g)
