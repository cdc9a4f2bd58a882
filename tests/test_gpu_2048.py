"""The 2048^3 polygonization (bench.py's config4_2048) against the reference, crop by crop (tests/crops.py).

At 2048^3 the linear voxel offset (z * n + y) * n + x passes 2^31 at z = 512 and 2^32 at z = 1024, there are 8 levels
(coarse levels 4-7), and byte offsets into the default index arena pass 2^32; none of that happens at 1024^3.  A full
reference run at this size does not fit a test, so the reference runs on crops: 256^3 and 512^3 cubes of the same voxels,
whose selected blocks must equal the big run's.  Levels 5-7 are out of every crop's reach and get the size-independent
properties of the whole output instead.  One context runs the whole module (the grid alone is 24 GiB)."""
import os
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import crops
import golden_hash
import gridgen

pytestmark = pytest.mark.gpu

N = 2048
LEVELS = 8
# 256^3 crops (x, y, z) of the terrain; z = None centres the crop on the surface band found in the level-0 records.
# Their crops straddle z = 512 (offset 2^31; the terrain is solid there) and z = 1024 (2^32), and two lie in z >= 1024.
CROPS_256 = [(0, 0, None), (1792, 1792, None), (1024, 1024, 896), (512, 512, 384), (768, 1280, None), (0, 1024, None),
             (1024, 1792, None), (1792, 256, None)]
CROPS_512 = [(512, 512, None), (1536, 1024, 1024)]


def _t0():
    return time.perf_counter()


@pytest.fixture(scope="module")
def ctx():
    import voxels_b200
    c = voxels_b200.Context(0)
    yield c
    c.close()


def _volumes(ctx):
    """The device grid's three channels as [z, y, x] torch views (no copy)."""
    import torch
    from voxels_b200 import capi
    dev = torch.device("cuda", 0)
    return tuple(torch.as_tensor(capi.DevicePointer(p, N ** 3), device=dev).view(N, N, N) for p in ctx.device_pointers())


def _crop(ctx, origin, w):
    """(dist, mat, blend) numpy copies of the device grid's crop [origin, origin + w)^3, origin (x, y, z)."""
    import torch
    x, y, z = origin
    torch.cuda.synchronize()
    d, m, b = (v[z:z + w, y:y + w, x:x + w].contiguous().cpu().numpy() for v in _volumes(ctx))
    return d.view(np.int8), m, b


def _blocks_of(res):
    cache = {}

    def level(l):
        if l not in cache:
            cache[l] = crops.Blocks.from_result(res, l)
        return cache[l]
    return level


@pytest.fixture(scope="module")
def terrain(ctx):
    """The bench's input and run: vxb_grid_fill of the terrain, all 8 levels with transitions, downloaded."""
    from voxels_b200 import capi
    t = _t0()
    ctx.set_materials(None, None)
    ctx.fill(N, capi.Surface.terrain(N))
    info = ctx.polygonize()
    res = ctx.download()
    print("2048^3 fill + full run + download: %.1f s, %d blocks, %d vertices, %d indices" % (
        _t0() - t, info.block_count, info.vertex_total, info.index_total))
    return info, res


def _origins(res, crops_, w):
    """Crop origins with z = None resolved: the crop centred on the surface band of its columns, at a multiple of w / 4."""
    rec = res.records[res.records["level"] == 0]
    c = rec["coord_id"].astype(np.int64)
    nb = N // 16
    bx, by, bz = c % nb, (c // nb) % nb, c // (nb * nb)
    out = []
    for x, y, z in crops_:
        if z is None:
            cols = (bx * 16 >= x) & (bx * 16 < x + w) & (by * 16 >= y) & (by * 16 < y + w)
            assert cols.any(), "no surface over the columns of crop (%d, %d)" % (x, y)
            mid = (bz[cols].min() + bz[cols].max() + 1) * 8
            z = int(np.clip(round((mid - w // 2) / (w // 4)) * (w // 4), 0, N - w))
        out.append((x, y, z))
    return out


def _has_level0_blocks(res, o, w):
    rec = res.records[res.records["level"] == 0]
    c = rec["coord_id"].astype(np.int64)
    nb = N // 16
    b = np.stack([c % nb, (c // nb) % nb, c // (nb * nb)], axis=1) * 16
    return bool(np.all((b >= np.array(o)) & (b < np.array(o) + w), axis=1).any())


def test_fill_crops_equal_reference_constructor(reference, ctx, terrain):
    """vxb_grid_fill at 2048^3 against Grid::Create(w, w, w, start = origin, &terrain) on 256^3 crops across the 2^31 and
    2^32 voxel offsets."""
    from voxels_b200 import capi
    _, res = terrain
    origins = _origins(res, CROPS_256, 256)
    assert sum(z >= 1024 for _, _, z in origins) >= 2
    assert any(z < 512 < z + 256 for _, _, z in origins) and any(z < 1024 < z + 256 for _, _, z in origins)
    surface = capi.Surface.terrain(N)

    def want(o):   # the reference's constructor is serial: the crops are built side by side
        g = reference.grid_create_builtin(256, surface, start=tuple(float(v) for v in o))
        try:
            return reference.grid_to_dense(g)
        finally:
            reference.grid_destroy(g)
    t = _t0()
    with ThreadPoolExecutor(min(len(origins), os.cpu_count() or 1)) as pool:
        wants = list(pool.map(want, origins))
    for o, w in zip(origins, wants):
        for a, b, ch in zip(w, _crop(ctx, o, 256), ("distance", "material", "blend")):
            if not np.array_equal(a, b):
                bad = np.argwhere(a != b)
                raise AssertionError("crop %s: %s differs at %d voxels, first crop-local (z, y, x) %s" % (o, ch, len(bad), bad[0]))
    print("fill crops %s equal the reference constructor (%.1f s)" % (origins, _t0() - t))


def test_full_run_crops_against_reference(reference, ctx, terrain):
    """Every selected block of 8 crops of 256^3 and 2 of 512^3, all levels, against the reference's run of the crop's voxels
    (the device grid's own bytes, which the fill test pins to the reference's constructor)."""
    _, res = terrain
    big = _blocks_of(res)
    t = _t0()
    for w, crops_ in ((256, CROPS_256), (512, CROPS_512)):
        for o in _origins(res, crops_, w):
            g = reference.grid_from_dense(*_crop(ctx, o, w))
            lv = crops.reference_levels(reference, g, w)
            reference.grid_destroy(g)
            counts, problems = crops.compare_crop(lambda l: lv[l], big, o, w, len(lv))
            print("terrain crop %d^3 at %s: blocks compared per level %s" % (w, o, counts))
            assert not problems, "\n".join(problems[:10])
            if not _has_level0_blocks(res, o, w):
                continue           # solid (the crop across z = 512): no block on either side
            # a level-l block needs a margin of one block inside the crop on every side: 256^3 crops reach level 2,
            # 512^3 crops level 3
            for l in range(3 if w == 256 else 4):
                assert counts[l] > 0, "crop %d^3 at %s compared no level-%d block" % (w, o, l)
    print("terrain crops: %.1f s" % (_t0() - t))


def test_whole_output_properties(terrain):
    """Size-independent properties of every block of all 8 levels (the only check that reaches levels 5-7)."""
    info, res = terrain
    recs = res.records
    assert info.levels_total == LEVELS and info.block_count == len(recs)
    levels = recs["level"].astype(np.int64)
    assert set(np.unique(levels)) == set(range(LEVELS)), np.unique(levels)
    key = levels * (1 << 32) + recs["coord_id"]
    assert np.all(np.diff(key) > 0)                                       # the reference's order: level, then z, y, x
    base = np.array([crops.level_base(N, l) for l in range(LEVELS + 1)], np.int64)
    assert np.array_equal(recs["id"].astype(np.int64), base[levels] + recs["coord_id"])
    assert np.all(recs["coord_id"].astype(np.int64) < ((N // 16) >> levels) ** 3)
    st = res.stats.astype(np.int64)
    assert st[0] == base[LEVELS]                                          # BlocksCalculated: every block of every level
    assert st[4:].sum() == st[2]                                          # the per-class histogram sums to NonTrivialCells
    assert (st[1] + st[2]) % 4096 == 0
    vc, ic = recs["vertex_count"].astype(np.int64), recs["index_count"].astype(np.int64)
    assert info.vertex_total == vc.sum() and info.index_total == ic.sum()
    assert info.trans_vertex_total == recs["trans_vertex_count"].astype(np.int64).sum()
    assert info.trans_index_total == recs["trans_index_count"].astype(np.int64).sum()
    assert np.all(ic % 3 == 0) and np.all(recs["trans_index_count"] % 3 == 0)
    # the ranges lie inside the arenas and do not overlap
    for off, cnt, span in ((recs["vertex_offset"], vc, info.vertex_span), (recs["index_offset"], ic, info.index_span)):
        o = off.astype(np.int64)
        assert np.all(o + cnt <= span)
        order = np.argsort(o, kind="stable")
        assert np.all((o + cnt)[order][:-1] <= o[order][1:])
    # per chunk of blocks: indices address their own block's vertices, vertices lie in their block's box, every kept
    # triangle passes the reference's degenerate test, normals are unit (or zero)
    nb = (N // 16) >> levels
    m = (16 << levels).astype(np.float32)
    c = recs["coord_id"].astype(np.int64)
    lo = (np.stack([c % nb, c // (nb * nb), (c // nb) % nb], axis=1) * m[:, None]).astype(np.float32)   # output axes (x, z, y)
    for s in range(0, len(recs), 20000):
        sl = slice(s, s + 20000)
        vg = crops._gather(recs["vertex_offset"][sl], vc[sl])
        v = res.verts[vg]
        vblk = np.repeat(np.arange(len(vc[sl])), vc[sl])
        assert np.all(v["pos"] >= lo[sl][vblk] - 1e-3) and np.all(v["pos"] <= lo[sl][vblk] + m[sl][vblk, None] + 1e-3)
        nl = np.linalg.norm(v["nrm"].astype(np.float64), axis=1)
        assert np.all((np.abs(nl - 1) < 1e-5) | (nl == 0))
        ix = res.idx[crops._gather(recs["index_offset"][sl], ic[sl])].astype(np.int64)
        iblk = np.repeat(np.arange(len(ic[sl])), ic[sl])
        assert np.all(ix < vc[sl][iblk])
        p = (res.verts["pos"][recs["vertex_offset"][sl].astype(np.int64)[iblk] + ix][:, [0, 2, 1]] * np.float32(256)).astype(np.float32)
        a, b, cc = p[0::3], p[1::3], p[2::3]
        cr = np.cross((b - a).astype(np.float32), (cc - a).astype(np.float32)).astype(np.float64)
        assert np.all((cr ** 2).sum(axis=1) >= 1.1920928955078125e-07 * 0.5)
        tvc = recs["trans_vertex_count"][sl].astype(np.int64).ravel(); tic = recs["trans_index_count"][sl].astype(np.int64).ravel()
        tix = res.tidx[crops._gather(recs["trans_index_offset"][sl], tic)].astype(np.int64)
        assert np.all(tix < np.repeat(tvc, tic))
        tv = res.tverts[crops._gather(recs["trans_vertex_offset"][sl], tvc)]
        tl = np.linalg.norm(tv["nrm"].astype(np.float64), axis=1)
        assert np.all((np.abs(tl - 1) < 1e-5) | (tl == 0))


def test_level0_alone_and_repeatable(ctx, terrain):
    """polygonize(1, FLAG_NO_TRANSITIONS) gives the full run's level 0; a second full run gives the first's bytes."""
    import voxels_b200
    _, res = terrain
    want = [golden_hash.level_digests(res.level(l)) for l in range(LEVELS)]
    ctx.polygonize(1, voxels_b200.FLAG_NO_TRANSITIONS)
    assert golden_hash.level_digests(ctx.download().level(0)) == want[0]
    ctx.polygonize()
    again = ctx.download()
    for l in range(LEVELS):
        assert golden_hash.level_digests(again.level(l)) == want[l], "level %d differs in a second run" % l
    assert np.array_equal(again.stats, res.stats)


def test_edits_in_the_upper_half(reference, ctx, terrain):
    """8 sphere brushes at integer centres in z >= 1024 (vxb_grid_inject_surface + vxb_polygonize_region) against the
    reference's InjectSurface on the crop with the brush translated, and the re-created level-0 blocks against the
    reference's fresh run of the edited crop.  (Levels >= 1 of an incremental run are not a fresh run's by design.)"""
    from voxels_b200 import capi
    _, res = terrain
    w = 256
    o = _origins(res, [(0, 0, None)], w)[0]
    assert o[2] >= 1024
    cut = _crop(ctx, o, w)
    g = reference.grid_from_dense(*cut)
    rng = np.random.RandomState(2048)
    edits = []
    while len(edits) < 8:
        x, y, z = (int(v) for v in rng.randint(40, w - 40, size=3))
        if abs(int(cut[0][z, y, x])) >= 4:
            continue
        r = float(rng.choice([4, 6, 8, 10]))
        edits.append((np.array([x, y, z], np.float32), np.full(3, 2 * r + 4, np.float32), capi.Surface.sphere((0, 0, 0), r),
                      0 if len(edits) % 2 == 0 else 2))
    shift = np.array([o[0], o[2], o[1]] * 2, np.float32)      # boxes are in output axes (x, z, y)
    try:
        for i, (pos, ext, sph, kind) in enumerate(edits):
            box = reference.grid_inject_builtin(g, pos, ext, sph, kind)
            got = ctx.inject_surface(pos + np.array(o, np.float32), ext, sph, kind)
            assert np.array_equal(got, box + shift), "edit %d: box %s vs the reference's %s + %s" % (i, got, box, shift)
            for a, b, ch in zip(reference.grid_to_dense(g), _crop(ctx, o, w), ("distance", "material", "blend")):
                assert np.array_equal(a, b), "edit %d: %s of the crop differs from the reference's" % (i, ch)
            ctx.polygonize_region(got[:3], got[3:])
            part = ctx.download()
            region = ctx.region_info()
            fresh = crops.reference_levels(reference, g, w)[0]
            mn, mx = np.array(region.min_dirty[0]), np.array(region.max_dirty[0])
            b = fresh.coord
            wb = w // 16
            bmin = np.stack([b % wb * 16 + o[0], b // (wb * wb) * 16 + o[2], (b // wb) % wb * 16 + o[1]], axis=1)
            inside = np.all((bmin >= mn) & (bmin < mx), axis=1)
            k, problems = crops.compare_level(fresh.subset(inside), crops.Blocks.from_result(part, 0), o, w, big_ids=False)
            print("edit %d at %s: %d re-created level-0 blocks compared" % (i, pos + np.array(o, np.float32), k))
            assert not problems, "\n".join(problems[:10])
            assert k > 0
    finally:
        reference.grid_destroy(g)


def test_hostile_content_above_2_to_32(reference, ctx):
    """synth.terrain(2048) written by torch into the device grid, with patchwork(256) pasted into the far corner (z >= 1792,
    whose 512^3 corner crop reaches level 4) and hostile(256) pasted across z = 1024 and across z = 512, handed to the
    context with vxb_grid_set_device; each paste's 512^3 crop against the reference (the hostile ones at level 0)."""
    import torch
    from voxels_b200 import synth
    d, m, b = _volumes(ctx)
    synth.terrain(N, "cuda:0", z_chunk=8, out=(d.view(torch.int8), m, b))
    torch.cuda.empty_cache()
    pastes = [("patchwork", (1792, 1792, 1792), gridgen.patchwork(256), (1536, 1536, 1536)),
              ("hostile", (640, 1152, 896), gridgen.hostile(256), (512, 1024, 768)),
              ("hostile", (1152, 384, 384), gridgen.hostile(256, seed=11), (1024, 256, 256))]
    for _, (x, y, z), arrays, _ in pastes:
        for v, a in zip((d, m, b), arrays):
            v[z:z + 256, y:y + 256, x:x + 256] = torch.from_numpy(np.ascontiguousarray(a).view(np.uint8)).to(v.device)
    torch.cuda.synchronize()
    ctx.set_materials(None, None)
    ctx.set_device_grid(N, d.data_ptr(), m.data_ptr(), b.data_ptr(), keep=(d, m, b))
    ctx.polygonize()
    res = ctx.download()
    big = _blocks_of(res)
    for name, _, _, o in pastes:
        cut = _crop(ctx, o, 512)
        g = reference.grid_from_dense(*cut)
        lv = crops.reference_levels(reference, g, 512)
        reference.grid_destroy(g)
        # the hostile pastes' faces meet the terrain's uniform blocks of the other sign, so a surface runs between two
        # BF_Empty blocks: the reference skips them at level 0 and its coarse cells over them read an uninitialised
        # material (DESIGN.md section 2), so only their level 0 is defined.  The patchwork paste sits in air: all levels.
        levels = len(lv) if name == "patchwork" else 1
        counts, problems = crops.compare_crop(lambda l: lv[l], big, o, 512, levels)
        print("%s paste, crop 512^3 at %s: blocks compared per level %s" % (name, o, counts))
        assert not problems, "\n".join(problems[:10])
        assert all(counts[l] > 0 for l in range(min(levels, 4))), counts
        if name == "patchwork":
            assert counts[4] > 0, "the corner crop compared no level-4 block"
            # a level-0 block with more than 1024 non-trivial cells (a big block) is among the compared ones
            bx, by, bz = crops.selected(o, 512, N, 0)
            nt = gridgen.nontrivial_cells_per_block(cut[0], 0)
            assert (nt[bz, by, bx] > 1024).any(), "no selected level-0 big block in the patchwork crop"
