"""Numpy oracle of the mesh's bounds and of the culled select (include/vxb200.h "bounds and the culled select").

  block_boxes     the box of every block of a downloaded mesh: min / max of pos and sec[0..2] over its regular vertices and
                  the transition vertices of all six faces
  box_passes      the p-vertex test of the header, float32, products and sums in the header's order (numpy does not fuse)
  cut             the LOD cut and block_adj of tests/test_gpu_draws.py, restated over arrays and in the kernel's float32
                  (test_gpu_cull.py ties the two statements together on a grid)
  expected_draws  per view the set of regular and of transition draws
  draw_sets       the same sets from downloaded lists
"""
import numpy as np

F = np.float32
FACES = np.array([(0, 0, -1), (0, -1, 0), (-1, 0, 0), (0, 0, 1), (0, 1, 0), (1, 0, 0)], np.int64)
EMPTY_BOX = np.array([np.inf, np.inf, np.inf, -np.inf, -np.inf, -np.inf], F)


def block_box(res, r):
    parts = [res.verts[r["vertex_offset"]:r["vertex_offset"] + r["vertex_count"]]]
    parts += [res.tverts[o:o + c] for o, c in zip(r["trans_vertex_offset"], r["trans_vertex_count"])]
    pts = np.concatenate([np.concatenate([p["pos"], p["sec"][:, :3]]) for p in parts])
    if not len(pts):
        return EMPTY_BOX.copy()
    assert np.isfinite(pts).all()
    return np.concatenate([pts.min(axis=0), pts.max(axis=0)]).astype(F)


def block_boxes(res, which=None):
    """(blocks, 6) float32 {min xyz, max xyz} of res.records[which] (all records when None), in that order."""
    recs = res.records if which is None else res.records[which]
    return np.stack([block_box(res, r) for r in recs]) if len(recs) else np.zeros((0, 6), F)


def lattice_boxes(records, n):
    """The blocks' lattice boxes in output axes (x, z, y): NOT a bound of the vertices at levels >= 1."""
    level = records["level"].astype(np.int64)
    nb = (n // 16) >> level
    cid = records["coord_id"].astype(np.int64)
    m = (16 << level).astype(np.float64)
    lo = np.stack([cid % nb, cid // (nb * nb), (cid // nb) % nb], axis=1) * m[:, None]
    return np.concatenate([lo, lo + m[:, None]], axis=1)


def box_passes(boxes, planes):
    """boxes: (blocks, 6) float32; planes: (6, 4) float32.  True where the box passes every plane:
    c_i = n_i >= 0 ? max_i : min_i;  s = ((nx*cx + ny*cy) + nz*cz) + d;  pass iff s >= 0."""
    boxes = np.asarray(boxes, F).reshape(-1, 6)
    planes = np.asarray(planes, F).reshape(6, 4)
    nrm = planes[None, :, :3]
    with np.errstate(invalid="ignore", over="ignore"):
        c = np.where(nrm >= 0, boxes[:, None, 3:], boxes[:, None, :3])
        p = nrm * c
        s = ((p[..., 0] + p[..., 1]) + p[..., 2]) + planes[None, :, 3]
        return (s >= 0).all(axis=1)


def _stops(level, b, cam, base, top):
    """vxb_lod_stops for an array of grid block coordinates (x, y, z) of one level."""
    if level == top:
        return np.ones(len(b), bool)
    c = (b.astype(F) + F(0.5)) * F(16 << level)
    dx, dy, dz = c[:, 0] - cam[0], c[:, 2] - cam[1], c[:, 1] - cam[2]         # output axes (x, z, y)
    lim = F(base) * F(1 << level)
    return (dx * dx + dy * dy) + dz * dz >= lim * lim


def _descends_from(first, level, b, cam, base, top):
    """No node of levels [first, top] above (or at) the blocks stops."""
    ok = np.ones(len(b), bool)
    for l in range(first, top + 1):
        ok &= ~_stops(l, b >> (l - level), cam, base, top)
    return ok


def cut(records, n, levels, camera, base):
    """(selected, block_adj) per record: the cut of vxb_mesh_select_lod."""
    cam = np.asarray(camera, F)
    top = levels - 1
    selected = np.zeros(len(records), bool)
    adj = np.zeros(len(records), np.uint32)
    for level in range(levels):
        at = np.nonzero(records["level"] == level)[0]
        if not len(at):
            continue
        nb = (n // 16) >> level
        cid = records["coord_id"][at].astype(np.int64)
        b = np.stack([cid % nb, (cid // nb) % nb, cid // (nb * nb)], axis=1)
        sel = _descends_from(level + 1, level, b, cam, base, top)
        if level > 0:
            sel &= _stops(level, b, cam, base, top)
            a = np.zeros(len(at), np.uint32)
            for f, d in enumerate(FACES):
                nbr = b + d
                inside = ((nbr >= 0) & (nbr < nb)).all(axis=1)
                finer = _descends_from(level, level, np.clip(nbr, 0, nb - 1), cam, base, top)
                a |= (inside & finer).astype(np.uint32) << np.uint32(f)
            adj[at] = a
        selected[at] = sel
    adj[~selected] = 0
    return selected, adj


def draws_of(records, drawn, adj):
    """The draw sets of the records `drawn` (a mask): regular {(block_id, level, block_adj, index_count, first_index,
    base_vertex)} and transition {(block_id, level, block_adj, face, index_count, first_index, base_vertex)}."""
    regular, transition = set(), set()
    for k in np.nonzero(drawn)[0]:
        r, a = records[k], int(adj[k])
        regular.add((int(r["id"]), int(r["level"]), a, int(r["index_count"]), int(r["index_offset"]), int(r["vertex_offset"])))
        for f in range(6):
            if (a >> f) & 1 and r["trans_index_count"][f]:
                transition.add((int(r["id"]), int(r["level"]), a, f, int(r["trans_index_count"][f]), int(r["trans_index_offset"][f]),
                                int(r["trans_vertex_offset"][f])))
    return regular, transition


def expected_draws(records, boxes, n, levels, camera, base, views):
    """Per view the (regular, transition) sets: the cut of (camera, base), culled by box_passes."""
    selected, adj = cut(records, n, levels, camera, base)
    return [draws_of(records, selected & box_passes(boxes, v), adj) for v in np.asarray(views, F).reshape(-1, 6, 4)]


def draw_sets(lists):
    """The sets of draws_of from downloaded lists (commands, infos, transition commands, transition infos); asserts what
    every list must hold: first_instance indexes the list's own info array, one instance, the regular face marker."""
    rc, ri, tc, ti = lists
    assert np.array_equal(rc["first_instance"], np.arange(len(rc))) and np.array_equal(tc["first_instance"], np.arange(len(tc)))
    assert (rc["instance_count"] == 1).all() and (tc["instance_count"] == 1).all() and (ri["face"] == 0xFFFFFFFF).all()
    regular = set(zip(ri["block_id"].tolist(), ri["level"].tolist(), ri["block_adj"].tolist(), rc["index_count"].tolist(),
                      rc["first_index"].tolist(), rc["base_vertex"].tolist()))
    transition = set(zip(ti["block_id"].tolist(), ti["level"].tolist(), ti["block_adj"].tolist(), ti["face"].tolist(),
                         tc["index_count"].tolist(), tc["first_index"].tolist(), tc["base_vertex"].tolist()))
    assert len(regular) == len(rc) and len(transition) == len(tc), "a draw appears twice"
    return regular, transition


# ---- planes for the tests and tools/bench_cull.py (the API takes planes, not matrices) ----
def plane(normal, point):
    """{n, d} of the plane through `point` whose inside is the side `normal` points to."""
    nrm = np.asarray(normal, np.float64)
    return np.array([nrm[0], nrm[1], nrm[2], -float(nrm @ np.asarray(point, np.float64))], F)


PASS_ALL = np.tile(np.array([0, 0, 0, 1], F), (6, 1))


def perspective(eye, forward, up, fov_x_deg, fov_y_deg, near, far):
    """Six inward planes of a symmetric perspective frustum."""
    eye = np.asarray(eye, np.float64)
    f = np.asarray(forward, np.float64); f = f / np.linalg.norm(f)
    r = np.cross(f, np.asarray(up, np.float64)); r = r / np.linalg.norm(r)
    u = np.cross(r, f)
    tx, ty = np.tan(np.radians(fov_x_deg) / 2), np.tan(np.radians(fov_y_deg) / 2)
    return np.stack([plane(f, eye + near * f), plane(-f, eye + far * f),
                     plane(f * tx + r, eye), plane(f * tx - r, eye), plane(f * ty + u, eye), plane(f * ty - u, eye)])


def box_planes(lo, hi):
    """Six axis-aligned inward planes of the box [lo, hi] (an orthographic view volume)."""
    out = []
    for a in range(3):
        e = np.zeros(3); e[a] = 1
        out += [plane(e, e * lo[a]), plane(-e, e * hi[a])]
    return np.stack(out)
