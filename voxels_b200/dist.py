"""torch.distributed plumbing for the multi-GPU runs (one process per GPU; NCCL on the GPU box, gloo in the CPU tests).

ONE grid polygonized by all ranks (`ShardedGrid`, SURVEY.md section 8e / BASELINE configs[3], include/vxb200.h "Sharded
runs"): work is dealt by blocks; the read-only volumes are replicated in every rank's HBM (default) or sharded as a cube
whose z-pieces are mapped into every peer over NVLink (file descriptors travel over Unix sockets, `exchange_fds`); the
data path has two exchanges (an ncclAllGather of the per-block info, peer stores of the material pages ordered by a
second tiny all-gather), both issued by libvxb200.so itself on the context's stream, so a step is one CUDA graph.
torch.distributed carries the rendezvous: the NCCL id broadcast, barriers, the max-reduction of device times and the
all-gather of the block directories.  `tile_origin` / `whole_job_throughput`: the independent-tiles weak-scaling mode
kept as a secondary bench line."""
import os
import socket
import threading


class Ranks:
    def __init__(self, backend=None, device=None):
        self.rank = int(os.environ.get("RANK", "0"))
        self.world = int(os.environ.get("WORLD_SIZE", "1"))
        self.local_rank = int(os.environ.get("LOCAL_RANK", "0"))
        self.device = device
        self.td = None
        if self.world > 1:
            import torch.distributed as td
            self.td = td
            if not td.is_initialized():
                kw = {"device_id": device} if (backend == "nccl" and device is not None) else {}
                td.init_process_group(backend=backend or "nccl", **kw)

    def barrier(self):
        if self.td is not None:
            if self.device is not None and self.device.type == "cuda":
                self.td.barrier(device_ids=[self.local_rank])
            else:
                self.td.barrier()

    def max_over_ranks(self, value):
        """The slowest rank's value (multi-GPU times are reported as the max over ranks)."""
        if self.td is None:
            return float(value)
        import torch
        t = torch.tensor([float(value)], dtype=torch.float64, device=self.device if self.device is not None else "cpu")
        self.td.all_reduce(t, op=self.td.ReduceOp.MAX)
        return float(t.item())

    def sum_over_ranks(self, value):
        if self.td is None:
            return float(value)
        import torch
        t = torch.tensor([float(value)], dtype=torch.float64, device=self.device if self.device is not None else "cpu")
        self.td.all_reduce(t, op=self.td.ReduceOp.SUM)
        return float(t.item())

    def close(self):
        if self.td is not None and self.td.is_initialized():
            self.td.destroy_process_group()


def bind_to_gpu_numa_node(device_index):
    """Pins this process (its threads, and through first-touch its page-locked buffers) to the CPUs of the NUMA node the GPU
    hangs off, so that N ranks do not fight over one socket's memory controllers during their host<->device copies.
    Returns the node number, or None when the topology cannot be read (then nothing is changed)."""
    try:
        import torch
        p = torch.cuda.get_device_properties(device_index)
        bdf = "%04x:%02x:%02x.0" % (p.pci_domain_id, p.pci_bus_id, p.pci_device_id)
        with open("/sys/bus/pci/devices/%s/numa_node" % bdf) as f:
            node = int(f.read().strip())
        if node < 0:
            return None
        with open("/sys/devices/system/node/node%d/cpulist" % node) as f:
            cpus = parse_cpulist(f.read())
        allowed = sorted(set(cpus) & set(os.sched_getaffinity(0)))
        if not allowed:
            return None
        os.sched_setaffinity(0, allowed)
        return node
    except Exception:
        return None


def parse_cpulist(text):
    """'0-3,8,10-11' -> [0, 1, 2, 3, 8, 10, 11] (the format of /sys/devices/system/node/node*/cpulist)."""
    out = []
    for part in text.strip().split(","):
        if not part:
            continue
        if "-" in part:
            a, b = part.split("-")
            out += list(range(int(a), int(b) + 1))
        else:
            out.append(int(part))
    return out


def tile_origin(rank, n):
    """(x, y) origin of rank's tile in the endless terrain: tiles are laid out along x, n voxels apart."""
    return (rank * n, 0)


def whole_job_throughput(n, world, ms_per_step):
    """Mvoxels/s of the whole job: every rank polygonizes its own n^3 tile per step."""
    return float(n) ** 3 * world / (ms_per_step * 1e-3) / 1e6


# ---------------------------------------------------------------------------------------------------------------------
# one grid, all ranks
# ---------------------------------------------------------------------------------------------------------------------

def default_group_planes(n, world):
    """Planes per piece: 32 (the finest the block walk allows) when the pieces still meet the 2 MiB allocation granularity
    for the volumes AND the even-lattice channel (an eighth of a volume piece), else the smallest multiple that does;
    never more than n / world."""
    g = 32
    while g * n * n // 8 % (2 << 20) != 0 and g < n // world:
        g *= 2
    return min(g, n // world)


def owned_pieces(n, rank, world, group_planes):
    """[(piece, z0, z1)] of the pieces rank backs with its own HBM (cyclic deal)."""
    pieces = n // group_planes
    return [(p, p * group_planes, (p + 1) * group_planes) for p in range(rank, pieces, world)]


def exchange_fds(rank, world, fds, key):
    """Every rank offers `fds` (a list of open file descriptors) to every peer; returns {peer: [fds...]} with this
    process's duplicates of the peers' descriptors.  Unix sockets in the abstract namespace + SCM_RIGHTS; all ranks run
    on one host (one process per GPU of a box)."""
    if world == 1:
        return {}
    name = lambda r: "\0vxb200-%s-%d" % (key, r)  # noqa: E731
    server = socket.socket(socket.AF_UNIX, socket.SOCK_STREAM)
    server.bind(name(rank))
    server.listen(world)

    def serve():
        for _ in range(world - 1):
            conn, _addr = server.accept()
            with conn:
                conn.recv(1)
                socket.send_fds(conn, [b"f"], list(fds))
    t = threading.Thread(target=serve, daemon=True)
    t.start()
    got = {}
    for peer in range(world):
        if peer == rank:
            continue
        c = socket.socket(socket.AF_UNIX, socket.SOCK_STREAM)
        for attempt in range(600):  # the peer may not be listening yet
            try:
                c.connect(name(peer))
                break
            except (ConnectionRefusedError, FileNotFoundError):
                import time
                time.sleep(0.05)
        else:
            raise RuntimeError("exchange_fds: rank %d never reached rank %d" % (rank, peer))
        with c:
            c.send(b"r")
            _msg, received, _flags, _addr = socket.recv_fds(c, 1, len(fds))
        if len(received) != len(fds):
            raise RuntimeError("exchange_fds: expected %d descriptors from rank %d, got %d" % (len(fds), peer, len(received)))
        got[peer] = list(received)
    t.join()
    server.close()
    return got


def gather_directories(ranks, records):
    """All-gather of the per-rank block directories (numpy RECORD_DTYPE arrays): counts first, then the padded payload.
    Returns (records of all ranks sorted by (level, coord_id), owner rank of each)."""
    import numpy as np
    import torch
    if ranks.td is None:
        order = np.lexsort((records["coord_id"], records["level"]))
        return records[order], np.zeros(len(records), np.int32)
    dev = ranks.device if ranks.device is not None else torch.device("cpu")
    counts = torch.zeros(ranks.world, dtype=torch.int64, device=dev)
    mine = torch.tensor([len(records)], dtype=torch.int64, device=dev)
    ranks.td.all_gather_into_tensor(counts, mine)
    counts = counts.cpu().numpy()
    width = int(counts.max())
    item = records.dtype.itemsize
    payload = np.zeros(width * item, np.uint8)
    payload[:len(records) * item] = records.view(np.uint8).reshape(-1)
    out = torch.zeros(ranks.world * width * item, dtype=torch.uint8, device=dev)
    ranks.td.all_gather_into_tensor(out, torch.from_numpy(payload).to(dev))
    out = out.cpu().numpy().reshape(ranks.world, width * item)
    parts, owners = [], []
    for r in range(ranks.world):
        parts.append(out[r, :int(counts[r]) * item].copy().view(records.dtype))
        owners.append(np.full(int(counts[r]), r, np.int32))
    allrec, owner = np.concatenate(parts), np.concatenate(owners)
    order = np.lexsort((allrec["coord_id"], allrec["level"]))
    return allrec[order], owner[order]


class ShardedGrid:
    """One n^3 grid polygonized by all ranks (one GPU each).  Usage:
        sg = ShardedGrid(ranks, n)            # mode "replicated" (default) or "cube"
        sg.fill(surface)  |  sg.upload_packed(blob_ptr, nbytes)     # every rank: the whole grid (replicated) / its pieces (cube)
        sg.ready()                            # page buffers exchanged, NCCL communicator, barrier: every rank's data is in place
        info = sg.polygonize()                # one stream-ordered step (two exchanges inside); this rank's blocks
        directory, owner = sg.directory()     # every rank's blocks (all-gather), reference order

    replicated: every rank holds the three read-only volumes in its own HBM (24 GB at 2048^3) and the WORK is sharded - every
                load of a kernel is local.  Default, because peer loads over NVLink are not cached in the local L2, and the
                sparse 1-byte taps of the vertex / vote / transition code live on L2 hits.
    cube:       the volumes themselves are sharded: z-pieces of group_planes planes live in the ranks' HBM (cyclic deal) and
                are mapped into every peer over NVLink.  For grids that do not fit one GPU.
    """

    def __init__(self, ranks, n, device_index=None, key=None, group_planes=None, mode="replicated"):
        import torch
        from . import capi
        assert mode in ("replicated", "cube")
        self.ranks, self.n, self.mode = ranks, n, mode
        self.rank, self.world = ranks.rank, ranks.world
        self.group_planes = (default_group_planes(n, self.world) if mode == "cube" else min(32, n // self.world)) if group_planes is None else int(group_planes)
        self.device_index = ranks.local_rank if device_index is None else device_index
        self.device = torch.device("cuda", self.device_index)
        self.key = "%s-%d-%s" % (key or os.environ.get("MASTER_PORT", "0"), n, mode)
        self.ctx = capi.Context(self.device_index)
        self._configured = False
        self.last_attempts = 0
        if mode == "cube":
            self.ctx.cube_create(n, self.rank, self.world, self.group_planes)
            self.pieces, self.channels, _ = self.ctx.cube_info()
            if self.world > 1:
                mine = [p for p, _, _ in owned_pieces(n, self.rank, self.world, self.group_planes)]
                fds = [self.ctx.cube_export(c, p) for p in mine for c in range(self.channels)]
                got = exchange_fds(self.rank, self.world, fds, self.key + "-cube")
                for peer, theirs in got.items():
                    it = iter(theirs)
                    for p, _, _ in owned_pieces(n, peer, self.world, self.group_planes):
                        for c in range(self.channels):
                            fd = next(it)
                            self.ctx.cube_import(c, p, fd)
                            os.close(fd)
                for fd in fds:
                    os.close(fd)

    def fill(self, surface, start=(0.0, 0.0, 0.0), step=1.0):
        """Grid::Create(..., &surface) on the device: the whole grid (replicated) or this rank's pieces (cube)."""
        self.ctx.fill(self.n, surface, start, step)

    def fill_program(self, ops, start=(0.0, 0.0, 0.0), step=1.0):
        """fill() with an SDF program (a list of capi.Op): the whole grid (replicated) or this rank's pieces (cube)."""
        self.ctx.fill_program(self.n, ops, start, step)

    def upload_packed(self, blob_ptr, nbytes):
        """The grid's PackForSave bytes from (pinned) host memory: decoded on the GPU, whole (replicated) or this rank's pieces."""
        self.ctx.upload_packed(blob_ptr, nbytes)

    def _configure(self):
        from . import capi
        self.ctx.shard_configure(self.rank, self.world, self.group_planes)
        if self.world > 1:
            fd = self.ctx.shard_export()
            got = exchange_fds(self.rank, self.world, [fd], self.key + "-pages")
            for peer, theirs in got.items():
                self.ctx.shard_import(peer, theirs[0])
                os.close(theirs[0])
            os.close(fd)
            # the communicator of the two in-step all-gathers: id from rank 0, carried by torch.distributed
            ids = [capi.nccl_unique_id() if self.rank == 0 else None]
            self.ranks.td.broadcast_object_list(ids, src=0)
            self.ctx.shard_nccl_init(ids[0], self.rank, self.world)
        self._configured = True

    def piece_tensors(self):
        """cube mode: [(z0, z1, (dist, mat, blend))] torch views of this rank's pieces."""
        import torch
        from . import capi
        out = []
        for p, z0, z1 in owned_pieces(self.n, self.rank, self.world, self.group_planes):
            d, m, b, size = self.ctx.cube_piece(p)
            shape = (z1 - z0, self.n, self.n)
            view = lambda ptr: torch.as_tensor(capi.DevicePointer(ptr, size), device=self.device).view(shape)  # noqa: E731
            out.append((z0, z1, (view(d).view(torch.int8), view(m), view(b))))
        return out

    def ready(self):
        import torch
        if not self._configured:
            self._configure()
        torch.cuda.synchronize(self.device)
        self.ranks.barrier()

    def polygonize(self, flags=0, max_attempts=4):
        from . import capi
        for attempt in range(max_attempts):
            rc = self.ctx.polygonize_sharded(3, flags)
            # an overflow on any rank repeats the run on every rank (the exchanges are collective)
            if self.ranks.max_over_ranks(1.0 if rc != 0 else 0.0) == 0.0:
                self.last_attempts = attempt + 1
                return self.ctx.info()
        raise capi.VxbError("sharded run: output arenas kept overflowing")

    def directory(self):
        import numpy as np
        from . import capi
        info = self.ctx.info()
        records = np.zeros(info.block_count, capi.RECORD_DTYPE)
        self.ctx._check(self.ctx.L.vxb_result_download(self.ctx.h, capi._ptr(records), None, None, None, None), "vxb_result_download")
        return gather_directories(self.ranks, records)

    def close(self):
        self.ctx.close()
