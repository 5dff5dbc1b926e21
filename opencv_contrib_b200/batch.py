"""Batched frame-pair front end: shards independent image pairs over streams on one GPU and over
ranks on one node (one process per GPU).

The reference has no batching or multi-GPU layer -- callers loop over ``calc`` and pick a device
with ``cv::cuda::setDevice`` (modules/cudaoptflow/test/test_optflow.cpp:58-63, and the 16-stream
``cv::parallel_for_`` pattern of test_optflow.cpp:468-528).  Frame pairs are independent problems,
so the path shards with NO data-path collective: rank r of R owns the contiguous block
[r*N/R, (r+1)*N/R) of pair indices (SURVEY.md §8e); NCCL appears only in ``gather_flows``, the
result gather to rank 0.

torch is plumbing here (device tensors, streams, torch.distributed); all compute is in
libb200flow.so.
"""
from __future__ import annotations

import threading
from typing import Callable, List, Sequence, Tuple


def shard_range(n_items: int, rank: int, world: int) -> Tuple[int, int]:
    """Contiguous block partition [lo, hi) of n_items over world ranks (remainder to low ranks)."""
    base, rem = divmod(n_items, world)
    lo = rank * base + min(rank, rem)
    hi = lo + base + (1 if rank < rem else 0)
    return lo, hi


class FlowBatcher:
    """Runs many independent pairs through ``n_streams`` engine instances (one handle per stream,
    as instances are not re-entrant: reference tvl1flow.cpp:141-167 caches buffers per instance)."""

    def __init__(self, factory: Callable[[], object], n_streams: int = 4, device=None):
        import torch
        self.torch = torch
        self.device = device if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.algs = [factory() for _ in range(n_streams)]
        self.streams = [torch.cuda.Stream(device=self.device) for _ in range(n_streams)]
        self._done = [torch.cuda.Event() for _ in range(n_streams)]
        self._start = torch.cuda.Event()

    @property
    def n_streams(self) -> int:
        return len(self.streams)

    def run_device(self, pairs: Sequence[Tuple[object, object]], flows: Sequence[object]) -> None:
        """Device-resident batch.  Work is forked from / joined to the CURRENT stream, so CUDA
        events recorded on it bracket the whole batch; no host synchronisation."""
        torch = self.torch
        cur = torch.cuda.current_stream(self.device)
        self._start.record(cur)
        used = min(self.n_streams, len(pairs))
        for s in self.streams[:used]:
            s.wait_event(self._start)
        for i, ((a, b), f) in enumerate(zip(pairs, flows)):
            k = i % self.n_streams
            self.algs[k].calc(a, b, f, self.streams[k])
        for k in range(used):
            self._done[k].record(self.streams[k])
            cur.wait_event(self._done[k])

    def run_host(self, pairs: Sequence[Tuple[object, object]], flows: Sequence[object]) -> None:
        """Host-resident batch (numpy arrays, ideally pinned): each stream's worker thread uploads,
        computes and downloads its share through b2f_calc_host, so copies of one pair overlap the
        compute of others.  Returns when every flow has landed in host memory."""
        errs: List[BaseException] = []

        def work(k: int):
            try:
                # the CUDA current device is per thread: a fresh thread starts on device 0
                self.torch.cuda.set_device(self.device)
                for i in range(k, len(pairs), self.n_streams):
                    a, b = pairs[i]
                    self.algs[k].calc_host(a, b, flows[i], self.streams[k])
            except BaseException as e:  # noqa: BLE001
                errs.append(e)

        threads = [threading.Thread(target=work, args=(k,)) for k in range(min(self.n_streams, len(pairs)))]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        if errs:
            raise errs[0]

    def launches(self) -> int:
        return sum(a.getStats()["launches"] for a in self.algs)

    def reset_stats(self) -> None:
        for a in self.algs:
            a.resetStats()


class NativeFlowBatch:
    """Same interface as FlowBatcher, but the stream fork / join, the round-robin deal and the host-path worker
    threads live in libb200flow.so (csrc/batch.cu, ``b2f_batch_*``): one C call per batch instead of one per pair.

        NativeFlowBatch("tvl1", dict(nscales=5, warps=10, epsilon=0.0, iterations=30), n_streams=4)
    """

    _ALGO = {"tvl1": 1, "farneback": 2, "brox": 3, "denselk": 4, "deepflow": 5, "dis": 6, "fastbm": 7, "varref": 8,
             "optflowgf": 9}

    def __init__(self, family: str, params: dict | None = None, n_streams: int = 4):
        import ctypes as C
        from . import _lib
        self._C, self._libmod = C, _lib
        self._lib = _lib.lib()
        struct = {"tvl1": _lib.b2f_tvl1_params, "farneback": _lib.b2f_farneback_params, "brox": _lib.b2f_brox_params,
                  "denselk": _lib.b2f_denselk_params, "deepflow": _lib.b2f_deepflow_params,
                  "dis": _lib.b2f_dis_params, "fastbm": _lib.b2f_fastbm_params,
                  "varref": _lib.b2f_varref_params, "optflowgf": _lib.b2f_farneback_params}[family]()
        preset = (1,) if family == "dis" else ()  # DIS defaults: the FAST preset
        # the video module's Farneback takes the cv::cuda class's parameter struct and defaults
        defaults = "farneback" if family == "optflowgf" else family
        getattr(self._lib, "b2f_%s_default_params" % defaults)(C.byref(struct), *preset)
        for k, v in (params or {}).items():
            if not hasattr(struct, k):
                raise AttributeError("%s has no parameter %r" % (family, k))
            setattr(struct, k, v)
        self._b = C.c_void_p()
        st = self._lib.b2f_batch_create(self._ALGO[family], C.byref(struct), n_streams, C.byref(self._b))
        if st != 0:
            self._b = None
            raise _lib.B2FError(st)
        self.n_streams = n_streams

    def close(self):
        b, self._b = getattr(self, "_b", None), None
        if b:
            self._lib.b2f_batch_destroy(b)

    __del__ = close

    def set_engine_option(self, name: str, value) -> None:
        st = self._lib.b2f_batch_set_param(self._b, self._libmod.PARAM["engine"][name], float(value))
        if st != 0:
            raise self._libmod.B2FError(st)

    def _arrays(self, pairs, flows, conv):
        n = len(pairs)
        arr = self._libmod.b2f_image * n
        a, b, f = arr(), arr(), arr()
        for i, ((x, y), fl) in enumerate(zip(pairs, flows)):
            a[i], b[i], f[i] = conv(x), conv(y), conv(fl, True)
        return n, a, b, f

    def run_device(self, pairs, flows, stream=None) -> None:
        import torch
        from .cudaoptflow import _image_from_tensor
        n, a, b, f = self._arrays(pairs, flows, _image_from_tensor)
        if stream is None:
            stream = torch.cuda.current_stream()
        st = self._lib.b2f_batch_run_device(self._b, n, a, b, f, self._C.c_void_p(stream.cuda_stream))
        if st != 0:
            raise self._libmod.B2FError(st)

    def run_host(self, pairs, flows) -> None:
        from .cudaoptflow import _image_from_numpy
        n, a, b, f = self._arrays(pairs, flows, _image_from_numpy)
        st = self._lib.b2f_batch_run_host(self._b, n, a, b, f)
        if st != 0:
            raise self._libmod.B2FError(st)

    def run_device_gather(self, pairs, flows, comm: "NativeComm", dst: int = 0, gathered=None, stream=None) -> None:
        """run_device + the native result gather (b2f_batch_run_device_gather): every flow goes to rank ``dst`` over NCCL
        as soon as its own solve has finished, on the library's communication stream.  ``gathered``: on ``dst`` a list of
        ``nranks`` stacked tensors (n, H, W, 2) (index = source rank; the entry for ``dst`` may be the tensor the
        ``flows`` views come from), None elsewhere.  Ordered on ``stream`` like run_device; nothing blocks the host."""
        import torch
        from .cudaoptflow import _image_from_tensor
        n, a, b, f = self._arrays(pairs, flows, _image_from_tensor)
        g = None
        if comm.rank == dst:
            if gathered is None or len(gathered) != comm.nranks:
                raise ValueError("rank dst needs one receive tensor per rank")
            g = (self._libmod.b2f_image * (n * comm.nranks))()
            for r, t in enumerate(gathered):
                for i in range(n):
                    g[r * n + i] = _image_from_tensor(t[i], True)
        if stream is None:
            stream = torch.cuda.current_stream()
        st = self._lib.b2f_batch_run_device_gather(self._b, n, a, b, f, comm._c, dst, g,
                                                   self._C.c_void_p(stream.cuda_stream))
        if st != 0:
            raise self._libmod.B2FError(st)

    def launches(self) -> int:
        return int(self._lib.b2f_batch_launches(self._b))

    def reset_stats(self) -> None:
        self._lib.b2f_batch_reset_stats(self._b)


class NativeComm:
    """NCCL communicator owned by libb200flow.so (csrc/comm.cu) for the per-pair result gather of
    ``NativeFlowBatch.run_device_gather``.  One per process / GPU; creation is collective.

        comm = NativeComm.from_torch_distributed()      # id made on rank 0, broadcast through the process group
    """

    def __init__(self, unique_id: bytes, rank: int, nranks: int):
        import ctypes as C
        from . import _lib
        self._C, self._libmod, self._lib = C, _lib, _lib.lib()
        self._c = C.c_void_p()
        buf = C.create_string_buffer(unique_id, 128) if nranks > 1 else None
        st = self._lib.b2f_comm_create(buf, 128, rank, nranks, C.byref(self._c))
        if st != 0:
            self._c = None
            raise _lib.B2FError(st)
        self.rank, self.nranks = rank, nranks

    @staticmethod
    def unique_id() -> bytes:
        import ctypes as C
        from . import _lib
        buf = C.create_string_buffer(128)
        st = _lib.lib().b2f_comm_unique_id(buf, 128)
        if st != 0:
            raise _lib.B2FError(st)
        return buf.raw

    @classmethod
    def from_torch_distributed(cls, group=None):
        """Bootstrap over an initialised torch.distributed process group (any backend): rank 0 creates the NCCL id
        and broadcasts its 128 bytes; every rank then joins on its CURRENT CUDA device.  Failures before the collective
        ncclCommInitRank are agreed on by all ranks first, so nobody is left waiting in it."""
        import torch.distributed as dist
        from . import _lib
        rank, world = dist.get_rank(group), dist.get_world_size(group)
        if world == 1:
            return cls(b"", 0, 1)
        avail = [None] * world
        dist.all_gather_object(avail, int(_lib.lib().b2f_comm_available()), group=group)
        if not all(avail):
            raise RuntimeError("libnccl.so.2 cannot be loaded on rank(s) %s" % [r for r, a in enumerate(avail) if not a])
        box = [b""]
        if rank == 0:
            try:
                box = [cls.unique_id()]
            except Exception:  # noqa: BLE001 -- reported below, on every rank
                box = [b""]
        dist.broadcast_object_list(box, src=0, group=group)
        if len(box[0]) != 128:
            raise RuntimeError("rank 0 could not create an NCCL unique id")
        return cls(box[0], rank, world)

    def close(self):
        c, self._c = getattr(self, "_c", None), None
        if c:
            self._lib.b2f_comm_destroy(c)

    __del__ = close


def gather_flows(local_flows, dst: int = 0, group=None, out=None):
    """Result gather to rank ``dst`` (NCCL on GPUs, gloo on CPU tensors).  ``local_flows`` is one
    stacked tensor (n_local, H, W, 2) with the same n_local on every rank.  Returns the list of
    per-rank tensors on ``dst`` (index = rank, i.e. global pair order) and None elsewhere.
    ``out``: optional preallocated list of ``world`` receive tensors on ``dst`` (reused across steps)."""
    import torch.distributed as dist
    if not dist.is_initialized() or dist.get_world_size(group) == 1:
        return [local_flows]
    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    if rank != dst:
        out = None
    elif out is None:
        out = [local_flows.new_empty(local_flows.shape) for _ in range(world)]
    dist.gather(local_flows, out, dst=dst, group=group)
    return out
