"""View-sharded multi-GPU step: one process per GPU, Gaussian parameters replicated, each rank renders its
own view(s); the per-Gaussian gradients of the rasterizer are summed over the ranks INSIDE the op's backward,
overlapped with it, over NCCL (NVLink 5 / NVSwitch) -- SURVEY.md section 8e.  The reference is strictly
1 view / 1 GPU (sugar_trainers/coarse_sdf.py:98,507), so this is new behaviour: loss = sum (or mean) over the
batch's views.

    vp = ViewParallel(scale=1.0 / world)          # one per model; owns the exchange state (no globals)
    with vp.context():                            # or: _C.use_context(vp.ctx)
        image, radii = rasterizer(means3D=..., shs=..., ...)      # the drop-in module, unchanged
        loss(image).backward()                    # gradients arrive already summed over the ranks

What the backward does when an exchange is attached (sugar_b200/_C.py, include/sugar_b200.h).  Common to both
implementations:

  * SH factor mode (default): 192 of the 236 B/Gaussian of gradients are dL_dsh, and each view's dL_dsh is an
    outer product  basis(dir_view)[M] x dL/dRGB[3]  (backward.cu:20-139).  Only the 12-byte factors dL/dRGB (the
    blend pass's colour accumulators, final when it ends) and the camera positions cross the wire; the summed
    dL_dsh is rebuilt from them.
  * The other 11 floats (means3D 3, opacity 1, scales 3, rotations 4) are written by the per-Gaussian pass as
    one 44-byte record per Gaussian, in `chunks` Gaussian ranges; each range is exchanged while the next one is
    computed, so only the last range's exchange is exposed.
  * Because the sum happens on the rasterizer's OUTPUT gradients, anything in front of the op (exp / sigmoid /
    normalize / cat of SuGaR's raw parameters) just backpropagates the summed gradient: inputs need not be
    leaves, and several backwards per step (several views per rank) each do their own exchange.
  * dL_dmeans2D and radii are per-view densification statistics (sugar_scene/sugar_densifier.py:156-164) and
    are NOT summed here: each rank accumulates them locally, and densify.Densifier(group=...) reduces them and
    shares the split's normals when it densifies, so the replicated parameters stay replicas.
  * Losses that reach the parameters without going through the rasterizer (density / SDF regularisation,
    evaluated per view on its rank) are summed with `reduce_grad(tensor)`: identity in the forward, all-reduce of
    the incoming gradient in the backward.

Over peer memory (`peer=True`, or "auto" on PEER_AUTO_WORLDS; csrc/sgr_peer.cu, DESIGN.md section 5a): the ranks map
each other's exchange buffers with CUDA IPC once; a backward is then ONE C call, no NCCL call, no host callback:

    main   blend ─ signal ─ wait(all ranks) ─ per-Gaussian pass <MULTI> chunk 0 ─ chunk 1 ─ ...       (+ signals on a 3rd stream)
                                               TMA-loads the other ranks' factor blocks (NVLink), writes the SUMMED dL_dsh,
                                               TMA-stores its records into the staging array of the rank that owns them
    side                                       [chunk 0 signalled] reduce owned slice, post sums to every rank ─ split ─ ...

Over NCCL (`peer=False`, and on the world sizes "auto" does not give to the peer exchange; DESIGN.md section 5b):

    blend pass ─► hook BLEND_DONE ─► per-Gaussian pass, chunk 0 ─► hook ─► chunk 1 ─► hook ─► ... ─► finalize
                     │ all-gather of the SH factors                │ all-reduce of chunk 0's records
                     └─ runs underneath the per-Gaussian pass       └─ runs underneath chunk 1 ...

    the per-Gaussian pass does not write dL_dsh; `sgr_view_grad_finalize` rebuilds the sum over the views from the
    gathered factors and splits the reduced records into the arrays autograd expects (and applies `scale`).

`GradArena` is the plain utility underneath the CPU tests and for callers that prefer one explicit all-reduce
of leaf gradients after the backward (236 B/Gaussian, not overlapped).
"""
import contextlib
import ctypes as C
import os
from typing import Dict, Optional

import torch
import torch.distributed as dist

ARENA_FIELDS = ("means3D", "opacities", "scales", "rotations", "shs")


def shard_views(num_views: int, rank: int, world: int):
    """Views rendered by `rank`: {rank, rank+world, ...} (round-robin keeps ranks balanced)."""
    return list(range(rank, num_views, world))


def _world(group=None) -> int:
    return dist.get_world_size(group) if (dist.is_available() and dist.is_initialized()) else 1


class _ReduceGrad(torch.autograd.Function):
    @staticmethod
    def forward(ctx, t, scale, group):
        ctx.scale, ctx.group = scale, group
        return t.view_as(t)

    @staticmethod
    def backward(ctx, g):
        g = g.contiguous().clone()
        if _world(ctx.group) > 1:
            dist.all_reduce(g, op=dist.ReduceOp.SUM, group=ctx.group)
        if ctx.scale != 1.0:
            g.mul_(ctx.scale)
        return g, None, None


def reduce_grad(t: torch.Tensor, scale: float = 1.0, group=None) -> torch.Tensor:
    """Identity whose backward sums the incoming gradient over the ranks (x scale): wrap the tensors that feed
    per-view losses which do not go through the rasterizer."""
    return _ReduceGrad.apply(t, scale, group)


_SLOT_BLEND, _SLOT_CHUNK0, _SLOT_REDUCED0, _PEER_MAX_CHUNKS = 0, 1, 17, 16   # flag slots (csrc/sgr_peer.cu)
PEER_AUTO_WORLDS = (2,)   # beyond two ranks the peer pass waits on several remote factor blocks per CTA (DESIGN.md 5b)


def _peer_auto_worlds():
    e = os.environ.get("SGR_PEER_WORLDS")
    return tuple(int(x) for x in e.split(",") if x.strip()) if e else PEER_AUTO_WORLDS


class _DevMem:
    """A raw device range as seen by torch.as_tensor (the CUDA array interface)."""

    def __init__(self, ptr: int, nfloats: int):
        self.__cuda_array_interface__ = {"shape": (nfloats,), "typestr": "<f4", "data": (ptr, False), "version": 2}


class _PeerState:
    """One rank's peer-visible exchange buffer for P Gaussians and the mappings of the other ranks' buffers
    (layout: csrc/sgr_peer.cu).  Building it is collective (the IPC handles travel in one all-gather)."""

    def __init__(self, lib, check, P, rank, world, group, dev, nstage=None):
        self.P, self.rank, self.world, self.dev, self.seq = P, rank, world, dev, 0
        nstage = nstage or world
        up = lambda n: (n + 255) // 256 * 256
        fl, fb, rb = int(lib.sgr_peer_flag_bytes()), up(4 * (3 * P + 4)), up(4 * 11 * P + 64)
        off = {"flags": 0, "F0": fl, "F1": fl + fb, "S": fl + 2 * fb, "STAGE": fl + 2 * fb + rb}
        self.off, self.stage_stride = off, rb
        total = off["STAGE"] + nstage * rb
        self.imported, self.base, self.F_local = [], 0, []
        try:
            self._build(lib, check, P, rank, world, group, dev, nstage, off, rb, total)
        except BaseException:
            self.close(lib)   # nothing half-mapped or allocated is left behind
            raise
        self._streams = None

    def _build(self, lib, check, P, rank, world, group, dev, nstage, off, rb, total):
        with torch.cuda.device(dev):
            # A rank that cannot allocate / export still takes part in the handle all-gather (with an all-zero handle):
            # every rank then fails the same way and the caller's agreement step falls back to NCCL on all of them.
            handle, local_err = (C.c_ubyte * 64)(), None
            try:
                base = C.c_void_p()
                check(lib.sgr_peer_alloc(total, C.byref(base)))
                self.base = base.value
                check(lib.sgr_peer_export(self.base, handle))
            except Exception as e:
                local_err, handle = e, (C.c_ubyte * 64)()
            bases = [self.base]
            if world > 1:
                mine = torch.tensor(list(bytes(handle)), dtype=torch.uint8, device=dev)
                every = torch.empty(world * 64, dtype=torch.uint8, device=dev)   # flat: the form every backend takes
                dist.all_gather_into_tensor(every, mine, group=group)
                every = every.view(world, 64).cpu()
                if local_err is None and not bool(every.any(dim=1).all()):
                    local_err = RuntimeError("a peer rank could not allocate / export its exchange buffer")
                bases = []
                for j in range(world):
                    if local_err is not None:
                        break
                    if j == rank:
                        bases.append(self.base)
                        continue
                    h = (C.c_ubyte * 64)(*every[j].tolist())
                    q = C.c_void_p()
                    check(lib.sgr_peer_import(h, C.byref(q)))
                    self.imported.append(q.value)
                    bases.append(q.value)
            if local_err is not None:
                raise local_err
            i64 = lambda ptrs: torch.tensor(ptrs, dtype=torch.int64, device=dev)
            tab = lambda name: i64([b + off[name] for b in bases])
            self.flag_tab, self.S_tab = tab("flags"), tab("S")
            self.F_tab = [tab("F0"), tab("F1")]
            # records: rank j's staging array number `rank` receives what this rank's per-Gaussian pass computes for the
            # blocks j owns; this rank's own arrays 0 .. world-1 receive every rank's records of the blocks IT owns
            self.stage_tab = i64([b + off["STAGE"] + rank * rb for b in bases])
            self.rec_tab = i64([self.base + off["STAGE"] + j * rb for j in range(nstage)])
            self.flags_ptr, self.S_ptr = self.base, self.base + off["S"]
            self.counters_ptr = self.base + 63 * 64 * 4   # flag row 63: the fused kernels' CTA counters (local use only)
            self.R_ptr = self.base + off["STAGE"] + rank * rb
            self.F_local = [torch.as_tensor(_DevMem(self.base + off[k], 3 * P + 4), device=dev) for k in ("F0", "F1")]
            torch.cuda.synchronize(dev)

    def streams(self, dev):
        """(side stream of the record exchange, stream of the backward's own signal kernels, start event)"""
        if self._streams is None:
            self._streams = (torch.cuda.Stream(device=dev, priority=-1), torch.cuda.Stream(device=dev, priority=-1),
                             torch.cuda.Event())
        return self._streams

    def close(self, lib):
        for q in self.imported:
            lib.sgr_peer_close(q)
        self.imported = []
        self.F_local = []
        if self.base:
            lib.sgr_peer_free(self.base)
            self.base = 0


class ViewParallel:
    """Exchange state of one model's view-parallel step (see the module docstring).

    sh_factors  exchange 12 B/Gaussian/view SH factors instead of all-reducing dL_dsh (default True)
    chunks      Gaussian ranges of the per-Gaussian pass; each range's all-reduce overlaps the next range
    scale       multiplies every summed gradient (1/num_views for a mean over the batch)
    force       run the record / finalize path even with a single rank (tests; no collectives are issued)
    side_stream (NCCL exchange) finalize range c on a second (high-priority) stream as soon as its collective is done,
                concurrently with the per-Gaussian pass of the ranges behind it, instead of after the whole pass
    peer        "auto" (default): the peer-memory exchange on the world sizes in PEER_AUTO_WORLDS (a design
                choice, not timed on H100; override SGR_PEER_WORLDS), NCCL elsewhere or if the ranks cannot map each other's memory; True / False
    peer_timeout_s  a flag wait of the peer exchange traps after this long (a lost rank must not hang the others)
    taper       peer exchange: chunk c+1 is half the size of chunk c (the exposed tail is the last chunk's reduce + split)
    """

    def __init__(self, sh_factors: bool = True, chunks: int = 4, scale: float = 1.0, group=None, force: bool = False,
                 side_stream: bool = False, peer="auto", peer_timeout_s: float = 8.0, taper: bool = True):
        from . import _C
        self.sh_factors, self.chunks, self.scale, self.group, self.force = bool(sh_factors), int(chunks), float(scale), group, force
        self.side_stream = bool(side_stream)
        self.peer, self.peer_timeout_s, self.taper = peer, float(peer_timeout_s), bool(taper)
        self.peer_error = None   # why "auto" fell back to the NCCL exchange, if it did
        self._peer_states = {}   # (P, device) -> _PeerState
        self._emulated = ()      # tests: other ranks whose record slices this process reduces as well (see tests/test_gpu_parallel.py)
        self._side = {}     # device -> (stream, [events])
        self.ctx = _C.Context()
        self.ctx.exchange = self
        self.stats = {"backwards": 0, "collectives": 0}

    # -- selection ---------------------------------------------------------------------------------------
    @contextlib.contextmanager
    def context(self):
        from . import _C
        with _C.use_context(self.ctx):
            yield self

    def enabled(self) -> bool:
        return self.force or _world(self.group) > 1

    def uses_peer_memory(self, M: int, has_cov_precomp: bool) -> bool:
        """Peer mode serves the common case: SH colours exchanged as factors, covariances computed in the op.
        peer=True: always (raises if the buffers cannot be mapped); False: never; "auto" (default): on the world sizes
        the design gives to it (PEER_AUTO_WORLDS, not timed on H100; override: SGR_PEER_WORLDS="2,4,8"),
        falling back to NCCL if the ranks cannot map each other's memory."""
        if not self.peer or not M or not self.sh_factors or has_cov_precomp or self.chunks > _PEER_MAX_CHUNKS:
            return False
        if self.peer == "auto" and not self.force:
            return _world(self.group) in _peer_auto_worlds()
        return True

    # -- the exchange, driven from _C.rasterize_gaussians_backward ------------------------------------------
    def run_backward(self, launch, bufs, P, M, degree, means3D, campos, has_cov_precomp):
        """`launch(plan, *, dL_dcolors=ptr, dL_dsh=ptr)` enqueues this view's sgr_rasterize_backward_staged under
        `plan`, with the two gradient outputs optionally redirected; `bufs`: dict of the gradient tensors +
        "records" f32[P,11].  Returns nothing: bufs hold the reduced gradients when the enqueued work completes."""
        from ._lib import SGR_STAGE_BLEND_DONE, SGR_STAGE_CHUNK_DONE, SgrBackwardPlan, SgrStageHook, check, lib
        if self.uses_peer_memory(M, has_cov_precomp):
            st = self._peer_state(lib, check, P, means3D.device)
            if st is not None:
                return self._run_backward_peer(st, launch, bufs, P, means3D, campos)
        if "records" not in bufs:   # "auto" just fell back to the NCCL exchange: the arena was sized for peer mode
            bufs["records"] = torch.empty((P, 11), dtype=torch.float32, device=means3D.device)
        world = _world(self.group)
        multi = world > 1
        dev = means3D.device
        factor = bool(M) and self.sh_factors
        nchunks = max(1, self.chunks)
        taper = 0   # equal chunks here: the halving taper is for the peer exchange's exposed tail (not timed on H100)
        if getattr(self, "_ranges_key", None) != (P, nchunks, taper):
            self._ranges_key = (P, nchunks, taper)
            self._ranges = [self._range(lib, check, P, nchunks, c, taper) for c in range(nchunks)]
        ranges = self._ranges
        pending = {c: [] for c in range(nchunks)}
        early = []
        failure = []
        side = chunk_done = None
        if self.side_stream:
            if dev not in self._side:
                self._side[dev] = (torch.cuda.Stream(device=dev, priority=-1), [])
            side, chunk_done = self._side[dev]
            while len(chunk_done) < nchunks:
                chunk_done.append(torch.cuda.Event())
        stride = 3 * P + 4   # a view's factor block: dL/dRGB [P,3] followed by its camera position (+ 1 pad)
        d_all = None
        if factor:
            block = bufs["colors_block"]
            block[3 * P:3 * P + 3].copy_(campos.reshape(3))   # rides in the same all-gather as the factors
            d_all = self._gather_buffer(world, stride, dev) if multi else block.view(1, stride)

        def on_stage(_ctx, stage):
            try:
                if stage == SGR_STAGE_BLEND_DONE:  # dL_dcolors is final
                    if factor and multi:
                        early.append(dist.all_gather_into_tensor(d_all, bufs["colors_block"], group=self.group,
                                                                 async_op=True))
                    elif not M and multi:  # colours were precomputed: their gradient is an ordinary sum
                        early.append(dist.all_reduce(bufs["colors"], group=self.group, async_op=True))
                elif stage >= SGR_STAGE_CHUNK_DONE and side is not None and not multi:
                    # what the side stream's finalize of this range waits for
                    chunk_done[stage - SGR_STAGE_CHUNK_DONE].record()
                elif stage >= SGR_STAGE_CHUNK_DONE and multi:
                    c = stage - SGR_STAGE_CHUNK_DONE
                    p0, p1 = ranges[c]
                    if p1 > p0:
                        pending[c].append(dist.all_reduce(bufs["records"][p0:p1], group=self.group, async_op=True))
                        if M and not factor:
                            pending[c].append(dist.all_reduce(bufs["sh"][p0:p1], group=self.group, async_op=True))
                        if has_cov_precomp:
                            pending[c].append(dist.all_reduce(bufs["cov3D"][p0:p1], group=self.group, async_op=True))
            except BaseException as e:  # never unwind through the C frame
                failure.append(e)

        cb = SgrStageHook(on_stage)
        launch(SgrBackwardPlan(hook=cb, num_chunks=nchunks, chunk_taper=taper, reduce_records=bufs["records"].data_ptr()))
        if failure:
            raise failure[0]
        main = torch.cuda.current_stream(dev)
        d_ptr = d_all.data_ptr() if factor else None
        # stream-ordered waits: the host never blocks.  With a side stream every range is finalized as soon as ITS
        # collective is done, while the caller's stream is still in the per-Gaussian pass of later ranges.
        with (torch.cuda.stream(side) if side is not None else contextlib.nullcontext()):
            cur = side if side is not None else main
            for h in early:
                h.wait()
            for c in range(nchunks):
                p0, p1 = ranges[c]
                for h in pending[c]:
                    h.wait()
                if side is not None and not multi:
                    side.wait_event(chunk_done[c])   # single rank: the range's producer is the caller's stream itself
                if p1 > p0:
                    check(lib.sgr_view_grad_finalize(
                        P, p0, p1, M, degree, world, means3D.data_ptr(), (d_ptr + 12 * P) if factor else None, d_ptr,
                        stride, stride, bufs["sh"].data_ptr() if factor else None, bufs["records"].data_ptr(), self.scale,
                        bufs["means3D"].data_ptr(), bufs["opacity"].data_ptr(), bufs["scales"].data_ptr(),
                        bufs["rotations"].data_ptr(), cur.cuda_stream))
        if side is not None:
            main.wait_stream(side)   # everything after the backward (and the allocator's reuse of bufs) is ordered behind
        if self.scale != 1.0:  # what the finalize kernel did not touch
            if M and not factor:
                bufs["sh"].mul_(self.scale)
            if not M:
                bufs["colors"].mul_(self.scale)
            if has_cov_precomp:
                bufs["cov3D"].mul_(self.scale)
        self.stats["backwards"] += 1
        self.stats["collectives"] += len(early) + sum(len(v) for v in pending.values())

    # -- the exchange over peer memory (csrc/sgr_peer.cu): no NCCL call, no host callback in a backward ---------
    def _peer_state(self, lib, check, P, dev):
        key = (P, dev)
        if key not in self._peer_states:
            world = _world(self.group)
            rank = dist.get_rank(self.group) if world > 1 else 0
            st, err = None, None
            try:
                st = _PeerState(lib, check, P, rank, world, self.group, dev, nstage=getattr(self, "_nstage", None))
            except Exception as e:  # no IPC / no peer access on this box: every rank must take the same branch
                err = e
            if world > 1:
                ok = torch.tensor([0 if st is None else 1], device=dev, dtype=torch.int32)
                dist.all_reduce(ok, op=dist.ReduceOp.MIN, group=self.group)
                if int(ok.item()) == 0:
                    if st is not None:
                        st.close(lib)
                    st = None
            if st is None:
                if self.peer != "auto":
                    raise RuntimeError(f"peer-memory exchange unavailable: {err!r}")
                self.peer, self.peer_error = False, repr(err) if err else "a peer rank could not map the buffers"
            self._peer_states[key] = st
        return self._peer_states[key]

    def _run_backward_peer(self, st, launch, bufs, P, means3D, campos):
        from ._lib import SgrBackwardPlan, SgrPeerPlan
        dev = means3D.device
        world, rank = st.world, st.rank
        nchunks = max(1, self.chunks)
        taper = int(self.taper)
        st.seq += 1
        seq, par = st.seq, st.seq & 1
        main = torch.cuda.current_stream(dev)
        B, Csig, ev = st.streams(dev)
        F = st.F_local[par]
        F[3 * P:3 * P + 3].copy_(campos.reshape(3))     # the camera position rides behind the factors
        # main stream, all inside the C call: blend -> signal(BLEND) -> wait(BLEND, every rank) -> per-Gaussian pass in
        # chunks: TMA-loads the other ranks' factor blocks over NVLink, writes the summed dL_dsh, TMA-stores each CTA's
        # 44-byte records into the staging array of the rank that owns them -> signal(CHUNK c) after each chunk
        emulate = 0
        for r in self._emulated:
            emulate |= 1 << r
        peer = SgrPeerPlan(peer_flag_tab=st.flag_tab.data_ptr(), peer_nranks=world, peer_rank=rank,
                           peer_slot_blend=_SLOT_BLEND, peer_slot_chunk0=_SLOT_CHUNK0, peer_seq=seq,
                           peer_view_blocks=st.F_tab[par].data_ptr(), peer_flags=st.flags_ptr, peer_dsh_scale=self.scale,
                           peer_timeout_s=self.peer_timeout_s, peer_record_stages=st.stage_tab.data_ptr(),
                           peer_signal_stream=Csig.cuda_stream, peer_side_stream=B.cuda_stream,
                           peer_rec_tab=st.rec_tab.data_ptr(), peer_sum_tab=st.S_tab.data_ptr(), peer_sums=st.S_ptr,
                           peer_slot_reduced0=_SLOT_REDUCED0, peer_emulate_ranks=emulate)
        plan = SgrBackwardPlan(num_chunks=nchunks, chunk_taper=taper, reduce_records=st.R_ptr, peer=C.pointer(peer))
        # ... and on the side stream, also enqueued by the C call, chunk by chunk underneath the per-Gaussian pass of the
        # later chunks: [wait(CHUNK c, every rank) -> sum the slice this rank owns over the staging arrays (local loads)
        # -> store the sums into every rank's S (posted NVLink writes) -> signal(REDUCED c)] as ONE kernel, then behind
        # the next chunk's reduce: wait(REDUCED c) -> split S into the four gradient arrays (x scale)
        # dL_dcolors: the blend pass accumulates straight into the peer-visible factor block; dL_dsh: written by the
        # per-Gaussian pass, summed over ALL views
        launch(plan, dL_dcolors=F.data_ptr(), dL_dsh=bufs["sh"].data_ptr())
        main.wait_stream(B)
        main.wait_stream(Csig)
        self.stats["backwards"] += 1

    def close(self):
        """Unmap / free the peer buffers (collective: every rank calls it).  Optional -- process exit does the same."""
        from ._lib import lib
        for st in self._peer_states.values():
            if st is not None:
                torch.cuda.synchronize(st.dev)
                if st.world > 1:
                    dist.barrier(group=self.group)
                st.close(lib)
        self._peer_states = {}

    def _gather_buffer(self, world, stride, dev):
        """[world, 3P+4] receive buffer of the factor all-gather, kept across backwards (its readers, the finalize
        kernels, are enqueued on the compute stream before the next backward's gather is)."""
        key = (world, stride, dev)
        if getattr(self, "_gather_key", None) != key:
            self._gather_key, self._gather = key, torch.empty((world, stride), dtype=torch.float32, device=dev)
        return self._gather

    @staticmethod
    def _range(lib, check, P, nchunks, c, taper=0):
        p0, p1 = C.c_int32(0), C.c_int32(0)
        check(lib.sgr_backward_chunk_range(P, nchunks, c, taper, C.byref(p0), C.byref(p1)))
        return p0.value, p1.value


def sh_grad_from_factors(means3D: torch.Tensor, campos_all: torch.Tensor, dRGB_all: torch.Tensor, M: int,
                         sh_degree: int, out: torch.Tensor = None) -> torch.Tensor:
    """dL_dsh [P,M,3] = sum_v basis(normalize(means3D - campos_all[v])) (x) dRGB_all[v]  (CUDA kernel)."""
    from ._lib import check, lib, stream
    P, V = means3D.shape[0], campos_all.shape[0]
    if out is None:
        out = torch.empty((P, M, 3), dtype=torch.float32, device=means3D.device)
    assert out.is_contiguous() and out.numel() == P * M * 3 and dRGB_all.is_contiguous() and campos_all.is_contiguous()
    with torch.cuda.device(means3D.device):
        check(lib.sgr_view_grad_finalize(P, 0, P, M, sh_degree, V, means3D.contiguous().data_ptr(), campos_all.data_ptr(),
                                         dRGB_all.data_ptr(), 3 * P, 3, out.data_ptr(), None, 1.0, None, None, None, None,
                                         stream(means3D.device)))
    return out


class GradArena:
    """Flat per-Gaussian gradient buffer [means3D 3 | opacities 1 | scales 3 | rotations 4 | shs 3M] x P for ONE
    explicit all-reduce of leaf gradients after the backward (backend "nccl", or "gloo" in the CPU tests)."""

    def __init__(self, P: int, M: int, device, fields=ARENA_FIELDS):
        widths = {"means3D": 3, "shs": 3 * M, "opacities": 1, "scales": 3, "rotations": 4}
        self.fields = [f for f in fields]
        self.P = P
        self.offsets = {}
        off = 0
        for f in self.fields:
            self.offsets[f] = (off, widths[f] * P)
            off += widths[f] * P
        self.numel = off
        self.device = device
        self._flat = None

    @property
    def flat(self) -> torch.Tensor:
        if self._flat is None:
            self._flat = torch.zeros(self.numel, dtype=torch.float32, device=self.device)
        return self._flat

    def view(self, name: str) -> torch.Tensor:
        o, n = self.offsets[name]
        return self.flat[o:o + n]

    def pack(self, params: Dict[str, torch.Tensor]) -> None:
        for f in self.fields:
            g = params[f].grad
            v = self.view(f)
            if g is None:
                v.zero_()
            else:
                v.copy_(g.reshape(-1))

    def all_reduce_from(self, params: Dict[str, torch.Tensor], scale: float = 1.0, group=None) -> torch.Tensor:
        """Pack the leaves' gradients, sum them over the ranks, scale.  Returns the reduced flat arena."""
        self.pack(params)
        buf = self.flat
        if _world(group) > 1:
            dist.all_reduce(buf, op=dist.ReduceOp.SUM, group=group)
        if scale != 1.0:
            buf.mul_(scale)
        return buf

    def unpack_to(self, params: Dict[str, torch.Tensor]) -> None:
        """Write the reduced gradients back as .grad of the (replicated) parameters."""
        for f in self.fields:
            o, n = self.offsets[f]
            params[f].grad = self.flat[o:o + n].view_as(params[f]).clone()
