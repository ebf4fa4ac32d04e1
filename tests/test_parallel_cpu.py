"""Host-side multi-rank logic on CPU (gloo, world_size 2): view sharding and the flat gradient
arena all-reduce of sugar_b200.parallel.  No CUDA involved."""
import os
import sys

import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from sugar_b200 import parallel
    P, M = 50, 16
    g = torch.Generator().manual_seed(100 + rank)
    shapes = dict(means3D=(P, 3), shs=(P, M, 3), opacities=(P, 1), scales=(P, 3), rotations=(P, 4))
    params = {k: torch.zeros(s, requires_grad=True) for k, s in shapes.items()}
    for k, p in params.items():
        p.grad = torch.randn(p.shape, generator=g)
    local = {k: p.grad.clone() for k, p in params.items()}
    arena = parallel.GradArena(P, M, "cpu")
    arena.all_reduce_from(params, 1.0 / world)
    arena.unpack_to(params)
    # numpy, not torch tensors: a tensor travels as a file descriptor that the parent must still be able
    # to open after this process has exited (ConnectionResetError when the worker wins the race)
    q.put((rank, {k: v.numpy().copy() for k, v in local.items()},
           {k: p.grad.detach().numpy().copy() for k, p in params.items()}, parallel.shard_views(8, rank, world)))
    dist.barrier()
    dist.destroy_process_group()
    q.close()
    q.join_thread()  # the feeder thread has written everything before the process exits


def test_arena_allreduce_gloo_world2():
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    import socket
    with socket.socket() as sk:  # a free port for the rendezvous
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = [q.get(timeout=120) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    res.sort(key=lambda r: r[0])
    for k in res[0][1]:
        mean = (res[0][1][k] + res[1][1][k]) / world
        for r in res:
            assert torch.allclose(torch.from_numpy(r[2][k]), torch.from_numpy(mean), atol=1e-7), k
    assert res[0][3] == [0, 2, 4, 6] and res[1][3] == [1, 3, 5, 7]
    assert 59 * 50 == sum(n for _, n in __import__("sugar_b200.parallel", fromlist=["x"]).GradArena(50, 16, "cpu").offsets.values())


def _rg_worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from sugar_b200 import parallel
    x = torch.arange(6, dtype=torch.float32).reshape(2, 3).requires_grad_(True)
    y = parallel.reduce_grad(x * 2.0, scale=0.5)          # not a leaf: the sum happens on its gradient
    (y * (rank + 1)).sum().backward()
    q.put((rank, x.grad.numpy().copy()))
    dist.barrier()
    dist.destroy_process_group()
    q.close()
    q.join_thread()


def test_reduce_grad_sums_incoming_gradient_gloo_world2():
    """parallel.reduce_grad: identity forward; backward = all-reduce(sum) of the incoming gradient x scale, so
    per-view losses that do not pass through the rasterizer still reach the parameters summed over the ranks."""
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    import socket
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    procs = [ctx.Process(target=_rg_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=120) for _ in range(world))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    import numpy as np
    want = np.full((2, 3), (1 + 2) * 0.5 * 2.0, np.float32)  # sum over ranks of (rank+1), x scale, x d(2x)/dx
    for r in range(world):
        assert np.allclose(res[r], want), (r, res[r])


def test_reduce_grad_single_process_is_identity_times_scale():
    from sugar_b200 import parallel
    x = torch.ones(4, requires_grad=True)
    parallel.reduce_grad(x, scale=0.25).sum().backward()
    assert torch.allclose(x.grad, torch.full((4,), 0.25))
    assert parallel.shard_views(5, 1, 2) == [1, 3]


def test_exchange_policy_without_a_process_group(monkeypatch):
    """ViewParallel.uses_peer_memory: "auto" follows PEER_AUTO_WORLDS / SGR_PEER_WORLDS, True / False force, and the cases
    the peer exchange does not serve (no SH factors, precomputed covariances, > 16 chunks) go to NCCL."""
    from sugar_b200 import parallel
    assert parallel.PEER_AUTO_WORLDS == (2,)
    vp = parallel.ViewParallel()                       # "auto", world size 1 here
    assert vp.peer == "auto" and not vp.enabled()
    assert not vp.uses_peer_memory(16, False)
    monkeypatch.setenv("SGR_PEER_WORLDS", "1, 4")
    assert vp.uses_peer_memory(16, False)
    assert not vp.uses_peer_memory(16, True) and not vp.uses_peer_memory(0, False)
    monkeypatch.delenv("SGR_PEER_WORLDS")
    assert parallel.ViewParallel(peer=True).uses_peer_memory(16, False)
    assert not parallel.ViewParallel(peer=False, force=True).uses_peer_memory(16, False)
    assert parallel.ViewParallel(force=True).uses_peer_memory(16, False)          # forced single-rank runs (tests)
    assert not parallel.ViewParallel(peer=True, sh_factors=False).uses_peer_memory(16, False)
    assert not parallel.ViewParallel(peer=True, chunks=17).uses_peer_memory(16, False)


def test_record_ownership_of_producer_and_reducer_agree():
    """Peer exchange: the per-Gaussian pass sends CTA b of a chunk's nb CTAs to rank  b * N // nb  (sgr_backward.cu,
    PreBwdArgs::stage_tab); sgr_peer_reduce_records_synced lets rank r sum the blocks [ceil(r nb / N), ceil((r + 1) nb / N))
    (sgr_peer.cu).  Both are restated here: every block has exactly one owner and the two formulas name the same one."""
    for N in (1, 2, 3, 4, 7, 8, 16, 64):
        for nb in (1, 2, 3, 5, 8, 63, 64, 65, 1000, 11719, 46875):
            owner = [b * N // nb for b in range(nb)]
            seen = [0] * nb
            for r in range(N):
                bs, be = (nb * r + N - 1) // N, (nb * (r + 1) + N - 1) // N
                assert 0 <= bs <= be <= nb
                for b in range(bs, be):
                    assert owner[b] == r, (N, nb, b)
                    seen[b] += 1
            assert all(s == 1 for s in seen), (N, nb)


def _peer_setup_worker(rank, world, port, q, fail_rank):
    """Set-up of the peer-memory exchange (parallel._PeerState / ViewParallel._peer_state) over gloo with a stand-in for
    the five sgr_peer_* entry points: addresses are just numbers, nothing touches CUDA."""
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    import contextlib
    from sugar_b200 import parallel

    class FakeLib:
        def __init__(self):
            self.log = []

        def sgr_peer_flag_bytes(self):
            return 16384

        def sgr_peer_alloc(self, nbytes, out):
            if rank == fail_rank:
                return -1
            self.log.append(("alloc", int(nbytes)))
            out._obj.value = 0x100000000 * (rank + 1)
            return 0

        def sgr_peer_export(self, ptr, handle):
            handle[0], handle[1] = rank + 1, 0xAB          # "IPC handle": who owns the allocation
            return 0

        def sgr_peer_import(self, handle, out):
            self.log.append(("import", int(handle[0])))
            out._obj.value = 0x100000000 * int(handle[0]) + 0x1000   # the owner's buffer as mapped HERE
            return 0

        def sgr_peer_close(self, ptr):
            self.log.append(("close", int(ptr)))
            return 0

        def sgr_peer_free(self, ptr):
            self.log.append(("free", int(ptr)))
            return 0

    def check(status):
        if status:
            raise RuntimeError("stand-in library error")

    fake, dev, P = FakeLib(), torch.device("cpu"), 1000
    real = (parallel.torch.cuda.device, parallel.torch.cuda.synchronize, parallel.torch.as_tensor)
    parallel.torch.cuda.device = lambda d: contextlib.nullcontext()
    parallel.torch.cuda.synchronize = lambda d=None: None
    parallel.torch.as_tensor = lambda obj, device=None: torch.zeros(obj.__cuda_array_interface__["shape"])
    try:
        vp = parallel.ViewParallel(peer="auto")
        st = vp._peer_state(fake, check, P, dev)
    finally:
        parallel.torch.cuda.device, parallel.torch.cuda.synchronize, parallel.torch.as_tensor = real
    out = {"rank": rank, "ok": st is not None, "peer": vp.peer, "error": vp.peer_error, "log": fake.log}
    if st is not None:
        out.update(flag_tab=st.flag_tab.tolist(), stage_tab=st.stage_tab.tolist(), rec_tab=st.rec_tab.tolist(),
                   S_tab=st.S_tab.tolist(), F_tab=[t.tolist() for t in st.F_tab], R_ptr=st.R_ptr, base=st.base,
                   off=dict(st.off), stride=st.stage_stride, imported=list(st.imported))
    q.put(out)
    dist.barrier()
    dist.destroy_process_group()
    q.close()
    q.join_thread()


def _run_peer_setup(fail_rank):
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    import socket
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    procs = [ctx.Process(target=_peer_setup_worker, args=(r, world, port, q, fail_rank)) for r in range(world)]
    for p in procs:
        p.start()
    res = sorted((q.get(timeout=120) for _ in range(world)), key=lambda r: r["rank"])
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    return res


def test_peer_state_setup_gloo_world2():
    """Both ranks map each other's buffer: the pointer tables name rank j's regions as seen from each rank."""
    res = _run_peer_setup(fail_rank=-1)
    for me, r in enumerate(res):
        other = 1 - me
        assert r["ok"] and r["peer"] == "auto" and r["error"] is None
        own, mapped = 0x100000000 * (me + 1), 0x100000000 * (other + 1) + 0x1000
        bases = [own, mapped] if me == 0 else [mapped, own]
        assert r["base"] == own and r["imported"] == [mapped] and ("import", other + 1) in r["log"]
        assert r["flag_tab"] == bases
        off, rb = r["off"], r["stride"]
        assert r["S_tab"] == [b + off["S"] for b in bases]
        assert r["F_tab"] == [[b + off["F0"] for b in bases], [b + off["F1"] for b in bases]]
        # rank j's staging array number `me` receives my records; my own arrays 0..1 are what my reduce reads
        assert r["stage_tab"] == [b + off["STAGE"] + me * rb for b in bases]
        assert r["rec_tab"] == [own + off["STAGE"] + j * rb for j in range(2)]
        assert r["R_ptr"] == r["rec_tab"][me] == r["stage_tab"][me]
        assert off["F0"] % 256 == 0 and off["S"] % 256 == 0 and off["STAGE"] % 256 == 0 and rb % 256 == 0
        assert r["log"][0][0] == "alloc" and r["log"][0][1] == off["STAGE"] + 2 * rb


def test_peer_state_setup_falls_back_on_every_rank_when_one_cannot_allocate():
    """Rank 1 cannot allocate: it still joins the handle all-gather, rank 0 sees the zero handle, frees its own buffer
    without mapping anything, and BOTH fall back to the NCCL exchange (no rank is left waiting in a collective)."""
    res = _run_peer_setup(fail_rank=1)
    for r in res:
        assert not r["ok"] and r["peer"] is False and r["error"]
    assert ("free", 0x100000000) in res[0]["log"] and not any(c[0] == "import" for c in res[0]["log"])
    assert res[1]["log"] == []
