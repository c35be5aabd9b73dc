"""Multi-GPU probe (torchrun, one rank per GPU): row-sharded HGEMM with the NCCL and the fused
(multicast / P2P epilogue) transports, checked against a single-GPU product and timed."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch
import torch.distributed as dist

from leetcuda_b200 import hgemm
from leetcuda_b200.dist import RowShardedHgemm


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    rows, N, K = (int(x) for x in (sys.argv[1:4] if len(sys.argv) > 3 else (8192, 8192, 8192)))
    torch.manual_seed(7)
    a_full = torch.randn(rows * world, K, device=dev, dtype=torch.half)   # same on every rank
    b = torch.randn(K, N, device=dev, dtype=torch.half)
    a_shard = a_full[rank * rows:(rank + 1) * rows].contiguous()
    want = torch.empty(rows * world, N, device=dev, dtype=torch.half)
    for r in range(world):   # single-GPU truth with the same kernel
        hgemm.hgemm(a_full[r * rows:(r + 1) * rows].contiguous(), b, want[r * rows:(r + 1) * rows])
    torch.cuda.synchronize()

    # a second problem (A negated) to check that back-to-back steps do not trample each other's C
    a_shard2 = (-a_shard).contiguous()
    modes = [("nccl", {}), ("fused", {})]                      # fused: epilogue stores to every peer mapping
    if world > 1:
        # epilogue stores through the NVLS multicast mapping (multimem.st; peer stores where the fabric has none)
        modes.append(("fused-direct", {"B200_FUSED_EPILOGUE": "direct"}))
    only = os.environ.get("B200_DIST_PROBE_MODES")
    if only:
        modes = [m for m in modes if m[0] in only.split(",")]
    for name, env in modes:
        os.environ.update(env)
        try:
            sh = RowShardedHgemm(rows, N, K, world, rank, dev, transport="fused" if name.startswith("fused") else "nccl")
            for buf in (sh._bufs or [(sh.c_full,)]):
                buf[0].zero_()
            torch.cuda.synchronize()
            dist.barrier()
            # steps 1..4 alternate the two problems; every result is checked AFTER the next step was
            # issued (the ownership rule of RowShardedHgemm.fused: valid until the call after next)
            ok = True
            prev = None
            for it in range(4):
                out = sh(a_shard if it % 2 == 0 else a_shard2, b)
                if prev is not None:
                    ok = ok and torch.equal(prev[0], want if prev[1] % 2 == 0 else -want)
                prev = (out if sh.transport == "fused" else out.clone(), it)
            torch.cuda.synchronize()
            dist.barrier()
            ok = ok and torch.equal(prev[0], want if prev[1] % 2 == 0 else -want)
            mc = sh._bufs[0][2] if sh._bufs else 0
            for _ in range(3):
                sh(a_shard, b)
            torch.cuda.synchronize()
            dist.barrier()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            iters = 10
            e0.record()
            for _ in range(iters):
                sh(a_shard, b)
            e1.record()
            torch.cuda.synchronize()
            ms = torch.tensor([e0.elapsed_time(e1) / iters], device=dev)
            dist.all_reduce(ms, op=dist.ReduceOp.MAX)
            e0.record()
            for _ in range(iters):
                sh.compute_only(a_shard, b)
            e1.record()
            torch.cuda.synchronize()
            cms = e0.elapsed_time(e1) / iters
            if rank == 0:
                fl = 2.0 * rows * world * N * K
                print(f"[dist x{world}] {name:10s} bit-equal={ok} multicast={'yes' if mc else 'no'} "
                      f"{ms.item():.3f} ms/step {fl / ms.item() / 1e9:.0f} TFLOPS aggregate "
                      f"(compute only {cms:.3f} ms; gather bytes/rank {(world - 1) * rows * N * 2 / 2**20:.0f} MiB)", flush=True)
            okt = torch.tensor([int(ok)], device=dev)
            dist.all_reduce(okt, op=dist.ReduceOp.MIN)
            if rank == 0 and okt.item() != 1:
                print(f"[dist] {name}: MISMATCH on some rank", flush=True)
        except Exception as e:  # noqa
            if rank == 0:
                print(f"[dist] {name} failed: {type(e).__name__}: {str(e)[:300]}", flush=True)
        for k_ in env:
            os.environ.pop(k_, None)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
