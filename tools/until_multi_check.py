"""FullSystem::optimize's exit (gn_iterations_until) with the points sharded over GPUs and the device-side peer exchange, under
torchrun (one rank per GPU):

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29523 tools/until_multi_check.py

Every rank solves the replicated 68x68 system to the same bits, so every rank takes the same exit decision inside its graph and
leaves after the same body. Checked: equal body counts on all ranks, no peer error, the same bits as the host applying LDSO's rule
after every body on a second sharded context, and -- on rank 0 -- the unsharded single-GPU gn_iterations_until run of the whole
window: the same body count, energies to the 2e-3 bar (sharding reorders the accumulation, so the bits differ). Exit code != 0 on mismatch."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from ldso_b200 import capi, synth  # noqa: E402

WINDOW = dict(nF=3, pts_per_frame=250, seed=4)       # young window: budget 15, LDSO's exit fires after body 6


def sharded_ctx(full, win, rank, world, lr):
    ctx = capi.Context(win.w, win.h, win.levels, device=lr)
    ctx.set_stream(torch.cuda.current_stream().cuda_stream)
    ctx.load_synth_window(win)
    counts = [int(np.sum(synth.shard_window(full, r, world).res_target == full.nF - 1)) for r in range(world)]
    ctx.set_shard(int(np.sum(counts[:rank])), int(np.sum(counts)))
    handles = [None] * world
    dist.all_gather_object(handles, ctx.peer_export())
    ctx.peer_connect(rank, world, handles)
    dist.barrier()
    return ctx


def main():
    rank = int(os.environ["RANK"]); world = int(os.environ["WORLD_SIZE"]); lr = int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(lr)
    torch.cuda.set_stream(torch.cuda.Stream())      # a capturable stream: the exit then runs inside the CUDA graph
    dist.init_process_group("nccl", device_id=torch.device("cuda", lr))
    full = synth.make_window(**WINDOW)
    win = synth.shard_window(full, rank, world)
    budget = capi.optimize_iteration_budget(full.nF, 6)
    ok = True

    a = sharded_ctx(full, win, rank, world, lr)
    a.optimize_begin()
    a.gn_iterations_until(0, budget, 1)
    n = a.iterations_run()
    sol_a, e_a = a.last_solution(), a.energy()[0]
    pts_a = a.points()["idepth"]
    ok &= a.peer_error() == 0
    counts = [None] * world
    dist.all_gather_object(counts, n)
    ok &= len(set(counts)) == 1

    b = sharded_ctx(full, win, rank, world, lr)      # LDSO's rule applied on the host after every body
    b.optimize_begin()
    nb = 0
    for k in range(budget):
        b.gn_iterations(k, 1)
        nb += 1
        if b.energy()[1] and k >= 1:
            break
    sol_b, e_b = b.last_solution(), b.energy()[0]
    ok &= b.peer_error() == 0 and nb == n and e_a == e_b and np.array_equal(pts_a, b.points()["idepth"])
    for k in ("lastHS", "lastbS", "lastX"):
        ok &= bool(np.array_equal(sol_a[k], sol_b[k]))
    print(f"rank {rank}: bodies {n} (host rule {nb}), energy {e_a:.6f}, peer error {a.peer_error()}")
    torch.cuda.synchronize(); dist.barrier()

    if rank == 0:
        ref = capi.Context(full.w, full.h, full.levels, device=lr)
        ref.load_synth_window(full)
        ref.optimize_begin()
        ref.gn_iterations_until(0, budget, 1)
        n_ref, e_ref = ref.iterations_run(), ref.energy()[0]
        print(f"unsharded single GPU: bodies {n_ref}, energy {e_ref:.6f}")
        ok &= n_ref == n and abs(e_a - e_ref) <= 2e-3 * abs(e_ref)
        ref.close()
        print("UNTIL_MULTI_CHECK", "OK" if ok else "FAIL", "world", world)
    a.close(); b.close()
    flag = torch.tensor([1 if ok else 0], device="cuda")
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    dist.destroy_process_group()
    sys.exit(0 if int(flag.item()) == 1 else 1)


if __name__ == "__main__":
    main()
