"""One rank of the "glb" backend on FP8 tensors: usage pg_fp8_worker.py INIT_FILE RANK SIZE {cpu,cuda}.
Inputs are small integers, so every result is exact in both formats."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
os.environ.setdefault("CUDA_MODULE_LOADING", "EAGER")

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

import gloo_b200.parallel.process_group  # noqa: E402,F401  (registers "glb")


def main():
    path, rank, size, where = sys.argv[1], int(sys.argv[2]), int(sys.argv[3]), sys.argv[4]
    if where == "cuda":
        dev = torch.device("cuda", rank % torch.cuda.device_count())
        torch.cuda.set_device(dev)
    else:
        dev = torch.device("cpu")
    dist.init_process_group("glb", init_method=f"file://{path}", rank=rank, world_size=size)
    tri = size * (size + 1) // 2
    for fmt in (torch.float8_e4m3fn, torch.float8_e5m2):
        for n in (5, 4099):
            t = torch.full((n,), float(rank + 1), device=dev).to(fmt)
            dist.all_reduce(t)
            assert bool((t.float() == tri).all()), (fmt, n, t.float()[:4])
        # AVG: 2 * size / size = 2 (fused scale on CUDA, a float32 round trip on the host)
        t = torch.full((33,), 2.0, device=dev).to(fmt)
        dist.all_reduce(t, op=dist.ReduceOp.AVG)
        assert bool((t.float() == 2.0).all()), (fmt, t.float()[:4])
        t = torch.full((7,), float(rank + 1), device=dev).to(fmt)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        assert bool((t.float() == size).all())
        flat = torch.zeros(size * 3, device=dev).to(fmt)
        dist.all_gather_into_tensor(flat, torch.full((3,), float(rank), device=dev).to(fmt))
        assert flat.float().tolist() == [float(r) for r in range(size) for _ in range(3)]
        inp = (torch.arange(size * 2, dtype=torch.float32, device=dev) + 4 * rank).to(fmt)
        out = torch.zeros(size * 2, device=dev).to(fmt)
        dist.all_to_all_single(out, inp)
        want = torch.tensor([4.0 * r + 2 * rank + k for r in range(size) for k in range(2)]).to(fmt).float()
        assert out.float().tolist() == want.tolist()  # the bytes as sent
        if where == "cpu":
            out = torch.zeros(2, device=dev).to(fmt)
            dist.reduce_scatter_tensor(out, torch.full((2 * size,), 2.0).to(fmt), op=dist.ReduceOp.AVG)
            assert out.float().tolist() == [2.0, 2.0], out.float().tolist()
            b = torch.full((9,), float(rank), device=dev).to(fmt)
            dist.broadcast(b, src=size - 1)
            assert bool((b.float() == size - 1).all())
    if where == "cuda":
        torch.cuda.synchronize()
    dist.barrier()
    dist.destroy_process_group()
    print(f"rank {rank} ok", flush=True)


if __name__ == "__main__":
    main()
