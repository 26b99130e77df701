"""CPU, world_size 2 (gloo): the arithmetic of the tensor-parallel split that `-sm tensor` asks of the backend (src/llama-model.cpp:507-518,
610-664 through ggml-backend-meta.cpp:2080-2223), restated with the oracle.

  column-parallel (attn_q|k|v, ffn_gate|up): every rank owns M / n weight ROWS; outputs are concatenated -- exact.
  row-parallel (attn_output, ffn_down): every rank owns K / n of every row (a multiple of the 256-weight block, so the Q8_K activation blocks
      and their integers are those of the full product), computes a partial [N, M] and the partials are ALL-REDUCED.  The one-shot
      all-reduce (allreduce.cu) adds the partials in rank order on every rank, so every rank holds the same bits; against the
      single-device product only the fp32 summation order differs.

The ranks run the oracle on their slice, gloo carries the all-reduce / all-gather -- the same plumbing bench.py --gpus N uses between its ranks."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.oracle import BLOCK_BYTES, Oracle, Q4_K, Q6_K, random_blocks  # noqa: E402


def _worker(rank, world, port, t, M, K, N, out_path):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    orc = Oracle()
    rng = np.random.default_rng(123)                       # every rank draws the same full problem, then keeps its slice
    w = random_blocks(t, M, K, rng)
    x = rng.standard_normal((N, K)).astype(np.float32)
    full = orc.mul_mat(t, w, x)
    bb = BLOCK_BYTES[t]
    # ---- column-parallel: rows [rank * M / world, ...)
    m0, m1 = rank * M // world, (rank + 1) * M // world
    mine = torch.from_numpy(orc.mul_mat(t, np.ascontiguousarray(w[m0:m1]), x))
    parts = [torch.empty(N, (r + 1) * M // world - r * M // world) for r in range(world)]
    dist.all_gather(parts, mine)
    col = torch.cat(parts, dim=1).numpy()
    # ---- row-parallel: k-blocks [rank * nblk / world, ...) of every row
    nblk = K // 256
    b0, b1 = rank * nblk // world, (rank + 1) * nblk // world
    wk = np.ascontiguousarray(w.reshape(M, nblk, bb)[:, b0:b1].reshape(M, (b1 - b0) * bb))
    xk = np.ascontiguousarray(x[:, 256 * b0:256 * b1])
    partial = torch.from_numpy(orc.mul_mat(t, wk, xk))
    gathered = [torch.empty_like(partial) for _ in range(world)]
    dist.all_gather(gathered, partial)
    acc = gathered[0].clone()
    for r in range(1, world):
        acc = acc + gathered[r]                            # rank order, like the one-shot all-reduce
    row = acc.numpy()
    # every rank must hold the same bits
    chk = torch.from_numpy(row.copy())
    dist.broadcast(chk, src=0)
    same = bool(np.array_equal(chk.numpy(), row))
    if rank == 0:
        np.savez(out_path, full=full, col=col, row=row, same=np.array([same]))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("t,M,K,N", [(Q4_K, 96, 1024, 3), (Q6_K, 64, 2048, 2)])
def test_tensor_parallel_split_matches_single_device(tmp_path, t, M, K, N):
    out = str(tmp_path / "tp.npz")
    port = 29600 + (os.getpid() % 200)
    mp.spawn(_worker, args=(2, port, t, M, K, N, out), nprocs=2, join=True)
    z = np.load(out)
    assert bool(z["same"][0])                                               # bit-identical on both ranks
    assert np.array_equal(z["col"], z["full"])                              # column-parallel: exact
    scale = np.abs(z["full"]).max()
    assert np.abs(z["row"] - z["full"]).max() <= 4e-6 * max(scale, 1.0)     # row-parallel: fp32 summation order only
