"""The two exchange calls of sharded keep-all / kNN > 32 matching (include/line3d.h, setShard) through dist.exchange_rows on the CPU
(gloo, world_size 2): knn = 0 moves the counts and makes no record broadcast; the second call moves the rows at the common stride."""
import os
import socket
import subprocess
import sys
import textwrap

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

WORKER = textwrap.dedent("""
    import os, sys, numpy as np, torch, torch.distributed as dist
    sys.path.insert(0, %r)
    from line3dpp_b200 import dist as l3dist
    dist.init_process_group("gloo")
    rank, world = dist.get_rank(), dist.get_world_size()
    sizes = []
    broadcast = dist.broadcast
    def counting_broadcast(t, *a, **k):
        sizes.append(t.numel())
        return broadcast(t, *a, **k)
    dist.broadcast = counting_broadcast
    rows, bounds = 1000, [0, 377, 1000]
    rng = np.random.default_rng(11)
    full_counts = rng.integers(0, 50, rows).astype(np.int32)
    stride = int(full_counts.max())
    full_recs = rng.integers(0, 255, (rows * stride, l3dist.REC_BYTES)).astype(np.uint8)
    a, b = bounds[rank], bounds[rank + 1]
    counts = np.zeros_like(full_counts)
    counts[a:b] = full_counts[a:b]
    ct = torch.from_numpy(counts.view(np.uint8))
    l3dist.exchange_rows(ct, torch.empty(0, dtype=torch.uint8), bounds, 0)
    assert np.array_equal(counts, full_counts), "counts missing after the first call"
    assert sizes == [4 * 377, 4 * 623], sizes                  # one count broadcast per owner, no zero-byte record broadcast
    recs = np.zeros_like(full_recs)
    recs[a * stride:b * stride] = full_recs[a * stride:b * stride]
    l3dist.exchange_rows(ct, torch.from_numpy(recs.reshape(-1)), bounds, stride)
    assert np.array_equal(recs, full_recs), "rows missing after the second call"
    dist.barrier(); dist.destroy_process_group()
    print("rank", rank, "two-call exchange ok")
""")


def test_two_rank_gloo_counts_then_rows(tmp_path):
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    script = tmp_path / "worker.py"
    script.write_text(WORKER % ROOT)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", str(port), str(script)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
