"""Multi-GPU rebalance check (run under torchrun, one rank per GPU, NCCL; not collected by pytest): a keyed corpus held by
the collective corpus methods is skewed by removing most of rank 0's rows, then ShardedVectorEngine.rebalance() evens
the ranks out over NCCL, the vectors travelling as device tensors.  The MV2V bytes and the batched answers must be those
before the move, the ranks must end within one row of each other, and a second rebalance must move nothing.

    torchrun --nproc-per-node N tests/check_sharded_rebalance_torchrun.py [rows]

`rows` defaults to 200 000 (384 dims, cosine)."""
import os
import sys
from pathlib import Path

import numpy as np
import torch
import torch.distributed as dist

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from wax_b200 import VectorMetric, sharded  # noqa: E402

rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
dist.init_process_group("nccl", device_id=torch.device("cuda", local))
rows, dims = (int(sys.argv[1]) if len(sys.argv) > 1 else 200_000), 384
rng = np.random.default_rng(780)
eng = sharded.ShardedVectorEngine(VectorMetric.cosine, dims)
ids = np.arange(rows, dtype=np.uint64)
eng.add_batch(ids, rng.standard_normal((rows, dims), dtype=np.float32))
eng.set_groups(ids, ids // 7)
eng.set_attributes(ids, ids.astype(np.int64), ids % 4)
gone = [eng.engine.export_rows(0, eng.engine.count * 3 // 4, vectors=False)[0] if rank == 0 else None]
dist.broadcast_object_list(gone, src=0)
eng.remove_batch(gone[0])
qs = rng.standard_normal((16, dims), dtype=np.float32)
blob_before, answers_before = eng.serialize(), eng.search_batch(qs, 10)
counts_before = eng._counts.tolist()
moved = eng.rebalance()
ok = moved > 0 and int(eng._counts.max() - eng._counts.min()) <= 1 and eng.engine.count == eng._counts[rank]
ok = ok and eng.search_batch(qs, 10) == answers_before and eng.rebalance() == 0
blob_after = eng.serialize()
ok = ok and (rank != 0 or bytes(blob_after) == bytes(blob_before))
flag = torch.tensor([1 if ok else 0], device="cuda")
dist.all_reduce(flag, op=dist.ReduceOp.MIN)
if rank == 0:
    print(f"SHARDED REBALANCE {'PASS' if flag.item() == 1 else 'FAIL'} world={world} rows {counts_before} -> "
          f"{eng._counts.tolist()}, {moved} moved", flush=True)
eng.close()
dist.destroy_process_group()
sys.exit(0 if flag.item() == 1 else 1)
