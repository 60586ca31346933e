"""spectral_mode 2 (LLE's composite operator) on a multi-GPU communicator is refused with the documented message.  Launched
with torchrun, one rank per GPU:
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port P scripts/mgpu_lle_check.py
Rank 0 prints one JSON line; exit code != 0 on failure."""
import json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.distributed as dist
from gem_b200 import _native, synth, dist as gd
from gem_b200.embedding.lle import lle_composite_operator

rank, world, local = int(os.environ['RANK']), int(os.environ['WORLD_SIZE']), int(os.environ['LOCAL_RANK'])
torch.cuda.set_device(local)
dist.init_process_group('nccl', device_id=torch.device('cuda', local))
ctx = _native.Context(local)
gd.init_comm_from_torch(ctx, dist, rank, world)
P, PT = lle_composite_operator(synth.sbm(n=4096, block=512, seed=3))
r0, ip, ix, w = P.row_shard(rank, world)
_, ipt, ixt, wt = PT.row_shard(rank, world)
msg = ''
with _native.DeviceGraph(ctx, P.n, ip, ix, w.astype('float32'), ipt, ixt, wt.astype('float32'), row0=r0) as g:
    try:
        g.hope(9, 0.0, spectral_mode=2)
    except RuntimeError as exc:
        msg = str(exc)
ok = 'spectral_mode 2 (the composite operator -M^T M) is single-GPU' in msg
if rank == 0:
    print(json.dumps({'world': world, 'ok': ok, 'message': msg}))
dist.destroy_process_group()
sys.exit(0 if ok else 1)
