"""Worker of tests/test_gpu_scst.py::test_scst_dp2_equals_single_gpu -- two self-critical updates under torchrun (or a
plain single process): same seeded parameters and GLOBAL batch on every rank; each rank samples and trains on its shard
(parallel.shard_batch), its sources keyed by their place in the global batch, so both runs draw the same summaries.
Rank 0 writes the updated parameters."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main(out, steps=2):
    import torch
    world = int(os.environ.get('WORLD_SIZE', '1'))
    if world > 1:
        torch.cuda.set_device(int(os.environ['LOCAL_RANK']))
        torch.distributed.init_process_group('nccl', device_id=torch.device('cuda', int(os.environ['LOCAL_RANK'])))
    from nats_b200 import nats, parallel
    opts = dict(dim_word=24, dim=128, dim_att=20, n_words=300, encoder='gru', decoder='gru_cond')
    np.random.seed(78)
    params = nats.init_params(opts)
    tparams = nats.init_tparams(params)
    graph = nats.build_model(tparams, opts)[-1].mean()
    graph.clip_c = 1.0
    f_grad_shared, f_update = nats.adadelta('lr', tparams, graph, None, graph)
    f_init, f_next = nats.build_sampler(tparams, opts)
    rank, w = parallel.world()
    rng = np.random.RandomState(6)
    costs = []
    for s in range(steps):
        sx = [list(rng.randint(2, 300, size=rng.randint(5, 40))) for _ in range(7)]      # 7 pairs: uneven shards
        sy = [list(rng.randint(2, 300, size=rng.randint(3, 12))) for _ in range(7)]
        bx, by, n = parallel.shard_batch(sx, sy, rank, w)
        per = (n + w - 1) // w
        if len(bx) == 0:
            c = f_grad_shared(None, None, None, None, global_batch=n)
        else:
            c = nats.scst_step(tparams, f_init, f_next, opts, f_grad_shared, bx, by, 0.75, 3, 12, 99, s * 7 + rank * per,
                               global_batch=n)[0]
        f_update(0.01)
        costs.append(float(c))
    if rank == 0:
        np.savez(out, costs=np.array(costs), **nats.unzip(tparams))
    if world > 1:
        torch.distributed.destroy_process_group()


if __name__ == '__main__':
    main(sys.argv[1])
