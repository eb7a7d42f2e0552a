"""torchrun helper: a 2-rank EmbeddingRankingTrainer step must equal the 1-GPU step on the
concatenated batch (tables and tower after one Adagrad step).  Prints DP_EQUIVALENCE_OK."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.distributed as dist

local_rank = int(os.environ['LOCAL_RANK'])
torch.cuda.set_device(local_rank)
dist.init_process_group('nccl', device_id=torch.device('cuda', local_rank))
import ranking_b200 as tfr  # noqa: E402

world, rank = dist.get_world_size(), dist.get_rank()
b, n, d, v, e, t = 8 * world, 24, 8, 200, 12, 16
g = torch.Generator().manual_seed(7)
x = torch.randn(b, n, d, generator=g).cuda()
y = torch.randint(0, 5, (b, n), generator=g).float().cuda()
y[:, n - 6:] = -1.
q = torch.randint(-1, v, (b, 6), generator=g, dtype=torch.int32).cuda()
doc = torch.randint(-1, v, (b, n, t), generator=g, dtype=torch.int32).cuda()


def make(collective):
  emb = tfr.keras.layers.TokenEmbedding(v, e, seed=5)
  tower = tfr.keras.layers.create_tower([32, 16], 1, activation='relu', use_batch_norm=False,
                                        dropout=0, input_dim=d + 2 * e, seed=11,
                                        precision='tf32x3')
  tr = tfr.train.EmbeddingRankingTrainer(
      {'shared': emb}, {'context': {'q': 'shared'}, 'example': {'doc': 'shared'}}, tower,
      tfr.keras.losses.get('approx_ndcg_loss'), optimizer='adagrad', learning_rate=0.1,
      collective=collective)
  return tr


def tokens(sl):
  return {'context': {'q': q[sl]}, 'example': {'doc': doc[sl]}}


COLLECTIVE = os.environ.get('TFR_COLLECTIVE', 'fused')
trainer = make(COLLECTIVE)
tfr.dp.broadcast_(trainer.tower.flat.data)
sl = tfr.dp.shard_lists(b)
trainer.train_step(x[sl], y[sl], tokens=tokens(sl))
torch.cuda.synchronize()
if rank == 0:
  ref = make('nccl')
  ref.world = 1
  ref.group = None
  import ranking_b200.dp as dpmod
  saved = (dpmod.all_reduce_sum_, dpmod.replica_grad_scale)
  dpmod.all_reduce_sum_ = lambda t, group=None: t
  dpmod.replica_grad_scale = lambda group=None: 1.0
  ref.train_step(x, y, tokens=tokens(slice(None)))
  dpmod.all_reduce_sum_, dpmod.replica_grad_scale = saved
  torch.cuda.synchronize()
  err = float((trainer.tower.flat.data - ref.tower.flat.data).abs().max() /
              ref.tower.flat.data.abs().max())
  print('max rel param diff', err)
  assert err < 1e-5, err
  print('DP_EQUIVALENCE_OK', COLLECTIVE)
dist.barrier()
dist.destroy_process_group()
