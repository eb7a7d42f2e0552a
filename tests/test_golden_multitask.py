"""The multi-task recovery experiment of tests/_multitask_refs.py through the fp64 CPU oracle.
This run fixes the thresholds the fused trainer is held to in tests/test_multitask_gpu.py."""
import _multitask_refs as MR

# Set from the oracle run below (measured: validation NDCG@5 of the multi-task planes 0.993
# (relevance) and 0.994 (click); the models trained on the other task's labels alone reach 0.559
# and 0.537, gaps of 0.433 and 0.457), with a margin of about 2x on the gap.
DELTA = 0.2
FLOOR = 0.95


def test_multitask_recovery_oracle(tmp_path):
  batches, (vx, vy) = MR.synthetic(str(tmp_path))
  multi = MR.oracle_train(list(MR.LABELS), batches)(vx)
  planes = {t: multi[..., i] for i, t in enumerate(MR.LABELS)}
  single = {t: MR.oracle_train([t], batches)(vx)[..., 0] for t in MR.LABELS}
  for task, (own, other) in MR.margins(planes, single, vy).items():
    assert own >= FLOOR, (task, own)
    assert own >= other + DELTA, (task, own, other)
