"""ORACLE — TEST INFRASTRUCTURE ONLY.  Not product code.

CPU restatement (numpy / plain torch on CPU, fp64 where it matters) of the reference's data-parallel
hot path, used ONLY as the checker by `tests/`, `__graft_entry__.smoke()` and the `cpu_baseline` /
`--impl reference` legs of `bench.py`.  Nothing under `distributed_sod_project_b200/` may import it.

Parity status
-------------
* Reference-owned arithmetic (`loss/CEL.py:15-20`, `BCEWithLogitsLoss` at `train.py:203`,
  `utils/pipeline_ops.py` `get_total_loss` 19-43 / `CustomScheduler` 185-232 / `make_optimizer` 235-316,
  `utils/tensor_ops.py:60-64`, `network/TestModel.py`) is PINNED: `tools/make_golden.py` imports the
  unmodified reference modules from a checkout of the reference and writes
  `tests/golden/*.npz`; `tests/test_oracle_golden.py` checks every oracle function against them.
* The apex pieces (`apex.parallel.DistributedDataParallel`, `apex.parallel.SyncBatchNorm`, `apex.amp`;
  call sites `train.py:15-16,180-185,299`) are NOT in the reference repository (un-vendored, un-pinned:
  `readme.md:40-42`) and apex is not installed here: **parity unpinned** for those.  Their published
  semantics are restated here and cross-checked against the equivalent single-process computation
  (W-rank SyncBN+DDP == one process on the concatenated batch, see `oracle/syncbn.py`) and, on the GPU
  box, against `torch.nn.SyncBatchNorm` / `torch.distributed.all_reduce`.
"""
