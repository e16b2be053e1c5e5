"""The reference's command line (`python train.py -ng N`) drives the engine end to end."""
import json
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(ngpus, overrides, port):
    env = dict(os.environ, SOD_CONFIG_JSON=json.dumps(overrides))
    out = subprocess.run([sys.executable, os.path.join(ROOT, "train.py"), "-ng", str(ngpus), "-p", str(port)], cwd=ROOT, env=env,
                         capture_output=True, text=True, timeout=500)
    assert out.returncode == 0, out.stderr[-3000:]
    return out.stdout


def test_train_cli_single_gpu_multiscale(tmp_path):
    out = _run(1, {"epoch_num": 2, "synthetic_iters_per_epoch": 3, "batch_size": 4, "print_freq": 1, "save_freq": 0, "is_distributed": False,
                   "size_list": [128, 192], "input_size": 192, "model": "cp_res50", "output_name": "output", "synthetic_eval_images": 6}, 29701)
    assert "End Training" in out and out.count("[I:") == 6 and "Lr:0.0050000,0.0500000" in out
    ckpt = [l for l in out.splitlines() if "img/s" in l]
    assert len(ckpt) == 2
    # the final evaluation over every test set of the config (reference train.py:273-275), GPU metrics
    assert out.count("Results on the testset(") == 6 and "'MAE':" in out and "'SM':" in out


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_train_cli_two_gpus_graph():
    out = _run(2, {"epoch_num": 1, "synthetic_iters_per_epoch": 4, "batch_size": 8, "print_freq": 2, "save_freq": 0,
                   "input_size": 128, "model": "res50", "cuda_graph": True, "synthetic_eval_images": 7}, 29702)
    assert "End Training" in out and out.count("[I:") == 2
    assert out.count("Results on the testset(") == 6


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_train_cli_two_gpus_default_model_cp_res50():
    """the configuration a plain `python train.py -ng 2` runs (config.py defaults: cp_res50, CUDA graph, uint8 input pipeline,
    validation + final test), shrunk in size only: the activation-checkpointed model re-runs every SyncBN forward — and its
    cross-rank exchange — inside backward, all of it captured in the graph"""
    out = _run(2, {"epoch_num": 2, "synthetic_iters_per_epoch": 3, "batch_size": 8, "print_freq": 1, "save_freq": 1, "val_freq": 2,
                   "input_size": 128, "output_name": "output_cp2", "synthetic_eval_images": 5}, 29705)
    assert "End Training" in out and out.count("[I:") == 6
    assert out.count("Results on the valset(") == 1 and out.count("Results on the testset(") == 6
    losses = [float(l.split("Cur:")[1].split("|")[0]) for l in out.splitlines() if "Cur:" in l]
    assert len(losses) == 6 and all(0.1 < v < 5.0 for v in losses)


def test_train_cli_test_mode_evaluates_a_saved_checkpoint():
    """resume_mode == "test" (the reference's DEFAULT, config.py:28): load the saved weights, evaluate, exit"""
    common = {"epoch_num": 1, "synthetic_iters_per_epoch": 2, "batch_size": 4, "print_freq": 0, "save_freq": 1, "is_distributed": False,
              "input_size": 96, "model": "res50", "output_name": "output_testmode", "synthetic_eval_images": 5, "val_freq": 1}
    out = _run(1, dict(common, final_test=False), 29703)
    assert out.count("Results on the valset(") == 1 and "Results on the testset(" not in out
    out = _run(1, dict(common, resume_mode="test"), 29704)
    assert "Loaded checkpoint" in out and out.count("Results on the testset(") == 6 and "[I:" not in out
    # the reference's stand-alone evaluation script (test.py) on the same checkpoint: same numbers as train.py's test mode
    env = dict(os.environ, SOD_CONFIG_JSON=json.dumps(dict(common, resume_mode="test")))
    res = subprocess.run([sys.executable, os.path.join(ROOT, "test.py")], cwd=ROOT, env=env, capture_output=True, text=True, timeout=500)
    assert res.returncode == 0, res.stderr[-3000:]
    import ast
    import re
    dicts = lambda text: [ast.literal_eval(m) for m in re.findall(r"\{'MaxF'[^}]*\}", text)]     # noqa: E731
    mine, theirs = dicts(res.stdout), dicts(out)
    assert len(mine) == 6 == len(theirs)
    for a, b in zip(mine, theirs):      # test.py runs the network in fp32 (as the reference's does), train.py's test mode under bf16 autocast
        assert all(abs(a[k] - b[k]) < 3e-2 for k in ("MaxF", "MeanF", "MAE", "SM", "EM")), (a, b)
