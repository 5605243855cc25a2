"""N-rank run == N single-GPU runs (SURVEY.md section 4): the 2-rank NCCL launch of bench.py (weights broadcast from
rank 0 over NVLink, streams sharded rank + world * i) must return, for every stream, exactly the tokens one GPU
returns for that stream.  Needs two GPUs: `python -m pytest tests/test_gpu_multi.py -m gpu` on a machine with two or more."""
import json
import os
import subprocess
import sys

import pytest
import torch

from _wm_paths import ROOT

pytestmark = pytest.mark.gpu


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_rank_run_equals_single_gpu_runs(tmp_path):
    from whisper_medusa_b200 import WhisperMedusaModel
    from whisper_medusa_b200.synthetic import preset_config, synthetic_audio, synthetic_state_dict

    import bench

    dump = str(tmp_path / "tok")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29541", os.path.join(ROOT, "bench.py"), "--gpus", "2", "--steps", "2", "--warmup", "1",
           "--preset", "tiny.en", "--heads", "4", "--seconds", "5", "--no-extras", "--no-cpu-baseline", "--dump-tokens", dump]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    line = json.loads([l for l in r.stdout.splitlines() if l.startswith("{")][-1])
    assert line["n_gpus"] == 2 and line["config"]["streams_per_step"] == 2
    cfg = preset_config("tiny.en", heads=4)
    m = WhisperMedusaModel(cfg, synthetic_state_dict(cfg, seed=0)).to("cuda:0")
    seen = 0
    for rank in (0, 1):
        d = json.load(open(f"{dump}.rank{rank}"))
        for sid, toks in zip(d["stream_ids"], d["tokens"]):
            out = m.generate_from_pcm(synthetic_audio(5.0, stream_id=sid), exponential_decay_length_penalty=bench.PENALTY,
                                      posterior_alpha=bench.REGIMES["realistic"])[0].tolist()
            assert out == toks, (rank, sid)
            seen += 1
    assert seen == 4
    m.close()
