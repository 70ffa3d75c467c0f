"""`--hpconfig` of the LM1B example scripts: one parser (`models.lm1b.parse_hpconfig`) shared by
training, evaluation and generation, so a checkpoint trained with non-default sizes restores into
the evaluation and generation models built from the same flags."""
import argparse
import os
import subprocess
import sys

import pytest

from parallax_b200.models.lm1b import HPCONFIG_MODEL_KEYS, parse_hpconfig

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_parse_hpconfig_model_keys_and_flags():
    flags = argparse.Namespace(batch_size=128, learning_rate=0.2, datadir=None)
    kw = parse_hpconfig("projected_size=1024, emb_size=1024,keep_prob=0.5,num_sampled=0,"
                        "state_size=64,batch_size=8,learning_rate=0.1,datadir=/d,", flags)
    assert kw == {"projected_size": 1024, "emb_size": 1024, "keep_prob": 0.5, "num_sampled": 0,
                  "state_size": 64}
    assert set(kw) == set(HPCONFIG_MODEL_KEYS)
    assert type(kw["projected_size"]) is int and type(kw["keep_prob"]) is float
    assert (flags.batch_size, flags.learning_rate, flags.datadir) == (8, 0.1, "/d")
    assert parse_hpconfig("", flags) == {}


@pytest.mark.parametrize("spec", ["projected_sz=48", "vocab=10", "=3"])
def test_parse_hpconfig_unknown_key(spec):
    with pytest.raises(ValueError, match="unknown hyper-parameter"):
        parse_hpconfig(spec, argparse.Namespace(batch_size=1))


def test_eval_and_generate_restore_a_wider_checkpoint(tmp_path):
    """The driver trains `--tiny --hpconfig projected_size=48`; evaluation and generation with the
    same `--hpconfig` restore it, and without it the restore refuses the checkpoint's shapes."""
    env = {k: v for k, v in os.environ.items()
           if not k.startswith("PARALLAX_") and k not in ("RANK", "WORLD_SIZE", "LOCAL_RANK")}
    env.update(PARALLAX_FABRIC="host", CUDA_VISIBLE_DEVICES="", OMP_NUM_THREADS="2")
    ck = str(tmp_path / "ck")
    hp = ["--hpconfig", "projected_size=48"]

    def run(script, args):
        return subprocess.run([sys.executable, os.path.join(ROOT, "examples/lm1b", script),
                               "--use_synthetic", "--tiny"] + args, env=env, cwd=str(tmp_path),
                              capture_output=True, text=True, timeout=400)
    r = run("lm1b_distributed_driver.py", ["--max_steps", "2", "--ckpt_dir", ck,
                                           "--save_ckpt_steps", "2", "--logdir",
                                           str(tmp_path / "log")] + hp)
    assert r.returncode == 0, r.stderr[-1500:]
    r = run("lm1b_eval.py", ["--ckpt_dir", ck, "--max_batches", "1", "--batch_size", "4"] + hp)
    assert r.returncode == 0, r.stderr[-1500:]
    assert "global_step 2" in r.stderr + r.stdout and "perplexity" in r.stdout
    r = run("lm1b_generate.py", ["--ckpt_dir", ck, "--prefix", "5 17", "--num_words", "3",
                                 "--num_sequences", "2"] + hp)
    assert r.returncode == 0, r.stderr[-1500:]
    assert all(l.split()[:2] == ["5", "17"] for l in r.stdout.strip().splitlines()[-2:])
    r = run("lm1b_eval.py", ["--ckpt_dir", ck, "--max_batches", "1", "--batch_size", "4"])
    assert r.returncode != 0 and "size" in r.stderr
