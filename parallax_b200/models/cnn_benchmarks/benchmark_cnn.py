"""The CNN benchmark harness.

Parity: `examples/tf_cnn_benchmarks/benchmark_cnn.py:60-1014` — the parameter
table (`_DEFAULT_PARAMS`, `make_params`), `get_learning_rate` (`:444-484`: fixed
`--learning_rate` with optional staircase epoch decay and floor, else the
model's own schedule), `BenchmarkCNN` (`:487-1014`): dataset + model + optimizer
choice (momentum with Nesterov / sgd / rmsprop, `:805-818`), element-wise
`gradient_clip`, L2 `weight_decay`, reduced-precision compute with a loss scale,
training / forward-only / evaluation (top-1, top-5) modes, `--params_stat`, and
the images/sec report of the driver (`CNNBenchmark_distributed_driver.py:85-91`).

What a TF graph built implicitly is explicit here: `build_graph()` returns the
`parallax.Graph` handed to `parallel_run`, `sess_config()` the engine options
(compute dtype, CUDA-graph capture), and `input_iterator()` this worker's batches.
"""
import argparse
import collections
import time

import torch
import torch.nn as nn

from ... import optim
from ...graph import ClipByValue, Graph, ScaleGradients
from ...log import parallax_log as log
from . import datasets, model_config

ParamSpec = collections.namedtuple("ParamSpec", "type default help")

_DEFAULT_PARAMS = collections.OrderedDict([
    ("model", ParamSpec(str, "trivial", "name of the model to run")),
    ("eval", ParamSpec(bool, False, "evaluate instead of train")),
    ("forward_only", ParamSpec(bool, False, "only run the forward pass")),
    ("print_training_accuracy", ParamSpec(bool, False, "report top-1/top-5 while training")),
    ("batch_size", ParamSpec(int, 0, "batch size per compute device (0 = model default)")),
    ("num_batches", ParamSpec(int, 100, "number of batches to run (excluding warm-up)")),
    ("num_warmup_batches", ParamSpec(int, None, "warm-up batches (default 10)")),
    ("display_every", ParamSpec(int, 10, "steps between progress lines")),
    ("data_dir", ParamSpec(str, None, "dataset directory; synthetic data when unset")),
    ("data_name", ParamSpec(str, None, "imagenet | cifar10 (inferred from data_dir)")),
    ("resize_method", ParamSpec(str, "bilinear",
                                "round_robin | nearest | bilinear | bicubic | area")),
    ("distortions", ParamSpec(bool, True, "image distortions during training")),
    ("data_format", ParamSpec(str, "NHWC", "NHWC (channels_last, tensor-core layout) | NCHW")),
    ("params_stat", ParamSpec(bool, False, "print total parameter / gradient element counts")),
    ("optimizer", ParamSpec(str, "sgd", "momentum | sgd | rmsprop")),
    ("learning_rate", ParamSpec(float, None, "initial learning rate (model default if unset)")),
    ("num_epochs_per_decay", ParamSpec(float, 0, "epochs between staircase decays")),
    ("learning_rate_decay_factor", ParamSpec(float, 0, "decay factor")),
    ("minimum_learning_rate", ParamSpec(float, 0, "floor of the decayed learning rate")),
    ("momentum", ParamSpec(float, 0.9, "momentum")),
    ("rmsprop_decay", ParamSpec(float, 0.9, "RMSProp decay")),
    ("rmsprop_momentum", ParamSpec(float, 0.9, "RMSProp momentum")),
    ("rmsprop_epsilon", ParamSpec(float, 1.0, "RMSProp epsilon")),
    ("gradient_clip", ParamSpec(float, None, "clip gradients to [-x, x] element-wise")),
    ("weight_decay", ParamSpec(float, 0.00004, "L2 weight decay")),
    ("use_fp16", ParamSpec(bool, False, "reduced-precision compute (bf16 on Hopper)")),
    ("fp16_loss_scale", ParamSpec(float, None, "loss scale (default 1: bf16 needs none)")),
    ("tf_random_seed", ParamSpec(int, 1234, "random seed")),
    ("num_batches_for_eval", ParamSpec(int, 0, "evaluation batches (0 = one epoch)")),
    ("display_every_for_eval", ParamSpec(int, 10, "steps between evaluation progress lines")),
    ("checkpoint_dir", ParamSpec(str, None, "checkpoint directory (evaluation restores it)")),
    ("cuda_graph", ParamSpec(bool, True, "capture the training step into a CUDA graph")),
    ("deterministic", ParamSpec(bool, False, "fixed seeds for data order and augmentation")),
])

Params = collections.namedtuple("Params", list(_DEFAULT_PARAMS))


def make_params(**kwargs):
    """`Params` with defaults for everything not given; unknown names raise."""
    bad = [k for k in kwargs if k not in _DEFAULT_PARAMS]
    if bad:
        raise ValueError("Invalid parameter(s): %s" % ", ".join(sorted(bad)))
    vals = {k: spec.default for k, spec in _DEFAULT_PARAMS.items()}
    vals.update(kwargs)
    return Params(**vals)


def add_arguments(ap):
    for name, spec in _DEFAULT_PARAMS.items():
        if spec.type is bool:
            ap.add_argument("--" + name, type=lambda s: s.lower() in ("1", "true", "yes"),
                            nargs="?", const=True, default=spec.default, help=spec.help)
        else:
            ap.add_argument("--" + name, type=spec.type, default=spec.default, help=spec.help)
    return ap


def make_params_from_flags(flags):
    return make_params(**{k: getattr(flags, k) for k in _DEFAULT_PARAMS if hasattr(flags, k)})


def get_learning_rate(params, num_examples_per_epoch, model, batch_size):
    """→ float or callable lr(step).  `batch_size` is the GLOBAL batch."""
    steps_per_epoch = float(num_examples_per_epoch) / batch_size
    if not params.learning_rate:
        if params.num_epochs_per_decay > 0 or params.learning_rate_decay_factor > 0:
            raise ValueError("learning-rate decay needs an explicit --learning_rate")
        return model.get_learning_rate(batch_size, steps_per_epoch)
    base = float(params.learning_rate)
    if params.num_epochs_per_decay > 0 and params.learning_rate_decay_factor > 0:
        every = max(int(steps_per_epoch * params.num_epochs_per_decay), 1)
        factor = float(params.learning_rate_decay_factor)
        floor = float(params.minimum_learning_rate)

        def lr(step):
            return max(base * factor ** (max(int(step) - 1, 0) // every), floor)
        return lr
    return base


class _WithAccuracy(nn.Module):
    """classifier + in-graph top-1 / top-5 hit counts (`benchmark_cnn.py:935-947`)"""

    def __init__(self, net, channels_last=True, accuracy=False):
        super().__init__()
        self.net, self.channels_last, self.accuracy = net, channels_last, accuracy
        self.image_size = getattr(net, "image_size", 224)

    def forward(self, images, labels):
        if self.channels_last and images.dim() == 4:
            images = images.contiguous(memory_format=torch.channels_last)
        out = self.net(images, labels)
        if self.accuracy or not self.training:
            top5 = out["logits"].float().topk(min(5, out["logits"].shape[-1]), -1).indices
            hit = top5 == labels[:, None]
            out["top_1_accuracy"] = hit[:, 0].float().sum()
            out["top_5_accuracy"] = hit.float().sum()
        return out


class BenchmarkCNN(object):
    def __init__(self, params):
        self.params = p = params
        if p.eval and p.forward_only:
            raise ValueError("Only one of forward_only and eval parameters is true")
        if p.optimizer not in ("momentum", "sgd", "rmsprop"):
            raise ValueError('Optimizer "%s" was not recognized' % p.optimizer)
        if p.data_format not in ("NHWC", "NCHW"):
            raise ValueError("data_format must be NHWC or NCHW")
        if p.fp16_loss_scale and not p.use_fp16:
            raise ValueError("fp16_loss_scale requires use_fp16")
        self.dataset = datasets.create_dataset(p.data_dir, p.data_name)
        self.model_conf = model_config.get_model_config(p.model, self.dataset)
        self.batch_size = p.batch_size or self.model_conf.get_default_batch_size()
        self.model_conf.set_batch_size(self.batch_size)
        self.num_batches = p.num_batches
        self.num_warmup_batches = 10 if p.num_warmup_batches is None else p.num_warmup_batches
        self.loss_scale = float(p.fp16_loss_scale) if p.fp16_loss_scale else 1.0
        self.train = not (p.eval or p.forward_only)
        self.model = None

    # -- graph -------------------------------------------------------------------
    def build_model(self):
        torch.manual_seed(self.params.tf_random_seed)
        nclass = self.dataset.num_classes + 1          # class 0 = background, like the reference
        net = self.model_conf.build(nclass)
        self.model = _WithAccuracy(net, self.params.data_format == "NHWC",
                                   self.params.print_training_accuracy)
        return self.model

    def build_graph(self, num_workers=1):
        p = self.params
        model = self.model or self.build_model()
        if not self.train:
            return Graph(model, optimizer=None, name="cnn_eval")
        lr = get_learning_rate(p, self.dataset.num_examples_per_epoch("train"), self.model_conf,
                               self.batch_size * num_workers)
        wd = float(p.weight_decay or 0.0)
        if p.optimizer == "momentum":
            opt = optim.Momentum(lr, p.momentum, use_nesterov=True, weight_decay=wd)
        elif p.optimizer == "sgd":
            opt = optim.GradientDescent(lr, weight_decay=wd)
        else:
            opt = optim.RMSProp(lr, p.rmsprop_decay, p.rmsprop_momentum, p.rmsprop_epsilon,
                                weight_decay=wd)
        rules = [ScaleGradients(1.0 / self.loss_scale)] if self.loss_scale != 1.0 else []
        if p.gradient_clip:
            rules.append(ClipByValue(float(p.gradient_clip)))
        return Graph(model, optimizer=opt, loss="loss", loss_scale=self.loss_scale,
                     grad_rules=rules, name="cnn")

    def sess_config(self):
        sc = {"cuda_graph": bool(self.params.cuda_graph) and self.train}
        if self.params.use_fp16:
            sc["compute_dtype"] = "bf16"
        return sc

    # -- data ----------------------------------------------------------------------
    def input_iterator(self, subset=None, device=None):
        p = self.params
        subset = subset or ("validation" if p.eval else "train")
        size = self.model_conf.get_image_size()
        cls = self.dataset.get_image_preprocessor()
        pre = cls(size, size, self.batch_size, train=self.train, distortions=p.distortions,
                  resize_method=p.resize_method,
                  seed=p.tf_random_seed if p.deterministic else None)
        if self.dataset.use_synthetic_gpu_images():
            return pre.minibatch(self.dataset, subset, device=device)
        return pre.minibatch(self.dataset, subset)

    # -- loops -----------------------------------------------------------------------
    def print_info(self, num_workers):
        p = self.params
        log.info("Model:       %s", self.model_conf.name)
        log.info("Dataset:     %s (%s)", self.dataset.name,
                 "synthetic" if self.dataset.use_synthetic_gpu_images() else p.data_dir)
        log.info("Mode:        %s", "evaluation" if p.eval else
                 "forward-only" if p.forward_only else "training")
        log.info("Batch size:  %d global / %d per device", self.batch_size * num_workers,
                 self.batch_size)
        log.info("Data format: %s   Optimizer: %s   Precision: %s", p.data_format, p.optimizer,
                 "bf16" if p.use_fp16 else "fp32")

    def run(self, sess, num_workers=1, worker_id=0, device=None):
        if self.params.eval:
            return self.evaluate(sess, num_workers, worker_id)
        return self.benchmark(sess, num_workers, worker_id, device)

    def benchmark(self, sess, num_workers=1, worker_id=0, device=None):
        """warm-up + `num_batches` timed steps → dict(images_per_sec, steps_per_sec, …)"""
        p, chief = self.params, worker_id == 0
        if chief:
            self.print_info(num_workers)
            if p.params_stat:
                n = sum(q.numel() for q in self.model.parameters())
                log.info("total parameters / gradient elements: %d / %d", n, n)
            log.info("Step\tImg/sec\ttotal_loss" +
                     ("\ttop_1_accuracy\ttop_5_accuracy" if p.print_training_accuracy else ""))
        fetch = ["loss"] + (["train_op"] if self.train else [])
        if p.print_training_accuracy:
            fetch += ["top_1_accuracy", "top_5_accuracy"]
        it = self.input_iterator(device=device)
        total, losses = self.num_warmup_batches + self.num_batches, []
        t0 = window = time.time()                  # restarted when the warm-up ends
        for step in range(1, total + 1):
            images, labels = next(it)
            out = sess.run(fetch, {"images": [images], "labels": [labels]})
            if step == self.num_warmup_batches:
                t0 = window = time.time()
            if step > self.num_warmup_batches:
                losses.append(out[0][0])
                k = step - self.num_warmup_batches
                if chief and (k % p.display_every == 0 or k == self.num_batches):
                    now = time.time()
                    n = k % p.display_every or p.display_every
                    line = "%d\timages/sec: %.1f\t%.3f" % (
                        k, n * self.batch_size * num_workers / max(now - window, 1e-9), out[0][0])
                    if p.print_training_accuracy:
                        line += "\t%.3f\t%.3f" % (out[-2][0] / self.batch_size,
                                                  out[-1][0] / self.batch_size)
                    log.info(line)
                    window = now
        elapsed = time.time() - t0
        ips = self.num_batches * self.batch_size * num_workers / max(elapsed, 1e-9)
        if chief:
            log.info("-" * 64)
            log.info("total images/sec: %.2f", ips)
            log.info("-" * 64)
        return {"images_per_sec": ips, "steps_per_sec": self.num_batches / max(elapsed, 1e-9),
                "average_loss": float(sum(losses) / max(len(losses), 1)),
                "num_steps": self.num_batches}

    def evaluate(self, sess, num_workers=1, worker_id=0):
        """top-1 / top-5 accuracy over the validation set (`benchmark_cnn.py:560-640`)"""
        p = self.params
        self.model.eval()
        nb = p.num_batches_for_eval or int(
            self.dataset.num_examples_per_epoch("validation") / (self.batch_size * num_workers))
        it = self.input_iterator("validation")
        top1 = top5 = seen = 0.0
        t0 = time.time()
        for i in range(nb):
            try:
                images, labels = next(it)
            except StopIteration:
                break
            t1, t5 = sess.run(["top_1_accuracy", "top_5_accuracy"],
                              {"images": [images], "labels": [labels]})
            top1, top5, seen = top1 + t1[0], top5 + t5[0], seen + self.batch_size
            if worker_id == 0 and (i + 1) % p.display_every_for_eval == 0:
                log.info("%d\t%.1f examples/sec", i + 1, seen / (time.time() - t0))
        res = {"top_1_accuracy": top1 / max(seen, 1), "top_5_accuracy": top5 / max(seen, 1),
               "num_examples": int(seen)}
        if worker_id == 0:
            log.info("Accuracy @ 1 = %.4f Accuracy @ 5 = %.4f [%d examples]",
                     res["top_1_accuracy"], res["top_5_accuracy"], res["num_examples"])
        return res


def main(argv=None):          # pragma: no cover - thin CLI
    import parallax_b200 as parallax
    ap = add_arguments(argparse.ArgumentParser())
    ap.add_argument("--resource_info_file", default="localhost")
    ap.add_argument("--run_option", default="MPI")
    flags = ap.parse_args(argv)
    bench = BenchmarkCNN(make_params_from_flags(flags))
    cfg = parallax.Config(run_option=flags.run_option, search_partitions=False,
                          sess_config=bench.sess_config())
    if flags.checkpoint_dir:
        cfg.ckpt_config = parallax.CheckPointConfig(ckpt_dir=flags.checkpoint_dir)
    sess, nw, wid, _ = parallax.parallel_run(bench.build_graph(), flags.resource_info_file,
                                             parallax_config=cfg)
    bench.run(sess, nw, wid)
    sess.close()


if __name__ == "__main__":    # pragma: no cover
    main()
