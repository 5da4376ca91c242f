"""Training / evaluation loop with the interface of the reference's `pytorch_generative.trainer.Trainer`
(reference trainer.py:15-285), re-implemented for the CUDA path.

What is kept from the reference (so that a recipe written against it runs unchanged):
  * constructor arguments and defaults (`model, loss_fn, optimizer, train_loader, eval_loader, lr_scheduler,
    clip_grad_norm, skip_grad_norm, log_dir, sample_epochs, save_checkpoint_epochs, n_gpus, device_id`);
  * `loss_fn(inputs, targets, predictions)` returning a tensor or a dict with a "loss" entry; the overridable
    `train_one_batch` / `eval_one_batch` hooks;
  * the training step (trainer.py:173-193): train mode, host->device copy, zero_grad, forward, loss, backward,
    `clip_grad_norm_(params, clip or skip or 1e50)` (the norm is always computed: it is a logged metric), the step is
    skipped when the norm exceeds `skip_grad_norm`, the scheduler steps after every batch, metrics are read with
    `.item()`;
  * checkpoints `trainer_state_{epoch}.ckpt` with the keys `model, optimizer, step, epoch, examples_processed,
    time_taken, lr_scheduler` (trainer.py:98-148), written by rank 0 only, restored from the latest epoch.

What differs:
  * multi-GPU is one process per GPU launched by `torch.distributed.run`; gradients are averaged by
    `parallel.OverlappedGradAverager` (bucketed all-reduce inside the fused backward) instead of wrapping the model in
    DistributedDataParallel.  The reference's DDP wrap prefixes every checkpoint key with `module.`; checkpoints are
    written WITHOUT the prefix and `restore_checkpoint` accepts both spellings, so files move between the two
    implementations in either direction (`export_reference_checkpoint` writes the prefixed form on request);
  * with a `FusedAdam` optimizer the clip + Adam part of the step is two kernels over all parameters (`optim.py`);
  * TensorBoard is optional: scalars go to `SummaryWriter` when tensorboard is importable, and always to
    `metrics.jsonl` in the log directory.
"""

import collections
import glob
import json
import os
import re
import tempfile
import time

import torch

from . import parallel


class _Scalars:
    """Scalar / image sink: TensorBoard when available, plus a JSON-lines file."""

    def __init__(self, log_dir, purge_step=None):
        os.makedirs(log_dir, exist_ok=True)
        self._jsonl = open(os.path.join(log_dir, "metrics.jsonl"), "a")
        self._tb = None
        try:
            from torch.utils import tensorboard

            self._tb = tensorboard.SummaryWriter(log_dir, max_queue=100, purge_step=purge_step)
        except Exception:  # tensorboard not installed: the JSON-lines log is the record
            self._tb = None

    def add_scalars(self, tag, values, step):
        self._jsonl.write(json.dumps({"tag": tag, "step": step, **{k: float(v) for k, v in values.items()}}) + "\n")
        if self._tb is not None:
            self._tb.add_scalars(tag, values, step)

    def add_scalar(self, tag, value, step):
        self._jsonl.write(json.dumps({"tag": tag, "step": step, "value": float(value)}) + "\n")
        if self._tb is not None:
            self._tb.add_scalar(tag, value, step)

    def add_images(self, tag, tensor, step):
        if self._tb is not None:
            self._tb.add_images(tag, tensor, step)

    def close(self):
        self._jsonl.close()
        if self._tb is not None:
            self._tb.close()


def strip_ddp_prefix(state_dict):
    """`module.`-prefixed keys (a DistributedDataParallel-wrapped reference model, trainer.py:78-82,102) -> plain keys."""
    if state_dict and all(k.startswith("module.") for k in state_dict):
        return collections.OrderedDict((k[len("module."):], v) for k, v in state_dict.items())
    return state_dict


class Trainer:
    """Stateful train / eval loop; calling `interleaved_train_and_eval` again resumes where it stopped."""

    def __init__(self, model, loss_fn, optimizer, train_loader, eval_loader, lr_scheduler=None, clip_grad_norm=None,
                 skip_grad_norm=None, log_dir=None, sample_epochs=3, save_checkpoint_epochs=1, n_gpus=0, device_id=None):
        self.loss_fn = loss_fn
        self.train_loader = train_loader
        self.eval_loader = eval_loader
        self.clip_grad_norm = clip_grad_norm
        self.skip_grad_norm = skip_grad_norm
        self.log_dir = log_dir or tempfile.mkdtemp()
        self.save_checkpoint_epochs = save_checkpoint_epochs
        self.sample_epochs = sample_epochs

        self.device_id = 0 if device_id is None and n_gpus == 1 else device_id
        if n_gpus > 0:
            if n_gpus > 1:
                assert device_id is not None, "'device_id' must be provided if n_gpus > 1."
            self.device = torch.device("cuda", self.device_id or 0)
            torch.cuda.set_device(self.device)
        else:
            self.device = torch.device("cpu")
        self.model = model.to(self.device)
        self.optimizer = optimizer
        self.lr_scheduler = lr_scheduler
        self._params = [p for p in self.model.parameters()]
        self._grad_averager = None
        if n_gpus > 1:
            parallel.broadcast_parameters(self.model)
            self._grad_averager = parallel.OverlappedGradAverager(self.model, self._params)

        # state saved in checkpoints
        self._step = 0
        self._epoch = 0
        self._examples_processed = 0
        self._time_taken = 0

        self._summary_writer = _Scalars(self.log_dir)

    # ---- checkpoints (reference trainer.py:95-148) ----
    def _path(self, file_name):
        return os.path.join(self.log_dir, file_name)

    def _checkpoint(self):
        ckpt = {
            "model": self.model.state_dict(),
            "optimizer": self.optimizer.state_dict(),
            "step": self._step,
            "epoch": self._epoch,
            "examples_processed": self._examples_processed,
            "time_taken": self._time_taken,
        }
        if self.lr_scheduler is not None:
            ckpt["lr_scheduler"] = self.lr_scheduler.state_dict()
        return ckpt

    def _save_checkpoint(self):
        if self.device_id not in (0, None) or self._epoch % self.save_checkpoint_epochs != 0:
            return
        torch.save(self._checkpoint(), self._path(f"trainer_state_{self._epoch}.ckpt"))

    def export_reference_checkpoint(self, path, ddp_prefix=False):
        """Writes the current state in the reference's format; `ddp_prefix=True` spells the model keys the way a
        multi-GPU (DistributedDataParallel) reference run does."""
        ckpt = self._checkpoint()
        if ddp_prefix:
            ckpt["model"] = collections.OrderedDict(("module." + k, v) for k, v in ckpt["model"].items())
        torch.save(ckpt, path)

    def _find_latest_epoch(self):
        files = glob.glob(self._path("trainer_state_[0-9]*.ckpt"))
        epochs = sorted(int(re.findall(r"trainer_state_(\d+)\.ckpt", os.path.basename(f))[0]) for f in files)
        if not epochs:
            raise FileNotFoundError(f"No checkpoints found in {self.log_dir}.")
        print(f"Found {len(epochs)} saved checkpoints.")
        return epochs[-1]

    def restore_checkpoint(self, epoch=None):
        """Restores the trainer from `log_dir` (latest epoch unless given).  Accepts checkpoints written by the
        reference Trainer, single- or multi-GPU."""
        epoch = epoch or self._find_latest_epoch()
        name = f"trainer_state_{epoch}.ckpt"
        print(f"Restoring trainer state from checkpoint {name}.")
        ckpt = torch.load(self._path(name), map_location=self.device, weights_only=False)
        self.model.load_state_dict(strip_ddp_prefix(ckpt["model"]))
        self.optimizer.load_state_dict(ckpt["optimizer"])
        self._step = ckpt["step"]
        self._epoch = ckpt["epoch"]
        self._examples_processed = ckpt["examples_processed"]
        self._time_taken = ckpt["time_taken"]
        if self.lr_scheduler is not None:
            self.lr_scheduler.load_state_dict(ckpt["lr_scheduler"])
        self._summary_writer.close()
        self._summary_writer = _Scalars(self.log_dir, purge_step=self._step)

    # ---- one batch ----
    @staticmethod
    def _get_metrics_dict(loss_or_metrics):
        metrics = loss_or_metrics if isinstance(loss_or_metrics, dict) else {"loss": loss_or_metrics}
        assert "loss" in metrics, 'Metrics dictionary does not contain "loss" key.'
        return metrics

    def _log_metrics(self, metrics, training):
        for key, metric in metrics.items():
            self._summary_writer.add_scalars(f"metrics/{key}", {"train" if training else "eval": metric}, self._step)

    def train_one_batch(self, x, y):
        """Forward + loss of one training batch; override for custom training loops."""
        return self.loss_fn(x, y, self.model(x))

    def _train_one_batch(self, x, y):
        self.model.train()
        x = x.to(self.device, non_blocking=True)
        if y is not None:
            y = y.to(self.device, non_blocking=True)
        self.optimizer.zero_grad()
        metrics = self._get_metrics_dict(self.train_one_batch(x, y))
        metrics["loss"].backward()
        if self._grad_averager is not None:
            self._grad_averager.average_()

        # 1e50: the norm is logged even when the gradients are left alone (reference trainer.py:183-186)
        max_norm = self.clip_grad_norm or self.skip_grad_norm or 1e50
        fused = getattr(self.optimizer, "clip_and_step", None)
        if fused is not None:
            # norm, clip and Adam update in two kernels over all parameters; the skip rule is evaluated on the device
            norm = fused(max_norm, skip_above=self.skip_grad_norm)
            stepped = True if not self.skip_grad_norm else norm.item() <= self.skip_grad_norm
        else:
            norm = torch.nn.utils.clip_grad_norm_(self._params, max_norm)
            stepped = not self.skip_grad_norm or norm.item() <= self.skip_grad_norm
            if stepped:
                self.optimizer.step()
        metrics["grad_norm"] = norm
        if stepped and self.lr_scheduler is not None:
            self.lr_scheduler.step()
        return {k: v.item() for k, v in metrics.items()}

    def eval_one_batch(self, x, y):
        """Forward + loss of one evaluation batch; override for custom evaluation loops."""
        return self.loss_fn(x, y, self.model(x))

    @torch.no_grad()
    def _eval_one_batch(self, x, y):
        self.model.eval()
        x = x.to(self.device, non_blocking=True)
        if y is not None:
            y = y.to(self.device, non_blocking=True)
        metrics = self._get_metrics_dict(self.eval_one_batch(x, y))
        return {k: v.item() for k, v in metrics.items()}

    @torch.no_grad()
    def sample_one_batch(self):
        self.model.eval()
        try:
            self._summary_writer.add_images("sample", self.model.sample(n_samples=16), self._step)
        except Exception as exc:  # sampling is a convenience log, never fatal (reference trainer.py:213-220)
            print(f"Failed to sample from the model: {exc}")

    # ---- the loop (reference trainer.py:222-285) ----
    def interleaved_train_and_eval(self, max_epochs, restore=True):
        """Trains for up to `max_epochs` epochs, evaluating after each one; resumes from `log_dir` when `restore`."""
        if restore:
            try:
                self.restore_checkpoint()
            except FileNotFoundError:
                print(f"No checkpoint found in {self.log_dir}. Training from scratch.")

        for _ in range(max_epochs - self._epoch):
            start_time = time.time()
            for batch in self.train_loader:
                x, y = batch if isinstance(batch, (tuple, list)) else (batch, None)
                self._examples_processed += x.shape[0]
                lrs = {f"group_{i}": g["lr"] for i, g in enumerate(self.optimizer.param_groups)}
                self._summary_writer.add_scalars("metrics/lr", lrs, self._step)
                metrics = self._train_one_batch(x, y)
                self._log_metrics(metrics, training=True)

                self._time_taken += time.time() - start_time
                start_time = time.time()
                self._summary_writer.add_scalar("speed/examples_per_sec", self._examples_processed / self._time_taken,
                                                self._step)
                self._summary_writer.add_scalar("speed/millis_per_example",
                                                self._time_taken / self._examples_processed * 1000, self._step)
                self._summary_writer.add_scalar("speed/epoch", self._epoch, self._step)
                self._summary_writer.add_scalar("speed/step", self._step, self._step)
                self._step += 1

            n_examples, sums = 0, collections.defaultdict(float)
            for batch in self.eval_loader:
                x, y = batch if isinstance(batch, (tuple, list)) else (batch, None)
                n_examples += x.shape[0]
                for key, metric in self._eval_one_batch(x, y).items():
                    sums[key] += metric * x.shape[0]
            self._log_metrics({key: total / max(n_examples, 1) for key, total in sums.items()}, training=False)

            self._epoch += 1
            self._save_checkpoint()
            if self._epoch % self.sample_epochs == 0:
                self.sample_one_batch()

        self._summary_writer.close()
