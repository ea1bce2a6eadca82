"""Training / evaluation loop with the reference Trainer's interface (trainer/trainer/trainer.py:22-223) for this
package's entry points (row F4): fit / train_epoch / val_epoch, AdamW step with gradient clipping (35) and a
per-iteration OneCycleLR step, checkpoints in the reference's format ({"meta", "state_dict", "optimizer", "scheduler"},
trainer/utils/checkpoint.py:62-89, `module.` prefix stripped on load), detections gathered over the ranks and handed to
`dataset.evaluation`.  Differences that are the point of the GPU path: inputs move with non-blocking copies, the
gradient all-reduce is the bucketed / overlapped reducer of parallel.py instead of DDP, losses are logged from device
values read once per logging interval (the reference's `.cpu()` log values synchronise every iteration)."""
import logging
import os
import time

import torch
import torch.distributed as dist

from .parallel import BucketedGradAllReduce, default_buckets


def example_to_device(example, device, non_blocking=True):
    out = {}
    for k, v in example.items():
        if torch.is_tensor(v):
            out[k] = v.to(device, non_blocking=non_blocking)
        elif isinstance(v, list) and v and torch.is_tensor(v[0]):
            out[k] = [e.to(device, non_blocking=non_blocking) for e in v]
        else:
            out[k] = v
    return out


def save_checkpoint(model, filename, optimizer=None, scheduler=None, meta=None):
    sd = {k: v.detach().cpu() for k, v in model.state_dict().items()}
    ck = {"meta": meta or {}, "state_dict": sd}
    if optimizer is not None:
        ck["optimizer"] = optimizer.state_dict()
    if scheduler is not None:
        ck["scheduler"] = scheduler.state_dict()
    os.makedirs(os.path.dirname(os.path.abspath(filename)), exist_ok=True)
    torch.save(ck, filename)


def load_checkpoint(model, filename, map_location="cpu", strict=False):
    ck = torch.load(filename, map_location=map_location, weights_only=False)
    sd = ck.get("state_dict", ck.get("model", ck))
    sd = {(k[len("module."):] if k.startswith("module.") else k): v for k, v in sd.items()}
    model.load_state_dict(sd, strict=strict)
    return ck


class Trainer:
    def __init__(self, model, train_dataloader=None, val_dataloader=None, optimizer=None, lr_scheduler=None, clip_grad_val=0.0,
                 max_epochs=0, eval_every_nepochs=1, eval_epochs=None, logger=None, log_every_niters=50, work_dir="."):
        self.model, self.train_dataloader, self.val_dataloader = model, train_dataloader, val_dataloader
        self.optimizer, self.lr_scheduler = optimizer, lr_scheduler
        self.clip_grad_val, self.max_epochs = float(clip_grad_val), int(max_epochs)
        self.eval_every_nepochs, self.eval_epochs = eval_every_nepochs, eval_epochs
        self.logger = logger or logging.getLogger("pillarnext_b200")
        self.log_every_niters, self.work_dir = log_every_niters, work_dir
        self.rank = dist.get_rank() if dist.is_initialized() else 0
        self.world_size = dist.get_world_size() if dist.is_initialized() else 1
        self.epoch = self.global_step = 0
        self.reducer = BucketedGradAllReduce(default_buckets(model)) if (self.world_size > 1 and optimizer is not None) else None
        self.last_eval = None

    @property
    def device(self):
        return torch.device("cuda", torch.cuda.current_device())

    def load_checkpoint(self, filename, map_location="cpu", strict=False):
        self.logger.info("load checkpoint from %s", filename)
        return load_checkpoint(self.model, filename, map_location, strict)

    def save_checkpoint(self, filename_tmpl="epoch_{}.pth"):
        if self.rank == 0:
            save_checkpoint(self.model, os.path.join(self.work_dir, filename_tmpl.format(self.epoch)), self.optimizer,
                            self.lr_scheduler, dict(epoch=self.epoch, iter=self.global_step))

    def resume(self, filename):
        ck = self.load_checkpoint(filename, strict=True)
        self.epoch, self.global_step = ck["meta"]["epoch"], ck["meta"]["iter"]
        if "optimizer" in ck and self.optimizer is not None:
            self.optimizer.load_state_dict(ck["optimizer"])
        if "scheduler" in ck and self.lr_scheduler is not None:
            self.lr_scheduler.load_state_dict(ck["scheduler"])

    def train_iter(self, batch):
        ex = example_to_device(batch, self.device)
        loss, logs = self.model(ex)
        self.optimizer.zero_grad(set_to_none=True)
        loss.backward()
        if self.reducer is not None:
            self.reducer.finish()
        if self.clip_grad_val > 0:
            torch.nn.utils.clip_grad_norm_(self.model.parameters(), self.clip_grad_val)
        self.optimizer.step()
        if self.lr_scheduler is not None:
            self.lr_scheduler.step()
        self.global_step += 1
        return loss, logs

    def train_epoch(self):
        self.model.train()
        sampler = getattr(self.train_dataloader, "sampler", None)
        if hasattr(sampler, "set_epoch"):
            sampler.set_epoch(self.epoch)
        t0 = time.time()
        for i, batch in enumerate(self.train_dataloader):
            loss, logs = self.train_iter(batch)
            if self.rank == 0 and (i + 1) % self.log_every_niters == 0:
                self.logger.info("epoch %d iter %d/%d lr %.2e loss %.4f (%.1f it/s)", self.epoch + 1, i + 1, len(self.train_dataloader),
                                 self.optimizer.param_groups[0]["lr"], float(loss), (i + 1) / (time.time() - t0))
        self.epoch += 1
        self.save_checkpoint()

    @torch.no_grad()
    def val_epoch(self):
        self.model.eval()
        detections = {}
        for batch in self.val_dataloader:
            detections.update(self.model(example_to_device(batch, self.device)))
        if self.world_size > 1:
            dist.barrier()
            parts = [None] * self.world_size
            dist.all_gather_object(parts, detections)
            detections = {k: v for p in parts for k, v in p.items()}
        result = None
        if self.rank == 0:
            result = self.val_dataloader.dataset.evaluation(detections, output_dir=self.work_dir)
            self.logger.info("validation: %s", result)
        self.last_eval = result
        return result, detections

    def fit(self):
        while self.epoch < self.max_epochs:
            self.train_epoch()
            if self.val_dataloader is not None and self.eval_every_nepochs and self.epoch % self.eval_every_nepochs == 0:
                self.val_epoch()
