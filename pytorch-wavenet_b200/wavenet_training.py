"""The caller of the training hot path, with the reference's names (reference wavenet_training.py): ``WavenetTrainer`` with the
same constructor, ``train`` / ``validate`` and ``generate_audio`` -- SURVEY.md section 8 row f1.  What differs from upstream:

* the loss is ``fused_cross_entropy`` (wn_ce_fwd_bwd: loss and d(loss)/d(logits) in one pass over the logits instead of five
  eager passes), numerically F.cross_entropy(output, target) with mean reduction (wavenet_training.py:69);
* the default optimizer is ``FusedAdam`` (wn_adam_step: torch.optim.Adam's update for all tensors in one launch); any
  ``torch.optim`` class can still be passed, as in the reference;
* items may be class INDICES (``WavenetDataset(one_hot=False)``): they go through ``model.forward_indices``;
* items may be ``(x, condition, target)`` for a conditioned model (``WavenetDataset(condition_on_file=True)``): the
  condition (labels or vectors, one per item) goes to the model with its batch; ``condition`` may also be a dict with keys
  among ``condition`` and ``local_condition`` (a (C, F) frame-rate series per item), passed as the keyword arguments;
* when ``torch.distributed`` is initialised the loop is data parallel: the dataset is sharded with a DistributedSampler and
  gradients are averaged over the ranks block by block while the backward runs (data_parallel.make_data_parallel).
The Tensorboard side of the reference's Logger (model_logging.py) is out of scope; ``Logger`` here prints.
"""
import ctypes
import time

import numpy as np
import torch
import torch.distributed as dist
import torch.utils.data

import native


class _FusedCrossEntropy(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits, target):
        if logits.device.type != "cuda" or logits.dtype != torch.float32 or logits.dim() != 2:
            raise RuntimeError("fused_cross_entropy: logits must be a (N, classes) float32 CUDA tensor")
        logits = logits.contiguous()
        target = target.to(device=logits.device, dtype=torch.int64).contiguous().view(-1)
        n, c = logits.shape
        if target.numel() != n:
            raise RuntimeError(f"fused_cross_entropy: {n} rows of logits but {target.numel()} targets")
        lib = native.lib()
        with torch.cuda.device(logits.device):
            dlogits = torch.empty_like(logits)
            loss = torch.empty((), device=logits.device, dtype=torch.float32)
            work = torch.empty(lib.wn_ce_workspace_bytes() // 4, device=logits.device, dtype=torch.float32)
            stream = torch.cuda.current_stream(logits.device).cuda_stream
            native.check(lib.wn_ce_fwd_bwd(logits.data_ptr(), target.data_ptr(), dlogits.data_ptr(), loss.data_ptr(),
                                           work.data_ptr(), None, n, c, stream), "cross entropy")
        ctx.save_for_backward(dlogits)
        return loss

    @staticmethod
    def backward(ctx, grad_out):
        (dlogits,) = ctx.saved_tensors
        if getattr(ctx, "consumed", False):
            raise RuntimeError("fused_cross_entropy: backward called twice (the stored gradient is scaled in place; the "
                               "network's own autograd node does not support a second backward either)")
        ctx.consumed = True
        if ctx.needs_input_grad[0] and grad_out.numel() == 1 and grad_out.dtype == torch.float32 and dlogits.numel() % 4 == 0:
            # scale in place by the (device) scalar: no pass at all when it is 1, which is what loss.backward() passes
            with torch.cuda.device(dlogits.device):
                native.check(native.lib().wn_scale_by(dlogits.data_ptr(), dlogits.numel(), grad_out.contiguous().data_ptr(),
                                                      torch.cuda.current_stream(dlogits.device).cuda_stream), "scale dlogits")
            return dlogits, None
        return dlogits * grad_out, None


def fused_cross_entropy(logits, target):
    """F.cross_entropy(logits, target) (mean over rows) with the gradient computed in the same kernel."""
    return _FusedCrossEntropy.apply(logits, target)


class FusedAdam(torch.optim.Optimizer):
    """torch.optim.Adam (no amsgrad, L2 weight decay) with ONE native launch per step for all parameter tensors.

    As in torch, each parameter keeps its own step count (``state[p]["step"]``), which advances only on steps where the
    parameter has a gradient; parameters whose counts differ are updated by one launch per distinct count."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0, model=None):
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay))
        self._model = model              # its packed weight copies are invalidated after every step
        self._tables = {}

    def _table(self, params):
        key = tuple((p.data_ptr(), p.grad.data_ptr(), p.numel()) for p in params)
        t = self._tables.get(key)
        if t is not None:
            return t
        if len(self._tables) >= 16:      # parameter sets come and go (gradients that are None on some steps): keep a few
            self._tables.clear()
        dev = params[0].device
        segs, chunks = np.zeros((len(params), 5), dtype=np.int64), []
        for i, p in enumerate(params):
            st = self.state[p]
            if "exp_avg" not in st:
                st["exp_avg"], st["exp_avg_sq"] = torch.zeros_like(p), torch.zeros_like(p)
            segs[i] = (p.data_ptr(), p.grad.data_ptr(), st["exp_avg"].data_ptr(), st["exp_avg_sq"].data_ptr(), p.numel())
            chunks += [(i, c) for c in range((p.numel() + 4095) // 4096)]
        t = dict(segs=torch.from_numpy(segs).to(dev), n_chunks=len(chunks),
                 chunks=torch.tensor(chunks, dtype=torch.int32, device=dev).contiguous())
        self._tables[key] = t
        return t

    @torch.no_grad()
    def step(self, closure=None):
        loss = closure() if closure is not None else None
        lib = native.lib()
        for gi, group in enumerate(self.param_groups):
            params = [p for p in group["params"] if p.grad is not None]
            if not params:
                continue
            for p in params:
                if p.dtype != torch.float32 or not p.is_contiguous() or not p.grad.is_contiguous() or p.device.type != "cuda":
                    raise RuntimeError("FusedAdam handles contiguous float32 CUDA parameters")
            by_step = {}
            for p in params:
                st = self.state[p]
                st["step"] = int(st.get("step", 0)) + 1
                by_step.setdefault(st["step"], []).append(p)
            dev = params[0].device
            for step, ps in by_step.items():
                t = self._table(ps)
                with torch.cuda.device(dev):
                    native.check(lib.wn_adam_step_f64(t["segs"].data_ptr(), t["chunks"].data_ptr(), t["n_chunks"],
                                                      float(group["lr"]), float(group["betas"][0]), float(group["betas"][1]),
                                                      float(group["eps"]), float(group["weight_decay"]), step,
                                                      torch.cuda.current_stream(dev).cuda_stream), "adam step")
        if self._model is not None:
            self._model.invalidate_packed_weights()        # the kernel wrote the parameters behind autograd's version counters
        return loss


class Logger:
    """Console stand-in for the reference's Logger (model_logging.py:9-60): same call points, prints instead of Tensorboard."""

    def __init__(self, log_interval=50, validation_interval=200, generate_interval=500, trainer=None, generate_function=None):
        self.trainer = trainer
        self.log_interval, self.validation_interval, self.generate_interval = log_interval, validation_interval, generate_interval
        self.accumulated_loss = 0
        self.generate_function = generate_function

    def log(self, current_step, current_loss):
        self.accumulated_loss += current_loss
        if current_step % self.log_interval == 0:
            print("loss at step " + str(current_step) + ": " + str(self.accumulated_loss / self.log_interval))
            self.accumulated_loss = 0
        if current_step % self.validation_interval == 0 and self.trainer is not None and self.trainer.dataloader is not None:
            avg_loss, avg_accuracy = self.trainer.validate()
            print("validation loss: " + str(avg_loss) + "  validation accuracy: " + str(avg_accuracy * 100) + "%")
        if self.generate_function is not None and current_step % self.generate_interval == 0:
            self.generate_function(current_step)


class WavenetTrainer:
    def __init__(self, model, dataset, optimizer=FusedAdam, lr=0.001, weight_decay=0, gradient_clipping=None, logger=None,
                 snapshot_path=None, snapshot_name='snapshot', snapshot_interval=1000, dtype=torch.FloatTensor,
                 ltype=torch.LongTensor, num_workers=8):
        self.model = model
        self.dataset = dataset
        self.dataloader = None
        self.lr = lr
        self.weight_decay = weight_decay
        self.clip = gradient_clipping
        self.optimizer_type = optimizer
        kw = dict(model=model) if optimizer is FusedAdam else {}
        self.optimizer = optimizer(params=self.model.parameters(), lr=self.lr, weight_decay=self.weight_decay, **kw)
        self.logger = logger if logger is not None else Logger()
        self.logger.trainer = self
        self.snapshot_path = snapshot_path
        self.snapshot_name = snapshot_name
        self.snapshot_interval = snapshot_interval
        self.dtype, self.ltype = dtype, ltype                # kept for signature compatibility; tensors follow the model's device
        self.num_workers = num_workers
        self.world = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1
        self.rank = dist.get_rank() if self.world > 1 else 0
        if self.world > 1:
            import data_parallel
            data_parallel.make_data_parallel(self.model)

    def _device(self):
        return next(self.model.parameters()).device

    def _logits(self, x, condition=None):
        dev = self._device()
        if isinstance(condition, dict):              # {"condition": ..., "local_condition": ...}, batched by the default collate
            unknown = set(condition) - {"condition", "local_condition"}
            if unknown:
                raise ValueError(f"a condition dict may hold 'condition' and 'local_condition', not {sorted(unknown)}")
            kw = dict(condition)
        else:
            kw = dict(condition=condition)
        if x.dtype in (torch.uint8, torch.int64) and x.dim() == 2:
            return self.model.forward_indices(x.to(dev, non_blocking=True), **kw)
        return self.model(x.to(dev, torch.float32, non_blocking=True), **kw)

    @staticmethod
    def _unpack(batch):
        """(x, target) or (x, condition, target) -> x, condition or None, target"""
        if len(batch) == 3:
            return batch[0], batch[1], batch[2]
        x, target = batch
        return x, None, target

    def _loader(self, batch_size, shuffle):
        sampler = None
        if self.world > 1:
            sampler = torch.utils.data.distributed.DistributedSampler(self.dataset, num_replicas=self.world, rank=self.rank,
                                                                      shuffle=shuffle)
        return torch.utils.data.DataLoader(self.dataset, batch_size=batch_size, shuffle=shuffle and sampler is None,
                                           sampler=sampler, num_workers=self.num_workers, pin_memory=True,
                                           drop_last=self.world > 1)

    def train(self, batch_size=32, epochs=10, continue_training_at_step=0, max_steps=None):
        self.model.train()
        self.dataloader = self._loader(batch_size, shuffle=True)
        step = continue_training_at_step
        for current_epoch in range(epochs):
            if self.rank == 0:
                print("epoch", current_epoch)
            if self.world > 1:
                self.dataloader.sampler.set_epoch(current_epoch)
            tic = time.time()
            for batch in iter(self.dataloader):
                x, condition, target = self._unpack(batch)
                target = target.view(-1).to(self._device(), non_blocking=True)
                loss = fused_cross_entropy(self._logits(x, condition), target)
                self.optimizer.zero_grad()
                loss.backward()
                if self.clip is not None:
                    torch.nn.utils.clip_grad_norm_(self.model.parameters(), self.clip)
                self.optimizer.step()
                if not isinstance(self.optimizer, FusedAdam):
                    self.model.invalidate_packed_weights()
                step += 1
                if step == 100 and self.rank == 0:
                    print("one training step does take approximately " + str((time.time() - tic) * 0.01) + " seconds)")
                if step % self.snapshot_interval == 0 and self.snapshot_path is not None and self.rank == 0:
                    time_string = time.strftime("%Y-%m-%d_%H-%M-%S", time.gmtime())
                    torch.save(self.model, self.snapshot_path + '/' + self.snapshot_name + '_' + time_string)
                if self.rank == 0:
                    self.logger.log(step, float(loss.detach()))
                if max_steps is not None and step - continue_training_at_step >= max_steps:
                    return step
        return step

    def validate(self):
        self.model.eval()
        self.dataset.train = False
        total_loss, accurate, batches = 0.0, 0, 0
        loader = self._loader(self.dataloader.batch_size if self.dataloader is not None else 32, shuffle=False)
        with torch.no_grad():
            for batch in iter(loader):
                x, condition, target = self._unpack(batch)
                target = target.view(-1).to(self._device())
                output = self._logits(x, condition)
                total_loss += float(torch.nn.functional.cross_entropy(output, target))
                accurate += int((output.argmax(1) == target).sum())
                batches += 1
        avg_loss = total_loss / max(batches, 1)
        avg_accuracy = accurate / max(len(self.dataset) * self.dataset.target_length, 1)
        self.dataset.train = True
        self.model.train()
        return avg_loss, avg_accuracy


def generate_audio(model, length=8000, temperatures=[0., 1.]):
    return np.stack([model.generate_fast(length, temperature=temp) for temp in temperatures], axis=0)
