"""Whole-step CUDA-graph capture of the VxmDense training step.

The reference's loop (scripts/torch/train.py:199-220: forward, losses, backward, Adam) issues ~100 kernels per step
here; at ~10 ms per step the launch gaps are worth a millisecond.  `lr`, `lam` and the gradient scale are baked into the captured kernels' arguments: build a new GraphedTrainStep to change
them (an LR schedule needs a re-capture per change).  `GraphedTrainStep` captures ONE full step
(zero-grad, forward, NCC/MSE + Grad losses, backward, the single gradient allreduce, fused Adam) into a CUDA graph on
static input buffers and replays it; nothing in the captured region reads host state (the Adam step count lives on
the device, packed bf16 weights are re-derived inside the graph).
"""
import torch

from . import dist as vdist
from . import losses


class GraphedTrainStep:
    """`loss_fn(model, *inputs) -> loss` is the forward + loss of one step; the default is train.py's
    image loss (NCC, MutualInformation for image_loss="mi", or MSE) + lam * Grad('l2') on (source, target).  Any number of input tensors can be declared
    through `capture(*inputs)` (e.g. the two one-hot segmentations of the semi-supervised step)."""

    def __init__(self, model, optimizer, image_loss="ncc", lam=0.01, int_downsize=2, warmup=3, keep_warmup=False, loss_fn=None):
        self.model, self.opt = model, optimizer
        if image_loss == "ncc":
            self.img = losses.NCC().loss
        elif image_loss == "mi":   # cross-contrast: MutualInformation() with its defaults (16 bins, intensities in [0, 1])
            self.img = losses.MutualInformation().loss
        else:
            self.img = losses.MSE().loss
        self.grad = losses.Grad("l2", loss_mult=int_downsize).loss
        self.lam = lam
        self.warmup = warmup
        self.keep_warmup = keep_warmup
        self.loss_fn = loss_fn
        self.graph = None
        self.inputs = None
        self.loss = None

    # kept for callers that read the static buffers
    @property
    def src(self):
        return self.inputs[0]

    @property
    def trg(self):
        return self.inputs[1]

    def _forward_loss(self):
        if self.loss_fn is not None:
            return self.loss_fn(self.model, *self.inputs)
        y, flow = self.model(self.inputs[0], self.inputs[1])
        return self.img(self.inputs[1], y) + self.lam * self.grad(None, flow)

    def _step(self):
        self.opt.zero_grad()
        loss = self._forward_loss()
        loss.backward()
        vdist.allreduce_grads(self.opt.fp.grad)
        self.opt.step()
        return loss.detach()

    def capture(self, *inputs):
        """Warm up eagerly on a side stream, then capture one step.  `inputs` fix the static shapes."""
        self.inputs = [torch.empty_like(x) for x in inputs]
        for dst, x in zip(self.inputs, inputs):
            dst.copy_(x)
        # the warm-up steps are real optimizer steps on the first inputs: snapshot the optimizer state and put it back, so
        # that a captured run follows the same trajectory as an eager run from the same seed (keep_warmup=True keeps
        # them, e.g. to compare with an eager loop that also took them).  The model's buffers (a TemplateCreation's mean
        # stream) are state the warm-up advances too
        snap = None if self.keep_warmup else self.opt.snapshot()
        bufs = None if self.keep_warmup else [(b, b.clone()) for b in self.model.buffers()]
        dev = inputs[0].device
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(self.warmup):
                self._step()
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        if snap is not None:
            self.opt.restore(snap)
            with torch.no_grad():
                for b, saved in bufs:
                    b.copy_(saved)
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self.loss = self._step()
        return self

    def __call__(self, *inputs):
        """Replay.  Given inputs are copied into the static buffers first (device or pinned host tensors)."""
        for dst, x in zip(self.inputs, inputs):
            if x is not None:
                dst.copy_(x, non_blocking=True)
        self.graph.replay()
        # the captured Adam kernel rewrote the fp32 parameters behind torch's version counters: packed bf16 copies used
        # by a later EAGER forward (validation, registration) must be rebuilt
        from . import engine_bf16
        engine_bf16.bump_weights_epoch()
        return self.loss
