"""Whole-step CUDA graph for the launch-bound configurations (PixelCNN / ImageGPT on MNIST-sized inputs).

`Trainer._train_one_batch` (reference trainer.py:173-193) of a small model is a few milliseconds of GPU work behind
several hundred kernel launches; replaying the step as one CUDA graph removes the per-launch host cost.  The kernels
already take the stream explicitly and keep no host-side state per call, so the autograd step captures as is.  The
captured region is zero_grad -> forward -> loss -> backward -> clip_grad_norm_ -> Adam; the learning-rate decay of the
recipes' MultiplicativeLR is applied in place on the (tensor) learning rate between replays, and the two `.item()`
reads of the reference happen on the static outputs after the replay.
"""

import torch


class GraphedTrainStep:
    def __init__(self, model, params, loss_fn, example_x, lr, lr_gamma, max_norm=1e50, warmup=3):
        self.model, self.params, self.loss_fn = model, list(params), loss_fn
        self.lr0 = float(lr)
        self.lr = torch.tensor(float(lr), device=example_x.device)
        self.lr_gamma, self.max_norm = lr_gamma, max_norm
        self.opt = torch.optim.Adam(self.params, lr=self.lr, capturable=True)
        self.static_x = example_x.clone()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):  # warm-up on a side stream, as CUDA-graph capture of autograd requires
            for _ in range(warmup):
                self._eager_step()
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        self.opt.zero_grad(set_to_none=True)
        with torch.cuda.graph(self.graph):
            self.static_loss, self.static_norm, self.static_preds = self._eager_step()

    def _eager_step(self):
        """One training step; returns the loss, the gradient norm and the logits (the graph's static outputs)."""
        self.opt.zero_grad(set_to_none=True)
        preds = self.model(self.static_x)
        loss = self.loss_fn(preds, self.static_x)
        loss.backward()
        norm = torch.nn.utils.clip_grad_norm_(self.params, self.max_norm, foreach=True)
        self.opt.step()
        return loss.detach(), norm.detach(), preds.detach()

    @torch.no_grad()
    def reset(self, state_dict=None, lr=None):
        """Rewinds the step to a fresh optimizer (the capture's warm-up steps moved the weights and the Adam moments):
        optionally reloads `state_dict` into the model, zeroes the moments / step counters in place (the graph keeps
        reading the same tensors) and restores the learning rate."""
        if state_dict is not None:
            own = self.model.state_dict()
            for k, v in state_dict.items():
                if k in own:
                    own[k].copy_(v)
        for st in self.opt.state.values():
            for t in st.values():
                if torch.is_tensor(t):
                    t.zero_()
        if lr is not None:
            self.lr0 = float(lr)
        self.lr.fill_(self.lr0)

    def __call__(self, x):
        self.static_x.copy_(x, non_blocking=True)
        self.graph.replay()
        torch.autograd.graph.increment_version(self.params)  # the replay wrote them: stale bf16 copies must miss
        self.lr.mul_(self.lr_gamma)  # MultiplicativeLR of the recipes (image_gpt.py:156), in place for the graph
        return self.static_loss.item(), self.static_norm.item()
