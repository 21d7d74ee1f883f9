"""Fused tail of the training step: gradient-norm clip + SGD over flat buffers.

Drop-in for the pair the reference uses (train.py:32-35,95-97):

    grad_norm = nn.utils.clip_grad_norm(model.parameters(), 200)
    optimizer.step()                       # torch.optim.SGD(lr, momentum)

    opt = FlatSGD(model, lr=1e-3, momentum=0.0, max_grad_norm=200, world_size=1)
    opt.zero_grad(); loss = model.loss(batch); loss.backward()
    grad_norm = opt.step()                 # all-reduce (if world_size > 1) + clip + update

Parameters and gradients are re-pointed to views of two contiguous fp32 buffers (state_dict names
and values are unchanged), so zero_grad is one memset, the data-parallel all-reduce runs over
slices of one buffer (one per GRU layer, issued during backward so that it overlaps the remaining
layers, plus one for the rest), and clip + update are two kernels (csrc/elementwise.cu) with no host synchronisation: the
clip coefficient stays on the device.  `step()` returns the pre-clip gradient norm as a 0-dim
CUDA tensor (what train.py logs as grad_norm).
"""
import torch

from . import _lib, ops
from .parallel import BucketReducer


class FlatSGD:
    def __init__(self, model, lr, momentum=0.0, max_grad_norm=200.0, world_size=1, group=None,
                 overlap=True):
        self.lr = float(lr)
        self.momentum = float(momentum)
        self.max_norm = float(max_grad_norm)
        self.world = world_size
        self.group = group
        # flat order: the GRU parameters grouped per layer as [w_ih fwd|rev][w_hh fwd|rev]
        # [b_ih fwd|rev][b_hh fwd|rev], so that the direction-concatenated operands the kernels
        # take are plain VIEWS of the flat buffers; everything else in module order
        self.gru_groups = []
        ordered, seen = [], set()
        for mod in model.modules():
            if isinstance(mod, torch.nn.GRU) and mod.bias:
                ndir = 2 if mod.bidirectional else 1
                for l in range(mod.num_layers):
                    sfx = ["_l%d%s" % (l, "_reverse" if d else "") for d in range(ndir)]
                    grp = [[getattr(mod, kind + s_) for s_ in sfx]
                           for kind in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")]
                    flat = [q for part in grp for q in part]
                    if all(q.requires_grad and id(q) not in seen for q in flat):
                        self.gru_groups.append(grp)
                        for q in flat:
                            seen.add(id(q))
                            ordered.append(q)
        ordered += [p for p in model.parameters() if p.requires_grad and id(p) not in seen]
        self.params = ordered
        dev = self.params[0].device
        _lib.require_cuda(self.params[0], "model parameters")
        # 16-byte align every parameter inside the flat fp32 AND bf16 buffers (8 elements)
        offs, n = [], 0
        for p in self.params:
            offs.append(n)
            n += (p.numel() + 7) // 8 * 8
        self.n = n
        self.flat_p = torch.zeros(n, dtype=torch.float32, device=dev)
        self.flat_g = torch.zeros(n, dtype=torch.float32, device=dev)
        self.mom = torch.zeros(n, dtype=torch.float32, device=dev) if self.momentum != 0 else None
        self.sumsq = torch.zeros(1, dtype=torch.float32, device=dev)
        nb = _lib.workspace_size(_lib.load().sb_sumsq_workspace_size)
        self.sumsq_ws = torch.zeros(nb, dtype=torch.uint8, device=dev)
        self.spans = {}
        self.offs = {}
        for p, o in zip(self.params, offs):
            view = self.flat_p[o:o + p.numel()].view_as(p)
            view.copy_(p.data)
            p.data = view
            p.grad = self.flat_g[o:o + p.numel()].view_as(p)
            self.spans[id(p)] = (o, o + (p.numel() + 7) // 8 * 8)
            self.offs[id(p)] = o
        # bf16 shadow of the parameters, rewritten by every step(): the tensor-core operands
        self.flat_p16 = self.flat_p.to(torch.bfloat16)
        self._register_operands()
        self.reducer = BucketReducer(self.flat_g, world_size, group)
        # the weight-gradient GEMMs accumulate straight into the flat gradient buffer (opt-in)
        ops.set_grad_sink(True)
        if world_size > 1 and overlap:
            # GRU backward announces each layer's gradients as soon as they are final
            ops.set_grad_ready_hook(self._grads_ready, guard=self._guard_second_backward)

    def _register_operands(self):
        """Hand ops the per-layer GRU operands as views of the flat buffers (bf16 weights of both
        directions concatenated, fp32 biases): no per-step cast / cat kernels.  The cache entry
        carries the parameters' version counters; ops ignores it when a parameter was modified by
        anything but step() (load_state_dict, manual edits) until the next step() re-syncs it."""
        self._op_entries = []
        for grp in self.gru_groups:
            w_ih, w_hh, b_ih, b_hh = grp
            ndir = len(w_ih)

            def adjacent(ps):
                return all(self.offs[id(ps[d + 1])] == self.offs[id(ps[d])] + ps[d].numel()
                           for d in range(len(ps) - 1))
            if not all(adjacent(ps) for ps in grp) or w_ih[0].shape[1] % 8 != 0:
                continue
            H3, In = w_ih[0].shape
            H = w_hh[0].shape[1]
            o = self.offs
            entry = {
                "wih": self.flat_p16[o[id(w_ih[0])]:o[id(w_ih[0])] + ndir * H3 * In].view(ndir * H3, In),
                "whh": self.flat_p16[o[id(w_hh[0])]:o[id(w_hh[0])] + ndir * H3 * H].view(ndir, H3, H),
                "bih": self.flat_p[o[id(b_ih[0])]:o[id(b_ih[0])] + ndir * H3],
                "bhh": self.flat_p[o[id(b_hh[0])]:o[id(b_hh[0])] + ndir * H3].view(ndir, H3),
                "params": [q for part in grp for q in part],
            }
            entry["versions"] = [q._version for q in entry["params"]]
            self._op_entries.append(entry)
            ops.register_gru_operands(w_ih[0], entry)

    def refresh_operands(self):
        """re-derive the bf16 shadow from the fp32 parameters (after load_state_dict etc.)"""
        self.flat_p16.copy_(self.flat_p)
        for e in self._op_entries:
            e["versions"] = [q._version for q in e["params"]]

    def _guard_second_backward(self, params):
        spans = [self.spans.get(id(p)) for p in params]
        spans = [sp for sp in spans if sp is not None]
        if not spans:
            return
        lo, hi = min(sp[0] for sp in spans), max(sp[1] for sp in spans)
        if any(plo < hi and lo < phi for plo, phi, _ in self.reducer.pending):
            raise RuntimeError(
                "FlatSGD(overlap=True): a second backward pass before step() would add local "
                "gradients into slices that are already being all-reduced; use overlap=False "
                "for gradient accumulation")

    def _check_views(self):
        """model.cuda()/.to() or zero_grad(set_to_none=True) silently detach the flat views"""
        lo, hi = self.flat_p.data_ptr(), self.flat_p.data_ptr() + 4 * self.n
        glo, ghi = self.flat_g.data_ptr(), self.flat_g.data_ptr() + 4 * self.n
        for p in self.params:
            if not (lo <= p.data_ptr() < hi):
                raise RuntimeError("FlatSGD: a parameter no longer lives in the flat buffer "
                                   "(model moved after the optimizer was built?)")
            if p.grad is None or not (glo <= p.grad.data_ptr() < ghi):
                raise RuntimeError("FlatSGD: a .grad no longer lives in the flat gradient buffer "
                                   "(zero_grad(set_to_none=True)? use FlatSGD.zero_grad())")

    def state_dict(self):
        return {"lr": self.lr, "momentum": self.momentum, "max_grad_norm": self.max_norm,
                "mom": None if self.mom is None else self.mom.detach().cpu().clone()}

    def load_state_dict(self, state):
        self.lr = float(state["lr"])
        self.momentum = float(state["momentum"])
        self.max_norm = float(state.get("max_grad_norm", self.max_norm))
        mom = state.get("mom")
        if self.momentum != 0:
            if self.mom is None:
                self.mom = torch.zeros_like(self.flat_p)
            if mom is not None:
                if mom.numel() != self.n:
                    raise ValueError("FlatSGD.load_state_dict: momentum buffer size mismatch")
                self.mom.copy_(mom.to(self.mom.device))
        else:
            self.mom = None

    def _grads_ready(self, params):
        spans = [self.spans.get(id(p)) for p in params]
        if any(s is None for s in spans):
            return
        self.reducer.ready(min(s[0] for s in spans), max(s[1] for s in spans))

    def zero_grad(self, set_to_none=False):
        self.flat_g.zero_()

    def all_reduce(self):
        self.reducer.finish()

    def step(self):
        lib = _lib.load()
        self._check_views()
        self.all_reduce()
        sp = _lib.stream_ptr()
        ops._launch("sumsq", 0.0, lambda: lib.sb_sumsq(self.flat_g.data_ptr(), self.n,
                                                       self.sumsq.data_ptr(),
                                                       self.sumsq_ws.data_ptr(), sp))
        ops._launch("sgd_clip_step", 0.0,
                    lambda: lib.sb_sgd_clip_step(self.flat_p.data_ptr(), self.flat_g.data_ptr(),
                                                 _lib.ptr(self.mom), self.flat_p16.data_ptr(),
                                                 self.n, self.sumsq.data_ptr(), self.lr,
                                                 self.momentum, self.max_norm, sp))
        for e in self._op_entries:       # the kernel just re-derived every shadow value
            e["versions"] = [q._version for q in e["params"]]
        return self.sumsq.sqrt().squeeze(0)
