"""Drop-in for `functions.ctc` of the warp-ctc pytorch_binding the reference imports
(speech/models/ctc_model.py:9, call site :34-40; dependency cloned by Makefile:4-7).

    loss_fn = CTCLoss()
    loss = loss_fn(acts, labels, act_lens, label_lens)     # 1-element tensor, shape (1,)

    acts        FloatTensor (B, T, V) batch-first RAW logits on the CUDA device (softmax internal)
    labels      IntTensor  (sum(label_lens),)  flat, CPU or CUDA
    act_lens    IntTensor  (B,)  CPU or CUDA
    label_lens  IntTensor  (B,)  CPU or CUDA

The blank index defaults to the LAST class (V-1), which is what the reference's CTC model
assumes (ctc_model.py:18,59).  The minibatch reduction is a SUM (size_average=False), the
warp-ctc binding's default; both are constructor keywords because the un-vendored dependency
could not be inspected (SURVEY.md §8b).
"""
import torch

from .. import _lib


def ctc_costs_and_grads(acts, labels, act_lens, label_lens, blank=None, need_grad=True):
    """Run the fused sm_90a CTC kernel.  Returns (costs (B,), grads (B,T,V) or None)."""
    _lib.require_cuda(acts, "acts")
    lib = _lib.load()
    if acts.dtype != torch.float32:
        acts = acts.float()
    acts = acts.contiguous()
    B, T, V = acts.shape
    if blank is None:
        blank = V - 1
    dev = acts.device

    lab = labels.detach().to("cpu", torch.int32).reshape(-1)
    llen = label_lens.detach().to("cpu", torch.int32).reshape(-1)
    alen = act_lens.detach().to("cpu", torch.int32).reshape(-1)
    if llen.numel() != B or alen.numel() != B:
        raise ValueError("act_lens / label_lens must have one entry per utterance")
    if int(llen.sum()) != lab.numel():
        raise ValueError("labels has %d entries but label_lens sums to %d"
                         % (lab.numel(), int(llen.sum())))
    if lab.numel() and (int(lab.min()) < 0 or int(lab.max()) >= V):
        raise ValueError("label out of range")
    max_l = int(llen.max()) if B else 0
    offs = torch.zeros(B, dtype=torch.int32)
    if B > 1:
        offs[1:] = torch.cumsum(llen[:-1], 0)
    # one packed host->device copy: [labels | offsets | label_lens | act_lens]
    n_lab = lab.numel()
    packed = torch.cat([lab, offs, llen, alen]).pin_memory().to(dev, non_blocking=True)
    d_lab = packed[:n_lab]
    d_off = packed[n_lab:n_lab + B]
    d_llen = packed[n_lab + B:n_lab + 2 * B]
    d_alen = packed[n_lab + 2 * B:]

    import ctypes
    nbytes = ctypes.c_size_t(0)
    _lib.check(lib.sb_ctc_workspace_size(B, T, V, max_l, ctypes.byref(nbytes)),
               "sb_ctc_workspace_size")
    ws = torch.empty(nbytes.value, dtype=torch.uint8, device=dev)
    costs = torch.empty(B, dtype=torch.float32, device=dev)
    grads = torch.empty_like(acts) if need_grad else None
    from .. import ops
    with torch.cuda.device(dev):
        sp = _lib.stream_ptr()
        ops._launch("ctc_fwd_bwd", 0.0,
                    lambda: lib.sb_ctc_fwd_bwd(acts.data_ptr(), _lib.ptr(grads), d_lab.data_ptr(),
                                               d_off.data_ptr(), d_llen.data_ptr(),
                                               d_alen.data_ptr(), B, T, V, int(blank), max_l,
                                               costs.data_ptr(), ws.data_ptr(), nbytes.value, sp))
    return costs, grads


class _CTCFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, acts, labels, act_lens, label_lens, blank, size_average):
        need_grad = acts.requires_grad
        costs, grads = ctc_costs_and_grads(acts, labels, act_lens, label_lens, blank, need_grad)
        loss = costs.sum().reshape(1)
        if size_average:
            loss = loss / acts.shape[0]
            if grads is not None:
                grads = grads / acts.shape[0]
        ctx.grads = grads
        ctx.costs = costs
        return loss

    @staticmethod
    def backward(ctx, grad_out):
        g = ctx.grads
        if g is None:
            return None, None, None, None, None, None
        return g * grad_out.reshape(1, 1, 1), None, None, None, None, None


class CTCLoss(torch.nn.Module):
    def __init__(self, blank=None, size_average=False):
        super().__init__()
        self.blank = blank
        self.size_average = size_average

    def forward(self, acts, labels, act_lens, label_lens):
        return _CTCFunction.apply(acts, labels, act_lens, label_lens, self.blank,
                                  self.size_average)
