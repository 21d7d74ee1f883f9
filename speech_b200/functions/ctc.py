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

from .. import _lib, ops


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
    (d_lab, d_off, d_llen, d_alen), max_l = _lib.pack_labels(labels, label_lens, act_lens, B, dev,
                                                            num_classes=V)
    nbytes = _lib.workspace_size(lib.sb_ctc_workspace_size, B, T, V, max_l)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    costs = torch.empty(B, dtype=torch.float32, device=dev)
    grads = torch.empty_like(acts) if need_grad else None
    with torch.cuda.device(dev):
        sp = _lib.stream_ptr()
        ops._launch("ctc_fwd_bwd", 0.0,
                    lambda: lib.sb_ctc_fwd_bwd(acts.data_ptr(), _lib.ptr(grads), d_lab.data_ptr(),
                                               d_off.data_ptr(), d_llen.data_ptr(),
                                               d_alen.data_ptr(), B, T, V, int(blank), max_l,
                                               costs.data_ptr(), ws.data_ptr(), nbytes, sp))
    return costs, grads


def ctc_viterbi(acts, labels, act_lens, label_lens, blank=None):
    """Viterbi (forced) alignment of each transcript to its logits: the best single path through
    the lattice the loss sums over (sb_ctc_viterbi; same inputs as the loss, blank = last class by
    default).  Returns, on the device, path (B, T) int32 -- the index of the label each frame is
    aligned to, -1 for blank, -2 past act_lens[b] and everywhere for an utterance with no
    alignment -- and scores (B,) float64, the path's log-probability (-inf without alignment)."""
    _lib.require_cuda(acts, "acts")
    lib = _lib.load()
    if acts.dtype != torch.float32:
        acts = acts.float()
    acts = acts.contiguous()
    B, T, V = acts.shape
    if blank is None:
        blank = V - 1
    dev = acts.device
    (d_lab, d_off, d_llen, d_alen), max_l = _lib.pack_labels(labels, label_lens, act_lens, B, dev,
                                                            num_classes=V)
    nbytes = _lib.workspace_size(lib.sb_ctc_viterbi_workspace_size, B, T, V, max_l)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    path = torch.empty(B, T, dtype=torch.int32, device=dev)
    scores = torch.empty(B, dtype=torch.float64, device=dev)
    # no labels in the batch: an empty tensor has no address, and no label is read
    lab_ptr = d_lab.data_ptr() or d_off.data_ptr()
    with torch.cuda.device(dev):
        sp = _lib.stream_ptr()
        ops._launch("ctc_viterbi", 0.0,
                    lambda: lib.sb_ctc_viterbi(acts.data_ptr(), lab_ptr, d_off.data_ptr(),
                                               d_llen.data_ptr(), d_alen.data_ptr(), B, T, V,
                                               int(blank), max_l, path.data_ptr(),
                                               scores.data_ptr(), ws.data_ptr(), nbytes, sp))
    return path, scores


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
