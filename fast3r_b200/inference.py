"""Drop-in for ``fast3r.dust3r.inference_multiview`` (reference: fast3r/dust3r/inference_multiview.py:22-104,
collation helpers fast3r/dust3r/utils/device.py:52-95).  Same signatures, same result structure
``{"views": [...], "preds": [...], "loss": None}`` moved to CPU, same optional ``profiling_info``.

Precision mapping (SURVEY.md Q1; reference: inference_multiview.py:41-49).  The reference disables autocast only
for the *string* "32" (true fp32); ``torch.bfloat16`` selects bf16 autocast and anything else the default autocast
dtype.  Here:
  * ``"32"`` and ``torch.float32`` -> the parity path (``precision="fp32"``: fp32 activations, hi/lo-split bf16
    tensor-core products; ~1e-5 rel-L2 of the reference's fp32 result).  ``torch.float32`` is what README/demo pass
    and clearly intend fp32, although the reference then silently runs its default autocast dtype (Q1).
  * everything else (``torch.bfloat16``, ``torch.float16``, "bf16", "16", ...) -> the fast path (``precision="bf16"``:
    bf16 operands, fp32 accumulation / residual stream / statistics), closer to fp32 than the reference's own
    bf16-autocast path.  On a model set to ``precision="fp16"`` (``model.set_precision("fp16")``) the fast path runs
    fp16 operands instead; ``torch.float16`` does not select fp16 by itself.
Preds always come back fp32.
"""
from __future__ import annotations

import numpy as np
import torch

_MOVE_KEYS = "img pts3d valid_mask camera_pose camera_intrinsics F_matrix corres".split()
_KEEP_HOST_REFS = False  # set by _forward_to_host around the model call


def _map_leaves(obj, leaf_fn):
    """Applies leaf_fn to every non-container leaf of a nested dict / list / tuple structure (structure preserved)."""
    if isinstance(obj, dict):
        return {key: _map_leaves(val, leaf_fn) for key, val in obj.items()}
    if isinstance(obj, (list, tuple)):
        return type(obj)(_map_leaves(val, leaf_fn) for val in obj)
    return leaf_fn(obj)


def todevice(batch, device, callback=None, non_blocking=False):
    """Behaviour of fast3r/dust3r/utils/device.py:14-49: move every tensor / ndarray leaf to ``device``
    ("numpy" converts tensors to ndarrays instead); other leaves pass through."""
    if callback:
        batch = callback(batch)

    def move(leaf):
        if device == "numpy":
            return leaf.detach().cpu().numpy() if isinstance(leaf, torch.Tensor) else leaf
        if isinstance(leaf, np.ndarray):
            leaf = torch.from_numpy(leaf)
        return leaf.to(device, non_blocking=non_blocking) if torch.is_tensor(leaf) else leaf

    return _map_leaves(batch, move)


def to_cpu(x):
    return todevice(x, "cpu")


def listify(elems):
    return [x for e in elems for x in e]


def _stack_arrays(samples, lists):
    """Tensors / ndarrays of the samples of one field: concatenated along dim 0 (or flattened into a list).
    A one-sample "batch" (what inference() builds) is returned as is instead of torch.cat([x]): same values, but no
    2.26 MB host copy per view, and the caller's page-locked buffers stay page-locked for the async H2D."""
    tensors = [torch.from_numpy(x) if isinstance(x, np.ndarray) else x for x in samples]
    if lists:
        return listify(tensors)
    return tensors[0] if len(tensors) == 1 else torch.cat(tensors)


def collate_with_cat(whatever, lists=False):
    """Behaviour of fast3r/dust3r/utils/device.py:60-91: merge a sequence of samples field by field.  The first sample
    decides how a field is merged: None -> None; python scalars / strings -> the sequence itself; tuples -> merged
    column-wise; dicts -> merged key-wise; tensors / ndarrays -> concatenated; anything else -> sequences chained."""
    if isinstance(whatever, dict):
        return {key: collate_with_cat(vals, lists=lists) for key, vals in whatever.items()}
    if not isinstance(whatever, (tuple, list)) or len(whatever) == 0:
        return whatever
    first, seq_type = whatever[0], type(whatever)
    if first is None:
        return None
    if isinstance(first, (bool, float, int, str)):
        return whatever
    if isinstance(first, tuple):
        return seq_type(collate_with_cat(column, lists=lists) for column in zip(*whatever))
    if isinstance(first, dict):
        return {key: collate_with_cat([sample[key] for sample in whatever], lists=lists) for key in first}
    if isinstance(first, (torch.Tensor, np.ndarray)):
        return _stack_arrays(whatever, lists)
    return sum(whatever, seq_type())


def check_if_same_size(imgs):
    shapes = [img["img"].shape[-2:] for img in imgs]
    return all(shape == shapes[0] for shape in shapes)


class _HostSink:
    """Receives finished chunks of the model's output buffers and copies them to page-locked host memory on a side
    stream while the model keeps computing (used by _forward_to_host; the model calls chunk_done per head chunk)."""
    _streams = {}

    def __init__(self, device):
        self.host = {}  # device storage ptr -> pinned uint8 host buffer of the same size
        if device.index is None:
            device = torch.device("cuda", torch.cuda.current_device())
        self.device = device
        key = (device.type, device.index)
        if key not in _HostSink._streams:
            _HostSink._streams[key] = torch.cuda.Stream(device=device)
        self.stream = _HostSink._streams[key]

    def chunk_done(self, tensors, start, count):
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(self.device))  # the stream the head kernels of this chunk were enqueued on
        self.stream.wait_event(ev)
        with torch.cuda.stream(self.stream):
            for t in tensors:
                st = t.untyped_storage()
                k = st.data_ptr()
                if k not in self.host:
                    self.host[k] = torch.empty(st.nbytes(), dtype=torch.uint8, pin_memory=True)
                row = t[0].numel() * t.element_size()
                lo, hi = t.storage_offset() * t.element_size() + start * row, t.storage_offset() * t.element_size() + (start + count) * row
                dev_bytes = torch.empty(0, dtype=torch.uint8, device=t.device).set_(st)
                self.host[k][lo:hi].copy_(dev_bytes[lo:hi], non_blocking=True)

    def finish(self):
        self.stream.synchronize()
        return self.host


def _preds_to_cpu(preds, prefilled=None):
    """D2H of the predictions (§8 f1).  The per-view tensors are slices of a few large device buffers; each
    distinct buffer is copied ONCE, asynchronously, into page-locked host memory (torch's caching host allocator
    recycles the blocks, results own their memory) and the per-view CPU tensors are rebuilt as views of it.
    Same values / shapes / dtypes as the reference's per-tensor ``.to("cpu")`` (utils/device.py:52)."""
    groups = {}
    for p in preds:
        for v in p.values():
            if torch.is_tensor(v) and v.is_cuda:
                st = v.untyped_storage()
                groups.setdefault(st.data_ptr(), (st, v.device))
    if not groups:
        return to_cpu(preds)
    host = dict(prefilled or {})
    devices = set()
    for key, (st, dev) in groups.items():
        devices.add(dev)
        if key in host:
            continue  # already streamed to the host chunk by chunk during the forward
        dev_bytes = torch.empty(0, dtype=torch.uint8, device=dev).set_(st)
        h = torch.empty(dev_bytes.numel(), dtype=torch.uint8, pin_memory=True)
        h.copy_(dev_bytes, non_blocking=True)
        host[key] = h
    for dev in devices:
        torch.cuda.current_stream(dev).synchronize()
    out = []
    for p in preds:
        q = {}
        for k, v in p.items():
            if torch.is_tensor(v) and v.is_cuda:
                h = host[v.untyped_storage().data_ptr()]
                q[k] = torch.empty(0, dtype=v.dtype).set_(h.untyped_storage(), v.storage_offset(), v.shape, v.stride())
            else:
                q[k] = to_cpu(v)
        out.append(q)
    return out


def precision_of(dtype) -> str:
    """Kernel precision for an ``inference(dtype=...)`` / ``loss_of_one_batch(precision=...)`` value (module docstring)."""
    if dtype == "32" or dtype is torch.float32 or dtype == "fp32" or dtype == "float32":
        return "fp32"
    return "bf16"


class _precision_scope:
    """Runs the model at the precision of ``dtype`` (precision_of) for the duration of a call.  A model set to "fp16"
    keeps it for every dtype that selects the fast path: its fast path is fp16."""

    def __init__(self, model, dtype):
        self.model, self.want = model, precision_of(dtype)

    def __enter__(self):
        self.prev = getattr(self.model, "precision", None)
        if self.prev is not None:
            self.model.precision = "fp16" if (self.want == "bf16" and self.prev == "fp16") else self.want

    def __exit__(self, *exc):
        if self.prev is not None:
            self.model.precision = self.prev


def _upload(batch, model, device):
    """H2D of the view tensors of one collated sample, in place."""
    sharded = getattr(model, "sp_group", None) is not None  # sequence parallel: the model uploads only its own views
    for view in batch:
        for name in _MOVE_KEYS:
            if name not in view or (sharded and name == "img"):
                continue
            src = view[name]
            view[name] = src.to(device, non_blocking=True)
            if _KEEP_HOST_REFS and src.device.type == "cpu" and device.type != "cpu":
                view.setdefault("_host_copy", {})[name] = src  # lets inference() hand the same host tensor back


def _views_to_cpu(views):
    """The views of a result on the host.  The reference copies the (just uploaded) inputs back to the host (to_cpu(res),
    inference_multiview.py:92); the bytes are identical to the caller's host tensors, so those are returned instead of a
    second PCIe transfer.  NOTE: the returned views' "img" therefore ALIASES the caller's input tensor (the reference
    returns a copy)."""
    views_cpu = []
    for view in views:
        host = view.pop("_host_copy", {})
        views_cpu.append({k: (host[k] if k in host else to_cpu(v)) for k, v in view.items()})
    return views_cpu


def loss_of_one_batch(batch, model, criterion, device, precision, symmetrize_batch=False, use_amp=False, ret=None,
                      profiling=False):
    """fast3r/dust3r/inference_multiview.py:22-67 (H2D of the view tensors, precision selection, model call, optional
    criterion)."""
    device = torch.device(device)
    _upload(batch, model, device)
    views = batch
    with _precision_scope(model, precision):
        if profiling:
            preds, profiling_info = model(views, profiling=profiling)
        else:
            preds = model(views, profiling=profiling)
    loss = criterion(views, preds) if criterion is not None else None
    result = dict(views=views, preds=preds, loss=loss)
    if profiling:
        result["profiling_info"] = profiling_info
    return result[ret] if ret else result


def _forward_to_host(model, device, call):
    """Runs ``call()``, which uploads views (_upload), runs the model and returns (one preds list per sample, the rest),
    with the uploaded views' host tensors kept for _views_to_cpu and each finished head chunk streamed to page-locked
    host memory (_HostSink).  Returns (the preds lists on the host, the rest)."""
    global _KEEP_HOST_REFS
    _KEEP_HOST_REFS = True
    dev = torch.device(device)
    sink = _HostSink(dev) if (dev.type == "cuda" and hasattr(model, "_host_sink")) else None
    try:
        if sink is not None:
            model._host_sink = sink
        preds, rest = call()
    finally:
        _KEEP_HOST_REFS = False
        if sink is not None:
            model._host_sink = None
    # one D2H pass over all samples: the predictions of a shape group share their device buffers across samples
    flat = iter(_preds_to_cpu([p for sample in preds for p in sample], sink.finish() if sink is not None else None))
    return [[next(flat) for _ in sample] for sample in preds], rest


@torch.no_grad()
def inference(multiple_views_in_one_sample, model, device, dtype, verbose=True, profiling=False):
    """fast3r/dust3r/inference_multiview.py:70-99."""
    if verbose:
        print(f">> Inference with model on {len(multiple_views_in_one_sample)} images")

    def call():
        res = loss_of_one_batch(collate_with_cat([tuple(multiple_views_in_one_sample)]), model, None, device, dtype,
                                profiling=profiling)
        return [res["preds"]], res

    (preds,), res = _forward_to_host(model, device, call)
    result = collate_with_cat([dict(views=_views_to_cpu(res["views"]), preds=preds, loss=to_cpu(res["loss"]))],
                              lists=not check_if_same_size(multiple_views_in_one_sample))
    profiling_info = res.get("profiling_info")
    if profiling_info is not None:
        return result, profiling_info
    return result


@torch.no_grad()
def inference_many(samples, model, device, dtype, verbose=True, profiling=False):
    """Several scenes in one model call (Fast3R.forward_many).  ``samples``: a list of view lists, one per scene.
    Returns a list whose element i has the structure of ``inference(samples[i], model, device, dtype)``: ``views``,
    ``preds`` and ``loss=None``, on the host; with ``profiling``, (that list, one profiling_info for the whole call).
    The image ids are drawn per scene in scene order, as a loop of inference() calls draws them."""
    if verbose:
        print(f">> Inference with model on {len(samples)} samples, {sum(len(s) for s in samples)} images")
    batches = [collate_with_cat([tuple(views)]) for views in samples]

    def call():
        for batch in batches:
            _upload(batch, model, torch.device(device))
        with _precision_scope(model, dtype):
            out = model.forward_many(batches, profiling=profiling)
        return out if profiling else (out, None)

    preds, profiling_info = _forward_to_host(model, device, call)
    result = [collate_with_cat([dict(views=_views_to_cpu(batch), preds=sample, loss=None)],
                               lists=not check_if_same_size(views))
              for views, batch, sample in zip(samples, batches, preds)]
    if profiling:
        return result, profiling_info
    return result
