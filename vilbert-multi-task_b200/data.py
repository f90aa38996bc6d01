"""Input-pipeline edge of the hot path (SURVEY.md §8 f3): what sits between the reference's data loaders and `model(...)` in
vilbert/task_utils.py:186-310 — moving a batch to the GPU and reshaping / expanding it per task `process` type.

* `PinnedBatchPrefetcher`: double-buffered pinned-host -> device copies on a copy stream, one batch ahead of the compute stream
  (the reference does `t.cuda(non_blocking=True)` from pageable memory inside the step, task_utils.py:187). This is the code path
  `bench.py` times as `e2e`.
* `expand_batch`: the four `process` variants of task_utils.py:198-310. `retrieval` and `nlvr` are pure views; `expand` / `dialog`
  replicate every image's 2048-d region features, boxes and mask once per answer option — done here by ONE device kernel per
  tensor (`vb_repeat_rows`) instead of `unsqueeze().expand().contiguous()` chains.
"""
import torch

from . import _lib as L


def repeat_rows(x, repeats):
    """x [B, ...] -> [B * repeats, ...] with every item repeated consecutively (== x.unsqueeze(1).expand(B, repeats, ...).reshape)."""
    if repeats == 1:
        return x
    x = x.contiguous()
    item_bytes = x[0].numel() * x.element_size()
    if not x.is_cuda or item_bytes % 16 or x.data_ptr() % 16:
        return x.unsqueeze(1).expand(x.shape[0], repeats, *x.shape[1:]).reshape(x.shape[0] * repeats, *x.shape[1:])
    out = torch.empty((x.shape[0] * repeats,) + tuple(x.shape[1:]), dtype=x.dtype, device=x.device)
    L.call(L.lib().vb_repeat_rows, x, out, item_bytes, x.shape[0], repeats)
    return out


def expand_batch(process, features, spatials, image_mask, question, input_mask, segment_ids, co_attention_mask=None):
    """Returns (features, spatials, image_mask, question, input_mask, segment_ids, co_attention_mask, batch_size, num_options) shaped
    as `model(...)` expects, following task_utils.py:198-310 for process in {"normal", "expand", "retrieval", "nlvr", "dialog"}."""
    B = features.size(0)
    num_options = 1
    if process == "dialog":
        nround, num_options = question.size(1), question.size(2)
        R = nround * num_options
        features, spatials, image_mask = repeat_rows(features, R), repeat_rows(spatials, R), repeat_rows(image_mask, R)
        question = question.reshape(-1, question.size(3))
        input_mask = input_mask.reshape(-1, input_mask.size(3))
        segment_ids = segment_ids.reshape(-1, segment_ids.size(3))
        if co_attention_mask is not None:
            co_attention_mask = co_attention_mask.reshape(-1, co_attention_mask.size(3), co_attention_mask.size(4))
        B = B * nround
    elif process == "expand":
        num_options = question.size(1)
        features, spatials, image_mask = repeat_rows(features, num_options), repeat_rows(spatials, num_options), repeat_rows(image_mask, num_options)
        question = question.reshape(-1, question.size(2))
        input_mask = input_mask.reshape(-1, input_mask.size(2))
        segment_ids = segment_ids.reshape(-1, segment_ids.size(2))
        if co_attention_mask is not None:
            co_attention_mask = co_attention_mask.reshape(-1, co_attention_mask.size(2), co_attention_mask.size(3))
    elif process == "retrieval":
        num_options = question.size(1)
        features = features.reshape(-1, features.size(2), features.size(3))
        spatials = spatials.reshape(-1, spatials.size(2), spatials.size(3))
        image_mask = image_mask.reshape(-1, image_mask.size(2))
        question = question.reshape(-1, question.size(2))
        input_mask = input_mask.reshape(-1, input_mask.size(2))
        segment_ids = segment_ids.reshape(-1, segment_ids.size(2))
        if co_attention_mask is not None:
            co_attention_mask = co_attention_mask.reshape(-1, co_attention_mask.size(2), co_attention_mask.size(3))
    elif process == "nlvr":
        features = features.reshape(B * 2, features.size(1) // 2, features.size(2))
        spatials = spatials.reshape(B * 2, spatials.size(1) // 2, spatials.size(2))
        image_mask = image_mask.reshape(B * 2, image_mask.size(1) // 2)
        question = question.repeat(1, 2).reshape(B * 2, question.size(1))
        input_mask = input_mask.repeat(1, 2).reshape(B * 2, input_mask.size(1))
        segment_ids = segment_ids.repeat(1, 2).reshape(B * 2, segment_ids.size(1))
        if co_attention_mask is not None:
            co_attention_mask = co_attention_mask.reshape(B * 2, co_attention_mask.size(1) // 2, co_attention_mask.size(2))
    elif process != "normal":
        raise ValueError(f"unknown process {process!r}")
    return features, spatials, image_mask, question, input_mask, segment_ids, co_attention_mask, B, num_options


class PinnedBatchPrefetcher:
    """Iterates over `batches` (an iterable of tuples / dicts of CPU tensors, e.g. a DataLoader) and yields them on the GPU one
    batch ahead: each batch is staged in pinned host buffers (allocated once per shape) and copied on a dedicated copy stream while
    the previous batch computes; the consumer's stream waits on the copy's event only. A yielded batch lives in one of
    `depth + 1` rotating device buffers: it stays valid until `depth` further batches have been requested (consume it, or clone)."""

    def __init__(self, batches, device=None, depth=2):
        self.it = iter(batches)
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.stream = torch.cuda.Stream(device=self.device)
        self.depth = depth
        self._pinned = {}
        self._slot_event = {}
        self._queue = []
        for _ in range(depth):
            self._enqueue()

    def _stage(self, slot, key, t):
        k = (slot, key, tuple(t.shape), t.dtype)
        if k not in self._pinned:
            self._pinned[k] = (torch.empty(t.shape, dtype=t.dtype).pin_memory(), torch.empty(t.shape, dtype=t.dtype, device=self.device))
        host, dev = self._pinned[k]
        host.copy_(t)
        dev.copy_(host, non_blocking=True)
        return dev

    def _enqueue(self):
        try:
            batch = next(self.it)
        except StopIteration:
            return
        slot = getattr(self, "_n", 0) % (self.depth + 1)
        self._n = getattr(self, "_n", 0) + 1
        if slot in self._slot_event:
            self._slot_event[slot].synchronize()     # the previous H2D out of this slot's pinned buffers has finished
        with torch.cuda.stream(self.stream):
            if isinstance(batch, dict):
                out = {k: (self._stage(slot, k, v) if torch.is_tensor(v) else v) for k, v in batch.items()}
            else:
                out = tuple(self._stage(slot, i, v) if torch.is_tensor(v) else v for i, v in enumerate(batch))
            ev = torch.cuda.Event()
            ev.record(self.stream)
        self._slot_event[slot] = ev
        self._queue.append((out, ev))

    def __iter__(self):
        return self

    def __next__(self):
        if not self._queue:
            raise StopIteration
        out, ev = self._queue.pop(0)
        torch.cuda.current_stream().wait_event(ev)
        self._enqueue()
        return out
