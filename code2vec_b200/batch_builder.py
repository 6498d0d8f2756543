"""Device-resident corpus + on-GPU batch construction: the drop-in for `DatasetBuilder.refresh_train_dataset` /
`build_data` + the `DataLoader(shuffle=True)` of the reference's epoch loop (model/dataset_builder.py:55-63, :112-204,
main.py:160-169) for the method-name task (`build`, `epoch`) and the variable-name task (`build_vars`, `epoch_vars`), each
also as packed batches (`build_packed`, `epoch_packed`, `build_vars_packed`, `epoch_vars_packed`).  All arithmetic happens in libc2v_b200.so (`c2v_build_batch`); there is no
CPU fallback.

    corpus = DeviceCorpus.from_reader(reader, builder.train_items, device)          # once
    for starts, paths, ends, label in corpus.epoch(batch_size, max_path_length, seed=epoch):
        preds, _, _ = model.forward(starts, paths, ends, label)                      # main.py:172
"""
import ctypes

import numpy as np
import torch

from . import _lib
from .functional import PackedBags


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def packed_offsets(counts, item_ids, max_path_length):
    """Bag offsets (numpy int64 [B + 1]) of the packed batch of items `item_ids` (host int array [B]) over a corpus whose
    item i holds counts[i] contexts: bag b holds min(counts[id], L) contexts, and one (a pad context) when the item has
    none or the id is outside [0, len(counts)).  A pure host function: no device copy."""
    counts = np.asarray(counts, dtype=np.int64)
    ids = np.asarray(item_ids, dtype=np.int64).reshape(-1)
    ok = (ids >= 0) & (ids < counts.size)
    n = np.zeros(ids.size, np.int64)
    n[ok] = counts[ids[ok]]
    off = np.zeros(ids.size + 1, np.int64)
    np.cumsum(np.clip(n, 1, int(max_path_length)), out=off[1:])
    return off


def _upload(a, device):
    """host int64 array -> device tensor through pinned memory, without blocking the host"""
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.int64)).pin_memory().to(device, non_blocking=True)


class DeviceCorpus:
    """CSR image of `reader.items` in HBM: offsets int64 [n+1], contexts int32 [total, 3], labels int64 [n]."""

    def __init__(self, offsets, contexts, labels, method_token, question_token, device):
        dev = torch.device(device)
        if dev.type != "cuda":
            raise _lib.C2VError("DeviceCorpus lives on a CUDA device (sm_100a); there is no CPU path")
        host_offsets = (offsets.cpu().numpy() if isinstance(offsets, torch.Tensor) else np.asarray(offsets)).astype(np.int64).reshape(-1)
        self.counts = np.diff(host_offsets)           # contexts per item, on the host: packed bag offsets need no copy
        self.offsets = torch.as_tensor(offsets, dtype=torch.int64).contiguous().to(dev)
        self.contexts = torch.as_tensor(contexts, dtype=torch.int32).reshape(-1, 3).contiguous().to(dev)
        self.labels = None if labels is None else torch.as_tensor(labels, dtype=torch.int64).contiguous().to(dev)
        self.n_items = int(self.offsets.numel() - 1)
        if self.n_items < 1 or int(self.offsets[-1]) != self.contexts.shape[0]:
            raise ValueError("offsets / contexts do not describe a CSR corpus")
        self.method_token, self.question_token = int(method_token), int(question_token)
        self.device = dev

    @classmethod
    def from_reader(cls, reader, items, device):
        """`reader`: the reference's DatasetReader (dataset_reader.py:44-128); `items`: e.g. builder.train_items."""
        import numpy as np
        off = np.zeros(len(items) + 1, dtype=np.int64)
        for i, it in enumerate(items):
            off[i + 1] = off[i] + len(it.path_contexts)
        ctx = np.asarray([pc for it in items for pc in it.path_contexts], dtype=np.int32).reshape(-1, 3)
        lab = np.asarray([reader.label_vocab.stoi[it.normalized_label] for it in items], dtype=np.int64)
        return cls(off, ctx, lab, reader.terminal_vocab.stoi["@method_0"], reader.QUESTION_TOKEN_INDEX, device)

    @classmethod
    def from_corpus(cls, reader, device, item_indices=None):
        """`reader`: code2vec_b200.corpus.CorpusReader (the C++ parser's CSR arrays go to HBM as they are);
        item_indices: subset / order of items (e.g. the train split), default all."""
        import numpy as np
        if item_indices is None:
            off, ctx, lab = reader.ctx_offsets, reader.contexts, reader.item_labels
        else:
            idx = np.asarray(item_indices, dtype=np.int64)
            n = (reader.ctx_offsets[idx + 1] - reader.ctx_offsets[idx])
            off = np.zeros(len(idx) + 1, np.int64); np.cumsum(n, out=off[1:])
            take = np.concatenate([np.arange(reader.ctx_offsets[i], reader.ctx_offsets[i + 1]) for i in idx]) if len(idx) else np.zeros(0, np.int64)
            ctx, lab = reader.contexts[take], reader.item_labels[idx]
        c = cls(off, ctx, lab, reader.terminal_vocab.stoi["@method_0"], reader.QUESTION_TOKEN_INDEX, device)
        if reader.infer_variable:
            ui, uv, ul = reader.variable_units(item_indices)
            c.set_variable_units(ui, uv, ul, reader.variable_indexes, reader.terminal_vocab.len(),
                                 reader.shuffle_variable_indexes)
        return c

    def set_variable_units(self, unit_item, unit_var, unit_label, variable_indexes, terminal_count, shuffle_variable_indexes=False):
        """The bags of the variable-name task (dataset_builder.py:152-204): unit u = (item unit_item[u] of THIS corpus,
        terminal index unit_var[u] of its @var alias, label unit_label[u])."""
        import numpy as np
        dev = self.device
        self.unit_item = torch.as_tensor(np.asarray(unit_item), dtype=torch.int64).contiguous().to(dev)
        self.unit_var = torch.as_tensor(np.asarray(unit_var), dtype=torch.int64).contiguous().to(dev)
        self.unit_label = torch.as_tensor(np.asarray(unit_label), dtype=torch.int64).contiguous().to(dev)
        self.n_units = int(self.unit_item.numel())
        var = np.asarray(variable_indexes, dtype=np.int64)
        pos = np.full(int(terminal_count), -1, np.int32)
        pos[var] = np.arange(len(var), dtype=np.int32)
        self.var_pos = torch.from_numpy(pos).to(dev)
        self.variable_indexes = torch.from_numpy(var).to(dev)
        self.terminal_count, self.shuffle_variable_indexes = int(terminal_count), bool(shuffle_variable_indexes)
        self.unit_counts = np.zeros(0, np.int64)      # matching contexts per unit, on the host: packed bag offsets
        if self.n_units:
            counts = torch.empty((self.n_units,), dtype=torch.int64, device=dev)
            with torch.cuda.device(dev):
                rc = _lib.load().c2v_count_unit_contexts(_ptr(self.offsets), _ptr(self.contexts), self.n_items,
                                                         _ptr(self.unit_item), _ptr(self.unit_var), self.n_units, _ptr(counts),
                                                         ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream))
                _lib.check(rc, "c2v_count_unit_contexts")
            self.unit_counts = counts.cpu().numpy()

    def build_vars(self, unit_ids, max_path_length, seed):
        """-> (starts, paths, ends, label) of the variable-name bags `unit_ids` (int64 [B] into the units)."""
        lib = _lib.load()
        if getattr(self, "unit_item", None) is None:
            raise ValueError("no variable units: build the corpus from a reader with infer_variable=True")
        ids = unit_ids.to(device=self.device, dtype=torch.int64).contiguous()
        B, L = int(ids.numel()), int(max_path_length)
        with torch.cuda.device(self.device):
            starts = torch.empty((B, L), dtype=torch.int64, device=self.device)
            paths = torch.empty_like(starts); ends = torch.empty_like(starts)
            label = torch.empty((B,), dtype=torch.int64, device=self.device)
            rc = lib.c2v_build_batch_vars(_ptr(self.offsets), _ptr(self.contexts), self.n_items, _ptr(self.unit_item),
                                          _ptr(self.unit_var), _ptr(self.unit_label), self.n_units, _ptr(ids), B, L,
                                          int(seed) & 0xFFFFFFFFFFFFFFFF, self.question_token, _ptr(self.var_pos),
                                          self.terminal_count, _ptr(self.variable_indexes), int(self.variable_indexes.numel()),
                                          1 if self.shuffle_variable_indexes else 0,
                                          _ptr(starts), _ptr(paths), _ptr(ends), _ptr(label),
                                          ctypes.c_void_p(torch.cuda.current_stream(self.device).cuda_stream))
            _lib.check(rc, "c2v_build_batch_vars")
        return starts, paths, ends, label

    def build(self, item_ids, max_path_length, seed, check=False):
        """-> (starts, paths, ends, label): int64 [B, L] x3 and [B], like `build_data` + the DataLoader collate."""
        lib = _lib.load()
        ids = item_ids.to(device=self.device, dtype=torch.int64).contiguous()
        if check and ids.numel() and (int(ids.min()) < 0 or int(ids.max()) >= self.n_items):
            raise IndexError("item id out of range")
        B, L = int(ids.numel()), int(max_path_length)
        with torch.cuda.device(self.device):
            starts = torch.empty((B, L), dtype=torch.int64, device=self.device)
            paths = torch.empty_like(starts); ends = torch.empty_like(starts)
            label = torch.empty((B,), dtype=torch.int64, device=self.device)
            rc = lib.c2v_build_batch(_ptr(self.offsets), _ptr(self.contexts), self.n_items, _ptr(ids), _ptr(self.labels),
                                     B, L, int(seed) & 0xFFFFFFFFFFFFFFFF, self.method_token, self.question_token,
                                     _ptr(starts), _ptr(paths), _ptr(ends), _ptr(label),
                                     ctypes.c_void_p(torch.cuda.current_stream(self.device).cuda_stream))
            _lib.check(rc, "c2v_build_batch")
        return starts, paths, ends, label

    def epoch(self, batch_size, max_path_length, seed, shuffle=True, rank=0, world=1):
        """One pass over the corpus in random order (main.py:160-162); with world > 1 each rank takes its strided shard
        of the same permutation.  Every (epoch seed, item) pair draws a fresh context subset, like the per-epoch
        `refresh_train_dataset` of the reference."""
        g = torch.Generator(device=self.device).manual_seed(int(seed))
        order = torch.randperm(self.n_items, generator=g, device=self.device) if shuffle else \
            torch.arange(self.n_items, device=self.device)
        order = order[rank::world]
        for lo in range(0, order.numel(), batch_size):          # last batch ragged (drop_last unset, main.py:162)
            yield self.build(order[lo:lo + batch_size], max_path_length, seed)

    def build_packed(self, item_ids, max_path_length, seed):
        """-> (PackedBags, label [B]): the bags `build` returns for the same ids and seed, without the zero suffix.  Bag b
        holds min(n, L) contexts of its item (n = the item's context count); an empty item or an id outside the corpus is a
        bag of one pad context (0, 0, 0).  item_ids: host ints (a list, numpy array or CPU tensor: ids and bag offsets go to
        the device in one pinned, asynchronous copy) or a CUDA tensor (one device-to-host copy of the ids, because the bag
        offsets are computed on the host)."""
        L = int(max_path_length)
        return self._build_packed(*self._stage_packed(item_ids, self.counts, L), L, seed)

    def _stage_packed(self, ids, counts, L):
        """-> (device ids [B], host bag offsets, device bag offsets) of a packed batch over bags of counts[id] contexts"""
        if isinstance(ids, torch.Tensor) and ids.is_cuda:
            ids = ids.to(dtype=torch.int64).reshape(-1).contiguous()
            off = packed_offsets(counts, ids.cpu().numpy(), L)
            return ids, off, _upload(off, self.device)
        host_ids = (ids.numpy() if isinstance(ids, torch.Tensor) else np.asarray(ids)).astype(np.int64).reshape(-1)
        off = packed_offsets(counts, host_ids, L)
        staged = _upload(np.concatenate([host_ids, off]), self.device)
        return staged[:host_ids.size], off, staged[host_ids.size:]

    def _epoch_staged(self, n, counts, batch_size, L, seed, shuffle, rank, world):
        """the permutation of `epoch` over n ids, staged for packed batches -> (device ids, host offsets, device offsets)
        per batch.  Per epoch, not per batch: one device-to-host copy of the permutation (the bag offsets are computed on
        the host) and one pinned, asynchronous copy of every batch's offsets to the device; each batch takes its ids and
        offsets as slices of device tensors."""
        g = torch.Generator(device=self.device).manual_seed(int(seed))
        order = torch.randperm(n, generator=g, device=self.device) if shuffle else torch.arange(n, device=self.device)
        order = order[rank::world].contiguous()
        host = order.cpu().numpy()
        spans = [(lo, min(lo + batch_size, host.size)) for lo in range(0, host.size, batch_size)]
        offs = [packed_offsets(counts, host[lo:hi], L) for lo, hi in spans]
        if not offs:
            return
        all_dev = _upload(np.concatenate(offs), self.device)        # batch i's B + 1 offsets start at lo + i
        for i, ((lo, hi), off) in enumerate(zip(spans, offs)):
            yield order[lo:hi], off, all_dev[lo + i:hi + i + 1]

    def _empty_packed(self, B, off, off_dev, L):
        """-> (PackedBags, label [B]) to be filled by a packed builder: N = off[-1] rows"""
        starts = torch.empty((int(off[-1]),), dtype=torch.int64, device=self.device)
        bags = PackedBags(starts, torch.empty_like(starts), torch.empty_like(starts), off, L, device_offsets=off_dev)
        return bags, torch.empty((B,), dtype=torch.int64, device=self.device)

    def _build_packed(self, ids, off, off_dev, L, seed):
        """c2v_build_batch_packed for device ids [B] and bag offsets given on the host (off) and on the device (off_dev)"""
        lib = _lib.load()
        B = int(ids.numel())
        with torch.cuda.device(self.device):
            bags, label = self._empty_packed(B, off, off_dev, L)
            rc = lib.c2v_build_batch_packed(_ptr(self.offsets), _ptr(self.contexts), self.n_items, _ptr(ids), _ptr(self.labels),
                                            B, L, int(seed) & 0xFFFFFFFFFFFFFFFF, self.method_token, self.question_token,
                                            _ptr(bags.offsets), _ptr(bags.starts), _ptr(bags.paths), _ptr(bags.ends),
                                            _ptr(label), ctypes.c_void_p(torch.cuda.current_stream(self.device).cuda_stream))
            _lib.check(rc, "c2v_build_batch_packed")
        return bags, label

    def epoch_packed(self, batch_size, max_path_length, seed, shuffle=True, rank=0, world=1):
        """`epoch` with packed batches: the same permutation, the same items in the same order -> (PackedBags, label) per
        batch, as build_packed makes them, with the transfers of `_epoch_staged`."""
        L = int(max_path_length)
        for ids, off, off_dev in self._epoch_staged(self.n_items, self.counts, batch_size, L, seed, shuffle, rank, world):
            yield self._build_packed(ids, off, off_dev, L, seed)

    def build_vars_packed(self, unit_ids, max_path_length, seed):
        """-> (PackedBags, label [B]): the bags `build_vars` returns for the same unit ids and seed, without the zero
        suffix.  Bag b holds min(n, L) contexts (n = unit_counts[u], the unit's matching contexts); a unit without a match
        or an id outside the units is a bag of one pad context (0, 0, 0).  unit_ids: host ints (one pinned, asynchronous
        copy of ids and bag offsets) or a CUDA tensor (one device-to-host copy of the ids)."""
        self._need_units()
        L = int(max_path_length)
        return self._build_vars_packed(*self._stage_packed(unit_ids, self.unit_counts, L), L, seed)

    def _need_units(self):
        if getattr(self, "unit_item", None) is None:
            raise ValueError("no variable units: build the corpus from a reader with infer_variable=True")

    def _build_vars_packed(self, ids, off, off_dev, L, seed):
        """c2v_build_batch_vars_packed for device unit ids [B] and bag offsets on the host (off) and the device (off_dev)"""
        lib = _lib.load()
        B = int(ids.numel())
        with torch.cuda.device(self.device):
            bags, label = self._empty_packed(B, off, off_dev, L)
            rc = lib.c2v_build_batch_vars_packed(_ptr(self.offsets), _ptr(self.contexts), self.n_items, _ptr(self.unit_item),
                                                 _ptr(self.unit_var), _ptr(self.unit_label), self.n_units, _ptr(ids), B, L,
                                                 int(seed) & 0xFFFFFFFFFFFFFFFF, self.question_token, _ptr(self.var_pos),
                                                 self.terminal_count, _ptr(self.variable_indexes),
                                                 int(self.variable_indexes.numel()), 1 if self.shuffle_variable_indexes else 0,
                                                 _ptr(bags.offsets), _ptr(bags.starts), _ptr(bags.paths), _ptr(bags.ends),
                                                 _ptr(label), ctypes.c_void_p(torch.cuda.current_stream(self.device).cuda_stream))
            _lib.check(rc, "c2v_build_batch_vars_packed")
        return bags, label

    def epoch_vars_packed(self, batch_size, max_path_length, seed, shuffle=True, rank=0, world=1):
        """`epoch_vars` with packed batches: the same units in the same order -> (PackedBags, label) per batch, as
        build_vars_packed makes them, with the transfers of `_epoch_staged`."""
        self._need_units()
        L = int(max_path_length)
        for ids, off, off_dev in self._epoch_staged(self.n_units, self.unit_counts, batch_size, L, seed, shuffle, rank,
                                                    world):
            yield self._build_vars_packed(ids, off, off_dev, L, seed)

    def epoch_vars(self, batch_size, max_path_length, seed, shuffle=True, rank=0, world=1):
        """the same pass over the variable-name units (dataset_builder.py:152-204)"""
        g = torch.Generator(device=self.device).manual_seed(int(seed))
        order = torch.randperm(self.n_units, generator=g, device=self.device) if shuffle else \
            torch.arange(self.n_units, device=self.device)
        order = order[rank::world]
        for lo in range(0, order.numel(), batch_size):
            yield self.build_vars(order[lo:lo + batch_size], max_path_length, seed)
