"""ddstore_b200/dataset.py -- the loader side of the hot path (SURVEY.md 8f, rank 1).

`DistDataset` is the reference's `examples/vae/distdataset.py:13-92` re-built on the batched fetch:
same constructor shape (`data, label, comm, ddstore_width`), same per-sample `__getitem__` contract, plus
`__getitems__` -- which torch's DataLoader calls with the whole index batch -- so a batch costs one kernel
launch per variable and lands packed in HBM instead of one blocking round trip per sample followed by
`torch.tensor` + collate + `.to(device)` copies (`examples/vae/distdataset.py:84-88`, `vae-ddp.py:244`).

Epoch shuffle is the caller's sampler exactly as in the reference (`DistributedSampler`, `vae-ddp.py:216`):
`make_loader()` wires `DistributedSampler(shuffle=True)` + `set_epoch` + the identity collate.

(The reference flattens every sample into a disp=1 variable and then passes the SAMPLE index as the ROW index
(`distdataset.py:63,70,84`), so it returns floats [idx, idx+784) rather than image idx; here a sample is one row
of width `sample_size`, which is what the reference evidently meant.)
"""
import numpy as np
import torch
from torch.utils.data import DataLoader, Dataset
from torch.utils.data.distributed import DistributedSampler

from .comm import as_dds_comm
from .store import PyDDStore, _conversion, _pad_bits


def nsplit(a, n):
    """contiguous near-equal split (same arithmetic as examples/vae/distdataset.py:9-11)"""
    k, m = divmod(len(a), n)
    return (a[i * k + min(i, m):(i + 1) * k + min(i + 1, m)] for i in range(n))


def _norm_spec(spec):
    """(mean, std[, inner]) of a dataset's `normalize` -> set_normalization's (mean, std, inner); lists become float32"""
    if not isinstance(spec, (tuple, list)) or len(spec) not in (2, 3):
        raise ValueError("normalize takes (mean, std) or (mean, std, inner)")
    def f32(t):
        return t if torch.is_tensor(t) or isinstance(t, np.ndarray) else np.asarray(t, dtype=np.float32).reshape(-1)
    return f32(spec[0]), f32(spec[1]), int(spec[2]) if len(spec) == 3 else 1


class DistDataset(Dataset):
    """Fixed-shape samples + integer labels, sharded over the ranks of `comm` by contiguous blocks.

    data: sequence of (tensor/ndarray, label) pairs -- every rank passes the same sequence (like the reference) and
    keeps only its block; or pass `local_only=True` when `data` already is this rank's block.
    out_dtype / lut: batches (__getitems__, PrefetchLoader) deliver the samples converted to `out_dtype` inside the
    gather (float32 -> bfloat16 / float16, float64 -> float32, uint8 -> bfloat16 / float16 / float32 through `lut`, 256
    entries of out_dtype, default the plain value cast); the labels are never converted. The per-sample get() keeps
    the stored dtype.
    normalize=(mean, std[, inner]): batches deliver (x - mean[ch]) / std[ch] per channel, computed in float32 inside the
    gather (see PyDDStore.set_normalization for the channel rule), as out_dtype (default float32). A uint8 source is
    decoded through `lut` (256 float32 entries, default the plain value: pass torch.arange(256).float().div(255) for
    ToTensor() + Normalize()). The labels are never normalised.
    placement="host": the samples and labels live in pinned host memory every rank of the box maps instead of HBM (a
    dataset larger than the HBM the model leaves free); batches are still gathered on the GPU, over PCIe.
    """

    def __init__(self, data, label, comm=None, ddstore_width=None, device=None, local_only=False, out_dtype=None, lut=None,
                 normalize=None, placement="hbm"):
        super().__init__()
        self.label = label
        self.comm = as_dds_comm(comm)
        self.rank, self.comm_size = self.comm.Get_rank(), self.comm.Get_size()
        # replica groups exactly as the reference builds them (distdataset.py:25-30): consecutive ranks in groups of
        # `ddstore_width`, every group holding the WHOLE dataset sharded over its members (one group per NVSwitch box)
        self.ddstore_width = ddstore_width if ddstore_width is not None else self.comm_size
        if self.ddstore_width != self.comm_size:
            self.ddstore_comm = self.comm.Split(self.rank // self.ddstore_width, self.rank)
        else:
            self.ddstore_comm = self.comm
        self.ddstore_comm_rank, self.ddstore_comm_size = self.ddstore_comm.Get_rank(), self.ddstore_comm.Get_size()
        self.device = torch.device("cuda", torch.cuda.current_device() if device is None else device)
        self.ddstore = PyDDStore(self.ddstore_comm, device=self.device.index)

        if local_only:
            mine = list(range(len(data)))
            counts = [int(c) for c in self._allgather_int(len(data))]
            self.total_ns = sum(counts)
        else:
            self.total_ns = len(data)
            mine = list(nsplit(range(len(data)), self.ddstore_comm_size))[self.ddstore_comm_rank]
        vals, labels = [], []
        for i in mine:
            d, lab = data[i]
            d = d.cpu().numpy() if hasattr(d, "cpu") else np.asarray(d)
            vals.append(np.ascontiguousarray(d).reshape(-1))
            labels.append(lab)
        self.sample_shape = tuple(np.asarray(data[mine[0]][0]).shape) if mine else ()
        arr = np.stack(vals) if vals else np.zeros((0, 1), np.float32)
        self.sample_size = arr.shape[1]
        self.dtype = torch.from_numpy(arr[:0]).dtype
        self._np_dtype = arr.dtype
        # batch dtype: the stored one, or out_dtype converted in the gather (src_dtype = what the gather converts from)
        self.normalize = normalize is not None
        self.src_dtype = self.dtype if (out_dtype is not None or self.normalize) else None
        self.out_dtype = out_dtype if out_dtype is not None else (torch.float32 if self.normalize else self.dtype)
        self.lut = lut
        if self.src_dtype is not None:  # an unsupported pair fails here, not at the first batch
            _conversion(self.src_dtype, self.out_dtype, lut, self.normalize)
        self.ddstore.add(f"{self.label}data", np.ascontiguousarray(arr), placement=placement)
        if self.normalize:
            self.ddstore.set_normalization(f"{self.label}data", *_norm_spec(normalize))
        self.ddstore.add(f"{self.label}labels", np.ascontiguousarray(np.array(labels, dtype=np.int32).reshape(-1, 1)),
                         placement=placement)

    def _allgather_int(self, v):
        parts = self.ddstore_comm.allgather_bytes(int(v).to_bytes(8, "little"))
        return [int.from_bytes(p, "little") for p in parts]

    def len(self):
        return self.total_ns

    def __len__(self):
        return self.total_ns

    # ---- the reference's per-sample contract (distdataset.py:79-92): host buffers in, a CPU tensor + an int out
    def get(self, idx):
        val = np.empty((1, self.sample_size), dtype=self._np_dtype)
        lab = np.empty((1, 1), dtype=np.int32)
        self.ddstore.get(f"{self.label}data", val, int(idx))
        self.ddstore.get(f"{self.label}labels", lab, int(idx))
        return torch.from_numpy(val).view(self.sample_shape), int(lab[0, 0])

    def __getitem__(self, idx):
        return self.get(idx)

    # ---- the batched contract: DataLoader hands over the whole index list
    def __getitems__(self, indices):
        B = len(indices)
        idx = np.asarray(indices, dtype=np.int64)
        vals = torch.empty((B, self.sample_size), dtype=self.out_dtype, device=self.device)
        labs = torch.empty((B, 1), dtype=torch.int32, device=self.device)
        # on torch's CURRENT stream: the output tensors come from its caching allocator, whose blocks may still be in use
        # by work queued there, and the index copy + the gather are then ordered with everything the caller queued before
        st = torch.cuda.current_stream(self.device).cuda_stream
        self.ddstore.get_batch(f"{self.label}data", idx, out=vals, count=1, stream=st, src_dtype=self.src_dtype, lut=self.lut,
                               normalize=self.normalize)
        self.ddstore.get_batch(f"{self.label}labels", idx, out=labs, count=1, stream=st)
        return vals.view((B,) + self.sample_shape), labs.view(B)

    @staticmethod
    def collate(batch):
        """identity: __getitems__ already returns the collated, device-resident batch"""
        return batch

    def epoch_begin(self):
        self.ddstore.epoch_begin()

    def epoch_end(self):
        self.ddstore.epoch_end()

    def free(self):
        self.ddstore.free()


class RaggedDataset(Dataset):
    """Variable-length, multi-array samples (configs 3 and 4): every variable is a 2-D array of rows, and sample i
    owns rows [row_start[v][i], row_start[v][i] + row_count[v][i]) of variable v -- the HydraGNN-style layout the
    reference's get(name, arr, start) with count = arr.shape[0] implies (src/pyddstore.pyx:84-87).
    The (start, count) tables of ALL samples are kept on the device, so a batch needs only the sample ids."""

    def __init__(self, local_arrays, local_counts, comm=None, device=None, out_dtypes=None, luts=None, normalize=None,
                 pad=None, placement="hbm"):
        """local_arrays: {name: 2-D ndarray of this rank's rows}; local_counts: {name: int64[n_local_samples]}
        out_dtypes / luts: {name: dtype} / {name: 256-entry table}: those variables' batches are delivered converted in
        the gather (see DistDataset); their row offsets count rows as always.
        normalize: {name: (mean, std[, inner])}: those variables are delivered normalised per channel (see DistDataset),
        as out_dtypes[name] (default float32).
        pad: {name: max_rows | (max_rows, pad_value)}: those variables are delivered padded, as (tensor [B, max_rows,
        ...width] in their output dtype, int64 lengths [B]): each sample's first max_rows rows, then pad_value (default
        0) encoded in the output dtype. The other variables stay packed.
        placement="host": every variable lives in pinned host memory instead of HBM (see DistDataset)."""
        out_dtypes, luts, normalize = dict(out_dtypes or {}), dict(luts or {}), dict(normalize or {})
        super().__init__()
        self.comm = as_dds_comm(comm)
        self.rank, self.comm_size = self.comm.Get_rank(), self.comm.Get_size()
        self.device = torch.device("cuda", torch.cuda.current_device() if device is None else device)
        self.ddstore = PyDDStore(self.comm, device=self.device.index)
        self.names = list(local_arrays)
        self.row_bytes, self.dtypes, self.widths = {}, {}, {}
        self.counts = {}  # host copy of every sample's row count per variable (sizes the packed outputs)
        n_local = len(next(iter(local_counts.values())))
        for name in self.names:
            arr = np.ascontiguousarray(local_arrays[name])
            cnt = np.ascontiguousarray(local_counts[name], dtype=np.int64)
            assert cnt.sum() == arr.shape[0] and len(cnt) == n_local
            self.ddstore.add(name, arr, placement=placement)
            first_row = ([0] + self.ddstore.query(name)["lenlist"])[self.rank]
            local_start = first_row + np.concatenate([[0], np.cumsum(cnt)[:-1]])
            # every rank learns every sample's (start, count): 16 B per sample per variable
            blobs = self.comm.allgather_bytes(len(cnt).to_bytes(8, "little"))
            sizes = [int.from_bytes(b, "little") for b in blobs]
            most = max(sizes)
            buf = np.zeros((2, most), np.int64)
            buf[0, :len(cnt)], buf[1, :len(cnt)] = local_start, cnt
            parts = self.comm.allgather_bytes(buf.tobytes())
            tabs = [np.frombuffer(p, np.int64).reshape(2, most)[:, :n] for p, n in zip(parts, sizes)]
            all_start = np.concatenate([t[0] for t in tabs])
            all_count = np.concatenate([t[1] for t in tabs])
            self.ddstore.set_sample_index(name, all_start, all_count)  # device-resident (start, count) of every sample
            self.counts[name] = all_count
            self.row_bytes[name] = arr.dtype.itemsize * int(np.prod(arr.shape[1:], dtype=np.int64))
            self.dtypes[name] = torch.from_numpy(arr[:0]).dtype
            self.widths[name] = arr.shape[1:]
        # what the batches deliver: out_dtypes[name] converted (or normalised) from the stored dtype, else the stored bytes
        self.normalize = {n: n in normalize for n in self.names}
        self.src_dtypes = {n: (self.dtypes[n] if (n in out_dtypes or self.normalize[n]) else None) for n in self.names}
        self.out_dtypes = {n: out_dtypes.get(n, torch.float32 if self.normalize[n] else self.dtypes[n]) for n in self.names}
        self.luts = {n: luts.get(n) for n in self.names}
        self.out_row_bytes = {}
        for n in self.names:
            if self.src_dtypes[n] is not None:  # an unsupported pair fails here
                _conversion(self.src_dtypes[n], self.out_dtypes[n], self.luts[n], self.normalize[n])
            if self.normalize[n]:
                self.ddstore.set_normalization(n, *_norm_spec(normalize[n]))
            self.out_row_bytes[n] = self.row_bytes[n] // self.dtypes[n].itemsize * self.out_dtypes[n].itemsize
        self.pad = {}  # name -> (max_rows, pad_value) of the padded variables
        for n, spec in dict(pad or {}).items():
            if n not in self.names:
                raise KeyError(f"pad: no variable {n!r}")
            m, v = (spec if isinstance(spec, (tuple, list)) else (spec, 0))
            if int(m) < 0:
                raise ValueError("pad: max_rows must be >= 0")
            _pad_bits(v, self.out_dtypes[n])  # (a value the output dtype cannot hold fails here)
            self.pad[n] = (int(m), v)
        self.packed_names = [n for n in self.names if n not in self.pad]
        self.total_ns = int(len(self.counts[self.names[0]]))

    def __len__(self):
        return self.total_ns

    def __getitem__(self, idx):
        return self.__getitems__([idx])

    def __getitems__(self, indices):
        """-> {name: (packed rows tensor [sum(count), ...width], int64 row offsets per sample [B+1])}, and for a padded
        variable {name: (tensor [B, max_rows, ...width], int64 lengths [B])}.
        One launch chain per variable; the sample-id -> (start, count) lookup happens on the device."""
        ids = np.ascontiguousarray(indices, dtype=np.int64)
        # host ids go to the store as they are: it copies them on the stream the gather runs on (torch's current stream:
        # the outputs below come from that stream's allocator), so the kernel can never read them before they landed
        st = torch.cuda.current_stream(self.device).cuda_stream
        out = {}
        for name, (m, v) in self.pad.items():  # one padded launch per padded variable
            buf = torch.empty((len(ids), m) + tuple(self.widths[name]), dtype=self.out_dtypes[name], device=self.device)
            lengths = torch.empty(len(ids), dtype=torch.int64, device=self.device)
            self.ddstore.get_samples(name, ids, buf, stream=st, src_dtype=self.src_dtypes[name], lut=self.luts[name],
                                     normalize=self.normalize[name], pad_rows=m, pad_value=v, lengths=lengths)
            out[name] = (buf, lengths)
        names = self.packed_names
        if not names:
            return out
        bufs, offs, rows = [], [], []
        for name in names:
            r = int(self.counts[name][ids].sum())  # host-side size of the packed result (sizes only, no data)
            rows.append(r)
            bufs.append(torch.empty((max(r, 1),) + tuple(self.widths[name]), dtype=self.out_dtypes[name], device=self.device))
            offs.append(torch.empty(len(ids) + 1, dtype=torch.int64, device=self.device))
        conv = any(self.src_dtypes[n] is not None for n in names)
        if 1 < len(names) <= 4:
            # every packed variable of the batch in ONE launch (dds_get_samples_multi; a single variable takes
            # dds_get_samples, which the multi-array launch does not stand in for)
            kw = dict(src_dtypes=[self.src_dtypes[n] for n in names], luts=[self.luts[n] for n in names],
                      normalize=[self.normalize[n] for n in names]) if conv else {}
            self.ddstore.get_samples_multi(names, ids, bufs, offsets=offs, stream=st, **kw)
        else:
            for name, buf, off in zip(names, bufs, offs):
                self.ddstore.get_samples(name, ids, out=buf, offsets=off, stream=st, src_dtype=self.src_dtypes[name],
                                         lut=self.luts[name], normalize=self.normalize[name])
        for name, buf, off, r in zip(names, bufs, offs, rows):
            out[name] = (buf[:r], off // self.out_row_bytes[name])
        return out

    collate = staticmethod(lambda batch: batch)

    def free(self):
        self.ddstore.free()


def make_loader(dataset, batch_size, rank=0, world_size=1, shuffle=True, seed=0, drop_last=False):
    """DataLoader over a DistDataset/RaggedDataset with the reference's epoch shuffle (DistributedSampler,
    examples/vae/vae-ddp.py:216-219): call loader.sampler.set_epoch(e) at the top of every epoch."""
    sampler = DistributedSampler(dataset, num_replicas=world_size, rank=rank, shuffle=shuffle, seed=seed,
                                 drop_last=drop_last)
    return DataLoader(dataset, batch_size=batch_size, sampler=sampler, num_workers=0, collate_fn=dataset.collate,
                      drop_last=drop_last)


class PrefetchLoader:
    """Double-buffered batch prefetch (SURVEY.md 8f rank 4): while the consumer works on batch k, batch k+1 is
    already being gathered on a side stream into the other buffer set. The reference brackets every batch with
    epoch_begin/epoch_end around a blocking fetch (examples/vae/vae-ddp.py:240-265); here the fetch of the next
    batch hides under the training step and the consumer only waits on a CUDA event.

    dataset: a DistDataset; sampler: iterable of sample indices (e.g. DistributedSampler); yields (vals, labels)
    device tensors that stay valid until the next-but-one FETCH (depth = 2 buffer sets).
    group: small batches are launch-bound (a 2 MB batch costs more in launch + ramp than in HBM time), so
    `group` consecutive batches are fetched by ONE launch (one request list of group x batch_size ids, one packed buffer
    sliced back into the batches) -- a queue of small batches served by one kernel.
    """

    def __init__(self, dataset, sampler, batch_size, drop_last=False, depth=2, group=1):
        self.ds, self.sampler, self.bs, self.drop_last, self.depth = dataset, sampler, batch_size, drop_last, max(2, depth)
        self.group = max(1, int(group))
        dev = dataset.device
        self.stream = torch.cuda.Stream(device=dev)
        rows = batch_size * self.group
        self.bufs = [(torch.empty((rows, dataset.sample_size), dtype=dataset.out_dtype, device=dev),
                      torch.empty((rows, 1), dtype=torch.int32, device=dev),
                      torch.empty(rows, dtype=torch.int64, device=dev)) for _ in range(self.depth)]
        self.events = [torch.cuda.Event() for _ in range(self.depth)]

    def _batches(self):
        if isinstance(self.sampler, DeviceBatchSampler):
            # the epoch's permutation already lives on the device: batches are tensor slices, nothing to copy
            yield from self.sampler
            return
        cur = []
        for i in self.sampler:
            cur.append(int(i))
            if len(cur) == self.bs:
                yield cur
                cur = []
        if cur and not self.drop_last:
            yield cur

    def _issue(self, slot, idx):
        vals, labs, d_idx = self.bufs[slot]
        n = len(idx)
        if n > vals.shape[0]:
            raise ValueError(f"a fetch of {n} samples does not fit the loader's buffers ({vals.shape[0]} = batch_size x group)")
        keep = idx
        with torch.cuda.stream(self.stream):
            if torch.is_tensor(idx) and idx.is_cuda:
                ids = idx
            else:
                keep = torch.as_tensor(idx, dtype=torch.int64).pin_memory()
                d_idx[:n].copy_(keep, non_blocking=True)
                ids = d_idx[:n]
            st = self.stream.cuda_stream
            # independent batches into alternating buffer sets: let consecutive launches overlap (DDS_OVERLAP)
            self.ds.ddstore.get_batch(f"{self.ds.label}data", ids, out=vals[:n], count=1, stream=st, wait=False,
                                      overlap=True, src_dtype=self.ds.src_dtype, lut=self.ds.lut, normalize=self.ds.normalize)
            self.ds.ddstore.get_batch(f"{self.ds.label}labels", ids, out=labs[:n], count=1, stream=st, wait=False,
                                      overlap=True)
            self.events[slot].record(self.stream)
        return n, keep

    def _groups(self):
        """`group` consecutive batches as one fetch: (concatenated ids, [sizes of the batches])"""
        cur, sizes = [], []
        for idx in self._batches():
            cur.append(idx)
            sizes.append(len(idx))
            if len(cur) == self.group:
                yield cur, sizes
                cur, sizes = [], []
        if cur:
            yield cur, sizes

    def __iter__(self):
        consumer = torch.cuda.current_stream(self.ds.device)
        pending = []  # (slot, sizes, keepalive)
        slot = 0
        for parts, sizes in self._groups():
            if len(parts) == 1:
                idx = parts[0]
            elif torch.is_tensor(parts[0]):
                idx = torch.cat(parts)
            else:
                idx = [i for p in parts for i in p]
            # a slot is reused `depth` fetches later: make the side stream wait for whatever the consumer queued so far
            self.stream.wait_stream(consumer)
            _, keep = self._issue(slot, idx)
            pending.append((slot, sizes, keep))
            slot = (slot + 1) % self.depth
            if len(pending) == self.depth:
                yield from self._take(pending.pop(0), consumer)
        while pending:
            yield from self._take(pending.pop(0), consumer)
        self.ds.ddstore.wait()  # surface any fetch error of the epoch

    def _take(self, item, consumer):
        slot, sizes, _ = item
        consumer.wait_event(self.events[slot])
        vals, labs, _ = self.bufs[slot]
        b0 = 0
        for n in sizes:
            yield vals[b0:b0 + n].view((n,) + self.ds.sample_shape), labs[b0:b0 + n].view(n)
            b0 += n


class RaggedPrefetchLoader:
    """Double-buffered prefetch for a RaggedDataset (variable-length, multi-array samples): while the consumer works on
    batch k, batch k+1 -- every variable of it, ONE launch (`dds_get_samples_multi`) -- is planned and gathered on a side
    stream into the other buffer set. Consecutive fetches are queued with overlap=True, so the plan of batch k+1 runs
    under the gather of batch k (the kernel enforces that batch k+2 writes nothing before batch k has retired).

    sampler: iterable of sample ids on the host (e.g. DistributedSampler): the packed sizes come from the host copy of
    the row counts. Yields {name: (packed rows tensor [sum(count), ...width], int64 row offsets [B+1])}; a batch stays
    valid until the next-but-one fetch. The dataset's padded variables (RaggedDataset(pad=...)) are queued beside that
    launch, one padded launch each (also overlap=True), into fixed-size per-slot buffers, and yielded as
    {name: (tensor [B, max_rows, ...width], int64 lengths [B])}."""

    def __init__(self, dataset, sampler, batch_size, drop_last=False, depth=2):
        if len(dataset.names) > 4:
            raise ValueError("RaggedPrefetchLoader fetches all variables in one launch (<= 4 variables)")
        self.ds, self.sampler, self.bs, self.drop_last, self.depth = dataset, sampler, batch_size, drop_last, max(2, depth)
        dev = dataset.device
        self.stream = torch.cuda.Stream(device=dev)
        self.events = [torch.cuda.Event() for _ in range(self.depth)]
        self.bufs = [None] * self.depth   # per slot: {name: uint8 buffer}, grown on demand
        self.offs = [[torch.empty(batch_size + 1, dtype=torch.int64, device=dev) for _ in dataset.packed_names] for _ in range(self.depth)]
        self.d_ids = [torch.empty(batch_size, dtype=torch.int64, device=dev) for _ in range(self.depth)]
        self.pbufs = [{name: (torch.empty((batch_size, m) + tuple(dataset.widths[name]), dtype=dataset.out_dtypes[name],
                                          device=dev), torch.empty(batch_size, dtype=torch.int64, device=dev))
                       for name, (m, _) in dataset.pad.items()} for _ in range(self.depth)]

    def _batches(self):
        cur = []
        for i in self.sampler:
            cur.append(int(i))
            if len(cur) == self.bs:
                yield cur
                cur = []
        if cur and not self.drop_last:
            yield cur

    def _issue(self, slot, idx):
        ds = self.ds
        names = ds.packed_names
        ids = np.asarray(idx, dtype=np.int64)
        rows = [int(ds.counts[name][ids].sum()) for name in names]  # host-side sizes only
        need = [max(r, 1) * ds.out_row_bytes[name] for r, name in zip(rows, names)]
        if self.bufs[slot] is None or any(b.numel() < n for b, n in zip(self.bufs[slot], need)):
            # (grown rarely; a fresh buffer cannot still be in use by an earlier fetch)
            # (whole 8-byte words, so a converting fetch can view them in its output dtype)
            self.bufs[slot] = [torch.empty((int(n * 1.25) + 64 + 7) // 8 * 8, dtype=torch.uint8, device=ds.device) for n in need]
        keep = torch.from_numpy(ids).pin_memory()
        n = len(ids)
        with torch.cuda.stream(self.stream):
            self.d_ids[slot][:n].copy_(keep, non_blocking=True)
            for name, (buf, lengths) in self.pbufs[slot].items():
                m, v = ds.pad[name]
                ds.ddstore.get_samples(name, self.d_ids[slot][:n], buf[:n], stream=self.stream.cuda_stream, wait=False,
                                       overlap=True, src_dtype=ds.src_dtypes[name], lut=ds.luts[name],
                                       normalize=ds.normalize[name], pad_rows=m, pad_value=v, lengths=lengths[:n])
            kw = {}
            if any(ds.src_dtypes[m] is not None for m in names):  # (the uint8 buffers are viewed as out_dtypes)
                kw = dict(src_dtypes=[ds.src_dtypes[m] for m in names], luts=[ds.luts[m] for m in names],
                          normalize=[ds.normalize[m] for m in names])
            bufs = [b.view(ds.out_dtypes[m]) if kw else b for b, m in zip(self.bufs[slot], names)]
            if len(names) > 1:
                ds.ddstore.get_samples_multi(names, self.d_ids[slot][:n], bufs, offsets=[o[:n + 1] for o in self.offs[slot]],
                                             stream=self.stream.cuda_stream, wait=False, overlap=True, **kw)
            elif names:  # (a single packed variable: dds_get_samples)
                m = names[0]
                ds.ddstore.get_samples(m, self.d_ids[slot][:n], bufs[0], offsets=self.offs[slot][0][:n + 1],
                                       stream=self.stream.cuda_stream, wait=False, overlap=True, src_dtype=ds.src_dtypes[m],
                                       lut=ds.luts[m], normalize=ds.normalize[m])
            self.events[slot].record(self.stream)
        return n, rows, keep

    def __iter__(self):
        consumer = torch.cuda.current_stream(self.ds.device)
        pending, slot = [], 0
        for idx in self._batches():
            self.stream.wait_stream(consumer)  # the slot's previous tenant has been consumed by whatever is queued so far
            pending.append((slot,) + self._issue(slot, idx))
            slot = (slot + 1) % self.depth
            if len(pending) == self.depth:
                yield self._take(pending.pop(0), consumer)
        while pending:
            yield self._take(pending.pop(0), consumer)
        self.ds.ddstore.wait()  # surface any fetch error of the epoch

    def _take(self, item, consumer):
        slot, n, rows, _ = item
        consumer.wait_event(self.events[slot])
        ds, out = self.ds, {}
        for name, (buf, lengths) in self.pbufs[slot].items():
            out[name] = (buf[:n], lengths[:n])
        for k, name in enumerate(ds.packed_names):
            nb = rows[k] * ds.out_row_bytes[name]
            buf = self.bufs[slot][k][:nb].view(ds.out_dtypes[name]).view((rows[k],) + tuple(ds.widths[name]))
            out[name] = (buf, self.offs[slot][k][:n + 1] // ds.out_row_bytes[name])
        return out


def ingest_chunks(store, name, chunks, first_row=0):
    """Streaming ingest (SURVEY.md 8f rank 3): fill a pre-`init`'d shard from an iterator of host arrays (the
    reference's init + update-in-chunks pattern, include/ddstore.hpp:110-195). Every chunk goes through the library's
    pipelined path (`dds_ingest`: worker threads stage slices of the chunk into pinned buffers while the copy engine
    moves the previous buffer), so producing / reading chunk k+1 on the host overlaps the H2D copy of chunk k's tail.
    Returns rows written."""
    row = int(first_row)
    for chunk in chunks:
        arr = np.ascontiguousarray(chunk)
        store.ingest(name, arr, row)  # bounds-checked; returns when `arr` has been consumed
        row += arr.shape[0]
    store.ingest_wait()
    return row - int(first_row)


class DeviceBatchSampler:
    """Epoch shuffle with the indices resident on the device: the permutation of an epoch is EXACTLY
    torch's DistributedSampler order (same generator seeding: seed + epoch, same padding / striding,
    examples/vae/vae-ddp.py:216), computed once per epoch and moved to the GPU in one copy; batches are then
    slices of that tensor, so the per-batch index H2D copy and its sync disappear from the step.

        sampler = DeviceBatchSampler(len(ds), batch_size, rank, world_size, seed=0)
        for epoch in range(E):
            sampler.set_epoch(epoch)
            for ids in sampler:                       # int64 CUDA tensor views
                store.get_batch("x", ids, out=buf[:len(ids)], count=1)
    """

    def __init__(self, dataset_len, batch_size, rank=0, world_size=1, shuffle=True, seed=0, drop_last=False, device=None):
        class _Len:
            def __init__(self, n):
                self.n = n

            def __len__(self):
                return self.n

        self._ds = DistributedSampler(_Len(dataset_len), num_replicas=world_size, rank=rank, shuffle=shuffle, seed=seed,
                                      drop_last=False)
        self.batch_size, self.drop_last = batch_size, drop_last
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self._ids = None
        self.set_epoch(0)

    def set_epoch(self, epoch):
        self._ds.set_epoch(epoch)
        order = torch.tensor(list(iter(self._ds)), dtype=torch.int64)
        self._ids = order.to(self.device, non_blocking=False)

    def __len__(self):
        n = self._ids.numel()
        return n // self.batch_size if self.drop_last else (n + self.batch_size - 1) // self.batch_size

    def __iter__(self):
        n = self._ids.numel()
        for b0 in range(0, n, self.batch_size):
            if self.drop_last and b0 + self.batch_size > n:
                return
            yield self._ids[b0:b0 + self.batch_size]
