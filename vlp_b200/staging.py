"""Input staging for the H100 hot path (SURVEY.md §8f-4): what sits between the data loader and `model(...)`.

The reference loader (vlp/seq2seq_loader.py:229-359, stacked by vlp/loader_utils.py) hands the training loop, per step and per GPU,
fp32 region features [B,100,2048] + [B,100,1607] and an int64 [B,123,123] self-attention mask — 1.58 MB per sample, 101 MB per
64-sample batch — which run_img2txt_dist.py:463 copies synchronously (`t.to(device)`).  At 6.7 ms per step that copy is a
quarter of the PCIe budget and the int64 mask is pure redundancy.  This module provides the H100-first replacement:

  * `mask_descriptor` / `PackedAttentionMask.synthesize`: the mask travels as three integers per sample (len_a, len_b, mode) and
    is synthesised on the device, directly in the packed form (S = 128 * ceil(L / 128) bits per row) the attention kernels consume (`vlpk_mask_synth`,
    bit-identical to packing the loader's matrix — tests/test_staging_gpu.py);
  * features are staged as bf16 (the dtype the region projections read; feature files / loader workers should emit bf16 — a
    one-time dataset conversion — fp32 host tensors are accepted and converted on the host as a fallback);
  * `BatchStager`: pinned host slots + a copy stream, `depth`-deep: batch i+1's host->device copies overlap batch i's compute;
    `get()` makes the compute stream wait for the copy event only.

The staged batch feeds the unchanged module surface: `model(img, vis_pe, input_ids, segment_ids, input_mask, ...)` where
`input_mask` may be the loader's int64 tensor or a `PackedAttentionMask`.
"""
import torch

from . import _lib as L
from . import ops

BF16 = torch.bfloat16
FIELDS = ("input_ids", "segment_ids", "input_mask", "masked_ids", "masked_pos", "masked_weights", "is_next", "task_idx", "img",
          "vis_masked_pos", "vis_pe", "ans_labels")          # order of Preprocess4Seq2seq.__call__'s tuple (seq2seq_loader.py:359)


def mask_descriptor(len_b, mode):
    """(len_b [B] int32, mode [B] int32: 0 = bidirectional, 1 = seq2seq) host tensors for `PackedAttentionMask.synthesize`.
    len_b = number of text tokens (tokens_b) per sample; the region prefix length len_a is a per-model constant."""
    lb = torch.as_tensor(len_b, dtype=torch.int32)
    md = torch.as_tensor([1 if (m == "s2s" or m == 1) else 0 for m in mode] if not torch.is_tensor(mode) else mode, dtype=torch.int32)
    return lb, md


def loader_mask(len_b, mode, len_a, L_):
    """bool [B, L, L]: the self-attention mask seq2seq_loader.py:291-301 builds for text lengths len_b [B] and modes [B] (1 = seq2seq,
    0 = bidirectional) — the matrix the packed mask of `mask_descriptor(len_b, mode)` stands for."""
    len_b, mode = torch.as_tensor(len_b), torch.as_tensor(mode)
    st = len_a + 2
    en = (st + 1 + len_b.to(torch.int64)).view(-1, 1, 1)
    i = torch.arange(L_, device=len_b.device).view(1, -1, 1)
    j = torch.arange(L_, device=len_b.device).view(1, 1, -1)
    s2s = (j < st) | ((i >= st) & (i < en) & (j >= st) & (j <= i))
    bi = (j < en).expand(-1, L_, -1)
    return torch.where(mode.view(-1, 1, 1) != 0, s2s, bi)


def describe_mask(input_mask, len_a):
    """Recover (len_b, mode) from a loader-built [B,L,L] 0/1 mask (seq2seq_loader.py:291-301) — for callers that still receive the
    matrix from an unmodified loader.  s2s rows past the text keep only the prefix, bi rows are all identical.  ValueError unless the
    matrix is exactly loader_mask(len_b, mode): a matrix of another form — one that blocks the key columns of masked regions (what
    seq2seq_loader.py:303-304 means to do for --vis_mask_prob), or one whose layout len_a does not describe — has no (len_b, mode)
    descriptor, and reading one off it would stand for a different mask.  O(B*L*L) work on the matrix's device."""
    m = input_mask
    B, Lm, _ = m.shape
    st = len_a + 2
    last_row = m[:, Lm - 1]                                   # bi: [1]*en + [0]*pad ; s2s: prefix only (unless the text fills L)
    diag = m[:, torch.arange(Lm), torch.arange(Lm)]           # s2s: ones on [0, en) ... bi: ones on [0, en)
    en = diag.sum(-1)
    first_text_row = m[:, st]                                  # s2s: attends to [0, st]; bi: [0, en)
    s2s = (first_text_row.sum(-1) == st + 1) & (en > st + 1) | ((en == st + 1) & (last_row.sum(-1) == st) & (Lm > st + 1))
    len_b = (en - len_a - 3).clamp_min(0)
    bad = (m != loader_mask(len_b, s2s, len_a, Lm).to(m.dtype)).flatten(1).any(1) | (en < st + 1)
    if bool(bad.any()):
        raise ValueError(f"vlp_b200: the attention mask of sample(s) {bad.nonzero().flatten().tolist()[:8]} is not a loader mask of "
                         f"{len_a} regions (seq2seq_loader.py:291-301) — a matrix with blocked region columns has no "
                         f"(len_b, mode) descriptor")
    return len_b.to(torch.int32), s2s.to(torch.int32)


class PackedAttentionMask:
    """The self-attention mask of one batch in the form the attention kernels read: int32 [B, L, 4] (bit j of row i = query i
    attends to key j).  Accepted wherever the module surface takes `attention_mask` / `input_mask`."""

    def __init__(self, bits, L_):
        self._vlpk_bits = bits
        self.L = L_

    @property
    def bits(self):
        return self._vlpk_bits

    @property
    def is_cuda(self):
        return self._vlpk_bits.is_cuda

    @property
    def device(self):
        return self._vlpk_bits.device

    def dim(self):
        return 3

    @classmethod
    def synthesize(cls, len_b, mode, len_a, L_, out=None):
        """len_b, mode: int32 CUDA tensors [B].  One kernel launch, no [B,L,L] tensor exists anywhere."""
        if not (len_b.is_cuda and mode.is_cuda and len_b.dtype == torch.int32 and mode.dtype == torch.int32):
            raise RuntimeError("vlp_b200.staging: len_b / mode must be int32 CUDA tensors")
        B = len_b.shape[0]
        shape = (B, int(L_), ops.key_slots(int(L_)) // 32)
        if out is not None and not (tuple(out.shape) == shape and out.dtype == torch.int32 and out.is_cuda and out.is_contiguous()):
            raise ValueError(f"vlp_b200.staging: out must be a contiguous int32 CUDA tensor of shape {shape}")
        bits = out if out is not None else torch.empty(shape, device=len_b.device, dtype=torch.int32)
        L.call("vlpk_mask_synth", len_b.data_ptr(), mode.data_ptr(), int(len_a), B, int(L_), bits.data_ptr(), L.stream())
        return cls(bits, L_)


class GroupedCaptionMask:
    """The packed self-attention mask of G seq2seq captions per image (vlpk_mask_synth_grouped): int32 [B, L', S' / 32] for B images,
    L' = P + G * T with P = len_a + 2 prefix rows shared by the image's captions and T = L - P text rows per caption.  Passed as
    `attention_mask` with `captions_per_image=G` to BertForPreTrainingLossMask.forward."""

    def __init__(self, bits, G, T, len_a, L_):
        self._vlpk_bits = bits
        self.G, self.T, self.len_a, self.L = int(G), int(T), int(len_a), int(L_)

    @property
    def bits(self):
        return self._vlpk_bits

    @property
    def packed_len(self):
        return self.len_a + 2 + self.G * self.T

    @property
    def is_cuda(self):
        return self._vlpk_bits.is_cuda

    @property
    def device(self):
        return self._vlpk_bits.device

    def dim(self):
        return 3

    @staticmethod
    def check(G, len_a, L_):
        """(T, L') of G captions of L-row samples with len_a regions; ValueError when G < 1 or L' exceeds ops.MAX_SEQ."""
        G, len_a, L_ = int(G), int(len_a), int(L_)
        T = L_ - len_a - 2
        if G < 1 or T < 1 or len_a < 0:
            raise ValueError(f"vlp_b200: captions_per_image={G} with len_a={len_a}, L={L_} describes no packed sequence")
        Lp = len_a + 2 + G * T
        if Lp > ops.MAX_SEQ:
            raise ValueError(f"vlp_b200: {G} captions per image pack to {Lp} rows; the attention kernels take up to {ops.MAX_SEQ}")
        return T, Lp

    @classmethod
    def synthesize(cls, len_b, G, len_a, L_, out=None):
        """len_b: int32 CUDA tensor [B * G], the text tokens of pair b * G + g.  One kernel launch."""
        ops._require_cuda(len_b, "len_b")
        if not (len_b.dtype == torch.int32 and len_b.dim() == 1):
            raise RuntimeError("vlp_b200.staging: len_b must be a 1-d int32 CUDA tensor")
        T, Lp = cls.check(G, len_a, L_)
        if len_b.numel() == 0 or len_b.numel() % int(G):
            raise ValueError(f"vlp_b200.staging: {len_b.numel()} pairs do not form whole images of {G} captions")
        B = len_b.numel() // int(G)
        shape = (B, Lp, ops.key_slots(Lp) // 32)
        if out is not None and not (tuple(out.shape) == shape and out.dtype == torch.int32 and out.is_cuda and out.is_contiguous()):
            raise ValueError(f"vlp_b200.staging: out must be a contiguous int32 CUDA tensor of shape {shape}")
        bits = out if out is not None else torch.empty(shape, device=len_b.device, dtype=torch.int32)
        L.call("vlpk_mask_synth_grouped", len_b.contiguous().data_ptr(), int(G), int(len_a), B, T, bits.data_ptr(), L.stream())
        return cls(bits, G, T, len_a, L_)

    @classmethod
    def from_pair_masks(cls, input_mask, G, len_a):
        """The loader's [B * G, L, L] 0/1 masks (host or device) of B images x G seq2seq pairs -> the packed mask, via describe_mask.
        ValueError if any pair is bidirectional: its prefix rows see its text, so it cannot share a prefix."""
        len_b, s2s = describe_mask(input_mask.cpu(), len_a)
        if not bool(s2s.all()):
            raise ValueError("vlp_b200: only seq2seq pairs can share an image prefix; the batch holds a bidirectional pair")
        dev = input_mask.device if input_mask.is_cuda else torch.device("cuda", torch.cuda.current_device())
        return cls.synthesize(len_b.to(dev), G, len_a, input_mask.shape[-1])


class BatchStager:
    """Pinned, `depth`-deep host->device staging of training batches.

        stager = BatchStager(device, len_vis_input=100, max_len=123)
        stager.put(batch0)                       # dict with FIELDS keys (or the loader's 12-tuple); host tensors
        for step in range(n):
            if step + 1 < n: stager.put(next_batch)       # copies overlap the current step's compute
            b = stager.get()                     # device dict; b["input_mask"] is a PackedAttentionMask when the host batch
            loss = model(b["img"], b["vis_pe"], b["input_ids"], b["segment_ids"], b["input_mask"], ...)   # carried len_b / mode

    Host batches may carry either "input_mask" (the loader's int64 matrix: copied as is, 121 KB per sample) or "len_b" + "mode"
    (int32 [B]: the mask is synthesised on the device).  Features are staged in `feature_dtype`.

    captions_per_image=G > 1: batches of B images x G seq2seq captions for BertForPreTrainingLossMask(..., captions_per_image=G).
    "img" / "vis_pe" have B rows, the text fields B * G rows (pair b * G + g is image b's caption g), and either "len_b" (int32
    [B * G], with "mode" if the loader gives it) or the loader's "input_mask" matrices (read on the host through describe_mask, not
    copied); a bidirectional pair is refused with ValueError.  b["input_mask"] is a GroupedCaptionMask.  Reading matrices costs host
    time on the step's path — describe_mask compares every element, about 8 ms of one Xeon core for 64 pairs at L = 123 — so loaders
    that can should pass "len_b"."""

    def __init__(self, device, len_vis_input=100, max_len=123, feature_dtype=BF16, depth=2, captions_per_image=1):
        self.device = torch.device(device)
        self.G = int(captions_per_image)
        if self.G > 1:
            GroupedCaptionMask.check(self.G, len_vis_input, max_len)
        self.len_a, self.max_len, self.fdt, self.depth = int(len_vis_input), int(max_len), feature_dtype, int(depth)
        self.copy_stream = torch.cuda.Stream(device=self.device)
        self._slots = [None] * self.depth            # pinned host mirrors, allocated on first use per slot
        self._dev = [None] * self.depth
        self._ready = [torch.cuda.Event() for _ in range(self.depth)]
        self._consumed = [torch.cuda.Event() for _ in range(self.depth)]
        self._put = self._got = 0
        self.h2d_bytes = 0                           # bytes of the last put()
        for ev in self._consumed:
            ev.record(torch.cuda.current_stream(self.device))

    def _as_dict(self, batch):
        if isinstance(batch, dict):
            return batch
        return dict(zip(FIELDS, batch))

    def put(self, batch):
        if self._put - self._got >= self.depth:
            raise RuntimeError("BatchStager: all slots in flight; call get() first")
        hb = self._as_dict(batch)
        if self.G > 1:
            hb = dict(hb)
            if "input_mask" in hb:                   # the loader's matrices: their (len_b, mode), checked like from_pair_masks
                len_b, s2s = describe_mask(torch.as_tensor(hb.pop("input_mask")), self.len_a)
                if not bool(s2s.all()):
                    raise ValueError("BatchStager: only seq2seq pairs can share an image prefix; the batch holds a bidirectional pair")
                if "len_b" in hb and not torch.equal(torch.as_tensor(hb["len_b"]).to(torch.int32), len_b):
                    raise ValueError("BatchStager: len_b disagrees with the text lengths of input_mask")
                hb["len_b"] = len_b
            if "len_b" not in hb:
                raise ValueError("BatchStager: captions_per_image > 1 needs len_b (int32 [B * G]) or input_mask in every batch")
            if "mode" in hb and not bool((torch.as_tensor(hb.pop("mode")) == 1).all()):
                raise ValueError("BatchStager: only seq2seq pairs can share an image prefix; the batch holds a bidirectional pair")
        s = self._put % self.depth
        self._put += 1
        pinned = self._slots[s]
        if pinned is None:
            pinned = self._slots[s] = {}
        nbytes = 0
        staged = {}
        for k, v in hb.items():
            if not torch.is_tensor(v):
                v = torch.as_tensor(v)
            if k in ("img", "vis_pe") and v.dtype != self.fdt:
                v = v.to(self.fdt)                   # fallback: loaders should emit feature_dtype already
            buf = pinned.get(k)
            if buf is None or buf.shape != v.shape or buf.dtype != v.dtype:
                buf = pinned[k] = torch.empty(v.shape, dtype=v.dtype).pin_memory()
            if buf.data_ptr() != v.data_ptr():
                buf.copy_(v)                         # callers that fill the pinned slot in place (see slot()) skip this copy
            staged[k] = buf
            nbytes += buf.numel() * buf.element_size()
        self.h2d_bytes = nbytes
        with torch.cuda.stream(self.copy_stream):
            self.copy_stream.wait_event(self._consumed[s])       # the previous occupant of this slot has been consumed
            dev = {k: v.to(self.device, non_blocking=True) for k, v in staged.items()}
            if self.G > 1:
                dev["input_mask"] = GroupedCaptionMask.synthesize(dev["len_b"], self.G, self.len_a, self.max_len)
            elif "input_mask" not in dev:
                dev["input_mask"] = PackedAttentionMask.synthesize(dev["len_b"], dev["mode"], self.len_a, self.max_len)
            self._ready[s].record(self.copy_stream)
        self._dev[s] = dev

    def slot(self, fields):
        """Pinned host tensors of the next slot (allocated from `fields`: name -> (shape, dtype)) for loaders that write into them
        directly; pass the returned dict to put()."""
        s = self._put % self.depth
        if self._slots[s] is None:
            self._slots[s] = {}
        for k, (shape, dtype) in fields.items():
            buf = self._slots[s].get(k)
            if buf is None or tuple(buf.shape) != tuple(shape) or buf.dtype != dtype:
                self._slots[s][k] = torch.empty(shape, dtype=dtype).pin_memory()
        return {k: self._slots[s][k] for k in fields}

    def get(self):
        if self._got >= self._put:
            raise RuntimeError("BatchStager: get() without a pending put()")
        s = self._got % self.depth
        self._got += 1
        cur = torch.cuda.current_stream(self.device)
        cur.wait_event(self._ready[s])
        dev = self._dev[s]
        for v in dev.values():                        # the caching allocator must not recycle these before the compute stream is done
            t = v.bits if isinstance(v, (PackedAttentionMask, GroupedCaptionMask)) else v
            t.record_stream(cur)
        return _Staged(dev, self._consumed[s], cur)


class _Staged(dict):
    """Device batch; call done() (or let the next put() into the same slot wait) once the step's kernels have been enqueued."""

    def __init__(self, dev, consumed_event, stream):
        super().__init__(dev)
        self._ev, self._stream = consumed_event, stream

    def done(self):
        self._ev.record(self._stream)
