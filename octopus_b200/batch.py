"""Struct-of-arrays packing of haplotypes and reads — the memory layout of include/phmm_b200.h.

A *block* keeps every per-base array concatenated in one contiguous numpy array plus an int64 offset array, i.e.
exactly what ``phmm_haplotypes`` / ``phmm_reads`` point at. Blocks can be moved to the GPU as torch tensors
(``to_device``) so that a call can run on inputs already resident in HBM.
"""
import ctypes as C

import numpy as np

from . import _lib


def _u8(x):
    if isinstance(x, str):
        x = x.encode()
    if isinstance(x, (bytes, bytearray)):
        return np.frombuffer(bytes(x), dtype=np.uint8)
    return np.ascontiguousarray(np.asarray(x)).view(np.uint8).reshape(-1)


def pack_sequences(seqs, dtype=np.uint8):
    """One array per entry → (off[n+1] int64, the entries back to back). For uint8, str / bytes / arrays of any dtype give their bytes."""
    off = np.zeros(len(seqs) + 1, dtype=np.int64)
    parts = []
    for i, s in enumerate(seqs):
        a = _u8(s) if dtype == np.uint8 else np.ascontiguousarray(np.asarray(s, dtype=dtype)).reshape(-1)
        parts.append(a)
        off[i + 1] = off[i] + len(a)
    data = np.concatenate(parts) if parts else np.zeros(0, dtype=dtype)
    return off, np.ascontiguousarray(data.astype(dtype, copy=False))


class _Block:
    _fields = ()

    def arrays(self):
        return {f: getattr(self, f) for f in self._fields if getattr(self, f) is not None}

    def to_device(self, device="cuda:0"):
        """Copy of this block whose arrays are torch CUDA tensors (inputs resident in HBM)."""
        import torch
        out = object.__new__(type(self))
        out.__dict__.update(self.__dict__)
        for f in self._fields:
            a = getattr(self, f)
            if a is not None:
                t = torch.from_numpy(np.ascontiguousarray(a))
                setattr(out, f, t.to(device, non_blocking=False))
        out.on_device = True
        return out

    def pin(self):
        """Copy of this block in page-locked host memory (torch pinned tensors viewed as numpy)."""
        import torch
        out = object.__new__(type(self))
        out.__dict__.update(self.__dict__)
        keep = []
        for f in self._fields:
            a = getattr(self, f)
            if a is not None:
                t = torch.from_numpy(np.ascontiguousarray(a)).pin_memory()
                keep.append(t)
                setattr(out, f, t.numpy())
        out._pinned = keep
        return out


def _ptr(a):
    if a is None:
        return None
    if hasattr(a, "data_ptr"):
        return a.data_ptr()
    return a.ctypes.data


class HaplotypeBlock(_Block):
    """H haplotypes: what HaplotypeLikelihoodModel::reset computes per haplotype (haplotype_likelihood_model.cpp:60-78)."""
    _fields = ("off", "seq", "snv_mask_fwd", "snv_prior_fwd", "snv_mask_rev", "snv_prior_rev", "gap_open", "gap_extend", "begin")

    def __init__(self, off, seq, snv_mask_fwd, snv_prior_fwd, snv_mask_rev, snv_prior_rev, gap_open, gap_extend, begin=None):
        self.n = len(off) - 1
        self.off = np.ascontiguousarray(off, dtype=np.int64)
        self.seq = np.ascontiguousarray(seq, dtype=np.uint8)
        self.snv_mask_fwd = np.ascontiguousarray(snv_mask_fwd, dtype=np.uint8)
        self.snv_prior_fwd = np.ascontiguousarray(snv_prior_fwd, dtype=np.int8)
        self.snv_mask_rev = np.ascontiguousarray(snv_mask_rev, dtype=np.uint8)
        self.snv_prior_rev = np.ascontiguousarray(snv_prior_rev, dtype=np.int8)
        self.gap_open = np.ascontiguousarray(gap_open, dtype=np.int8)
        self.gap_extend = np.ascontiguousarray(gap_extend, dtype=np.int8)
        self.begin = None if begin is None else np.ascontiguousarray(begin, dtype=np.int64)
        self.on_device = False
        total = int(self.off[-1])
        for f in self._fields[1:8]:
            assert len(getattr(self, f)) == total, f

    @classmethod
    def of_device(cls, off, seq, snv_mask_fwd, snv_prior_fwd, snv_mask_rev, snv_prior_rev, gap_open, gap_extend, begin=None):
        """A block over torch CUDA tensors as they are (begin: host array or None, copied to the tensors' device)."""
        import torch
        out = object.__new__(cls)
        out.n = len(off) - 1
        out.off, out.seq = off, seq
        out.snv_mask_fwd, out.snv_prior_fwd, out.snv_mask_rev, out.snv_prior_rev = snv_mask_fwd, snv_prior_fwd, snv_mask_rev, snv_prior_rev
        out.gap_open, out.gap_extend = gap_open, gap_extend
        out.begin = None if begin is None else torch.as_tensor(np.ascontiguousarray(begin, dtype=np.int64), device=seq.device)
        out.on_device = True
        return out

    def c_struct(self):
        s = _lib.Haplotypes()
        s.n = self.n
        for f in self._fields:
            setattr(s, f, _ptr(getattr(self, f)))
        return s

    def length(self, h):
        return int(self.off[h + 1] - self.off[h])

    def hap(self, h):
        """Host-side view of haplotype h's arrays (dict of numpy slices)."""
        a, b = int(self.off[h]), int(self.off[h + 1])
        return {f: getattr(self, f)[a:b] for f in self._fields[1:8]}


class HaplotypeSequences(_Block):
    """H haplotypes as sequences only (phmm_haplotype_sequences): the populate calls with an error model derive the penalty arrays
    of a HaplotypeBlock from them on the GPU. ``is_substitution``: per-base flags (bases that are substitutions in
    Haplotype::cigar()) or None; ``begin``: mapped_begin per haplotype or None. Numpy arrays, or torch CUDA tensors."""
    _fields = ("off", "seq", "is_substitution", "begin")

    def __init__(self, off, seq, begin=None, is_substitution=None):
        self.n = len(off) - 1
        self.on_device = hasattr(seq, "data_ptr") and seq.is_cuda
        if self.on_device:
            self.off, self.seq, self.is_substitution, self.begin = off, seq, is_substitution, begin
            return
        self.off = np.ascontiguousarray(off, dtype=np.int64)
        self.seq = np.ascontiguousarray(seq, dtype=np.uint8)
        self.is_substitution = None if is_substitution is None else np.ascontiguousarray(is_substitution, dtype=np.uint8)
        self.begin = None if begin is None else np.ascontiguousarray(begin, dtype=np.int64)
        assert self.is_substitution is None or len(self.is_substitution) == int(self.off[-1])

    @classmethod
    def pack(cls, sequences, begin=None, is_substitution=None):
        """sequences (list of str / bytes / uint8 arrays), optional per-haplotype begins and per-haplotype flag arrays → block."""
        off, seq = pack_sequences(sequences)
        sub = None if is_substitution is None else pack_sequences([np.asarray(x, dtype=np.uint8) for x in is_substitution])[1]
        return cls(off, seq, begin, sub)

    def c_struct(self):
        s = _lib.HaplotypeSequences()
        s.n = self.n
        for f in self._fields:
            setattr(s, f, _ptr(getattr(self, f)))
        return s


class ReadBlock(_Block):
    """R reads: the AlignedRead fields the path consumes (basics/aligned_read.hpp:36-39,120-146)."""
    _fields = ("off", "bases", "quals", "mapq", "reverse", "begin")

    def __init__(self, off, bases, quals, mapq=None, reverse=None, begin=None):
        self.n = len(off) - 1
        self.off = np.ascontiguousarray(off, dtype=np.int64)
        self.bases = np.ascontiguousarray(bases, dtype=np.uint8)
        self.quals = np.ascontiguousarray(quals, dtype=np.uint8)
        self.mapq = np.full(self.n, 60, dtype=np.uint8) if mapq is None else np.ascontiguousarray(mapq, dtype=np.uint8)
        self.reverse = np.zeros(self.n, dtype=np.uint8) if reverse is None else np.ascontiguousarray(reverse, dtype=np.uint8)
        self.begin = np.zeros(self.n, dtype=np.int64) if begin is None else np.ascontiguousarray(begin, dtype=np.int64)
        self.on_device = False
        assert len(self.bases) == len(self.quals) == int(self.off[-1])

    def c_struct(self):
        s = _lib.Reads()
        s.n = self.n
        for f in self._fields:
            setattr(s, f, _ptr(getattr(self, f)))
        return s

    def length(self, r):
        return int(self.off[r + 1] - self.off[r])

    def read(self, r):
        a, b = int(self.off[r]), int(self.off[r + 1])
        return self.bases[a:b], self.quals[a:b]


def pack_haplotypes(seqs, snv_mask_fwd, snv_prior_fwd, snv_mask_rev, snv_prior_rev, gap_open, gap_extend, begin=None):
    """Lists (one entry per haplotype) → HaplotypeBlock."""
    off, seq = pack_sequences(seqs)
    _, mf = pack_sequences(snv_mask_fwd, np.uint8)
    _, pf = pack_sequences(snv_prior_fwd, np.int8)
    _, mr = pack_sequences(snv_mask_rev, np.uint8)
    _, pr = pack_sequences(snv_prior_rev, np.int8)
    _, go = pack_sequences(gap_open, np.int8)
    _, ge = pack_sequences(gap_extend, np.int8)
    return HaplotypeBlock(off, seq, mf, pf, mr, pr, go, ge, begin)


def pack_reads(bases, quals, mapq=None, reverse=None, begin=None):
    off, b = pack_sequences(bases)
    _, q = pack_sequences(quals)
    return ReadBlock(off, b, q, mapq, reverse, begin)


def pack_positions(position_lists, H, R):
    """position_lists[h][r] → (off[H*R+1] int64, pos int32) in [H][R] order (phmm_positions)."""
    off = np.zeros(H * R + 1, dtype=np.int64)
    flat = []
    i = 0
    for h in range(H):
        for r in range(R):
            p = position_lists[h][r]
            flat.extend(int(x) for x in p)
            off[i + 1] = off[i] + len(p)
            i += 1
    return off, np.asarray(flat if flat else [0], dtype=np.int32)[:max(len(flat), 1)]


def _cat_off(blocks):
    off, base = [np.zeros(1, dtype=np.int64)], 0
    for b in blocks:
        off.append(b.off[1:] + base)
        base += int(b.off[-1])
    return np.concatenate(off)


def _cat(blocks, f):
    return np.concatenate([getattr(b, f) for b in blocks])


def concat_sequences(blocks):
    """Host HaplotypeSequences back to back as one block (flags zero-filled where a block has none, begins 0 where it has none)."""
    total = [int(b.off[-1]) for b in blocks]
    sub = None
    if any(b.is_substitution is not None for b in blocks):
        sub = np.concatenate([b.is_substitution if b.is_substitution is not None else np.zeros(t, dtype=np.uint8) for b, t in zip(blocks, total)])
    begin = np.concatenate([b.begin if b.begin is not None else np.zeros(b.n, dtype=np.int64) for b in blocks])
    return HaplotypeSequences(_cat_off(blocks), _cat(blocks, "seq"), begin, sub)


def concat_reads(blocks):
    """Host read blocks back to back as one ReadBlock (the block itself when there is one)."""
    if len(blocks) == 1:
        return blocks[0]
    return ReadBlock(_cat_off(blocks), *[_cat(blocks, f) for f in ReadBlock._fields[1:]])


def concat_blocks(hap_blocks, read_blocks):
    """Regions back to back for PairHMMEngine.populate_regions: (HaplotypeBlock, ReadBlock, hap_first, read_first) (host blocks)."""
    haps = HaplotypeBlock(_cat_off(hap_blocks), *[_cat(hap_blocks, f) for f in HaplotypeBlock._fields[1:8]],
                          np.concatenate([b.begin if b.begin is not None else np.zeros(b.n, dtype=np.int64) for b in hap_blocks]))
    reads = concat_reads(read_blocks)
    hap_first = np.concatenate([[0], np.cumsum([b.n for b in hap_blocks])]).astype(np.int32)
    read_first = np.concatenate([[0], np.cumsum([b.n for b in read_blocks])]).astype(np.int32)
    return haps, reads, hap_first, read_first
