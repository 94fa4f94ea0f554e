"""Token n-gram LMs in ARPA text for the GPU prefix beam search (``ctc_crf.ctc_beam_search(..., lm=NGramLM(...))``).

``NGramLM`` wraps the native loader (``cat_b200/csrc/ngram.cc``); ``make_random_arpa`` writes valid ARPA files for tests and
benchmarks, as ``fst.make_random_lm`` does for den graphs.
"""
from __future__ import annotations

import ctypes as C
from typing import Sequence, Union

import numpy as np
import torch

from . import _lib

# ccb_ngram_copy codes (include/ctc_crf_b200.h) and their dtypes
_TABLES = {"tok2word": (0, np.int32), "root_p": (1, np.float32), "root_dst": (2, np.int32), "arc_off": (3, np.int32),
           "arc_word": (4, np.int32), "arc_p": (5, np.float32), "arc_dst": (6, np.int32), "bow": (7, np.float32),
           "back": (8, np.int32)}


class NGramLM:
    """A back-off n-gram LM over token labels, read from ARPA text (``lmplz --arpa``, ``cat/utils/pipeline/ngram.sh
    --arpa``).  ``labels[i]`` is the LM word of token i; ``labels[0]`` is the blank and is never scored, a label the LM does
    not list (or an empty one) scores as ``<unk>``, and ``<s>`` / ``</s>`` as a label is a ValueError.  A malformed file
    raises RuntimeError naming the line.  The tables live on the host until a search uses the LM on a device; dropping the
    object frees both (on the device with ``cudaFree``, which waits for the device)."""

    def __init__(self, path: str, labels: Sequence[str]):
        labels = [str(x) for x in labels]
        for i, w in enumerate(labels[1:], 1):
            if w in ("<s>", "</s>"):
                raise ValueError(f"NGramLM: label {i} is {w!r}; sentence boundaries cannot be tokens")
        arr = (C.c_char_p * len(labels))(*[w.encode() for w in labels])
        L = _lib.lib()
        h = L.ccb_ngram_create(str(path).encode(), arr, len(labels))
        if not h:
            raise RuntimeError(f"NGramLM: {_lib.last_error()}")
        self._h = h
        self.path = str(path)
        self.V = len(labels)
        info = (C.c_long * 18)()
        L.ccb_ngram_info(h, info)
        self.order = int(info[0])
        self.num_states, self.num_arcs = int(info[1]), int(info[2])
        self.unk_substituted = bool(info[3])
        self.num_words = int(info[4])
        self.bos, self.eos = int(info[6]), int(info[7])
        self.counts = [int(x) for x in info[8:8 + self.order]]

    @property
    def handle(self) -> int:
        return self._h

    def tables(self) -> dict:
        """The host tables as numpy arrays (ngram.h NGramHost): tok2word, root_p, root_dst, arc_off, arc_word, arc_p (NaN:
        a prefix the loader inserted, whose value is the back-off value), arc_dst, bow, back; plus bos and eos."""
        L = _lib.lib()
        sizes = {"tok2word": self.V, "root_p": self.num_words, "root_dst": self.num_words, "arc_off": self.num_states + 1,
                 "arc_word": self.num_arcs, "arc_p": self.num_arcs, "arc_dst": self.num_arcs, "bow": self.num_states,
                 "back": self.num_states}
        out = {}
        for name, (which, dt) in _TABLES.items():
            a = np.empty(sizes[name], dt)
            if L.ccb_ngram_copy(self._h, which, a.ctypes.data_as(C.c_void_p), a.nbytes) != 0:
                raise RuntimeError(f"ccb_ngram_copy({name}) failed")
            out[name] = a
        out["bos"], out["eos"] = self.bos, self.eos
        return out

    def score(self, input_ids, targets, input_lengths=None):
        """CAT's ``NGram.score`` (``AbsDecoder.score``): the (N,) fp32 natural-log score of each row's word string
        w_0 .. w_L, L = input_lengths[b] (the width U when None): w_i is the word of input_ids[b, i] for i < L, and w_L the
        word of ``targets[b, -1]``, the last column whatever L is (both CAT callers put token 0 there).  Token 0 is </s>,
        or <s> at position 0; every term is ARPA back-off from the empty history, as KenLM's score(bos=False, eos=False),
        summed in fp64 and rounded once (DESIGN.md §7 "N-gram sentence scoring").  One kernel launch.
        input_ids (N, U) and targets (N, U') are int32 or int64 on one device; input_lengths (N,) int32 or int64 on any.
        CUDA inputs: the result is on that device and nothing synchronises the host; a device token outside [0, V) or
        length outside [1, U] gives that row NaN.  CPU inputs: computed on the current CUDA device, returned on the CPU.
        ValueError: bad ranks, dtypes or shapes, host tokens or lengths out of range, or an LM whose file lists no <s> or
        no </s>."""
        ids, tgt = input_ids, targets
        ints = (torch.int32, torch.int64)
        if not isinstance(ids, torch.Tensor) or ids.dim() != 2 or ids.dtype not in ints or ids.shape[1] < 1:
            raise ValueError("NGramLM.score: input_ids must be an int32 or int64 (N, U) tensor with U >= 1")
        N, U = int(ids.shape[0]), int(ids.shape[1])
        if not isinstance(tgt, torch.Tensor) or tgt.dim() != 2 or tgt.dtype not in ints or tgt.shape[0] != N \
                or tgt.shape[1] < 1:
            raise ValueError(f"NGramLM.score: targets must be an int32 or int64 (N, U') tensor with N = {N}, U' >= 1")
        if tgt.device != ids.device:
            raise ValueError(f"NGramLM.score: targets is on {tgt.device}, input_ids on {ids.device}")
        lens = input_lengths
        if lens is not None and (not isinstance(lens, torch.Tensor) or lens.dtype not in ints or tuple(lens.shape) != (N,)):
            raise ValueError(f"NGramLM.score: input_lengths must be None or an int32 or int64 (N,) tensor with N = {N}")
        if lens is not None and lens.is_cuda and ids.is_cuda and lens.device != ids.device:
            raise ValueError(f"NGramLM.score: input_lengths is on {lens.device}, input_ids on {ids.device}")
        on_host = not ids.is_cuda
        if lens is not None and (on_host or not lens.is_cuda):     # host lengths are checked here
            lens = lens.cpu()
            if N and (int(lens.min()) < 1 or int(lens.max()) > U):
                raise ValueError(f"NGramLM.score: input_lengths must lie in [1, U = {U}]")
        last = tgt[:, -1]
        if on_host and N:
            used = ids if lens is None else ids[torch.arange(U)[None, :] < lens[:, None]]
            lo, hi = min(int(used.min()), int(last.min())), max(int(used.max()), int(last.max()))
            if lo < 0 or hi >= self.V:
                raise ValueError(f"NGramLM.score: tokens must lie in [0, V = {self.V})")
        if N == 0:
            return torch.empty(0, dtype=torch.float32, device=ids.device)
        entry = _lib.lib().ccb_ngram_score
        from .rnnt import _int32, _on_device
        dev = ids.device if not on_host else torch.device("cuda", torch.cuda.current_device())
        if on_host:
            ids, last = ids.to(dev), last.to(dev)
        if ids.stride(1) != 1 or ids.stride(0) < U:
            ids = ids.contiguous()
        if lens is not None:
            if lens.is_cuda:
                lens = lens.contiguous()
            else:
                lens = lens.to(dev) if on_host else _on_device(dev, _int32(lens))[0]
        out = torch.empty(N, dtype=torch.float32, device=dev)
        i64 = lambda t: int(t.dtype == torch.int64)
        with torch.cuda.device(dev):
            rc = entry(self._h, N, U, ids.data_ptr(), ids.stride(0), i64(ids), last.data_ptr(),
                                   last.stride(0), i64(last), lens.data_ptr() if lens is not None else None,
                                   i64(lens) if lens is not None else 0, out.data_ptr(),
                                   torch.cuda.current_stream(dev).cuda_stream)
        if rc:
            msg = _lib.last_error()
            raise (ValueError if "lists no" in msg else RuntimeError)(f"NGramLM.score: {msg}")
        return out.cpu() if on_host else out

    def __del__(self):
        h = getattr(self, "_h", None)
        if h:
            self._h = None
            try:
                _lib.lib().ccb_ngram_destroy(h)
            except Exception:      # interpreter shutdown: module globals may already be gone
                pass


def make_random_arpa(path: str, V: int, order: int, counts: Union[int, Sequence[int]], seed: int = 0, *,
                     pruned_prefixes: float = 0.0, missing_suffixes: bool = False, unk: bool = True, bos: bool = True,
                     extra_words: int = 0) -> str:
    """Write a random back-off LM of the given order over the token words "2" .. str(V-1) (CAT's token-level labels, where
    label 1 is "<unk>") as ARPA text.  counts: n-grams of each order 2..order (one int for all).  Every word is a unigram;
    an n-gram of order k extends a (k-1)-gram by a random word.  Options:
      pruned_prefixes  fraction of the n-grams of orders 2..order-1 dropped although a longer n-gram extends them (the
                       loader must insert them again);
      missing_suffixes False: every n-gram's suffix is listed, as KenLM writes; True: suffixes are left as drawn;
      unk, bos         list <unk> / <s>;
      extra_words      words no label names, with n-grams of their own.
    log10 probabilities lie in [-3, -0.05], back-off weights in [-1.2, 0.2]; <s> gets -99, as lmplz writes."""
    rng = np.random.default_rng(seed)
    words = [str(i) for i in range(2, V)] + [f"x{j}" for j in range(extra_words)] + ["</s>"]
    if unk:
        words.append("<unk>")
    counts = [counts] * (order - 1) if isinstance(counts, int) else list(counts)
    grams = [set(), {(w,) for w in words} | ({("<s>",)} if bos else set())]
    for k in range(2, order + 1):
        ctx = sorted(g for g in grams[k - 1] if g[-1] != "</s>")     # </s> ends an n-gram; <s> can only start one
        want = counts[k - 2]
        got = set()
        for _ in range(20):
            if len(got) >= want:
                break
            n = want - len(got)
            for h, w in zip(rng.integers(len(ctx), size=n), rng.integers(len(words), size=n)):
                got.add(ctx[h] + (words[w],))
        grams.append(got)
    if not missing_suffixes:
        for k in range(order, 1, -1):
            grams[k - 1] |= {g[1:] for g in grams[k]}
    if pruned_prefixes > 0:
        for k in range(2, order):
            prefixes = sorted({g[:-1] for g in grams[k + 1]} & grams[k])
            drop = rng.random(len(prefixes)) < pruned_prefixes
            grams[k] -= {p for p, d in zip(prefixes, drop) if d}
    with open(path, "w") as f:
        f.write("\\data\\\n")
        for k in range(1, order + 1):
            f.write(f"ngram {k}={len(grams[k])}\n")
        for k in range(1, order + 1):
            f.write(f"\n\\{k}-grams:\n")
            for g in sorted(grams[k]):
                p = -99.0 if g == ("<s>",) else -float(rng.uniform(0.05, 3.0))
                line = f"{p:.6f}\t{' '.join(g)}"
                if k < order:
                    line += f"\t{-float(rng.uniform(-0.2, 1.2)):.6f}"
                f.write(line + "\n")
        f.write("\n\\end\\\n")
    return path
