"""SURVEY.md 8f-3 -- the op under its real caller, restated.

The reference trainer cannot be imported offline (`import cat` -> cat/shared/tokenizer.py:19 `import jieba`:
ModuleNotFoundError in this image, and /root/reference is absent on the GPU box), so the pieces of it that touch the loss
are restated here in behaviour, each with its source line:

  * ``AMTrainer``            cat/ctc/train.py:101-197 -- ``from ctc_crf import CTC_CRF_LOSS as CRFLoss`` (:118), lazy
    ``CRFContext(den_lm, device.index)`` on first forward (:137-141,:180-182), ``log_softmax`` (:174), labels/lx/ly moved to
    the CPU (:176-178), ``autocast(enabled=False)`` around ``criterion(logits.float(), labels.int(), lx.int(), ly.int())``
    (:184-190);
  * the unified trainer's SECOND criterion call on the same batch inside one step (cat/ctc/train_unified.py:248,267);
  * the step: ``autocast(enabled=use_amp)`` around the model, ``loss.data = loss.detach() * (local_bs * world / global_bs)``
    then ``backward()`` (cat/shared/manager.py:524-547);
  * CAT's mixed precision, with ``--amp --amp-dtype float16``: fp16, not bf16.  The manager imports ``autocast, GradScaler``
    from ``torch.cuda.amp`` (manager.py:29) and builds ``GradScaler(enabled=args.amp)`` (:280); ``autocast(enabled=use_amp)``
    (:533) is fp16 by default, so the encoder's last Linear returns fp16 logits; the step is ``scaler.scale(loss).backward()``
    (:547), then ``scaler.unscale_(optimizer)``, ``clip_grad_norm_(..., grad_norm)`` (default 2.0, coreutils.py:277-280),
    ``scaler.step(optimizer)``, ``scaler.update()`` (:620-627).  ``--amp`` alone keeps a bf16 autocast and a plain
    ``backward()`` + ``step()``;
  * process spawning: one process per GPU with ``mp.spawn``, ``torch.cuda.set_device(gpu)``, ``init_process_group('nccl')``,
    DistributedDataParallel (cat/shared/coreutils.py:493-504, cat/ctc/train.py:45-56,352).

``from ctc_crf import ...`` resolves to THIS repository.  Data: a synthetic "yesno"-shaped task (V = 5 tokens incl. blank;
features are noisy embeddings of the frame's token, so a 1-layer LSTM can learn it in a few steps), den graph = T o LM of a
small random phone LM composed natively (cat_b200.fst.compose_ctc_lm).

    python tools/trainer_smoke.py --steps 30                    # 1 GPU
    python tools/trainer_smoke.py --steps 30 --gpus 8           # DDP x 8 (mp.spawn, NCCL)
    python tools/trainer_smoke.py --steps 30 --from-logits      # CTC_CRF_LOSS(from_logits=True): raw encoder outputs in
    python tools/trainer_smoke.py --steps 30 --from-logits --amp --amp-dtype float16   # CAT's --amp: fp16 logits, GradScaler
"""
from __future__ import annotations

import argparse
import os
import sys
import tempfile
from typing import List

import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn as nn
from torch.amp import autocast

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

V = 5          # <blk>, a, c, s, t  (src/ctc_crf/test/main.py:6-11)
FEAT = 16


class TinyEncoder(nn.Module):
    """Stands in for cat.shared.encoder.*: (feats, lx) -> (logits (N,T,V), lx)."""

    def __init__(self, hidden: int = 48):
        super().__init__()
        self.lstm = nn.LSTM(FEAT, hidden, batch_first=True, bidirectional=True)
        self.out = nn.Linear(2 * hidden, V)

    def forward(self, feats, lx):
        h, _ = self.lstm(feats)
        return self.out(h), lx


class AMTrainer(nn.Module):
    """cat/ctc/train.py:101-197 restated (CRF branch), plus the second criterion call of train_unified.py:243-273."""

    def __init__(self, encoder: nn.Module, den_lm: str, lamb: float = 0.01, from_logits: bool = False, unified: bool = True):
        super().__init__()
        self.encoder = encoder
        self.den_lm = den_lm
        assert den_lm is not None and os.path.isfile(den_lm)
        from ctc_crf import CTC_CRF_LOSS as CRFLoss            # train.py:118
        self.criterion = CRFLoss(lamb=lamb, from_logits=from_logits) if from_logits else CRFLoss(lamb=lamb)
        self.from_logits = from_logits
        self.unified = unified
        self._crf_ctx = None

    def register_crf_ctx(self, den_lm=None):
        from ctc_crf import CRFContext                         # train.py:137
        self._crf_ctx = CRFContext(den_lm, next(iter(self.encoder.parameters())).device.index)

    def forward(self, feats, lx, labels, ly):
        logits, lx = self.encoder(feats, lx)
        if not self.from_logits:
            logits = torch.log_softmax(logits, dim=-1)         # train.py:174
        labels = labels.cpu()
        lx = lx.cpu()
        ly = ly.cpu()
        if self._crf_ctx is None:                              # lazy init, train.py:180-182
            self.register_crf_ctx(self.den_lm)
        with autocast("cuda", enabled=False):                  # train.py:184
            # the reference passes logits.float(); the raw-logit entry takes the encoder's own dtype (bf16 or fp16 under AMP)
            loss = self.criterion(logits if self.from_logits else logits.float(),
                                  labels.to(torch.int), lx.to(torch.int), ly.to(torch.int))
        if self.unified:                                       # train_unified.py:248-273: a second pass over the same batch
            chunk_out, _ = self.encoder(feats + 0.05 * torch.randn_like(feats), lx)
            chunk_logits = chunk_out if self.from_logits else torch.log_softmax(chunk_out, dim=-1)
            with autocast("cuda", enabled=False):
                chunk_loss = self.criterion(chunk_logits if self.from_logits else chunk_logits.float(),
                                            labels.to(torch.int), lx.to(torch.int), ly.to(torch.int))
            loss = loss + chunk_loss
        return loss


def make_den_lm(path: str, seed: int = 0) -> None:
    from cat_b200 import fst
    # every state has an arc for every phone and may end: the LM accepts every label sequence (a proper den graph)
    lm = fst.make_random_lm(H=6, V=V, d=V - 1, seed=seed)
    lm.final[:] = np.float32(-np.log(0.2))
    fst.write_fst(path, fst.compose_ctc_lm(lm))


def make_batch(rng: np.random.Generator, emb: np.ndarray, n: int, tmax: int = 48):
    """Sorted-by-length padded batch like sortedPadCollateASR (cat/shared/data.py:397-412): feats (N,T,F), lx, flat labels, ly."""
    lens = np.sort(rng.integers(tmax // 2, tmax + 1, size=n))[::-1]
    feats = np.zeros((n, int(lens[0]), FEAT), np.float32)
    labels: List[int] = []
    ly = []
    for i, T in enumerate(lens):
        L = int(rng.integers(2, 5))
        seq = rng.integers(1, V, size=L)
        bounds = np.sort(rng.choice(np.arange(2, T - 1), size=2 * L - 1, replace=False)) if T > 2 * L + 2 else np.arange(1, 2 * L)
        frame_tok = np.zeros(T, np.int64)
        for j in range(L):                       # label j occupies [b_{2j-1}, b_{2j}) ; blanks in between
            lo = 0 if j == 0 else bounds[2 * j - 1]
            hi = bounds[2 * j] if 2 * j < len(bounds) else T
            frame_tok[lo:hi] = seq[j]
            if 2 * j + 1 < len(bounds):
                frame_tok[bounds[2 * j]:bounds[2 * j + 1]] = 0
        feats[i, :T] = emb[frame_tok] + 0.3 * rng.standard_normal((T, FEAT)).astype(np.float32)
        labels.extend(int(k) for k in seq)
        ly.append(L)
    return (torch.tensor(feats), torch.tensor(lens.copy(), dtype=torch.int64), torch.tensor(labels, dtype=torch.int64),
            torch.tensor(ly, dtype=torch.int64))


def train(gpu: int, world: int, args, den_lm: str, log: List[float]) -> None:
    torch.manual_seed(1234 + gpu)
    torch.cuda.set_device(gpu)                                  # train.py:49
    if world > 1:
        dist.init_process_group(backend="nccl", init_method=f"tcp://127.0.0.1:{args.port}", world_size=world, rank=gpu)
    model = AMTrainer(TinyEncoder(), den_lm, lamb=0.01, from_logits=args.from_logits, unified=not args.no_unified).cuda(gpu)
    net = nn.parallel.DistributedDataParallel(model, device_ids=[gpu]) if world > 1 else model   # train.py:352
    opt = torch.optim.Adam(net.parameters(), lr=5e-3)
    amp_dtype = getattr(torch, args.amp_dtype)
    cat_amp = args.amp and amp_dtype == torch.float16          # CAT's fp16 step with its GradScaler (manager.py:29,280)
    scaler = torch.amp.GradScaler("cuda", enabled=cat_amp)
    rng = np.random.default_rng(100 + gpu)
    emb = np.random.default_rng(7).standard_normal((V, FEAT)).astype(np.float32)
    local_bs, global_bs = args.batch, args.batch * world
    for step in range(args.steps):
        feats, lx, labels, ly = make_batch(rng, emb, local_bs)
        feats = feats.cuda(gpu, non_blocking=True)
        with autocast("cuda", dtype=amp_dtype, enabled=args.amp):            # manager.py:533
            loss = net(feats, lx, labels, ly)
        raw = loss.detach().clone()
        loss.data = loss.detach() * (feats.size(0) * world / global_bs)       # manager.py:546
        opt.zero_grad(set_to_none=True)
        if cat_amp:
            scaler.scale(loss).backward()                                     # manager.py:547
            scaler.unscale_(opt)                                              # manager.py:620-627
            torch.nn.utils.clip_grad_norm_(net.parameters(), args.grad_norm, error_if_nonfinite=False)
            scaler.step(opt)
            scaler.update()
        else:
            loss.backward()
            opt.step()
        if world > 1:
            dist.all_reduce(raw)
            raw /= world
        val = float(raw.item())
        if not np.isfinite(val):
            raise RuntimeError(f"step {step}: loss {val}")
        log.append(val)
        if gpu == 0:
            print(f"[trainer_smoke] world={world} step {step:3d} loss {val:9.4f}", flush=True)
    if world > 1:
        dist.destroy_process_group()


def _worker(gpu: int, world: int, args, den_lm: str, out_path: str) -> None:
    log: List[float] = []
    train(gpu, world, args, den_lm, log)
    if gpu == 0:
        np.save(out_path, np.array(log))


def run(args) -> List[float]:
    tmp = tempfile.mkdtemp(prefix="ccb_trainer_")
    den_lm = os.path.join(tmp, "den_lm.fst")
    make_den_lm(den_lm)
    if args.gpus <= 1:
        log: List[float] = []
        train(0, 1, args, den_lm, log)
    else:
        out = os.path.join(tmp, "log.npy")
        mp.spawn(_worker, nprocs=args.gpus, args=(args.gpus, args, den_lm, out))   # coreutils.py:493-504
        log = list(np.load(out))
    first, last = float(np.mean(log[:5])), float(np.mean(log[-5:]))
    print(f"[trainer_smoke] gpus={args.gpus} amp={args.amp and args.amp_dtype} from_logits={args.from_logits} unified={not args.no_unified}: "
          f"loss {first:.4f} -> {last:.4f} over {len(log)} steps")
    if not last < first - 0.1 * abs(first):
        raise SystemExit(f"loss did not decrease: {first} -> {last}")
    return log


def parse(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--port", type=int, default=29531)
    ap.add_argument("--amp", action="store_true", help="autocast around the model (the loss stays under autocast(enabled=False))")
    ap.add_argument("--amp-dtype", default="bfloat16", choices=["bfloat16", "float16"],
                    help="autocast dtype of --amp; float16 is CAT's (torch.cuda.amp), with its GradScaler step")
    ap.add_argument("--grad-norm", type=float, default=2.0, help="gradient clipping of the float16 step (CAT's default)")
    ap.add_argument("--from-logits", action="store_true")
    ap.add_argument("--no-unified", action="store_true", help="one criterion call per step instead of two")
    return ap.parse_args(argv)


if __name__ == "__main__":
    run(parse())
