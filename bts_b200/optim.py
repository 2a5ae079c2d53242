"""Fused optimizer step of the BTS training loop (SURVEY 8f rank 1; reference pytorch/bts_main.py:371-373,456-460).

`FusedAdamW` is a drop-in for `torch.optim.AdamW` -- same constructor arguments, `param_groups` (so the reference's
poly-LR loop `for g in optimizer.param_groups: g['lr'] = ...` works unchanged), same `state` / `state_dict()` layout
(`step`, `exp_avg`, `exp_avg_sq` per parameter: checkpoints written by either optimizer load into the other) -- whose
`step()` is ONE multi-tensor CUDA kernel (csrc/optim.cu) over every parameter of every group, followed by ONE launch that
re-packs every cached conv operator of the wgmma engine (hi/lo split, swizzled tiles, forward and transposed) instead of
one pack launch per layer at the next forward pass (394 launches per step for DenseNet-161 + decoder).
"""
import ctypes

import torch

from . import _lib
from .ops import _stream


class FusedAdamW(torch.optim.AdamW):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2, repack=True):
        super().__init__(params, lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, amsgrad=False, foreach=False,
                         maximize=False, capturable=False, differentiable=False, fused=None)
        self.repack = repack
        self._plan = None

    def _build_plan(self, items):
        """static tables for the current set of (parameter, group) pairs: numel, hyper-group index, chunk map"""
        L = _lib.lib()
        chunk = L.bts_adamw_chunk()
        dev = items[0][0].device
        numel = [p.numel() for p, _ in items]
        ct, co = [], []
        for t, n in enumerate(numel):
            for o in range(0, n, chunk):
                ct.append(t)
                co.append(o)
        plan = {
            "key": tuple((id(p), gi) for p, gi in items),
            "numel": torch.tensor(numel, dtype=torch.int64, device=dev),
            "chunk_tensor": torch.tensor(ct, dtype=torch.int32, device=dev),
            "chunk_off": torch.tensor(co, dtype=torch.int64, device=dev),
            "n_chunks": len(ct),
            "ptrs_host": torch.empty(4 * len(items), dtype=torch.int64).pin_memory(),
            "ptrs": torch.empty(4 * len(items), dtype=torch.int64, device=dev),
        }
        return plan

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        items, steps = [], []
        for gi, group in enumerate(self.param_groups):
            if group.get("amsgrad") or group.get("maximize"):
                raise NotImplementedError("FusedAdamW: amsgrad / maximize are not used by BTS")
            for p in group["params"]:
                if p.grad is None:
                    continue
                if not (p.is_cuda and p.dtype == torch.float32 and p.grad.dtype == torch.float32 and p.is_contiguous()
                        and p.grad.is_contiguous() and not p.grad.is_sparse):
                    raise RuntimeError("FusedAdamW handles dense contiguous fp32 CUDA parameters (no fallback)")
                st = self.state[p]
                if len(st) == 0:
                    st["step"] = torch.tensor(0.0, dtype=torch.float32)             # torch.optim.AdamW's own state layout
                    st["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                    st["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                st["step"] += 1
                items.append((p, gi))
                steps.append(float(st["step"]))
        if not items:
            return loss
        # hyper groups: (param group, step count) -- normally one per param group
        hyper, hidx = {}, []
        for (p, gi), t in zip(items, steps):
            hidx.append(hyper.setdefault((gi, t), len(hyper)))
        if len(hyper) > 8:
            raise RuntimeError("FusedAdamW: more than 8 distinct (group, step) pairs")
        ng = len(hyper)
        sc = [0.0] * (7 * ng)
        for (gi, t), h in hyper.items():
            g = self.param_groups[gi]
            lr, (b1, b2), eps, wd = float(g["lr"]), g["betas"], float(g["eps"]), float(g["weight_decay"])
            bc1, bc2 = 1 - b1 ** t, 1 - b2 ** t
            vals = (1 - lr * wd, 1 - b1, b2, 1 - b2, bc2 ** 0.5, eps, (lr / bc1) * -1)
            for j, v in enumerate(vals):
                sc[j * ng + h] = v
        key = tuple((id(p), gi) for p, gi in items)
        if self._plan is None or self._plan["key"] != key:
            self._plan = self._build_plan(items)
        plan = self._plan
        n = len(items)
        ph = plan["ptrs_host"]
        if plan.get("ev") is not None:
            plan["ev"].synchronize()              # the previous step's async H2D copy of this pinned table has landed
        for i, (p, _) in enumerate(items):
            st = self.state[p]
            ph[i] = p.data_ptr()
            ph[n + i] = p.grad.data_ptr()
            ph[2 * n + i] = st["exp_avg"].data_ptr()
            ph[3 * n + i] = st["exp_avg_sq"].data_ptr()
        plan["ptrs"].copy_(ph, non_blocking=True)
        plan["ev"] = torch.cuda.Event()
        plan["ev"].record()
        grp = torch.tensor(hidx, dtype=torch.int32).pin_memory().to(plan["ptrs"].device, non_blocking=True) \
            if plan.get("hidx") != hidx else plan["grp"]
        plan["hidx"], plan["grp"] = hidx, grp
        scal = (ctypes.c_float * len(sc))(*sc)
        dev = items[0][0].device
        with torch.cuda.device(dev):
            rc = _lib.lib().bts_adamw_multi(plan["ptrs"].data_ptr(), plan["numel"].data_ptr(), grp.data_ptr(), n,
                                            plan["chunk_tensor"].data_ptr(), plan["chunk_off"].data_ptr(), plan["n_chunks"],
                                            scal, ng, _stream())
        _lib.check(rc, "bts_adamw_multi")
        _lib.count()
        _bump_versions([p for p, _ in items])
        if self.repack:
            from . import conv
            conv.repack_cached()
        return loss


def _bump_versions(params):
    """the kernel wrote the parameters behind autograd's back: bump their version counters (what an in-place torch op
    would have done) so that anything keyed on them -- e.g. the packed-operator cache -- notices"""
    setter = getattr(torch._C._autograd, "_unsafe_set_version_counter", None)
    if setter is not None:
        setter(list(params), [p._version + 1 for p in params])
    else:                                   # older torch: a no-op in-place op per parameter does the same
        for p in params:
            p.add_(0)
