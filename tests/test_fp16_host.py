"""Host logic of fp16 training, without a GPU: the compute dtype follows the autocast state, and 16-bit weight shadows
are cached per type."""
import math

import torch

from olmoasr_b200 import _core


def test_compute_dtype_follows_the_autocast_state(monkeypatch):
    assert _core.compute_dtype() == torch.bfloat16
    state = {"on": True, "dtype": torch.float16}     # the CUDA autocast state, which needs no device to be read
    monkeypatch.setattr(torch, "is_autocast_enabled", lambda dev: dev == "cuda" and state["on"])
    monkeypatch.setattr(torch, "get_autocast_dtype", lambda dev: state["dtype"])
    assert _core.compute_dtype() == torch.float16
    state["dtype"] = torch.bfloat16
    assert _core.compute_dtype() == torch.bfloat16
    state.update(on=False, dtype=torch.float16)
    assert _core.compute_dtype() == torch.bfloat16


def test_shadow_cache_is_keyed_by_dtype_and_version():
    p = torch.zeros(4)
    cache, builds = _core._ShadowCache(), []

    def build(dt):
        return lambda: builds.append(dt) or dt

    assert cache.get((p,), build(torch.bfloat16)) == torch.bfloat16
    assert cache.get((p,), build(torch.bfloat16)) == torch.bfloat16
    assert cache.get((p,), build(torch.float16), torch.float16) == torch.float16
    with torch.no_grad():
        p.add_(1)
    assert cache.get((p,), build(torch.float16), torch.float16) == torch.float16
    assert builds == [torch.bfloat16, torch.float16, torch.float16]


# ---- dtype-aware CPU stand-ins for the optimizer and cast entry points (restated from csrc/optimizer.cu) -------------
class _Device:
    """Resolves the raw pointers FusedAdamW passes to the tensors they point at, and runs the optimizer launches."""

    def __init__(self, tensors):
        self.t = {}
        for x in tensors:
            self.add(x)
        self.calls = []

    def add(self, x):
        self.t[x.data_ptr()] = x
        return x

    def __call__(self, name, *a):
        self.calls.append(name)
        T = lambda p: None if p is None else self.t[p]
        if name == "oasr_grad_sqnorm_flat":
            g, n, inv, out = T(a[0]), a[1], a[2], T(a[3])
            out[0] = ((g[:n] * inv) ** 2).sum()
        elif name in ("oasr_optim_prepare", "oasr_optim_prepare_amp"):
            if name == "oasr_optim_prepare":
                norm, found, st, inv, max_norm, b1, b2 = T(a[0]), T(a[1]), T(a[2]), *a[3:7]
                scale, ext = None, None
            else:
                norm, found, st, scale, ext, inv, max_norm, b1, b2 = T(a[0]), T(a[1]), T(a[2]), T(a[3]), T(a[4]), *a[5:9]
            nsq = float(norm.reshape(-1)[0])
            if scale is not None:
                nsq /= float(scale) ** 2
                inv /= float(scale)
            if (ext is not None and float(ext) != 0) or not math.isfinite(nsq):
                found.fill_(1.0)
                st[4] = 1.0
                return
            coef = inv * (min(1.0, max_norm / (math.sqrt(nsq) + 1e-6)) if max_norm > 0 else 1.0)
            st[0] += 1
            st[1], st[2], st[3], st[4], st[5] = coef, 1 - b1 ** float(st[0]), math.sqrt(1 - b2 ** float(st[0])), 0.0, math.sqrt(nsq)
        elif name in ("oasr_adamw_flat", "oasr_adamw_flat16"):
            p, g, m, v, sh, n, st = T(a[0]), T(a[1]), T(a[2]), T(a[3]), T(a[4]), a[5], T(a[6])
            lr, b1, b2, eps, wd = a[7:12]
            if float(st[4]) != 0:
                return
            gi = g * float(st[1])
            m.mul_(b1).add_((1 - b1) * gi)
            v.mul_(b2).add_((1 - b2) * gi * gi)
            p.mul_(1 - lr * wd).sub_(lr / float(st[2]) * (m / (v.sqrt() / float(st[3]) + eps)))
            shadow_dtype = torch.float16 if name == "oasr_adamw_flat16" else torch.bfloat16
            assert name != "oasr_adamw_flat16" or a[12] == 1       # OASR_DTYPE_F16
            sh.view(shadow_dtype).copy_(p.to(shadow_dtype))
        else:
            raise AssertionError(f"unexpected launch {name}")


def _slab_model(monkeypatch):
    from tests import cpu_backend
    from olmoasr_b200.slab import ParamSlabs

    cpu_backend.install(monkeypatch)
    torch.manual_seed(0)
    model = torch.nn.Sequential(torch.nn.Linear(16, 8), torch.nn.Linear(8, 4))
    return model, ParamSlabs(model)


def test_slab_shadow_recast_on_a_dtype_switch(monkeypatch):
    from olmoasr_b200 import kernels as K

    model, sl = _slab_model(monkeypatch)
    casts = []
    for name in ("cast_bf16", "convert"):
        fn = getattr(K, name)
        monkeypatch.setattr(K, name, lambda *a, _fn=fn, _n=name, **k: casts.append(_n) or _fn(*a, **k))
    sl.ensure_synced()
    assert sl.S_dtype == torch.bfloat16 and torch.equal(sl.S, sl.P.bfloat16()) and casts == ["cast_bf16"]
    sl.ensure_synced()                                        # nothing changed: no cast
    sl.ensure_synced(torch.float16)                           # fp16 forward: one flat re-cast into the same bytes
    assert sl.S_dtype == torch.float16 and casts == ["cast_bf16", "convert"]
    assert sl.S.dtype == torch.bfloat16 and torch.equal(sl.shadow_slab(), sl.P.half())
    sl.ensure_synced(torch.float16)
    assert casts == ["cast_bf16", "convert"]
    sl.ensure_synced(torch.bfloat16)                          # e.g. a bf16 evaluation after an fp16 step
    assert torch.equal(sl.S, sl.P.bfloat16()) and casts == ["cast_bf16", "convert", "cast_bf16"]


def _optimizer_run(monkeypatch, scale=None, found=None, inv_scale=1.0, grad_mult=1.0, shadow=torch.bfloat16):
    from olmoasr_b200 import optim

    model, sl = _slab_model(monkeypatch)
    sl.ensure_synced(shadow)
    opt = optim.FusedAdamW(model.parameters(), lr=1e-2, slabs=sl)
    torch.manual_seed(1)
    sl.G.copy_(torch.randn_like(sl.G) * grad_mult)
    opt._build()
    dev = _Device([sl.P, sl.G, sl.M, sl.V, sl.S, opt._norm_sq, opt._found_inf, opt._dev_state])
    monkeypatch.setattr(optim, "call", dev)
    monkeypatch.setattr(optim, "stream", lambda: None)
    if scale is not None or found is not None:            # what GradScaler.step attaches
        opt.grad_scale = None if scale is None else dev.add(torch.tensor(scale))
        opt.found_inf = dev.add(torch.tensor(float(found or 0.0)))
    opt.step(inv_scale=inv_scale)
    return sl, opt, dev.calls


def test_fused_adamw_grad_scaler_contract(monkeypatch):
    S = 1024.0
    plain, _, calls = _optimizer_run(monkeypatch)
    assert calls == ["oasr_grad_sqnorm_flat", "oasr_optim_prepare", "oasr_adamw_flat"]
    # grad_scale + found_inf: the scaled gradients are unscaled on the device
    scaled, opt, calls = _optimizer_run(monkeypatch, scale=S, found=0.0, grad_mult=S)
    assert calls == ["oasr_grad_sqnorm_flat", "oasr_optim_prepare_amp", "oasr_adamw_flat"]
    assert torch.allclose(scaled.P, plain.P, rtol=0, atol=1e-7) and float(opt._dev_state[0]) == 1
    # grad_scale None: scaler.unscale_(opt) already ran
    unscaled, _, calls = _optimizer_run(monkeypatch, scale=None, found=0.0)
    assert calls[1] == "oasr_optim_prepare_amp" and torch.equal(unscaled.P, plain.P)
    # found_inf set: no update, step not counted
    skipped, opt, _ = _optimizer_run(monkeypatch, scale=S, found=1.0, grad_mult=S)
    fresh = _slab_model(monkeypatch)[1]
    assert torch.equal(skipped.P, fresh.P) and float(opt._dev_state[0]) == 0 and float(opt._found_inf) == 1
    # inv_scale (1 / world of SlabGradSync) still multiplies in
    half_plain, _, _ = _optimizer_run(monkeypatch, inv_scale=0.5)
    half_scaled, _, _ = _optimizer_run(monkeypatch, scale=S, found=0.0, grad_mult=S, inv_scale=0.5)
    assert torch.allclose(half_scaled.P, half_plain.P, rtol=0, atol=1e-7) and not torch.equal(half_plain.P, plain.P)


def test_fused_adamw_refreshes_the_shadow_in_the_type_the_slab_holds(monkeypatch):
    sl, _, calls = _optimizer_run(monkeypatch, shadow=torch.float16)
    assert calls[-1] == "oasr_adamw_flat16"
    assert torch.equal(sl.shadow_slab(), sl.P.half())
