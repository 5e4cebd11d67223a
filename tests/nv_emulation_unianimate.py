"""Torch stand-ins for the UniAnimate window kernels of diffsynth._native (include/svi_b200_unianimate.h) — TEST
INFRASTRUCTURE ONLY.  `install(monkeypatch)` adds them to the DiT, VAE and conv stand-ins of nv_emulation, so the UniAnimate
pipelines run end to end on the CPU."""
import nv_emulation


def window_accumulate(win, skip, sum_, start):
    cs = win.shape[2]
    sum_[:, :, start + skip:start + cs] += win[:, :, skip:]
    return sum_


def window_normalize(sum_, count, out):
    out.copy_(sum_ / count.to(sum_.dtype).view(1, 1, -1, 1, 1))
    return out


def install(monkeypatch=None):
    from diffsynth import _native as nv
    nv_emulation.install(monkeypatch)
    put = (lambda n, v: monkeypatch.setattr(nv, n, v)) if monkeypatch is not None else (lambda n, v: setattr(nv, n, v))
    put("window_accumulate", window_accumulate)
    put("window_normalize", window_normalize)
