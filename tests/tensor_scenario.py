"""Tensor ingest (b2v_submit_tensor) through the two-sided driver of tests/scenario.py.

The direction matters: F / 255 in bf16 does not quantise back to F.  So the *tensor* is built first (from the scenario's BGRA
frame: F / 255 in the target dtype, plus noise of the dtype's size where wanted), quantised with the numpy statement of the
rule in DESIGN.md §3, and that quantised BGRA frame is what the oracle encodes; the GPU side is handed the tensor.  `run`
rewrites the picture events accordingly; the driver itself is untouched."""
from __future__ import annotations

import dataclasses
from dataclasses import dataclass, field

import numpy as np

from tests import scenario
from tests.device_scenario import CHANNELS, gpu_side

DTYPES = ["u8", "f16", "bf16", "f32"]


def torch_dtype(name: str):
    import torch
    return {"u8": torch.uint8, "f16": torch.float16, "bf16": torch.bfloat16, "f32": torch.float32}[name]


def quantise(x32: np.ndarray) -> np.ndarray:
    """The rule, in numpy: fp32 elements -> 8-bit samples."""
    assert x32.dtype == np.float32
    with np.errstate(invalid="ignore"):
        return np.rint(np.nan_to_num(np.clip(x32, 0, 1), nan=0) * np.float32(255)).astype(np.uint8)


def host_tensor(bgra: np.ndarray, dtype: str, channels: str = "RGB", noise_seed=None):
    """`bgra` as a CPU torch tensor (H, W, C) of `dtype` with its channels in the order `channels`, and the BGRA frame that
    tensor quantises to.  Floats hold F / 255 rounded to the dtype, with `noise_seed` plus uniform noise of up to +-0.6 / 255 (so
    that roundings land on both sides and values leave [0, 1] at the ends).  A fourth channel holds junk that must not matter."""
    import torch
    px = np.ascontiguousarray(bgra[..., CHANNELS[channels]])
    if len(channels) == 4:
        px[..., 3] = np.random.default_rng(5).integers(0, 256, px.shape[:2], dtype=np.uint8)
    if dtype == "u8":
        return torch.from_numpy(px), bgra
    x = px.astype(np.float32) / np.float32(255)
    if noise_seed is not None:
        x += np.random.default_rng(noise_seed).uniform(-0.6 / 255, 0.6 / 255, x.shape).astype(np.float32)
    t = torch.from_numpy(x).to(torch_dtype(dtype))
    q = quantise(t.float().numpy())
    out = np.empty(bgra.shape, np.uint8)
    out[..., 3] = 255
    out[..., CHANNELS[channels][:3]] = q[..., :3]
    return t, out


def device_tensor(hwc, form: str = "CHW", margin=(0, 0), device: int = 0):
    """The (H, W, C) CPU tensor on cuda:`device` at (x, y) = margin inside a larger surface, laid out as `form` says, and the
    `layout` keyword that describes the result to submit_tensor:
      "CHW"   planar, contiguous            "HWC"   interleaved, contiguous
      "NHWC"  picture 0 of a (1, C, H, W) channels_last batch: a (C, H, W) view whose channel stride is one element"""
    import torch
    h, w, c = hwc.shape
    mx, my = margin
    fill = 0x5A if hwc.dtype == torch.uint8 else 0.35
    dev = f"cuda:{device}"
    if form == "HWC":
        t = torch.full((h + 2 * my, w + 2 * mx, c), fill, dtype=hwc.dtype, device=dev)
        t[my:my + h, mx:mx + w] = hwc.to(dev)
        return t, "HWC"
    if form == "NHWC":
        t = torch.full((1, c, h + 2 * my, w + 2 * mx), fill, dtype=hwc.dtype, device=dev).contiguous(memory_format=torch.channels_last)[0]
    else:
        t = torch.full((c, h + 2 * my, w + 2 * mx), fill, dtype=hwc.dtype, device=dev)
    t[:, my:my + h, mx:mx + w] = hwc.to(dev).permute(2, 0, 1)
    return t, "CHW"


@dataclass
class TensorConfig(scenario.Config):
    dtype: str = "f16"
    channels: str = "RGB"
    form: str = "CHW"                  # device_tensor's `form`
    margin: tuple = (0, 0)
    noise: bool = True
    tensors: dict = field(default_factory=dict, repr=False, compare=False)    # id(quantised frame) -> (CPU tensor, frame)


class TensorGpuSide(scenario.GpuSide):
    def __init__(self, cfg: TensorConfig, device: int = 0):
        super().__init__(dataclasses.replace(cfg, entry="ring"), device)     # the session; pictures take the tensor path below
        self.cfg, self.device = cfg, device

    def tensor(self, frame):
        if id(frame) not in self.uploaded:       # held with the frame, so that its id stays unique; a resize clears it
            self.uploaded[id(frame)] = (device_tensor(self.cfg.tensors[id(frame)][0], self.cfg.form, self.cfg.margin, self.device), frame)
        return self.uploaded[id(frame)][0]

    def picture(self, frame):
        t, layout = self.tensor(frame)
        self.s.submit_tensor(t, channels=self.cfg.channels, layout=layout, origin=self.cfg.margin)


def tensorise(cfg: TensorConfig, events) -> list:
    """The events with every picture's frame replaced by the frame its tensor quantises to; the tensors go into cfg.tensors."""
    done, out = {}, []
    for ev in events:
        if ev[0] == "picture":
            f = ev[1]
            if id(f) not in done:
                t, q = host_tensor(f, cfg.dtype, cfg.channels, len(done) if cfg.noise else None)
                done[id(f)] = (q, f)
                cfg.tensors[id(q)] = (t, q)
            ev = scenario.picture(done[id(f)][0])
        out.append(ev)
    return out


def run(cfg: TensorConfig, events, cls=TensorGpuSide, **kw) -> list:
    """scenario.run with tensor submits on the GPU side."""
    with gpu_side(cls):
        return scenario.run(cfg, tensorise(cfg, events), **kw)
