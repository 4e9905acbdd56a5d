"""Host-side mirror of models/seed_qformer/qformer_quantizer.py (Blip2QformerQuantizer) on top of libseedb200.

Same public surface as the reference class on the inference path -- `from_pretrained`,
`get_codebook_indices(image) -> (embed_ind, query_output_up)`, `get_codebook_entry(indices)`, `n_embed`,
`codebook_embed_dim`, `.eval()/.half()/.to()` -- but every forward runs as hand-written sm_90a kernels behind
the C ABI (include/seedb200.h).  There is no eager-PyTorch path: without a CUDA device or without the built
library the constructor raises.
"""
from __future__ import annotations

import re
from typing import Dict, Optional, Tuple

import torch
import torch.nn as nn

from . import lib as L

# state-dict prefixes of the reference model that the inference path never reads
# (recon_s branch `pos_embed`/`blocks.*`, BERT text branch, LM head): qformer_quantizer.py:206-211,238-250
_UNUSED_PREFIXES = ("blocks.", "Qformer.cls", "Qformer.bert.embeddings.word_embeddings",
                    "Qformer.bert.embeddings.position_embeddings", "Qformer.bert.embeddings.position_ids")
_UNUSED_KEYS = ("pos_embed",)
_UNUSED_RE = re.compile(r"^Qformer\.bert\.encoder\.layer\.\d+\.(intermediate|output)\.")


def _depth(sd: Dict[str, torch.Tensor], pattern: str) -> int:
    rx = re.compile(pattern)
    idx = [int(m.group(1)) for k in sd for m in [rx.match(k)] if m]
    return max(idx) + 1 if idx else 0


class _DeviceStub(nn.Module):
    """Stands in for `model.visual_encoder` / `model.ln_vision`: callers only move them between devices
    (gradio_demo/seed_llama_flask.py:72).  The weights live inside the seedb200 handle."""

    num_features = 1408

    def forward(self, *a, **k):  # pragma: no cover
        raise RuntimeError("the ViT runs inside libseedb200; call get_codebook_indices()")


class Blip2QformerQuantizer(nn.Module):
    def __init__(self, state_dict: Dict[str, torch.Tensor], device="cuda", max_batch: int = 256,
                 vq_mode: int = L.VQ_FP16, gemm_ctas: int = 0, vit_precision: str = "fp16", **_ignored):
        super().__init__()
        if vit_precision != "fp16":
            raise ValueError("seed_b200 implements the reference's fp16 mode (configs/tokenizer/*.yaml `fp16: True`); "
                             "fp32 operands are not supported on this path")
        dev = torch.device(device)
        if dev.type != "cuda" or not torch.cuda.is_available():
            raise RuntimeError("Blip2QformerQuantizer (seed_b200) needs a CUDA device: there is no CPU path")
        used = {k: v for k, v in state_dict.items()
                if k not in _UNUSED_KEYS and not k.startswith(_UNUSED_PREFIXES) and not _UNUSED_RE.match(k)}
        self.vit_depth = _depth(used, r"visual_encoder\.blocks\.(\d+)\.")
        self.qformer_layers = _depth(used, r"Qformer\.bert\.encoder\.layer\.(\d+)\.")
        self.detok_depth = _depth(used, r"blocks_image\.(\d+)\.")
        cb = used["quantize.embedding.weight"]
        self.n_embed, self.codebook_embed_dim = int(cb.shape[0]), int(cb.shape[1])
        self.image_features_dim = 1024
        weights = {k: v.detach().to(device=dev, dtype=torch.float16).contiguous() for k, v in used.items()}
        self._enc = L.Encoder(weights, vit_depth=self.vit_depth, qformer_layers=self.qformer_layers,
                              detok_depth=self.detok_depth, n_codes=self.n_embed, max_batch=max_batch,
                              vq_mode=vq_mode, gemm_ctas=gemm_ctas)
        self._device = dev
        self.visual_encoder = _DeviceStub()
        self.ln_vision = _DeviceStub()

    # ---- reference API -----------------------------------------------------------------------
    @classmethod
    def from_pretrained(cls, pretrained_model_path, **kwargs):
        """qformer_quantizer.py:340-375: torch.load(seed_quantizer.pt) -> model (strict=False semantics: unknown
        keys are ignored, missing hot-path keys are an error raised by the C side)."""
        if str(pretrained_model_path).startswith("http"):
            raise RuntimeError("no network access: download seed_quantizer.pt and pass a local path")
        ckpt = torch.load(pretrained_model_path, map_location="cpu")
        if isinstance(ckpt, dict) and "model" in ckpt and isinstance(ckpt["model"], dict):
            ckpt = ckpt["model"]
        return cls(ckpt, **kwargs)

    @property
    def device(self):
        return self._device

    def get_codebook_indices(self, image: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        """qformer_quantizer.py:288-307: image [B,3,224,224] -> (embed_ind [B,32] int64, query_output_up [B,32,768])."""
        image = self._check_image(image)
        ids, _, qup = self._enc.encode(image, return_query_up=True)
        return ids, qup

    def encode_ids(self, image: torch.Tensor, return_z: bool = False):
        """get_codebook_indices without the (discarded) decode_task_layer branch -- what ImageTokenizer.encode uses."""
        image = self._check_image(image)
        ids, z, _ = self._enc.encode(image, return_z=return_z)
        return (ids, z) if return_z else ids

    def encode_tokens(self, image: torch.Tensor, image_id_shift: int, boi: int, eoi: int, out=None):
        """encode_ids fused with `<img>` + (shift + id) x 32 + `</img>` (seedb200_encoder_encode_tokens): [B,34] int64."""
        image = self._check_image(image)
        return self._enc.encode_tokens(image, image_id_shift, boi, eoi, out=out)

    def get_codebook_entry(self, indices: torch.Tensor) -> torch.Tensor:
        """qformer_quantizer.py:309-338: ids [B,32] -> image embeds [B,1024] (input of the unCLIP decoder)."""
        if self.detok_depth == 0:
            raise RuntimeError("checkpoint has no blocks_image.* weights: de-tokenizer head unavailable")
        idx = indices.to(device=self._device, dtype=torch.int64)
        if idx.numel() % 32 != 0:
            raise ValueError(f"expected 32 ids per image, got shape {tuple(indices.shape)}")
        if idx.numel() and (int(idx.min()) < 0 or int(idx.max()) >= self.n_embed):
            raise IndexError("index out of range in self")   # what F.embedding raises in the reference
        return self._enc.detokenize(idx)

    def _check_image(self, image: torch.Tensor) -> torch.Tensor:
        if image.dim() != 4 or tuple(image.shape[1:]) != (3, 224, 224):
            # PatchEmbed.forward asserts the size (eva_vit.py:226-228)
            raise AssertionError(f"Input image size ({tuple(image.shape)}) doesn't match model (B*3*224*224).")
        return image.to(device=self._device, dtype=torch.float16).contiguous()

    # nn.Module conveniences the reference callers use; parameters live in the C handle
    def half(self):
        return self

    def float(self):
        raise ValueError("seed_b200 implements the fp16 mode only")

    def to(self, *args, **kwargs):
        tgt = kwargs.get("device", args[0] if args else None)
        if tgt is not None and not isinstance(tgt, torch.dtype) and torch.device(tgt).type != "cuda":
            raise RuntimeError("seed_b200 tokenizer weights cannot be moved off the GPU")
        return self

    def eval(self):
        return self

    def taps(self, B: int):
        """parity taps of the last encode call: ViT output, ln_vision output, Q-Former output (fp16)."""
        return {"vit": self._enc.tap(0, B).view(B, 257, 1408), "image_embeds": self._enc.tap(2, B).view(B, 257, 1408),
                "qformer": self._enc.tap(1, B).view(B, 32, 768)}
