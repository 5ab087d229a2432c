"""`Sam` / `SamPredictor` duck types backed by libmsam_b200.so (include/msam_b200.h).

micro-sam never touches SAM internals except through the predictor object that `util.get_sam_model` returns
(reference: micro_sam/util.py:460-476; attribute census in SURVEY.md 8b).  `B200SamPredictor` offers exactly that
surface -- `set_image`, `set_torch_image`, `predict`, `predict_torch`, `get_image_embedding`, `reset_image`, the mutable
`features / original_size / input_size / is_image_set` attributes, `transform`, `device`, `model` -- while every FLOP
runs in the hand-written sm_90a kernels.  There is no PyTorch fallback: without the library / an H100 it raises.
"""
from __future__ import annotations

import ctypes
import types
from typing import Dict, Optional, Tuple

import numpy as np
import torch

from . import _lib

# micro_sam/models/build_sam.py:40-76
ARCH = {
    "vit_b": dict(embed_dim=768, depth=12, num_heads=12, global_attn_indexes=(2, 5, 8, 11)),
    "vit_l": dict(embed_dim=1024, depth=24, num_heads=16, global_attn_indexes=(5, 11, 17, 23)),
    "vit_h": dict(embed_dim=1280, depth=32, num_heads=16, global_attn_indexes=(7, 15, 23, 31)),
    # MobileSAM (micro_sam/util.py:35-43,436-441): TinyViT encoder, fixed architecture (csrc/tinyvit.cu); depth 0 selects it
    "vit_t": dict(embed_dim=320, depth=0, num_heads=10, global_attn_indexes=()),
    # tiny shapes for tests only
    "vit_test": dict(embed_dim=128, depth=2, num_heads=2, global_attn_indexes=(1,)),
    "vit_test80": dict(embed_dim=160, depth=2, num_heads=2, global_attn_indexes=(1,)),
}
_EMBED_TO_TYPE = {768: "vit_b", 1024: "vit_l", 1280: "vit_h", 128: "vit_test", 160: "vit_test80"}


def validate_model_type(state: Dict[str, torch.Tensor]) -> str:
    """micro_sam/models/build_sam.py:24-37."""
    if "image_encoder.patch_embed.proj.weight" in state:
        return _EMBED_TO_TYPE[state["image_encoder.patch_embed.proj.weight"].shape[0]]
    return "vit_t"


def get_preprocess_shape(oldh: int, oldw: int, long_side: int) -> Tuple[int, int]:
    scale = long_side * 1.0 / max(oldh, oldw)
    return int(oldh * scale + 0.5), int(oldw * scale + 0.5)


class ResizeLongestSide:
    """segment_anything.utils.transforms.ResizeLongestSide (host side; used at util.py:663, inference.py:227-233)."""

    def __init__(self, target_length: int):
        self.target_length = target_length

    def apply_image(self, image: np.ndarray) -> np.ndarray:
        th, tw = get_preprocess_shape(image.shape[0], image.shape[1], self.target_length)
        if (th, tw) == tuple(image.shape[:2]):
            return np.ascontiguousarray(image)
        from PIL import Image  # same PIL bilinear(+antialias) uint8 resize the reference reaches via torchvision
        if image.ndim == 3 and image.shape[2] == 3 and image.dtype == np.uint8 and \
                np.array_equal(image[..., 0], image[..., 1]) and np.array_equal(image[..., 0], image[..., 2]):
            # gray image replicated to RGB by _to_image (the usual microscopy input): PIL resamples the bands independently with the
            # same coefficients, so one band is resized and replicated -- bit-identical, a third of the work (host-bound e2e paths)
            band = np.asarray(Image.fromarray(np.ascontiguousarray(image[..., 0])).resize((tw, th), Image.BILINEAR))
            return np.stack([band, band, band], axis=2)      # (measured: 1 ms; a broadcast assignment takes 5 ms)
        return np.array(Image.fromarray(image).resize((tw, th), Image.BILINEAR))

    def apply_image_torch(self, image: torch.Tensor) -> torch.Tensor:
        """(B, C, H, W) float tensor -> longest side `target_length` (bilinear, antialiased), the torch twin used by
        training/trainable_sam.py:36 and prompt_based_segmentation.py:100."""
        th, tw = get_preprocess_shape(image.shape[2], image.shape[3], self.target_length)
        return torch.nn.functional.interpolate(image, (th, tw), mode="bilinear", align_corners=False, antialias=True)

    def apply_coords(self, coords: np.ndarray, original_size: Tuple[int, ...]) -> np.ndarray:
        old_h, old_w = original_size
        new_h, new_w = get_preprocess_shape(old_h, old_w, self.target_length)
        coords = np.array(coords, dtype=float, copy=True)
        coords[..., 0] = coords[..., 0] * (new_w / old_w)
        coords[..., 1] = coords[..., 1] * (new_h / old_h)
        return coords

    def apply_boxes(self, boxes: np.ndarray, original_size: Tuple[int, ...]) -> np.ndarray:
        return self.apply_coords(np.asarray(boxes).reshape(-1, 2, 2), original_size).reshape(-1, 4)

    def apply_coords_torch(self, coords: torch.Tensor, original_size) -> torch.Tensor:
        old_h, old_w = original_size
        new_h, new_w = get_preprocess_shape(old_h, old_w, self.target_length)
        coords = coords.clone().to(torch.float)
        coords[..., 0] = coords[..., 0] * (new_w / old_w)
        coords[..., 1] = coords[..., 1] * (new_h / old_h)
        return coords

    def apply_boxes_torch(self, boxes: torch.Tensor, original_size) -> torch.Tensor:
        return self.apply_coords_torch(boxes.reshape(-1, 2, 2), original_size).reshape(-1, 4)


class _EncoderFn(torch.autograd.Function):
    """image_encoder with a backward pass (cfg 5): forward = msam_encode_train (keeps the activations in the engine), backward =
    msam_encode_backward, which fills the engine's per-parameter gradients (read them with `B200Sam.encoder_grads()`); the image
    itself gets no gradient (trainable_sam.py never asks for one)."""

    @staticmethod
    def forward(ctx, x, anchor, sam):
        x = x.to(device=sam.device, dtype=torch.float32).contiguous()
        out = torch.empty(x.shape[0], 256, 64, 64, device=sam.device, dtype=torch.float32)
        _lib.check(_lib.lib().msam_encode_train(sam._h, _lib.ptr(x), x.shape[0], _lib.ptr(out), _lib.cur_stream()))
        ctx.sam = sam
        return out

    @staticmethod
    def backward(ctx, grad_out):
        g = grad_out.to(torch.float32).contiguous()
        _lib.check(_lib.lib().msam_encode_backward(ctx.sam._h, _lib.ptr(g), _lib.cur_stream()))
        ctx.sam._encoder_grads_valid = True
        return None, torch.zeros((), device=g.device), None


def prompt_table_index(point_labels: Optional[torch.Tensor], has_boxes: bool, n_prompts: int) -> torch.Tensor:
    """Which learned embedding sits behind each sparse prompt token (PromptEncoder._embed_points / _embed_boxes): label 0 / 1 ->
    point_embeddings[0 / 1], label -1 -> not_a_point_embed (index 4; a padding point with label -1 is appended when no box is given),
    box corners -> point_embeddings[2], [3].  (n_prompts, n_sparse) int64 -- the gradient routing table of the training decoder."""
    idx = []
    if point_labels is not None:
        lab = torch.as_tensor(point_labels).round().to(torch.int64).reshape(n_prompts, -1)
        if not has_boxes:
            lab = torch.cat([lab, torch.full((n_prompts, 1), -1, dtype=torch.int64, device=lab.device)], dim=1)
        idx.append(torch.where(lab < 0, torch.full_like(lab, 4), lab.clamp(max=1)))
    if has_boxes:
        dev = idx[0].device if idx else "cpu"
        idx.append(torch.tensor([[2, 3]], dtype=torch.int64, device=dev).expand(n_prompts, 2))
    if not idx:
        raise ValueError("training needs point and / or box prompts")
    return torch.cat(idx, dim=1)


class _DevBuf:
    """Exposes a raw device allocation through __cuda_array_interface__ so that torch can wrap it without a copy."""

    def __init__(self, ptr: int, n: int):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<f4", "data": (ptr, False), "version": 2}


def _device_view(ptr: int, n: int, device) -> torch.Tensor:
    return torch.as_tensor(_DevBuf(ptr, n), device=device)


class _DecoderFn(torch.autograd.Function):
    """prompt encoder + mask decoder of ONE image with a backward pass (csrc/decoder_train.cu): (embedding [256,64,64], sparse prompt
    embeddings [P,Ts,256], mask prompts [P,1,256,256] or None) -> (low-res logits [P,M,256,256], IoU predictions [P,M]).  backward
    fills / accumulates the decoder and prompt-encoder parameter gradients inside the engine (`B200Sam.decoder_grads()`) and returns
    dL/d embedding (the mask prompts get no gradient)."""

    @staticmethod
    def forward(ctx, emb, sparse, emb_index, sam, slot, multimask, masks):
        emb = emb.to(device=sam.device, dtype=torch.float32).contiguous()
        sparse = sparse.to(device=sam.device, dtype=torch.float32).contiguous()
        emb_index = emb_index.to(device=sam.device, dtype=torch.int32).contiguous()
        P, Ts = sparse.shape[:2]
        M = 3 if multimask else 1
        low = torch.empty(P, M, 256, 256, device=sam.device, dtype=torch.float32)
        iou = torch.empty(P, M, device=sam.device, dtype=torch.float32)
        _lib.check(_lib.lib().msam_decoder_train_forward_ex(sam._h, slot, _lib.ptr(emb), _lib.ptr(sparse), _lib.ptr(emb_index), Ts, P,
                                                            _lib.ptr(masks), int(bool(multimask)), _lib.ptr(low), _lib.ptr(iou),
                                                            _lib.cur_stream()))
        ctx.sam, ctx.slot, ctx.masked = sam, slot, masks is not None
        return low, iou

    @staticmethod
    def backward(ctx, d_low, d_iou):
        sam = ctx.sam
        d_low = None if d_low is None else d_low.to(torch.float32).contiguous()
        d_iou = None if d_iou is None else d_iou.to(torch.float32).contiguous()
        d_emb = torch.empty(256, 64, 64, device=sam.device, dtype=torch.float32)
        _lib.check(_lib.lib().msam_decoder_train_backward(sam._h, ctx.slot, _lib.ptr(d_low), _lib.ptr(d_iou), _lib.ptr(d_emb), _lib.cur_stream()))
        sam._decoder_grads_valid = True
        sam._mask_grads_valid = sam._mask_grads_valid or ctx.masked
        return d_emb, None, None, None, None, None, None


class _ImageEncoder:
    """Callable stand-in for `sam.image_encoder`: (B,3,1024,1024) fp32 preprocessed -> (B,256,64,64) fp32."""

    def __init__(self, sam: "B200Sam"):
        self._sam = sam
        self.img_size = sam.image_size

    def __call__(self, x: torch.Tensor) -> torch.Tensor:
        sam = self._sam
        if x.ndim != 4 or x.shape[1] != 3 or x.shape[2] != self.img_size or x.shape[3] != self.img_size:
            raise ValueError(f"image_encoder expects (B,3,{self.img_size},{self.img_size}), got {tuple(x.shape)}")
        if torch.is_grad_enabled() and sam.training:
            if getattr(sam, "_grad_anchor", None) is None:   # a leaf that makes the output part of the autograd graph
                sam._grad_anchor = torch.zeros((), device=sam.device, requires_grad=True)
            return _EncoderFn.apply(x, sam._grad_anchor, sam)
        x = x.to(device=sam.device, dtype=torch.float32).contiguous()
        out = torch.empty(x.shape[0], 256, 64, 64, device=sam.device, dtype=torch.float32)
        _lib.check(_lib.lib().msam_encode_f32(sam._h, _lib.ptr(x), x.shape[0], _lib.ptr(out), _lib.cur_stream()))
        return out


class _PromptEncoder:
    """Callable stand-in for `sam.prompt_encoder` (segment_anything PromptEncoder as used at
    micro_sam/training/trainable_sam.py:88-96): `(points=(coords, labels)|None, boxes=(P,4)|None, masks=(P,1,256,256)|None)`
    -> `(sparse (P, n, 256), dense (P, 256, 64, 64))`, plus `get_dense_pe()`."""
    embed_dim = 256

    def __init__(self, sam: "B200Sam"):
        self._sam = sam
        g = sam.image_size // 16
        self.image_embedding_size = (g, g)
        self.input_image_size = (sam.image_size, sam.image_size)
        self.mask_input_size = (4 * g, 4 * g)
        self._dense_pe = None
        nm = sam._state.get("prompt_encoder.no_mask_embed.weight")
        self._no_mask = None if nm is None else nm.to(sam.device, torch.float32).reshape(1, -1, 1, 1).contiguous()

    def get_dense_pe(self) -> torch.Tensor:
        if self._dense_pe is None:
            sam = self._sam
            g = self.image_embedding_size[0]
            pe = torch.empty(g * g, 256, device=sam.device, dtype=torch.float32)
            _lib.check(_lib.lib().msam_get_dense_pe(sam._h, _lib.ptr(pe), _lib.cur_stream()))
            self._dense_pe = pe.view(g, g, 256).permute(2, 0, 1)[None].contiguous()
        return self._dense_pe

    def is_no_mask_dense(self, dense: torch.Tensor) -> bool:
        """True if `dense` is the broadcast no-mask embedding this object handed out (the decoder's shared fast path)."""
        return (self._no_mask is not None and dense.device == self._no_mask.device
                and dense.untyped_storage().data_ptr() == self._no_mask.untyped_storage().data_ptr()
                and tuple(dense.stride()) == (0, 1, 0, 0))

    @torch.no_grad()
    def __call__(self, points=None, boxes=None, masks=None):
        sam, dev = self._sam, self._sam.device
        pts = lbl = bx = mk = None
        np_, P = 0, None
        if points is not None:
            coords, labels = points
            pts = coords.to(dev, torch.float32).contiguous()
            lbl = labels.to(dev, torch.float32).contiguous()
            P, np_ = pts.shape[0], pts.shape[1]
        if boxes is not None:
            bx = boxes.to(dev, torch.float32).reshape(-1, 4).contiguous()
            P = bx.shape[0]
        if masks is not None:
            mk = masks.to(dev, torch.float32).reshape(-1, *self.mask_input_size).contiguous()
            P = mk.shape[0] if P is None else P
        if P is None:
            P = 1   # PromptEncoder._get_batch_size
        n_sparse = (np_ + (0 if bx is not None else 1) if pts is not None else 0) + (2 if bx is not None else 0)
        sparse = torch.empty(P, n_sparse, 256, device=dev, dtype=torch.float32)
        g = self.image_embedding_size[0]
        dense = torch.empty(P, 256, g, g, device=dev, dtype=torch.float32) if mk is not None else None
        if n_sparse > 0 or mk is not None:
            _lib.check(_lib.lib().msam_prompt_encode(sam._h, _lib.ptr(pts), _lib.ptr(lbl), np_, _lib.ptr(bx), _lib.ptr(mk), P,
                                                     _lib.ptr(sparse) if n_sparse > 0 else None, _lib.ptr(dense),
                                                     _lib.cur_stream()))
        if dense is None:
            dense = self._no_mask.expand(P, -1, g, g)
        return sparse, dense

    forward = __call__


class _MaskDecoder:
    """Callable stand-in for `sam.mask_decoder` (kwargs as at micro_sam/training/trainable_sam.py:98-104)."""
    num_mask_tokens = 4
    num_multimask_outputs = 3
    transformer_dim = 256

    def __init__(self, sam: "B200Sam"):
        self._sam = sam

    @torch.no_grad()
    def __call__(self, image_embeddings: torch.Tensor, image_pe: torch.Tensor, sparse_prompt_embeddings: torch.Tensor,
                 dense_prompt_embeddings: torch.Tensor, multimask_output: bool):
        sam, dev = self._sam, self._sam.device
        if image_embeddings.numel() != 256 * 64 * 64:
            raise ValueError(f"mask_decoder expects ONE image embedding (1,256,64,64), got {tuple(image_embeddings.shape)}")
        if image_pe is not None and tuple(image_pe.shape[-3:]) != (256, 64, 64):
            raise ValueError(f"image_pe must have shape (1,256,64,64), got {tuple(image_pe.shape)}")
        sam.bind_embedding(image_embeddings)
        sp = sparse_prompt_embeddings.to(dev, torch.float32).contiguous()
        P, n_sparse = sp.shape[0], sp.shape[1]
        dn = dense_prompt_embeddings
        if sam.prompt_encoder.is_no_mask_dense(dn):
            dn = None
        else:
            dn = dn.to(dev, torch.float32).expand(P, -1, -1, -1).contiguous()
        M = 3 if multimask_output else 1
        low = torch.empty(P, M, 256, 256, device=dev, dtype=torch.float32)
        iou = torch.empty(P, M, device=dev, dtype=torch.float32)
        _lib.check(_lib.lib().msam_mask_decode(sam._h, _lib.ptr(sp) if n_sparse > 0 else None, n_sparse, _lib.ptr(dn), P,
                                               int(multimask_output), _lib.ptr(low), _lib.ptr(iou), _lib.cur_stream()))
        return low, iou

    forward = __call__


class B200Sam:
    """The model object (`predictor.model`).  Holds the upstream-keyed state dict (CPU) and the device engine."""

    mask_threshold: float = 0.0
    image_format: str = "RGB"

    def __init__(self, model_type: str, state_dict: Dict[str, torch.Tensor], device="cuda", max_batch: int = 16,
                 max_prompts: int = 256, image_size: int = 1024):
        if model_type not in ARCH:
            raise ValueError(f"unsupported model type {model_type!r} (have {sorted(ARCH)})")
        dev = torch.device(device)
        if dev.type != "cuda":
            raise RuntimeError(f"micro_sam_b200 runs on a CUDA (sm_90a) device only; got device={device!r}")
        if not torch.cuda.is_available():
            raise RuntimeError("micro_sam_b200: no CUDA device available and there is no CPU fallback")
        self.model_type = model_type
        self.image_size = image_size
        self.device = torch.device("cuda", dev.index if dev.index is not None else torch.cuda.current_device())
        a = ARCH[model_type]
        L = _lib.lib()
        ga = list(a["global_attn_indexes"]) + [-1] * (8 - len(a["global_attn_indexes"]))
        cfg = _lib.MsamConfig(a["embed_dim"], a["depth"], a["num_heads"], (ctypes.c_int32 * 8)(*ga), 14, image_size, 16,
                              256, max_batch, max_prompts)
        self._cfg = cfg
        self._h = None
        self._build_engine(state_dict)
        self.pixel_mean = torch.tensor([123.675, 116.28, 103.53], device=self.device).view(-1, 1, 1)
        self.pixel_std = torch.tensor([58.395, 57.12, 57.375], device=self.device).view(-1, 1, 1)

    def _build_engine(self, state_dict) -> None:
        """(Re)create the device engine from an upstream-keyed state dict: weights are packed (bf16 GEMM operands, fused /
        transposed layouts) at load time, so `load_state_dict` rebuilds the engine rather than patching buffers."""
        L = _lib.lib()
        if self._h:
            L.msam_destroy(self._h)
        self._h = ctypes.c_void_p()
        self._bound_key = self._bound_src = self._bound_tensor = None
        self._encoder_grads_valid = self._decoder_grads_valid = False   # a rebuilt engine has no training state yet
        self._mask_grads_valid = False   # mask_downscaling joins the trained tensors with the first masked backward
        with torch.cuda.device(self.device):
            _lib.check(L.msam_create(ctypes.byref(self._cfg), self.device.index, ctypes.byref(self._h)))
            self._state = {}
            for k, v in state_dict.items():
                v = v.detach().to("cpu", torch.float32).contiguous()
                self._state[k] = v
                shape = (ctypes.c_int64 * max(v.ndim, 1))(*v.shape)
                _lib.check(L.msam_load_weight(self._h, k.encode(), ctypes.c_void_p(v.data_ptr()), shape, v.ndim))
            _lib.check(L.msam_finalize_weights(self._h))
        self.image_encoder = _ImageEncoder(self)
        self.prompt_encoder = _PromptEncoder(self)
        self.mask_decoder = _MaskDecoder(self)

    # --- nn.Module-ish surface used by micro-sam (util.py:457-458, training/util.py:131, trainable_sam.py:40-106)
    def state_dict(self):
        return dict(self._state)

    def load_state_dict(self, state_dict, strict: bool = True):
        missing = [k for k in self._state if k not in state_dict]
        unexpected = [k for k in state_dict if k not in self._state]
        if strict and (missing or unexpected):
            raise RuntimeError(f"Error(s) in loading state_dict: missing {missing[:4]}..., unexpected {unexpected[:4]}...")
        merged = dict(self._state)
        merged.update({k: v for k, v in state_dict.items() if k in self._state})
        self._build_engine(merged)
        return missing, unexpected

    def named_parameters(self):
        """Host copies of the weights under their upstream names (frozen: the H100 core is an inference engine; the training
        surface of cfg 5 is documented in DESIGN.md)."""
        for k, v in self._state.items():
            yield k, torch.nn.Parameter(v, requires_grad=False)

    def parameters(self):
        for _, p in self.named_parameters():
            yield p

    training = False

    def eval(self):
        self.training = False
        return self

    def train(self, mode: bool = True):
        """Training mode switches `image_encoder(x)` (under grad mode) to the activation-keeping forward with a backward pass
        (csrc/encoder_train.cu); the prompt encoder / mask decoder are differentiated through `decoder_train`."""
        if mode and self.model_type == "vit_t":
            raise NotImplementedError("the TinyViT encoder has no backward pass")
        self.training = bool(mode)
        return self

    def decoder_train(self, emb: torch.Tensor, points, boxes, multimask_output: bool, slot: int = 0, masks=None):
        """mask_decoder(prompt_encoder(points, boxes, masks)) for ONE image in training mode: differentiable w.r.t. `emb` (256,64,64)
        and the decoder / prompt-encoder parameters.  points = (coords (P,n,2), labels (P,n)) in the 1024 frame or None; boxes (P,4)
        or None; masks = (P,1,256,256) low-res logits used as mask prompts, or None.  The masks get no gradient, so a `masks` tensor
        that requires grad is refused."""
        if not self.training:
            raise RuntimeError("decoder_train needs train() mode")
        if masks is not None:
            if masks.requires_grad:
                raise ValueError("decoder_train: masks must not require grad (no gradient w.r.t. the mask prompts is computed)")
            masks = masks.detach().to(self.device, torch.float32).contiguous()
        with torch.no_grad():
            sparse, _ = self.prompt_encoder(points=points, boxes=boxes, masks=None)
        P = sparse.shape[0]
        if masks is not None and tuple(masks.shape) != (P, 1, 256, 256):
            raise ValueError(f"decoder_train: masks must have shape ({P}, 1, 256, 256), got {tuple(masks.shape)}")
        emb_index = prompt_table_index(None if points is None else points[1], boxes is not None, P).to(self.device)
        assert emb_index.shape == sparse.shape[:2], (emb_index.shape, sparse.shape)
        return _DecoderFn.apply(emb, sparse, emb_index, self, int(slot), bool(multimask_output), masks)

    def decode_with_training_decoder(self, emb: torch.Tensor, points, boxes, multimask_output: bool, slot: int = 0, masks=None):
        """Forward pass only of `decoder_train` (no autograd record, any mode): the inference decoder takes at most 16 tokens per
        prompt, the training decoder up to 64, so prompts with more tokens (e.g. the later passes of iterative prompting) are decoded
        here.  Uses decoder slot `slot` like `decoder_train` (a pending backward pass of that slot is lost)."""
        with torch.no_grad():
            if masks is not None:
                masks = masks.detach().to(self.device, torch.float32).contiguous()
            sparse, _ = self.prompt_encoder(points=points, boxes=boxes, masks=None)
            emb_index = prompt_table_index(None if points is None else points[1], boxes is not None, sparse.shape[0]).to(self.device)
            return _DecoderFn.forward(types.SimpleNamespace(), emb.detach(), sparse, emb_index, self, int(slot), bool(multimask_output), masks)

    def zero_decoder_grads(self) -> None:
        _lib.check(_lib.lib().msam_decoder_zero_grads(self._h, _lib.cur_stream()))
        self._decoder_zeroings = getattr(self, "_decoder_zeroings", 0) + 1

    def decoder_grads(self) -> Dict[str, torch.Tensor]:
        """fp32 gradients of the mask-decoder / prompt-encoder parameters accumulated since `zero_decoder_grads()`, keyed and shaped
        like the upstream state dict.  The PE matrix is absent (it is not trained); mask_downscaling is present once a backward pass
        with mask prompts has run."""
        if not getattr(self, "_decoder_grads_valid", False):
            raise RuntimeError("no decoder gradients: run decoder_train(...) and backward() first")
        return self._decoder_tensors(_lib.lib().msam_decoder_grad)

    def _decoder_tensors(self, getter, params: bool = False) -> Dict[str, torch.Tensor]:
        """Decoder / prompt-encoder tensors (gradients or master weights) from the engine's packed layouts to upstream keys / shapes."""
        def fetch(name, n):
            g = torch.empty(n, device=self.device, dtype=torch.float32)
            _lib.check(getter(self._h, name.encode(), _lib.ptr(g), n, _lib.cur_stream()))
            return g
        out = {}
        for k, v in self._state.items():
            if not (k.startswith("mask_decoder.") or k.startswith("prompt_encoder.")):
                continue
            if k.endswith("positional_encoding_gaussian_matrix") or ("mask_downscaling" in k and not self._mask_grads_valid):
                continue
            if "output_upscaling.0" in k or "output_upscaling.3" in k:       # ConvTranspose2d [ci, co, 2, 2] <- GEMM layout [(dy,dx,co), ci]
                ci, co = self._state[k.rsplit(".", 1)[0] + ".weight"].shape[:2]
                if k.endswith(".weight"):
                    out[k] = fetch(k + "@gemm", 4 * co * ci).view(2, 2, co, ci).permute(3, 2, 0, 1).contiguous()
                else:
                    t4 = fetch(k + "@gemm", 4 * co).view(4, co)      # the bias is kept as 4 identical tiles, its gradient as 4 partial sums
                    out[k] = t4[0].clone() if params else t4.sum(0)
            elif "point_embeddings" in k:
                i = int(k.split(".")[2])
                out[k] = fetch("prompt_encoder.point_embeddings@stack", 4 * 256).view(4, 1, 256)[i]
            elif k == "mask_decoder.iou_token.weight":
                out[k] = fetch("mask_decoder.output_tokens@stack", 5 * 256).view(5, 256)[:1]
            elif k == "mask_decoder.mask_tokens.weight":
                out[k] = fetch("mask_decoder.output_tokens@stack", 5 * 256).view(5, 256)[1:]
            elif k.startswith("mask_decoder.iou_prediction_head.layers.2."):   # 4 outputs padded to 32 GEMM columns
                out[k] = (fetch(k, 32 * 256).view(32, 256)[:4] if k.endswith(".weight") else fetch(k, 32)[:4]).contiguous()
            else:
                out[k] = fetch(k, v.numel()).view(v.shape)
        return out

    def grad_views(self):
        """Zero-copy torch views of the engine's fp32 gradient buffers [(key, tensor)] (keys as in the C API: a few carry packed
        layouts, `@gemm` / `@stack`).  In-place operations on them (all-reduce, clipping, scaling) are seen by `optimizer_step()`."""
        L = _lib.lib()
        n = L.msam_train_tensor_count(self._h)
        out = []
        buf = ctypes.create_string_buffer(256)
        for i in range(max(n, 0)):
            g, w, cnt = ctypes.c_void_p(), ctypes.c_void_p(), ctypes.c_int64()
            _lib.check(L.msam_train_tensor_info(self._h, i, buf, 256, ctypes.byref(g), ctypes.byref(w), ctypes.byref(cnt)))
            out.append((buf.value.decode(), _device_view(g.value, cnt.value, self.device)))
        return out

    def allreduce_grads(self, world_size: int) -> int:
        """DDP semantics (micro_sam/training/training.py:train_sam): average every gradient over the ranks with ONE all-reduce of a
        flat fp32 buffer, written back into the engine's gradient buffers.  Returns the number of gradient elements."""
        from .distributed import allreduce_average_
        return allreduce_average_([v for _, v in self.grad_views()])

    def optimizer_step(self, lr: float = 1e-5, betas=(0.9, 0.999), eps: float = 1e-8, weight_decay: float = 0.01) -> None:
        """One AdamW update (torch.optim.AdamW semantics, the reference trainer's default) of every tensor that has gradients, on the
        device (csrc/train_opt.cu): fp32 master weights + moments, then the operands of the training paths are refreshed.  The fused
        inference decoder keeps its old operands until `load_state_dict(self.trained_state_dict())`."""
        _lib.check(_lib.lib().msam_optimizer_step(self._h, lr, betas[0], betas[1], eps, weight_decay, _lib.cur_stream()))

    def trained_state_dict(self) -> Dict[str, torch.Tensor]:
        """Upstream-keyed state dict with the fp32 master weights of the optimizer (CPU tensors); untouched tensors as loaded."""
        L = _lib.lib()
        out = dict(self._state)
        if getattr(self, "_decoder_grads_valid", False):
            out.update({k: v.cpu() for k, v in self._decoder_tensors(L.msam_train_param, params=True).items()})
        if getattr(self, "_encoder_grads_valid", False):
            for k, v in self._state.items():
                if k.startswith("image_encoder."):
                    g = torch.empty(v.shape, device=self.device, dtype=torch.float32)
                    _lib.check(L.msam_train_param(self._h, k.encode(), _lib.ptr(g), g.numel(), _lib.cur_stream()))
                    out[k] = g.cpu()
        return out

    def encoder_grads(self, names=None) -> Dict[str, torch.Tensor]:
        """fp32 gradients of the image-encoder parameters after a backward pass, keyed and shaped like the upstream state dict."""
        if not getattr(self, "_encoder_grads_valid", False):
            raise RuntimeError("no encoder gradients: run image_encoder(x) in train() mode and call backward() first")
        out = {}
        L = _lib.lib()
        for k, v in self._state.items():
            if not k.startswith("image_encoder.") or (names is not None and k not in names):
                continue
            g = torch.empty(v.shape, device=self.device, dtype=torch.float32)
            _lib.check(L.msam_encoder_grad(self._h, k.encode(), _lib.ptr(g), g.numel(), _lib.cur_stream()))
            out[k] = g
        return out

    def bind_embedding(self, f: torch.Tensor) -> None:
        """Bind a (1,256,64,64) image embedding as the decoder's current image (SamPredictor.features assignment).  The
        engine caches prompt-independent decoder state per bound embedding; the cache key lives HERE, with the engine it
        describes, so that several predictors sharing one model cannot decode against each other's image."""
        key = (f.data_ptr(), f._version, tuple(f.shape), str(f.device), f.dtype)
        if self._bound_key == key and self._bound_src is f:
            return
        feat = f.detach().to(self.device, torch.float32).contiguous()
        if feat.numel() != 256 * 64 * 64:
            raise ValueError(f"features must have shape (1,256,64,64), got {tuple(f.shape)}")
        _lib.check(_lib.lib().msam_set_image_embedding(self._h, _lib.ptr(feat), _lib.cur_stream()))
        self._bound_key, self._bound_src, self._bound_tensor = key, f, feat  # keeps both alive: the address cannot be reused

    def to(self, device):
        if torch.device(device).type != "cuda":
            raise RuntimeError("micro_sam_b200 models live on a CUDA device")
        return self

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                _lib.lib().msam_destroy(self._h)
                self._h = None
        except Exception:  # noqa: BLE001
            pass

    def preprocess(self, x: torch.Tensor) -> torch.Tensor:
        """Sam.preprocess: normalise + zero-pad to image_size (trainable_sam.py:24-47)."""
        x = (x.to(self.device, torch.float32) - self.pixel_mean) / self.pixel_std
        h, w = x.shape[-2:]
        return torch.nn.functional.pad(x, (0, self.image_size - w, 0, self.image_size - h))

    def encode_u8(self, images_u8: torch.Tensor) -> torch.Tensor:
        """Fused preprocess + encoder for a batch of already-resized uint8 HWC images [B,h,w,3] (h,w <= 1024)."""
        x = images_u8.to(self.device).contiguous()
        if x.dtype != torch.uint8 or x.ndim != 4 or x.shape[-1] != 3:
            raise ValueError("encode_u8 expects uint8 [B,h,w,3]")
        out = torch.empty(x.shape[0], 256, 64, 64, device=self.device, dtype=torch.float32)
        _lib.check(_lib.lib().msam_encode_u8(self._h, _lib.ptr(x), x.shape[0], x.shape[1], x.shape[2], _lib.ptr(out),
                                             _lib.cur_stream()))
        return out

    def postprocess_masks(self, masks: torch.Tensor, input_size, original_size) -> torch.Tensor:
        """Sam.postprocess_masks on (P,M,256,256) low-res logits -> (P,M,H,W) logits."""
        P, M = masks.shape[:2]
        lr = masks.to(self.device, torch.float32).contiguous().view(P * M, 256, 256)
        out = torch.empty(P * M, original_size[0], original_size[1], device=self.device, dtype=torch.float32)
        _lib.check(_lib.lib().msam_upsample_masks(_lib.ptr(lr), None, P * M, int(input_size[0]), int(input_size[1]),
                                                  int(original_size[0]), int(original_size[1]), self.mask_threshold,
                                                  _lib.ptr(out), None, _lib.cur_stream()))
        return out.view(P, M, original_size[0], original_size[1])


class B200SamPredictor:
    """Drop-in for segment_anything.SamPredictor (SURVEY.md A.1)."""

    def __init__(self, sam_model: B200Sam):
        self.model = sam_model
        self.transform = ResizeLongestSide(sam_model.image_size)
        self.reset_image()

    @property
    def device(self):
        return self.model.device

    def reset_image(self) -> None:
        self.is_image_set = False
        self.features = None
        self.orig_h = self.orig_w = self.input_h = self.input_w = None

    @torch.no_grad()
    def set_image(self, image: np.ndarray, image_format: str = "RGB") -> None:
        if image.dtype != np.uint8 or image.ndim != 3 or image.shape[-1] != 3:
            raise ValueError("set_image expects an HxWx3 uint8 image")
        if image_format != self.model.image_format:
            image = image[..., ::-1]
        x = self.transform.apply_image(image)
        self.reset_image()
        self.original_size = tuple(image.shape[:2])
        self.input_size = tuple(x.shape[:2])
        self.features = self.model.encode_u8(torch.from_numpy(np.ascontiguousarray(x))[None])
        self.is_image_set = True

    @torch.no_grad()
    def set_torch_image(self, transformed_image: torch.Tensor, original_image_size: Tuple[int, ...]) -> None:
        self.reset_image()
        self.original_size = tuple(original_image_size)
        self.input_size = tuple(transformed_image.shape[-2:])
        self.features = self.model.image_encoder(self.model.preprocess(transformed_image))
        self.is_image_set = True

    def get_image_embedding(self) -> torch.Tensor:
        if not self.is_image_set:
            raise RuntimeError("An image must be set with .set_image(...) to generate an embedding.")
        return self.features

    # -- re-bind when `features` was reassigned (by this or any other predictor of the same model)
    def _bind_features(self) -> None:
        f = self.features
        if f is None:
            raise RuntimeError("An image must be set with .set_image(...) before mask prediction.")
        self.model.bind_embedding(f)

    @torch.no_grad()
    def decode_low_res(self, point_coords: Optional[torch.Tensor], point_labels: Optional[torch.Tensor],
                       boxes: Optional[torch.Tensor] = None, multimask_output: bool = True,
                       mask_input: Optional[torch.Tensor] = None):
        """prompt_encoder + mask_decoder only: (low_res (P,M,256,256), iou (P,M)).  The hot AMG / batched-inference path
        stops here and post-processes with msam_mask_stats instead of materialising (P,M,H,W) logits."""
        if not self.is_image_set:
            raise RuntimeError("An image must be set with .set_image(...) before mask prediction.")
        self._bind_features()
        dev = self.device
        pts = lbl = bx = mk = None
        np_ = 0
        if point_coords is not None:
            if point_labels is None:
                raise ValueError("point_labels must be supplied with point_coords")
            pts = point_coords.to(dev, torch.float32).contiguous()
            lbl = point_labels.to(dev, torch.float32).contiguous()
            P, np_ = pts.shape[0], pts.shape[1]
        if boxes is not None:
            bx = boxes.to(dev, torch.float32).reshape(-1, 4).contiguous()
            P = bx.shape[0]
        if mask_input is not None:  # (P,1,256,256) low-res logits of a previous prediction (PromptEncoder._embed_masks)
            mk = mask_input.to(dev, torch.float32).reshape(-1, 256, 256).contiguous()
            if pts is None and bx is None:
                P = mk.shape[0]
            elif mk.shape[0] != P:
                raise ValueError(f"mask_input batch {mk.shape[0]} does not match the {P} prompts")
        if pts is None and bx is None and mk is None:
            raise ValueError("predict_torch needs point, box and/or mask prompts")
        M = 3 if multimask_output else 1
        low = torch.empty(P, M, 256, 256, device=dev, dtype=torch.float32)
        iou = torch.empty(P, M, device=dev, dtype=torch.float32)
        _lib.check(_lib.lib().msam_decode_ex(self.model._h, _lib.ptr(pts), _lib.ptr(lbl), np_, _lib.ptr(bx), _lib.ptr(mk), P,
                                             int(multimask_output), _lib.ptr(low), _lib.ptr(iou), _lib.cur_stream()))
        return low, iou

    @torch.no_grad()
    def predict_torch(self, point_coords, point_labels, boxes=None, mask_input=None, multimask_output: bool = True,
                      return_logits: bool = False):
        low, iou = self.decode_low_res(point_coords, point_labels, boxes, multimask_output, mask_input)
        P, M = low.shape[:2]
        H, W = self.original_size
        lr = low.view(P * M, 256, 256)
        if return_logits:
            masks = torch.empty(P * M, H, W, device=self.device, dtype=torch.float32)
            args = (_lib.ptr(masks), None)
        else:
            masks = torch.empty(P * M, H, W, device=self.device, dtype=torch.uint8)
            args = (None, _lib.ptr(masks))
        _lib.check(_lib.lib().msam_upsample_masks(_lib.ptr(lr), None, P * M, int(self.input_size[0]), int(self.input_size[1]),
                                                  int(H), int(W), self.model.mask_threshold, *args, _lib.cur_stream()))
        masks = masks.view(P, M, H, W)
        if not return_logits:
            masks = masks.bool()
        return masks, iou, low

    def predict(self, point_coords=None, point_labels=None, box=None, mask_input=None, multimask_output=True,
                return_logits=False):
        if not self.is_image_set:
            raise RuntimeError("An image must be set with .set_image(...) before mask prediction.")
        coords_t = labels_t = box_t = None
        if point_coords is not None:
            pc = self.transform.apply_coords(point_coords, self.original_size)
            coords_t = torch.as_tensor(pc, dtype=torch.float, device=self.device)[None]
            labels_t = torch.as_tensor(point_labels, dtype=torch.int, device=self.device)[None]
        if box is not None:
            box_t = torch.as_tensor(self.transform.apply_boxes(box, self.original_size), dtype=torch.float,
                                    device=self.device).reshape(1, 4)
        mask_t = None
        if mask_input is not None:
            mask_t = torch.as_tensor(mask_input, dtype=torch.float, device=self.device)[None]
        m, s, l = self.predict_torch(coords_t, labels_t, box_t, mask_t, multimask_output, return_logits)
        return m[0].cpu().numpy(), s[0].cpu().numpy(), l[0].cpu().numpy()


def local_otsu_threshold(low_res: torch.Tensor) -> torch.Tensor:
    """inference._local_otsu_threshold (inference.py:70-134) on (N,256,256) low-res logits -> fp32 thresholds [N]."""
    lr = low_res.reshape(-1, 256, 256).to(torch.float32).contiguous()
    if not lr.is_cuda:
        raise RuntimeError("local_otsu_threshold needs CUDA tensors")
    thr = torch.empty(lr.shape[0], device=lr.device, dtype=torch.float32)
    _lib.check(_lib.lib().msam_local_otsu_threshold(_lib.ptr(lr), lr.shape[0], _lib.ptr(thr), _lib.cur_stream()))
    return thr


def mask_stats(low_res: torch.Tensor, input_size, original_size, mask_threshold=0.0, stability_offset: float = 1.0):
    """Fused postprocess_masks + stability score + threshold + box + area on (N,256,256) low-res logits.
    `mask_threshold`: a float, or a device tensor [N] of per-mask thresholds (mask_threshold="auto").
    Returns (boxes int32 [N,4] xyxy, stability fp32 [N], area int32 [N]) on the device of `low_res`."""
    lr = low_res.reshape(-1, 256, 256)
    if not lr.is_cuda:
        raise RuntimeError("mask_stats needs CUDA tensors")
    lr = lr.to(torch.float32).contiguous()
    n = lr.shape[0]
    boxes = torch.empty(n, 4, device=lr.device, dtype=torch.int32)
    stab = torch.empty(n, device=lr.device, dtype=torch.float32)
    area = torch.empty(n, device=lr.device, dtype=torch.int32)
    if torch.is_tensor(mask_threshold):
        thr = mask_threshold.to(lr.device, torch.float32).reshape(-1).contiguous()
        assert thr.shape[0] == n
        _lib.check(_lib.lib().msam_mask_stats_ex(_lib.ptr(lr), n, int(input_size[0]), int(input_size[1]), int(original_size[0]),
                                                 int(original_size[1]), _lib.ptr(thr), float(stability_offset),
                                                 _lib.ptr(boxes), _lib.ptr(stab), _lib.ptr(area), _lib.cur_stream()))
        return boxes, stab, area
    _lib.check(_lib.lib().msam_mask_stats(_lib.ptr(lr), n, int(input_size[0]), int(input_size[1]), int(original_size[0]),
                                          int(original_size[1]), float(mask_threshold), float(stability_offset),
                                          _lib.ptr(boxes), _lib.ptr(stab), _lib.ptr(area), _lib.cur_stream()))
    return boxes, stab, area
