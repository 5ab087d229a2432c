"""micro-sam's automatic_segmentation.get_predictor_and_segmenter (automatic_segmentation.py:25-79): the segmentation mode
follows the checkpoint, AIS when it carries a `decoder_state`, AMG otherwise."""
from __future__ import annotations

from typing import Optional

from . import util
from .instance_segmentation import DEFAULT_SEGMENTATION_MODE_WITH_DECODER, get_decoder, get_instance_segmentation_generator


def get_predictor_and_segmenter(model_type: str, checkpoint=None, device=None, segmentation_mode: Optional[str] = None,
                                is_tiled: bool = False, predictor=None, state=None, **kwargs):
    """The predictor and the automatic instance segmentation class: `segmentation_mode` None or "auto" picks "ais" for a
    checkpoint with a decoder and "amg" otherwise."""
    if predictor is None:
        device = util.get_device(device)
        predictor, state = util.get_sam_model(model_type=model_type, device=device, checkpoint_path=checkpoint, return_state=True)
    elif state is None:
        raise ValueError("get_predictor_and_segmenter(predictor=...) needs the checkpoint's state as well")
    state = state or {}
    if segmentation_mode in (None, "auto"):
        segmentation_mode = DEFAULT_SEGMENTATION_MODE_WITH_DECODER if "decoder_state" in state else "amg"
    if segmentation_mode.lower() == "amg":
        decoder = None
    else:
        if "decoder_state" not in state:
            raise RuntimeError(f"You have passed 'segmentation_mode={segmentation_mode}', but your model does not contain a decoder.")
        decoder = get_decoder(None, state["decoder_state"], device=predictor.device)
    segmenter = get_instance_segmentation_generator(predictor=predictor, is_tiled=is_tiled, decoder=decoder,
                                                    segmentation_mode=segmentation_mode, **kwargs)
    return predictor, segmenter
