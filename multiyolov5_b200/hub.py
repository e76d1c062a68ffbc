"""The reference's hubconf.py `custom()` (reference hubconf.py:63-82) for local checkpoints:

    from multiyolov5_b200.hub import custom
    model = custom("best.pt")                  # autoShape on cuda: model([im1, im2], size=640) -> Detections
    model = custom("best.pt", autoshape=False) # the plain Model

The pretrained `yolov5s` ... entry points download weights and build the reference's plain detection yamls, which this multi-task
model does not parse; they are not built.
"""
import torch

from .models.experimental import attempt_load


def custom(path_or_model="path/to/model.pt", autoshape=True):
    """path_or_model: a checkpoint path (attempt_load: fp32, fused, eval), a loaded checkpoint dict (its 'ema' or 'model') or a Model.
    Returns the model, wrapped by Model.autoshape() when autoshape, on the current CUDA device."""
    if isinstance(path_or_model, str):
        model = attempt_load(path_or_model, map_location="cpu")
    else:
        model = path_or_model
        if isinstance(model, dict):
            model = model["ema" if model.get("ema") else "model"]
        model = model.float().eval()
    if autoshape:
        model = model.autoshape()
    return model.to(torch.device("cuda", torch.cuda.current_device()))
