"""``python -m e2fgvi_b200.inpaint`` — the reference's ``test.py`` with the same arguments and the same output file,
running the front end, the network and the window loop on the GPU.

    python -m e2fgvi_b200.inpaint -v video.mp4|frame_dir -c ckpt.pth -m mask_dir [--model e2fgvi|e2fgvi_hq]
                                  [--step 10] [--num_ref -1] [--neighbor_stride 5] [--savefps 24]
                                  [--set_size --width W --height H]

Decoding stays on the host exactly as test.py:56-94 does it (``cv2.VideoCapture`` for ``.mp4``, otherwise the sorted
directory through ``cv2.imread``; BGR -> RGB; the sorted mask directory through ``Image.open(...).convert('L')``).
The video is uploaded once; ``prepare_inputs`` resizes the frames (``--model e2fgvi``: 432x240; ``--set_size``:
``--width`` x ``--height``; otherwise native size) and prepares the masks, ``VideoInpainter`` runs the windows, and
the result is written to ``results/<name>_results.mp4`` with ``cv2.VideoWriter`` (``mp4v``).  There is no preview
window.  Producing the frames (``inpaint``) and writing them (``write_video``) are separate steps.
"""
import argparse
import importlib
import os
import sys

import numpy as np
import torch

from .video import VideoInpainter, prepare_inputs


def parser():
    p = argparse.ArgumentParser(description="E2FGVI")          # test.py:15-28, same names and defaults
    p.add_argument("-v", "--video", type=str, required=True)
    p.add_argument("-c", "--ckpt", type=str, required=True)
    p.add_argument("-m", "--mask", type=str, required=True)
    p.add_argument("--model", type=str, choices=["e2fgvi", "e2fgvi_hq"])
    p.add_argument("--step", type=int, default=10)
    p.add_argument("--num_ref", type=int, default=-1)
    p.add_argument("--neighbor_stride", type=int, default=5)
    p.add_argument("--savefps", type=int, default=24)
    p.add_argument("--set_size", action="store_true", default=False)
    p.add_argument("--width", type=int)
    p.add_argument("--height", type=int)
    return p


def target_size(args):
    """The frame size rule of test.py:110-115: ``(W, H)`` or None for the native size."""
    if args.model == "e2fgvi":
        return (432, 240)
    if args.set_size:
        return (args.width, args.height)
    return None


def output_path(video):
    """test.py:183-190: ``results/<last path component>_results.mp4`` (``x.mp4`` -> ``x_results.mp4``)."""
    base = video.split("/")[-1]
    name = base.replace(".mp4", "_results.mp4") if video.endswith(".mp4") else base + "_results.mp4"
    return os.path.join("results", name)


def read_frames(video):
    """(N,H,W,3) uint8 RGB, decoded as test.py:74-94 does."""
    import cv2
    frames = []
    if video.endswith(".mp4"):
        cap = cv2.VideoCapture(video)
        ok, img = cap.read()
        while ok:
            frames.append(cv2.cvtColor(img, cv2.COLOR_BGR2RGB))
            ok, img = cap.read()
    else:
        for name in sorted(os.listdir(video)):
            frames.append(cv2.cvtColor(cv2.imread(video + "/" + name), cv2.COLOR_BGR2RGB))
    if not frames:
        raise ValueError(f"no frames decoded from {video}")
    return np.stack(frames)


def read_masks(mask_dir):
    """The sorted mask files as 'L' planes (a list: their sizes may differ), decoded as test.py:58-64 does."""
    from PIL import Image
    return [np.array(Image.open(os.path.join(mask_dir, name)).convert("L")) for name in sorted(os.listdir(mask_dir))]


def load_model(args, device):
    net = importlib.import_module("e2fgvi_b200.model." + args.model)
    model = net.InpaintGenerator()
    model.load_state_dict(torch.load(args.ckpt, map_location="cpu"))
    return model.eval().to(device)


def inpaint(args, model=None, device=None):
    """Decode, prepare, inpaint: the composited video as (N,H,W,3) uint8 RGB on the GPU, before any encoding."""
    device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
    if model is None:
        model = load_model(args, device)
    frames, masks = prepare_inputs(read_frames(args.video), read_masks(args.mask), target_size(args), device)
    drv = VideoInpainter(model, neighbor_stride=args.neighbor_stride, ref_length=args.step, num_ref=args.num_ref)
    return drv(frames, masks)


def write_video(path, comp, fps):
    """test.py:188-196: ``mp4v`` at ``fps``, RGB frames written as BGR."""
    import cv2
    os.makedirs(os.path.dirname(path) or ".", exist_ok=True)
    comp = comp.cpu().numpy() if isinstance(comp, torch.Tensor) else comp
    h, w = comp.shape[1:3]
    writer = cv2.VideoWriter(path, cv2.VideoWriter_fourcc(*"mp4v"), fps, (w, h))
    for f in comp:
        writer.write(cv2.cvtColor(f, cv2.COLOR_RGB2BGR))
    writer.release()


def main(argv=None):
    args = parser().parse_args(argv)
    comp = inpaint(args)
    path = output_path(args.video)
    write_video(path, comp, args.savefps)
    print(f"Finish test! The result video is saved in: {path}.")
    return path


if __name__ == "__main__":
    main(sys.argv[1:])
