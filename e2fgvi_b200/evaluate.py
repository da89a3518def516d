"""``python -m e2fgvi_b200.evaluate`` — the reference's ``evaluate.py`` with the same arguments, output lines and files,
running the front end, the network, PSNR / SSIM and I3D on the GPU.

    python -m e2fgvi_b200.evaluate --dataset davis|youtube-vos --data_root R --model e2fgvi|e2fgvi_hq --ckpt CKPT
                                   [--save_results] [--num_workers N]

Per video of ``R/<dataset>/test.json`` (evaluate.py:70-161, core/dataset.py TestDataset):

* frames: ``R/<dataset>/JPEGImages/<video>.zip`` (sorted members, cv2.imdecode, BGR -> RGB; ``vfid.read_dataset_video``)
  and masks ``R/<dataset>/test_masks/<video>/%05d.png`` as 'L' planes, decoded on the host by a background thread
  while the GPU works on the previous video (evaluate.py's DataLoader workers overlap this step too);
* ``prepare_inputs`` resizes frames to 432x240 (Pillow bicubic) and masks (NEAREST, ``> 0``, 4x cross dilation);
* ``VideoInpainter.composite`` runs evaluate.py's windows (stride 5, every 10th frame as reference, no padding) and
  returns the float32 blended composite, on which ``frame_metrics`` computes PSNR and SSIM against the resized frames,
  as ``calc_psnr_and_ssim`` does;
* VFID uses the composite's uint8 truncation: the resized frames and it go through I3D as one batch of 2.

The result lines go to stdout and ``results/<model>_<dataset>/<model>_<dataset>_metrics.txt``; ``--save_results``
writes ``results/<model>_<dataset>/<video>/%05d.png`` (BGR) and, like evaluate.py, refuses an existing video folder.
``--num_workers`` is accepted for compatibility and unused: one decoding thread is always used.
"""
import argparse
import json
import os
import sys
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

from . import vfid
from .inpaint import load_model
from .metrics import frame_metrics
from .video import VideoInpainter, finalize, prepare_inputs

SIZE = (432, 240)                 # evaluate.py's (w, h)
NEIGHBOR_STRIDE, REF_LENGTH = 5, 10


def parser():
    p = argparse.ArgumentParser(description="E2FGVI")          # evaluate.py:164-175, same names and defaults
    p.add_argument("--dataset", choices=["davis", "youtube-vos"], type=str)
    p.add_argument("--data_root", type=str, required=True)
    p.add_argument("--model", choices=["e2fgvi", "e2fgvi_hq"], type=str)
    p.add_argument("--ckpt", type=str, required=True)
    p.add_argument("--save_results", action="store_true", default=False)
    p.add_argument("--num_workers", default=4, type=int, help="accepted for compatibility; unused")
    return p


def read_masks(data_root, dataset, name, count):
    """``R/<dataset>/test_masks/<name>/%05d.png`` for frames 0 .. count-1 as 'L' planes (a list)."""
    from PIL import Image
    out = []
    for i in range(count):
        path = os.path.join(data_root, dataset, "test_masks", name, f"{i:05d}.png")
        if not os.path.isfile(path):
            raise FileNotFoundError(f"evaluate: video {name!r}: mask {path} not found")
        out.append(np.array(Image.open(path).convert("L")))
    return out


def read_video(args, name, count):
    return (vfid.read_dataset_video(args.data_root, args.dataset, name, count),
            read_masks(args.data_root, args.dataset, name, count))


def evaluate_video(drv, i3d, frames, masks, device):
    """One video: ``(psnr, ssim)`` per frame (host float64), the uint8 composite on the GPU and the I3D features of
    the resized frames and of that composite."""
    frames, masks = prepare_inputs(frames, masks, SIZE, device)
    comp = drv.composite(frames, masks)
    psnr, ssim = frame_metrics(frames, comp)
    comp = finalize(comp)
    feats = i3d.features_u8(torch.stack([frames, comp])).cpu().numpy()
    return psnr, ssim, comp, feats[0].flatten(), feats[1].flatten()


def main(argv=None, model=None, i3d=None):
    """Run the evaluation; ``model`` / ``i3d`` replace the checkpoints when given.  Returns (average PSNR, average
    SSIM, VFID)."""
    import cv2
    args = parser().parse_args(argv)
    assert args.dataset in ("davis", "youtube-vos"), f"{args.dataset} dataset is not supported"
    with open(os.path.join(args.data_root, args.dataset, "test.json")) as f:
        videos = list(json.load(f).items())
    device = torch.device("cuda", torch.cuda.current_device())
    if model is None:
        model = load_model(args, device)
        print(f"Loading from: {args.ckpt}")
    else:
        device = next(model.parameters()).device
    drv = VideoInpainter(model, neighbor_stride=NEIGHBOR_STRIDE, ref_length=REF_LENGTH, num_ref=-1)

    print("Start evaluation...")
    result_path = os.path.join("results", f"{args.model}_{args.dataset}")
    os.makedirs(result_path, exist_ok=True)
    total_psnr, total_ssim, real, fake = [], [], [], []
    with open(os.path.join(result_path, f"{args.model}_{args.dataset}_metrics.txt"), "w") as summary, \
            ThreadPoolExecutor(max_workers=1) as pool:
        if i3d is None:
            i3d = vfid.init_i3d_model()
        pending = pool.submit(read_video, args, *videos[0]) if videos else None
        for index, (name, count) in enumerate(videos):
            frames, masks = pending.result()
            if index + 1 < len(videos):
                pending = pool.submit(read_video, args, *videos[index + 1])
            psnr, ssim, comp, f_real, f_fake = evaluate_video(drv, i3d, frames, masks, device)
            psnr, ssim = psnr.tolist(), ssim.tolist()
            total_psnr += psnr
            total_ssim += ssim
            real.append(f_real)
            fake.append(f_fake)
            cur_psnr, cur_ssim = sum(psnr) / len(psnr), sum(ssim) / len(ssim)
            # evaluate.py prints the DataLoader-collated name, a one-element list
            line = f"[{index + 1:3}/{len(videos)}] Name: {str([name]):25} | PSNR/SSIM: {cur_psnr:.4f}/{cur_ssim:.4f}"
            print(line)
            summary.write(line + "\n")
            if args.save_results:
                save_frame_path = os.path.join(result_path, name)
                os.makedirs(save_frame_path, exist_ok=False)
                for i, frame in enumerate(comp.cpu().numpy()):
                    cv2.imwrite(os.path.join(save_frame_path, str(i).zfill(5) + ".png"),
                                cv2.cvtColor(frame, cv2.COLOR_RGB2BGR))
        avg_psnr = sum(total_psnr) / len(total_psnr)
        avg_ssim = sum(total_ssim) / len(total_ssim)
        fid_score = vfid.calculate_vfid(real, fake)
        line = f"Finish evaluation... Average Frame PSNR/SSIM/VFID: {avg_psnr:.2f}/{avg_ssim:.4f}/{fid_score:.3f}"
        print(line)
        summary.write(line)
    return avg_psnr, avg_ssim, fid_score


if __name__ == "__main__":
    main(sys.argv[1:])
