"""Train a model file to its schedule, as the reference's train_convnet does:

    python -m convnet_b200.train MODEL.pbtxt --train train.npz [--valid valid.npz] [--checkpoint-dir D] [--resume CKPT]
                                 [--seed S]

The model file sets the schedule (max_iter, print_after, validate_after, save_after, reduce_lr_*, polyak_*,
checkpoint_dir; see net.model_schedule) and, in its train_dataset / valid_dataset blocks, the batch size, the batch order
and the crop of each data set.  Each .npz file holds `images` (float32 [N, C, H, W]) and `labels` (integers [N]) or
`targets` (float [N, F]) for an output layer trained on float targets.  --resume loads a checkpoint first: training
continues from its iteration and learning rates.  --seed seeds the net's initial weights and dropout (the model file's
seed is not used); the training and validation feeds are seeded with S + 1 and S + 2.  The conv arithmetic is the
library's (CONVNET_B200_PRECISION)."""
import argparse
import sys

import numpy as np


def load_npz(path):
    """(images, labels, targets) host tensors from an .npz file; labels or targets is None"""
    import torch
    with np.load(path) as d:
        if "images" not in d or ("labels" not in d and "targets" not in d):
            raise ValueError("%s: needs 'images' and 'labels' or 'targets' (it has %s)" % (path, ", ".join(d.files)))
        images = torch.from_numpy(np.ascontiguousarray(d["images"], dtype=np.float32))
        labels = torch.from_numpy(np.ascontiguousarray(d["labels"], dtype=np.int32)) if "labels" in d else None
        targets = torch.from_numpy(np.ascontiguousarray(d["targets"], dtype=np.float32)) if "targets" in d else None
    if images.dim() != 4:
        raise ValueError("%s: images must be [N, C, H, W], not %s" % (path, list(images.shape)))
    return images.pin_memory(), labels, targets


def main(argv=None):
    ap = argparse.ArgumentParser(prog="python -m convnet_b200.train", description=__doc__.split("\n\n")[0])
    ap.add_argument("model", help="a model file (.pbtxt) with a train_dataset block")
    ap.add_argument("--train", required=True, help=".npz training set")
    ap.add_argument("--valid", help=".npz validation set (the model needs a valid_dataset block)")
    ap.add_argument("--checkpoint-dir", help="where the run's files go (default: the model's checkpoint_dir, else .)")
    ap.add_argument("--resume", help="a checkpoint to continue from")
    ap.add_argument("--seed", type=int, default=42)
    a = ap.parse_args(argv)

    from . import net as N
    cfg = N.model_dataset(a.model, "train_dataset")
    if cfg is None:
        ap.error("%s has no train_dataset block (its batch_size is the net's)" % a.model)
    n = N.Net(a.model, cfg["batch_size"], seed=a.seed)
    handlers = []
    try:
        if a.resume:
            n.load(a.resume)
        images, labels, targets = load_npz(a.train)
        handlers.append(N.DataHandler.from_model(a.model, images, labels, "train_dataset", targets=targets, net=n,
                                                 seed=a.seed + 1))
        if a.valid:
            images, labels, targets = load_npz(a.valid)
            handlers.append(N.DataHandler.from_model(a.model, images, labels, "valid_dataset", targets=targets, net=n,
                                                     seed=a.seed + 2))
        n.train(handlers[0], handlers[1] if a.valid else None, checkpoint_dir=a.checkpoint_dir)
    except ValueError as e:
        print("error: %s" % e, file=sys.stderr)
        return 1
    finally:
        for h in handlers:
            h.close()
        n.close()
    print("End of training.")
    return 0


if __name__ == "__main__":
    sys.exit(main())
