"""Compare the training step of two builds of the library, output by output.

A change to the training path that is meant to keep its results (a refactor, a kernel cleanup) can be checked with this script:
`dump` runs a few seeded UNetTrainEngine steps (train-mode forward + backward, the third one replayed from a CUDA graph) with the
package of the checkout given by --root, which must have its librsb200.so built, and saves the logits of every step, the
parameter gradients, the BatchNorm running statistics and num_batches_tracked. `compare` reports, per output, whether the dumps
are byte-identical and otherwise the largest absolute difference. Dump the old build twice to see which outputs are bit-stable
from run to run (the fp64 atomics of the BatchNorm accumulators may not be), then the new build once:

  python scripts/train_step_equivalence.py dump --root OLD --out old1.pt
  python scripts/train_step_equivalence.py dump --root OLD --out old2.pt
  python scripts/train_step_equivalence.py dump --root . --out new.pt
  python scripts/train_step_equivalence.py compare old1.pt old2.pt new.pt

Configurations: 2 classes at 4 x 3 x 512 x 512 and 6 classes at 3 x 3 x 256 x 384.
"""

import argparse
import hashlib
import json
import os
import sys

CONFIGS = ((2, 4, 512, 512), (6, 3, 256, 384))  # classes, batch, height, width
STEPS = 3


def dump(root, out):
    sys.path.insert(0, os.path.abspath(root))
    import torch

    from robosat_b200 import synth
    from robosat_b200.train_engine import UNetTrainEngine

    dev = torch.device("cuda", 0)
    result = {}
    for classes, batch, h, w in CONFIGS:
        tag = "%dc_%dx%dx%d" % (classes, batch, h, w)
        params = {k[7:]: v.to(dev) for k, v in synth.make_state_dict(classes, seed=0).items()}
        eng = UNetTrainEngine(params, classes, batch, h, w, device=dev, loss_scale=1024.0)
        g = torch.Generator().manual_seed(11)
        for step in range(STEPS):
            x = synth.normalize_tiles(synth.make_tiles_u8(batch, max(h, w), seed=20 + step))[:, :, :h, :w].contiguous().to(dev)
            dlogits = (torch.randn((batch, classes, h, w), generator=g) * 1e-3).to(dev)
            result["%s/step%d/logits" % (tag, step)] = eng.forward(x).clone().cpu()
            grads = eng.backward(dlogits)
            torch.cuda.synchronize()
            if step < STEPS - 1:  # earlier steps' gradients by digest only: the whole set is ~130 MB per step
                flat = torch.cat([v.reshape(-1) for v in grads.values()]).cpu()
                result["%s/step%d/grads_sha256" % (tag, step)] = hashlib.sha256(flat.numpy().tobytes()).hexdigest()
        for k, v in grads.items():
            result["%s/grad/%s" % (tag, k)] = v.clone().cpu()
        for k, v in params.items():
            if k.endswith(("running_mean", "running_var", "num_batches_tracked")):
                result["%s/param/%s" % (tag, k)] = v.clone().cpu()
        del eng, params
        torch.cuda.empty_cache()
    torch.save(result, out)
    print("wrote %s: %d entries" % (out, len(result)))


def _group(key):
    """output kind of a dump key, for the summary"""
    tag, rest = key.split("/", 1)
    if rest.startswith("grad/"):
        kind = "grads"
    elif rest.startswith("param/"):
        kind = "num_batches_tracked" if rest.endswith("num_batches_tracked") else "bn_running_stats"
    elif rest.endswith("grads_sha256"):
        kind = "grads_sha256"
    else:
        kind = "logits"
    return tag + " " + kind


def compare(paths):
    import torch

    dumps = [torch.load(p) for p in paths]
    keys = sorted(dumps[0])
    for d, p in zip(dumps[1:], paths[1:]):
        assert sorted(d) == keys, "%s holds different outputs" % p
    summary = {}
    for k in keys:
        for j in range(1, len(dumps)):
            a, b = dumps[0][k], dumps[j][k]
            s = summary.setdefault((_group(k), j), {"outputs": 0, "identical": 0, "max_abs_diff": 0.0, "worst": None})
            s["outputs"] += 1
            if isinstance(a, str):
                same, diff = a == b, 0.0 if a == b else float("inf")
            else:
                same = a.dtype == b.dtype and a.shape == b.shape and torch.equal(a.view(-1).view(torch.uint8), b.view(-1).view(torch.uint8))
                diff = 0.0 if same else float((a.double() - b.double()).abs().max())
            s["identical"] += int(same)
            if diff > s["max_abs_diff"]:
                s["max_abs_diff"], s["worst"] = diff, k
    rows = []
    for (group, j), s in sorted(summary.items()):
        rows.append(dict(s, output=group, against=paths[j], reference=paths[0]))
        print("%-40s %-22s identical %4d / %-4d  max |diff| %.3g%s" % (group, os.path.basename(paths[j]), s["identical"], s["outputs"],
                                                                       s["max_abs_diff"], "  (%s)" % s["worst"] if s["worst"] else ""))
    return rows


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    sub = ap.add_subparsers(dest="cmd", required=True)
    d = sub.add_parser("dump")
    d.add_argument("--root", default=".", help="checkout whose robosat_b200 package (with librsb200.so built) runs the steps")
    d.add_argument("--out", required=True)
    c = sub.add_parser("compare")
    c.add_argument("dumps", nargs="+", help="the first dump is the reference the others are compared with")
    c.add_argument("--json", default=None, help="also write the summary rows here")
    args = ap.parse_args()
    if args.cmd == "dump":
        dump(args.root, args.out)
    else:
        rows = compare(args.dumps)
        if args.json:
            json.dump(rows, open(args.json, "w"), indent=1)


if __name__ == "__main__":
    main()
