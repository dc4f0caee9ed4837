"""L2 -> shared-memory operand traffic of the k_conv_tc launches in a `bench.py --profile-out` table.

For each tensor-core conv launch the table gives the time, the algorithmic FLOPs (2 * pixels * cout * cin * taps) and the
algorithmic bytes (4 * pixels * (cin + cout)).  With the layer's cout and kernel size (below, from net.cu's layer table)
those two numbers give the pixel count and cin, and with the feature resolution the tile count.  The operand bytes the
kernel moves from L2 into shared memory follow from its tiling:

  box (the kernel since A boxes are shared by the dy taps): per tile, one TW x (TH + 2) A box per (64-channel chunk, dx)
      for a 3x3 layer, the tile itself per chunk for a 1x1 layer; tiles of 16 x 8 pixels (8 x 16 below 12 columns)
  tap (the kernel before): per tile and K-block (tap x chunk), one TW x TH A tile; tiles of 32 x 4 from 24 columns on
  both: per tile and K-block, the tap's weights, 2 planes x npad x 128 bytes

Both planes (hi, lo) are counted.  The rate is bytes over the launch's measured time: a derived figure, not a counter.

    python tools/conv_tc_traffic.py PROFILE.csv [--layout box|tap] [--feat 32]
"""
import argparse
import csv
import math
from collections import OrderedDict

# tensor-core layers of the network: name -> (cout, kernel size); recons0 runs at twice the feature resolution
LAYERS = {
    "atten0": (1, 3), "pred_map0": (64, 3), "pred_map1": (1, 3), "local_fusion.res.conv1": (192, 3),
    "local_fusion.res.conv2": (192, 3), "local_fusion.conv": (64, 3), "gru.xconv": (64, 3), "gru.zr": (128, 3),
    "gru.out": (64, 3), "global_fusion": (64, 1), "offset0": (64, 3), "offset1": (64, 3), "conv_offset_mask": (216, 3),
    "dcn_gemm": (64, 1), "convblock0": (64, 3), "convblock1": (64, 3), "spatial_kernel": (2, 1), "dcn_fusion0": (64, 3),
    "dcn_fusion1": (64, 3), "dense_fusion0": (64, 3), "dense_fusion1": (64, 3), "recons0": (32, 3),
}


def tile_shape(W, layout):
    TW = (16 if W >= 12 else 8) if layout == "box" else (32 if W >= 24 else (16 if W >= 12 else 8))
    return TW, 128 // TW


def operand_bytes(n_img, H, W, cin, cout, k, layout):
    TW, TH = tile_shape(W, layout)
    tiles = n_img * math.ceil(W / TW) * math.ceil(H / TH)
    chunks, taps = cin // 64, k * k
    npad = (cout + 15) // 16 * 16
    b = chunks * taps * 2 * npad * 128
    if layout == "tap":
        a = chunks * taps * 2 * TW * TH * 128
    elif k == 3:
        a = chunks * 3 * 2 * TW * (TH + 2) * 128
    else:
        a = chunks * 2 * TW * TH * 128
    return tiles, tiles * a, tiles * b


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("profile", help="CSV written by bench.py --profile-out")
    ap.add_argument("--layout", choices=["box", "tap"], default="box")
    ap.add_argument("--feat", type=int, default=32, help="feature resolution (square), e.g. 32 for cfg2")
    args = ap.parse_args()
    agg = OrderedDict()                         # layer -> [launches, ms, flops, bytes]
    with open(args.profile) as f:
        rows = csv.reader(f)
        next(rows)                              # header (its class column name holds commas itself)
        for _, layer, cls, ms, fl, by in rows:  # idx, layer, class (0 = tensor-core conv), ms, FLOPs, bytes
            if int(cls) != 0 or layer not in LAYERS:
                continue
            a = agg.setdefault(layer, [0, 0.0, 0.0, 0.0])
            a[0] += 1
            a[1] += float(ms)
            a[2] += float(fl)
            a[3] += float(by)
    print(f"layout {args.layout}, features {args.feat}x{args.feat}")
    print(f"{'layer':<24}{'launches':>9}{'ms':>9}{'cin':>5}{'cout':>5}{'k':>3}{'images':>8}{'tiles':>8}"
          f"{'A MB':>9}{'B MB':>9}{'TB/s':>7}")
    tot_ms = tot_by = 0.0
    for name, (nl, ms, fl, by) in agg.items():
        cout, k = LAYERS[name]
        r = fl / by                             # = 2 cout cin k^2 / (4 (cin + cout))
        cin = round(4 * r * cout / (2 * cout * k * k - 4 * r))
        px = fl / (2.0 * cout * cin * k * k)
        side = 2 * args.feat if name == "recons0" else args.feat
        n_img = round(px / (side * side))
        tiles, a_by, b_by = operand_bytes(n_img, side, side, cin, cout, k, args.layout)
        tot_ms += ms
        tot_by += a_by + b_by
        print(f"{name:<24}{nl:>9}{ms:>9.4f}{cin:>5}{cout:>5}{k:>3}{n_img // nl:>8}{tiles // nl:>8}"
              f"{a_by / 1e6:>9.1f}{b_by / 1e6:>9.1f}{(a_by + b_by) / (ms * 1e-3) / 1e12:>7.2f}")
    print(f"{'total':<24}{'':>9}{tot_ms:>9.4f}{'':>29}{tot_by / 1e6:>18.1f}{tot_by / (tot_ms * 1e-3) / 1e12:>7.2f}")


if __name__ == "__main__":
    main()
