"""Bytes the 3x3 stride-1 convolutions of ResNet-50 bs256 request from L2, beside their measured time.

The im2col feed loads every 128-pixel tile once per filter tap and the weight tile once per k-block.  For comparison
the script also counts a slab of whole output rows, where each tile's input rows are loaded once with their halo and
the weights once per k-block, or once per CTA when they fit (DESIGN section 8, gap 2).  Each count is divided by the
measured launch time, which gives the L2 -> SM rate that feed would need.  The card's name and power limit are printed
with the table.

    python tests/profile_conv3x3_l2.py            (from the repository root, on an H100)
"""
import subprocess

import torch

from profile_gemm_shapes import conv_rows


def l2_bytes_3x3(n, h, c, sms=132):
    """Bytes a 3x3 stride-1 c -> c launch (fprop, or dgrad: the same shapes) requests from L2: im2col and slab."""
    bn = 64 if (c + 63) // 64 * 64 < (c + 127) // 128 * 128 else 128
    num_n, kb = (c + bn - 1) // bn, 9 * c // 64
    b_tile = kb * bn * 128
    im2col = -(-n * h * h // 128) * num_n * kb * (16384 + bn * 128)
    rows = 128 // h
    slab_rows = 0
    for g0 in range(0, n * h, rows):   # input rows per tile: its output rows + 2 halo rows per image it touches
        g1 = min(g0 + rows, n * h)
        slab_rows += g1 - g0 + 2 * ((g1 - 1) // h - g0 // h + 1)
    resident = num_n == 1 and b_tile <= 73728
    slab = num_n * (slab_rows * (c // 64) * (h + 2) * 128 + (0 if resident else -(-n * h // rows) * b_tile))
    if resident:
        slab += sms * b_tile
    return [('im2col', im2col), ('slab', slab)]


def main():
    card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                          capture_output=True, text=True).stdout.strip().splitlines()
    print(f'card: {card[torch.cuda.current_device()] if card else torch.cuda.get_device_name()} (name, power limit)')
    N = 256
    for h, c in ((56, 64), (28, 128), (14, 256), (7, 512)):
        l2 = l2_bytes_3x3(N, h, c)
        for what, flop, us in conv_rows(N, h, c, c, 3)[:2]:
            rates = ', '.join(f'{m} {b * 1e-9:.2f} GB ({b / us * 1e-6:.1f} TB/s)' for m, b in l2)
            print(f'conv 3x3 c{c} {h}x{h} {what:6s} {us:8.1f} us {flop / us * 1e-6:7.1f} TFLOP/s   L2 requested: {rates}',
                  flush=True)


if __name__ == '__main__':
    main()
