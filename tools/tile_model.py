"""Wave-quantised cost model of the twelve 3x3 convolutions (forward + dgrad) of one tiled rank, relative to 1/N of the
untiled run (DESIGN.md section 6).  A conv launch is `tiles` CTA tiles of 16 x (8 MT) pixels x BN channels walked by 132
persistent CTAs (one per H100 SM), so its time is ceil(tiles / 132) waves of one tile time.

  python tools/tile_model.py [size]

Columns: apron = every layer on own rows + 80-row aprons (what `STB_TILE=apron` runs), windowed = only the apron rows a
layer really needs (70 at the image, 0 at relu5_1), halo = own rows only (`STB_TILE=halo`, plus ~28 exchanges of ~13 us
each which this model does not contain); tile_h = 8 shows what 8-row tiles would change.
"""
import math
import sys

CONVS = [(3, 64, 0), (64, 64, 0), (64, 128, 1), (128, 128, 1), (128, 256, 2), (256, 256, 2), (256, 256, 2), (256, 256, 2),
         (256, 512, 3), (512, 512, 3), (512, 512, 3), (512, 512, 3), (512, 512, 4)]
# rows of halo (at the layer's own resolution) the OUTPUT of conv i needs so that every deeper own-row tap is exact
NEED = {1: 68, 2: 33, 3: 32, 4: 15, 5: 14, 6: 13, 7: 12, 8: 5, 9: 4, 10: 3, 11: 2, 12: 0}


def cost(size, rows_fn, tile_h=16):
    total = 0
    for i, (cin, cout, level) in enumerate(CONVS):
        if i == 0:
            continue
        w = size >> level
        rows = rows_fn(i, level)
        for c_out, c_in in ((cout, cin), (cin, cout)):          # forward, dgrad
            bn = 256 if c_out >= 256 else c_out
            mt = 1 if bn == 256 else 2
            tile_w = (8 if tile_h == 16 else 16) * mt
            tiles = math.ceil(w / tile_w) * math.ceil(rows / tile_h) * (c_out // bn)
            total += math.ceil(tiles / 132) * 132 * (2 * 9 * c_in * bn * 128 * mt)
    return total


def main():
    size = int(sys.argv[1]) if len(sys.argv) > 1 else 2048
    full = cost(size, lambda i, l: size >> l)
    print(f'{size}^2: conv cost of an interior band x N / cost of the untiled run (1.0 = perfect)')
    print(' N  tile_h   apron  windowed    halo')
    for n in (2, 4, 8):
        own = size // n
        for th in (16, 8):
            apron = cost(size, lambda i, l: (own + 160) >> l, th)

            def windowed(i, l):
                a, h = 80 >> l, NEED[i]
                start = ((a - h) // th) * th
                return math.ceil((a + (own >> l) + h - start) / th) * th
            halo = cost(size, lambda i, l: max(own >> l, 1), th)
            print(f'{n:2d}  {th:5d}  {apron / full * n:6.3f}  {cost(size, windowed, th) / full * n:8.3f}  {halo / full * n:6.3f}')


if __name__ == '__main__':
    main()
