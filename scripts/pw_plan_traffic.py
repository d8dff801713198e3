"""Shared-memory fill traffic of the pointwise GEMM (pointwise_tc) on the D0 640x640 batch-32 deep
backbone, computed from the shapes: for each launch the plan pwtc::run() picks on a 132-SM H100 at
the default options (tile rows, k-block width, resident or streamed W), the bytes its TMA loads
move from L2 into shared memory -- W tiles and A tiles -- next to the algorithmic HBM bytes, for
the shared-W plan and for the 64-row plan that pw_share_w = 1 forces.  Runs on the CPU; it mirrors
the plan rule of pointwise_tc.cu (block_n, block_k, kResidentWBytes, the shared-W rule) and
must be kept in step with it.
usage: python scripts/pw_plan_traffic.py"""

SMS = 132
RESIDENT_W = 108 * 1024
SHARE_RES_MIN_KBLOCKS = 10
BATCH = 32
MB = 1e6

# D0 (EfficientNet-B0 backbone) at 640x640: name, rows per image, K, N, per-image (SE) weights
LAYERS = []
for i, (rows_in, rows_out, cin, cout, nblk) in enumerate([
    (6400, 1600, 40, 80, 3),      # blocks_5-7: expand at 80x80 (block 5) / 40x40, project at 40x40
    (1600, 1600, 80, 112, 3),     # blocks_8-10
    (1600, 400, 112, 192, 4),     # blocks_11-14
    (400, 400, 192, 320, 1)]):    # blocks_15
  first = [5, 8, 11, 15][i]
  for b in range(first, first + nblk):
    k_in = cin if b == first else cout
    if b != 5:   # blocks_5/expand (K 40) is one of the thin-K layers
      LAYERS.append(('blocks_%d/expand' % b, rows_in if b == first else rows_out, k_in, 6 * k_in,
                     False))
    LAYERS.append(('blocks_%d/project' % b, rows_out, 6 * k_in, cout, True))


def ceil_div(a, b):
  return -(-a // b)


def plan(rows, k, n, per_image, residual, share_w):
  block_n = ceil_div(n, 32) * 32 if n <= 128 else 128
  nnb = ceil_div(n, block_n)

  def w_bytes(bk):
    return nnb * ceil_div(k, bk) * ceil_div(block_n * bk * 2, 1024) * 1024

  bk = 16 if k <= 16 else (32 if k <= 32 else 64)
  if bk == 64 and not per_image and w_bytes(64) > RESIDENT_W and w_bytes(32) <= RESIDENT_W:
    bk = 32
  resident = not per_image and w_bytes(bk) <= RESIDENT_W
  # shared-memory stage limits are not modelled: at the default budget they never decide these
  share_w = (share_w and not resident and BATCH * ceil_div(rows, 128) * nnb >= SMS and
             (not residual or ceil_div(k, bk) >= SHARE_RES_MIN_KBLOCKS))
  tile_m = 128 if share_w else 64
  return block_n, bk, resident, tile_m, nnb


def traffic(rows, k, n, per_image, residual, share_w):
  block_n, bk, resident, tile_m, nnb = plan(rows, k, n, per_image, residual, share_w)
  tiles = BATCH * ceil_div(rows, tile_m) * nnb
  nkb = ceil_div(k, bk)
  w = SMS * w_bytes_resident(nnb, nkb, block_n, bk) if resident else tiles * nkb * block_n * bk * 2
  a = tiles * nkb * tile_m * bk * 2
  return tile_m, bk, resident, w / MB, a / MB


def w_bytes_resident(nnb, nkb, block_n, bk):
  return nnb * nkb * ceil_div(block_n * bk * 2, 1024) * 1024


def main():
  print('| layer | K | N | plan | W from L2, MB (64-row) | A from L2, MB (64-row) | HBM MB |')
  print('|---|---|---|---|---|---|---|')
  tot = [0.0] * 5
  for name, rows, k, n, per_image in LAYERS:
    residual = 'project' in name and k // 6 == n   # the skip of a stride-1 block, same width
    hbm = 2 * (BATCH * rows * k + BATCH * rows * n * (2 if residual else 1) +
               (BATCH if per_image else 1) * n * k)
    tile_m, bk, resident, w, a = traffic(rows, k, n, per_image, residual, True)
    _, _, _, w0, a0 = traffic(rows, k, n, per_image, residual, False)
    how = 'resident W, bk %d' % bk if resident else '%d-row tiles, bk %d' % (tile_m, bk)
    print('| %s | %d | %d | %s | %.0f (%.0f) | %.0f (%.0f) | %.0f |' %
          (name, k, n, how, w, w0, a, a0, hbm / MB))
    for i, v in enumerate((w, w0, a, a0, hbm / MB)):
      tot[i] += v
  print('| total (%d launches) | | | | %.0f (%.0f) | %.0f (%.0f) | %.0f |' % ((len(LAYERS),) + tuple(tot)))


if __name__ == '__main__':
  main()
