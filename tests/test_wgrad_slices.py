"""The pixel split of the generic weight-gradient kernel (ops/igemm.py _wgrad_slices, the same
arithmetic as igemm_wgrad_kernel in csrc/igemm_wgrad.cu): every (output tile, pixel box) iteration
of a launch belongs to exactly one CTA, slices differ by at most one box, and each segment of a
slice stays inside one tile."""
import itertools

import pytest

from tensorflowonspark_b200.ops import igemm

TILES = [1, 2, 7, 8, 9, 16, 64, 128, 136, 288, 576]
BOXES = [1, 2, 3, 17, 98, 196, 392, 1568]
CTAS = [1, 5, 131, 132, 264]


@pytest.mark.parametrize("tiles,boxes,ctas", list(itertools.product(TILES, BOXES, CTAS)))
def test_wgrad_slices_cover_every_iteration_once(tiles, boxes, ctas):
  slices = igemm._wgrad_slices(tiles, boxes, ctas)
  assert len(slices) == min(ctas, tiles * boxes)
  seen = []
  lens = []
  for segs in slices:
    assert segs, "empty slice"
    n = 0
    for (t, b0, b1) in reversed(segs):   # the kernel walks a slice's segments last first
      assert 0 <= t < tiles and 0 <= b0 < b1 <= boxes
      seen.extend(t * boxes + b for b in range(b0, b1))
      n += b1 - b0
    lens.append(n)
    # a CTA adds its partial dW once per segment: at most 1 + ceil(slice / boxes) times
    assert len(segs) <= 1 + -(-n // boxes)
  # tiles outermost, a tile's boxes consecutive, slices in CTA order: the flat range in order
  assert seen == list(range(tiles * boxes))
  assert max(lens) - min(lens) <= 1


def test_wgrad_slices_resnet_l3c1_fills_the_sms():
  """ResNet-50 l3c1 (14 x 14, 1024 -> 256) at batch 256: 8 output tiles of 128 x 256 and 392
  boxes of 128 pixels.  Whole split-K work items of 1/17 of the pixels made 136 items, two rounds
  on 132 SMs with the second almost empty; the even split gives every CTA 23 or 24 boxes and adds
  at most one flush per tile."""
  tiles, boxes = 8, 392
  slices = igemm._wgrad_slices(tiles, boxes, 132)
  lens = [sum(b1 - b0 for (_, b0, b1) in s) for s in slices]
  assert len(slices) == 132 and min(lens) == 23 and max(lens) == 24
  flushes = sum(len(s) for s in slices)
  assert flushes <= 132 + tiles
