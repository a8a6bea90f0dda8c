"""aicb200.pixel_picker_order, the restatement of RaytraceToTexture's PixelPicker (raytrace_to_texture.rs:835-918) that
the GPU texture target's pick order is checked against: PixelPicker::new sorts the pixels stably by
`(square_radius + blend) as i64` (:861-876), takes the first min(60000, n / 4) as the centre (:877-880), and yields
sorted_pixels[Interleave(Cycle(0..central), Cycle(central..n))] (:882-886, 900-908).  itertools' Interleave toggles a
flag before every item, takes from the first iterator when it is set and from the second otherwise, and from the other
one whenever the one in turn has nothing; Cycle of an empty range never has anything."""
import numpy as np

import aicb200
from aicb200 import CENTRAL_PIXEL_LIMIT, pixel_picker_order


def central_of(w, h):
    return min(CENTRAL_PIXEL_LIMIT, w * h // 4)


def cycle_length_of(w, h):
    c = central_of(w, h)
    return 2 * max(c, w * h - c)


def sorted_pixels(w, h):
    """PixelPicker::new's sorted_pixels, scalar by scalar (Python's sort is stable, as sort_by_key is)."""
    cx, cy = w / 2.0 - 0.5, h / 2.0 - 0.5

    def key(i):
        x, y = i % w, i // w
        return int(max(abs(x - cx), abs(y - cy)) + ((x ^ y) % 4) * 2)

    return sorted(range(w * h), key=key)


def test_one_cycle_covers_every_pixel():
    for w, h in [(1, 1), (3, 2), (17, 9), (64, 48), (101, 37), (640, 360)]:
        picks = pixel_picker_order(w, h)
        assert picks.size == cycle_length_of(w, h)
        assert np.array_equal(np.unique(picks), np.arange(w * h)), (w, h)
        # as a sequence of distinct pixels, the first cycle is a permutation of the viewport
        first = dict.fromkeys(int(p) for p in picks)
        assert sorted(first) == list(range(w * h))


def test_the_centre_comes_first_and_repeats():
    for w, h in [(17, 9), (64, 48), (640, 360)]:
        order = sorted_pixels(w, h)
        c = central_of(w, h)
        picks = pixel_picker_order(w, h, 2 * cycle_length_of(w, h))
        even, odd = picks[0::2], picks[1::2]
        assert np.array_equal(even[:c], order[:c])                  # the centre, nearest first
        assert np.array_equal(even[c:2 * c], order[:c])             # and again: period 2 * central in the picks
        assert np.array_equal(odd[:w * h - c], order[c:])           # the rest, in sort order
        assert np.array_equal(odd[w * h - c:2 * (w * h - c)], order[c:])


def test_viewports_under_four_pixels_have_no_centre():
    """central = n / 4 = 0: Interleave goes on with the rest alone, one pixel per pick."""
    assert list(pixel_picker_order(1, 1, 5)) == [0, 0, 0, 0, 0]
    # 2 x 1: keys 0 (x=0: |0 - 0.5| + 0) and 2 (x=1: 0.5 + ((1 ^ 0) % 4) * 2)
    assert list(pixel_picker_order(2, 1, 6)) == [0, 1, 0, 1, 0, 1]
    # 3 x 1: keys 1, 2, 5
    assert list(pixel_picker_order(3, 1, 7)) == [0, 1, 2, 0, 1, 2, 0]
    # 1 x 3: centre (0, 1); keys 1 + 0, 0 + 2, 1 + 4
    assert list(pixel_picker_order(1, 3, 4)) == [0, 1, 2, 0]
    assert cycle_length_of(3, 1) == 6


def test_a_one_pixel_centre():
    """1 x 7: central = 7 / 4 = 1, so every even pick is the centre pixel.  Centre (0, 3); keys by row
    3, 2 + 2, 1 + 4, 0 + 6, 1 + 0, 2 + 2, 3 + 4 = [3, 4, 5, 6, 1, 4, 7] -> sorted [4, 0, 1, 5, 2, 3, 6]."""
    assert sorted_pixels(1, 7) == [4, 0, 1, 5, 2, 3, 6]
    assert list(pixel_picker_order(1, 7)) == [4, 0, 4, 1, 4, 5, 4, 2, 4, 3, 4, 6]
    assert cycle_length_of(1, 7) == 12


def test_the_centre_caps_at_60000():
    """480 x 500 = 240000 pixels: central = 60000 exactly; 500 x 500: 62500, capped to 60000; 479 x 500: 59875."""
    for w, h, c in [(480, 500, 60000), (500, 500, 60000), (479, 500, 59875)]:
        assert central_of(w, h) == c
        order = np.array(sorted_pixels(w, h))
        picks = pixel_picker_order(w, h, 2 * c + 2)
        assert np.array_equal(picks[0::2][:c], order[:c]), (w, h)
        assert picks[2 * c] == picks[0] == order[0]
        assert picks[2 * c + 1] == order[c + c % (w * h - c)]   # the rest is still going
        assert pixel_picker_order(w, h).size == 2 * (w * h - c)


def test_4x4_by_hand():
    """Centre (1.5, 1.5): square_radius is 0.5 for the middle 2 x 2 and 1.5 around it, blend = ((x ^ y) % 4) * 2.
    Keys, row by row:
        y=0: 1+0=1  1+2=3  1+4=5  1+6=7        (x ^ 0 = 0, 1, 2, 3)
        y=1: 1+2=3  0+0=0  0+6=6  1+4=5        (x ^ 1 = 1, 0, 3, 2)
        y=2: 1+4=5  0+6=6  0+0=0  1+2=3        (x ^ 2 = 2, 3, 0, 1)
        y=3: 1+6=7  1+4=5  1+2=3  1+0=1        (x ^ 3 = 3, 2, 1, 0)
    Stable by key: 0: 5 10 | 1: 0 15 | 3: 1 4 11 14 | 5: 2 7 8 13 | 6: 6 9 | 7: 3 12.  central = 16 / 4 = 4:
    [5 10 0 15] and the rest [1 4 11 14 2 7 8 13 6 9 3 12]; cycle_length = 2 * 12 = 24."""
    assert sorted_pixels(4, 4) == [5, 10, 0, 15, 1, 4, 11, 14, 2, 7, 8, 13, 6, 9, 3, 12]
    want = [5, 1, 10, 4, 0, 11, 15, 14, 5, 2, 10, 7, 0, 8, 15, 13, 5, 6, 10, 9, 0, 3, 15, 12]
    assert list(pixel_picker_order(4, 4)) == want
    assert list(pixel_picker_order(4, 4, 26)) == want + [5, 1]


def test_5x3_by_hand():
    """Centre (2, 1).  Keys, row by row:
        y=0: 2+0=2  1+2=3  1+4=5  1+6=7  2+0=2   (x ^ 0 = 0 1 2 3 4)
        y=1: 2+2=4  1+0=1  0+6=6  1+4=5  2+2=4   (x ^ 1 = 1 0 3 2 5)
        y=2: 2+4=6  1+6=7  1+0=1  1+2=3  2+4=6   (x ^ 2 = 2 3 0 1 6)
    i.e. [2 3 5 7 2 | 4 1 6 5 4 | 6 7 1 3 6].  Stable by key: 1: 6 12 | 2: 0 4 | 3: 1 13 | 4: 5 9 | 5: 2 8 |
    6: 7 10 14 | 7: 3 11.  central = 15 / 4 = 3: [6 12 0], the rest [4 1 13 5 9 2 8 7 10 14 3 11];
    cycle_length = 2 * 12 = 24."""
    assert sorted_pixels(5, 3) == [6, 12, 0, 4, 1, 13, 5, 9, 2, 8, 7, 10, 14, 3, 11]
    want = [6, 4, 12, 1, 0, 13, 6, 5, 12, 9, 0, 2, 6, 8, 12, 7, 0, 10, 6, 14, 12, 3, 0, 11]
    assert list(pixel_picker_order(5, 3)) == want


def test_the_restatement_matches_the_scalar_sort():
    for w, h in [(7, 5), (33, 20), (64, 48)]:
        order = sorted_pixels(w, h)
        c = central_of(w, h)
        k = np.arange(3 * cycle_length_of(w, h))
        lin = np.where(k % 2 == 0, (k // 2) % c, c + (k // 2) % (w * h - c))
        assert np.array_equal(pixel_picker_order(w, h, k.size), np.array(order)[lin])


def test_consistent_picks_wrap():
    """UpdateStrategy::Consistent's point_from_pixel_index (:912-918): x = i rem_euclid w,
    y = (i div_euclid w) rem_euclid h, so the index wraps at w * h."""
    w, h = 5, 3
    i = np.arange(40, dtype=np.uint64)
    assert np.array_equal(aicb200.consistent_picks(w, h, 0, 40), (i % (w * h)).astype(np.uint32))
    start = 2 ** 40 + 7
    got = aicb200.consistent_picks(w, h, start, 4)
    assert list(got) == [((start + j) % w) + ((start + j) // w % h) * w for j in range(4)]
