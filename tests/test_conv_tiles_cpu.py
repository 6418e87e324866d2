"""Tile choice of the convolution launches at the benchmark's 1080p shapes (output sides 544 x 960 at 1/2 resolution
down to 68 x 120 at 1/16): flat pixel tiles exactly at 1/16, the rectangles everywhere else, and the channel tile
that fills the waves of 132 SMs.  No GPU needed."""
from deva.model import native_ops as ops

SMS = 132
# the rectangles each resolution took before flat tiles existed (all exact fits except 1/16)
RECT = {(544, 960): (2, 64), (272, 480): (4, 32), (136, 240): (8, 16), (68, 120): (1, 128)}


def test_flat_tiles_exactly_at_one_sixteenth():
    for (ho, wo), rect in RECT.items():
        for stride in (1, 2):
            want = ops.FLAT if ((ho, wo) == (68, 120) and stride == 1) else rect
            assert ops.choose_tile(ho, wo, stride=stride) == want, (ho, wo, stride)
        assert ops.choose_tile(ho, wo, pool4=True) != ops.FLAT
    assert ops.choose_tile(68, 120, pool4=True) == (4, 32)
    assert ops.pixel_tiles(68, 120, ops.FLAT) == 64 and ops.pixel_tiles(68, 120, (1, 128)) == 68
    assert ops.choose_tile(30, 54) == ops.FLAT and ops.pixel_tiles(30, 54, ops.FLAT) == 13
    assert ops.choose_tile(32, 64) == (2, 64)  # an exact fit keeps its rectangle


def _units(b, ho, wo, cout_pad, nt, ksplit=1):
    return b * ops.pixel_tiles(ho, wo, ops.choose_tile(ho, wo)) * (cout_pad // nt) * ksplit


def _waves(units):
    return -(-units // SMS)


def test_batch1_sixteenth_launches():
    m = ops.pixel_tiles(68, 120, ops.choose_tile(68, 120))
    # layer3 c1 / c2 (256 channels): 64 units of 256 on 64 SMs -> 128 units of 128, one wave
    assert _units(1, 68, 120, 256, 256) == 64
    assert ops.choose_nt(256, 256, m, 1, SMS) == 128 and _units(1, 68, 120, 256, 128) == 128
    # proj1 / proj2 / fuser c1_x (512 channels): 128 units, one wave (136 and two waves with (1, 128) rectangles)
    assert ops.choose_nt(256, 512, m, 1, SMS) == 256 and _units(1, 68, 120, 512, 256) == 128
    # layer3 c3 (1024 channels) and the precise c2's 4 split-K chains: 256 units, two waves at 97 %
    assert ops.choose_nt(256, 1024, m, 1, SMS) == 256 and _units(1, 68, 120, 1024, 256) == 256
    assert ops.choose_nt(256, 256, m, 4, SMS) == 256 and _units(1, 68, 120, 256, 256, 4) == 256
    assert _waves(256) == 2 and 256 / (2 * SMS) > 0.96


def test_wide_launches_keep_their_channel_tile():
    # batch-16 launches at every resolution are many waves: the packed tile stays
    for (ho, wo) in RECT:
        for cout in (256, 512, 1024):
            m = 16 * ops.pixel_tiles(ho, wo, ops.choose_tile(ho, wo))
            assert ops.choose_nt(256, cout, m, 1, SMS) == 256, (ho, wo, cout)
    assert _units(16, 68, 120, 256, 256) == 1024  # 1088 with (1, 128) rectangles
    # batch-1 launches at 1/2 .. 1/8 resolution are four or more waves
    for (ho, wo) in ((544, 960), (272, 480), (136, 240)):
        m = ops.pixel_tiles(ho, wo, ops.choose_tile(ho, wo))
        for cout in (64, 128, 256, 512):
            nt = 256 if cout >= 256 else cout
            assert ops.choose_nt(nt, cout, m, 1, SMS) == nt, (ho, wo, cout)
    # ragged tiles (odd Cout, 160-wide) stay
    assert ops.choose_nt(160, 160, 64, 1, SMS) == 160


def test_narrower_tile_ties_go_to_the_wider():
    # 64 pixel tiles x 512 channels: 256 -> 128 units in one wave, 128 -> 256 units in two: same modelled time
    assert ops.choose_nt(256, 512, 64, 1, SMS) == 256
    # 128 channels at batch 1: 64 units of 128 or 128 units of 64, both one wave: 64 halves it
    assert ops.choose_nt(128, 128, 64, 1, SMS) == 64
