"""Launches of the exact convolution sweep (tests/test_conv_exact_gpu.py): a pairwise covering list, not the full product,
of filter size, stride (odd sides: the four stride-2 phase maps of unequal size), pixel tile (all six rectangles and
flat), channel tile (64 / 128 / 192 / 256 dividing cout_pad, and the ragged tiles of Cout 1, 33 and 129), images smaller
than a tile, ragged edges, grids with more work units than SMs, every operand mode and epilogue, and split-K chains.

Each case: batch b, input h x w, cin_pad, cout, filter k, stride s, tile ('flat' or (th, tw)), channel tile nt,
mode (operand passes: 'plain', 'x2', 'x_lo', 'w_lo' = split_mode 2, 'lo8' = split_mode 3), outs (requested outputs),
and optional extras: rank1, res ('own' / 'broadcast'), res_lo, head_n, gates, pool4, ksplit, g (the finest operand
grid is 2^-g; 10 unless the fused head's sums need a coarser one), sparse (one weight in 64 nonzero and activations
in {-1, 0, 1}, so that the gates' pre-activations stay where sigmoid and tanh are not flat).
cout_pad is cout rounded up to nt."""

RAW4 = ('raw', 'raw_lo', 'relu', 'relu_lo')


def _c(b, h, w, cin_pad, cout, k, s, tile, nt, mode='plain', outs=('raw',), **extra):
    return dict(b=b, h=h, w=w, cin_pad=cin_pad, cout=cout, k=k, s=s, tile=tile, nt=nt, mode=mode, outs=tuple(outs),
                **extra)


CASES = {
    # filter size x pixel tile x channel tile, plain passes
    'k1_flat_nt256': _c(2, 17, 23, 64, 256, 1, 1, 'flat', 256, outs=('raw', 'relu', 'f32')),
    'k3_r1x128_nt128': _c(1, 5, 130, 128, 256, 3, 1, (1, 128), 128),
    'k3_flat_nt64_edges': _c(2, 9, 70, 64, 128, 3, 1, 'flat', 64, outs=('relu',)),
    # stride 2 on odd sides, and images smaller than a tile (1 x 1, 1 x 200, 3 x 5).  An input one row high or one
    # column wide has no odd phase; its taps read phase 0's rows instead of the padding until conv.cu moved their
    # boxes out of the image (the three s2_image cases of one row or column failed before)
    'k3_s2_odd_r2x64': _c(2, 9, 13, 64, 64, 3, 2, (2, 64), 64, outs=('raw', 'relu', 'f32')),
    'k1_s2_odd_r4x32': _c(1, 15, 21, 128, 128, 1, 2, (4, 32), 128),
    's2_image_1x1': _c(3, 1, 1, 64, 64, 3, 2, (4, 32), 64, outs=('raw', 'f32')),
    's2_image_1x200': _c(1, 1, 200, 64, 128, 3, 2, (1, 128), 128, outs=('raw',)),
    's2_image_200x1': _c(1, 200, 1, 64, 64, 3, 2, (32, 4), 64, outs=('raw',)),
    's2_image_3x5_nt192': _c(2, 3, 5, 64, 192, 3, 2, (8, 16), 192),
    's1_image_1x1': _c(2, 1, 1, 128, 64, 3, 1, (16, 8), 64, outs=('raw', 'relu')),
    's1_image_1x200_flat': _c(1, 1, 200, 64, 64, 3, 1, 'flat', 64),
    # operand modes
    'x2_r4x32_nt192': _c(2, 11, 37, 128, 192, 3, 1, (4, 32), 192, 'x2', ('raw', 'relu')),
    'x_lo_r8x16': _c(2, 19, 21, 64, 128, 3, 1, (8, 16), 128, 'x_lo', RAW4),
    'x_lo_s2_r16x8': _c(1, 17, 15, 128, 64, 3, 2, (16, 8), 64, 'x_lo', ('f32',)),
    'w_lo_rank1_r32x4': _c(3, 33, 7, 128, 256, 1, 1, (32, 4), 256, 'w_lo', ('raw', 'relu', 'f32'), rank1=True),
    'rank1_flat_nt64': _c(2, 13, 19, 64, 128, 1, 1, 'flat', 64, outs=('raw', 'relu'), rank1=True),
    'lo8_flat': _c(1, 13, 20, 128, 128, 3, 1, 'flat', 128, 'lo8', ('relu', 'relu_lo8')),
    'lo8_res_lo_r2x64': _c(2, 9, 70, 256, 64, 3, 1, (2, 64), 64, 'lo8', ('raw', 'relu', 'relu_lo8'), res='own',
                           res_lo=True),
    # residuals: own and broadcast, with and without the low-order part
    'res_own_lo_flat_nt64': _c(2, 10, 30, 64, 128, 3, 1, 'flat', 64, outs=('raw', 'raw_lo', 'relu'), res='own',
                               res_lo=True),
    'res_own_r4x32': _c(2, 7, 9, 64, 256, 1, 1, (4, 32), 256, res='own'),
    'res_broadcast_lo_r1x128': _c(4, 6, 50, 64, 64, 3, 1, (1, 128), 64, outs=RAW4, res='broadcast', res_lo=True),
    'res_broadcast_flat_nt192': _c(3, 5, 40, 128, 192, 3, 1, 'flat', 192, outs=('relu',), res='broadcast'),
    'res_broadcast_lo_f32': _c(3, 6, 11, 64, 33, 3, 1, (8, 16), 64, outs=('raw', 'f32'), res='broadcast', res_lo=True),
    # fused head at N = 64 .. 256, with the 4x4 pool and the parity plan's operands
    'head64_r8x16': _c(2, 8, 16, 64, 64, 3, 1, (8, 16), 64, outs=('relu',), head_n=9, g=4),
    'head128_pool4_lo8_res': _c(2, 16, 32, 128, 128, 3, 1, (4, 32), 128, 'lo8', (), head_n=9, pool4=True,
                                res='own', res_lo=True, g=4),
    'head192_r16x8': _c(1, 12, 20, 64, 192, 1, 1, (16, 8), 192, head_n=3, g=4),
    'head256_flat': _c(1, 4, 40, 64, 256, 3, 1, 'flat', 256, outs=('relu', 'relu_lo'), head_n=1, g=4),
    # gates, pool4
    'gates_r8x16': _c(2, 9, 11, 64, 384, 3, 1, (8, 16), 192, 'x2', (), gates=True, sparse=True),
    'gates_flat': _c(1, 5, 40, 128, 192, 3, 1, 'flat', 192, 'x2', (), gates=True, sparse=True),
    'pool4_raw_r8x16': _c(2, 8, 24, 64, 128, 3, 1, (8, 16), 128, pool4=True),
    'pool4_only_r4x32_s2': _c(1, 16, 64, 64, 64, 3, 2, (4, 32), 64, outs=(), pool4=True),
    # ragged Cout: 1 (nt 32), 33 (nt 64), 129 (nt 160 -> wgmma width 192)
    'cout1': _c(2, 7, 9, 64, 1, 3, 1, (2, 64), 32, outs=('raw', 'relu', 'f32')),
    'cout33_x_lo': _c(2, 13, 17, 128, 33, 1, 1, (4, 32), 64, 'x_lo', RAW4 + ('f32',)),
    'cout129_nt160': _c(1, 11, 15, 64, 129, 3, 1, 'flat', 160, outs=('raw', 'relu', 'f32')),
    # more work units than SMs: 320 units
    'units_320_r8x16': _c(4, 40, 60, 64, 256, 3, 1, (8, 16), 64, outs=('relu',)),
    # split-K: chains of 11 of 54 k-iterations (boundaries inside a tap); 20 asked of 54 -> chains of 3 -> 18;
    # 7 asked of 36 -> chains of 6 -> 6
    'splitk_in_tap': _c(1, 9, 17, 128, 129, 3, 1, (4, 32), 160, 'x_lo', ('f32',), ksplit=5),
    'splitk_trailing_s2': _c(1, 13, 11, 128, 64, 3, 2, (8, 16), 64, 'x_lo', ('f32',), ksplit=20),
    'splitk_plain_flat': _c(2, 10, 12, 256, 256, 3, 1, 'flat', 128, 'plain', ('f32',), ksplit=7),
}

# chains each split-K case must produce
SPLIT_PARTS = {'splitk_in_tap': 5, 'splitk_trailing_s2': 18, 'splitk_plain_flat': 6}
