"""CPU: cotr_workspace_bytes counts the device workspace the library allocates (DESIGN section 2)."""

KTOKENS = 512
STEM_CANVAS_HALVES = 262 * 264 * 4          # bordered NHWC4 stem canvas, per image and plane (common.cuh)


def _split16(elems):
    return 4 * elems                         # two fp16 planes


def _encode_bytes_per_pair():
    img = 2                                  # images per pair
    backbone = _split16(img * (STEM_CANVAS_HALVES + 128 * 128 * 64 + 3 * 64 * 64 * 256 + 64 * 64 * 128 + 64 * 64 * 64))
    tokens = _split16(KTOKENS * (4 * 256 + 512 + 1024)) + _split16(256 * 512)     # src xa xb ao, qk, ffh; v transposed
    f32 = 4 * KTOKENS * 256 + 2 * 8 * KTOKENS * 16                                # LayerNorm scratch, two row-statistics buffers
    images = 8 * 132096                                                            # attention operand images of 8 heads
    pair_table = 2 * 4
    assert backbone + tokens + f32 == 48481792
    return backbone + tokens + f32 + images + pair_table


def test_workspace_bytes_per_pair(built_lib):
    from cotr_b200 import capi
    ws = capi.lib().cotr_workspace_bytes
    # both shapes decode 32768 rows at a time, so the difference is one pair's encoder workspace
    assert ws(2, 16384) - ws(1, 32768) == _encode_bytes_per_pair() == 48481792 + 1056768 + 8


def test_workspace_bytes_rounds_decode_rows_to_8(built_lib):
    from cotr_b200 import capi
    ws = capi.lib().cotr_workspace_bytes
    per_row = _split16(8 * 256 + 1536 + 1024) + 4 * 256 + 2 * 8 * 16      # split16 rows, LayerNorm scratch, statistics
    assert ws(1, 8) - ws(1, 0) == 8 * per_row
    assert ws(1, 1) == ws(1, 8)
    assert ws(1, 9) - ws(1, 0) == 16 * per_row
