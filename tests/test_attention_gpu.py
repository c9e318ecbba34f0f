"""Attention forward (csrc/attention_tc.cu) in the persistent regime and on crafted softmax inputs, against an fp64 reference
of the same bf16 inputs with the elementwise bounds derived in kernel_ref.attention_reference.

The kernel is persistent: min(items, SM count) CTAs, item = (image, head, pair of 128-query tiles), and barrier phases, the
double-buffered Q tile and the K/V ring carry over from one item of a CTA to the next.  The shapes below are scaled from the
device's SM count so that CTAs run several items (and one case exactly SM + 1), and each case asserts that it does.
"""
import pytest
import torch

from kernel_ref import ATT_KVTILE, attention_items, check_attention, crafted_qkv

pytestmark = pytest.mark.gpu


def sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def n_pairs(N):
    return (-(-N // 128) + 1) // 2


def batch_for(N, H, min_batch, per_cta=3):
    """The smallest batch >= min_batch whose item count gives every CTA at least `per_cta` items."""
    return max(min_batch, -(-per_cta * sm_count() // (n_pairs(N) * H)))


# (name, N, H, batch as a function of the SM count, items per CTA at least)
PERSISTENT = [
    ("vit_b_197", 197, 12, lambda sm: batch_for(197, 12, 64), 3),
    ("vit_l_577", 577, 16, lambda sm: batch_for(577, 16, 16), 3),   # three pairs: every third item holds one query tile
    ("one_tile_sm_plus_1", 128, 1, lambda sm: sm + 1, None),         # one CTA runs two items; warpgroup 1 idles in every item
    ("one_token", 1, 1, lambda sm: batch_for(1, 1, 3 * sm + 4), 3),
    ("pair2_one_row", 257, 8, lambda sm: batch_for(257, 8, 33), 3),  # the second pair is one tile holding one row
]


@pytest.mark.parametrize("name,N,H,batch,per_cta", PERSISTENT, ids=[c[0] for c in PERSISTENT])
def test_attention_persistent_matches_fp64(lib, name, N, H, batch, per_cta):
    """Random q, k, v (1.5 randn, bf16) at item counts above the SM count; out and lse2 within kernel_ref's bounds, guards
    untouched."""
    sm = sm_count()
    B = batch(sm)
    items, grid = attention_items(B, N, H, sm)
    if per_cta is None:
        assert items == sm + 1 and grid == sm
    else:
        assert items >= per_cta * grid and grid == sm, (items, grid)
    torch.manual_seed(N * 31 + H)
    qkv = (torch.randn(B, N, 3, H, 64, device="cuda") * 1.5).to(torch.bfloat16)
    check_attention(lib, qkv)


def test_attention_long_sequence_wraps_the_kv_ring(lib):
    """2049 tokens: 33 key tiles stream through the four-stage K/V ring of one item (eight wraps), and the last tile holds one
    key."""
    B, N, H = 2, 2049, 3
    assert -(-N // ATT_KVTILE) == 33
    torch.manual_seed(2049)
    qkv = (torch.randn(B, N, 3, H, 64, device="cuda") * 1.5).to(torch.bfloat16)
    check_attention(lib, qkv)


def _tiles(N, fn):
    j = torch.arange(N, device="cuda")
    return fn(j // ATT_KVTILE, j).float()


# A rescale happens when a row's maximum exceeds the reference by more than 8 in log2 units, i.e. 8 * 8 / log2(e) = 44.4
# raw score units (scores are scaled by 1/8).
CRAFTED = [
    # every key tile 48 raw units above the last: alpha 0.9375 grows 45 (8.11 log2: rescale each tile), 0.90625 grows 43.5
    # (7.85: the stale reference stands for a tile, P up to 2^7.85), 0 = all-equal scores (out = mean of v), -0.5 falls
    ("grow_below_and_above_8", 577, [0.90625, 0.9375, 0.0, -0.5], lambda t, j: 48.0 * t),
    # the ragged last tile jumps by 1000: alpha = 2^-180 underflows to 0 (alpha 1), 31 units stay below the rescale threshold
    # (1/32), -1 sends the last tile's P to exact 0
    ("jump_1000_in_last_tile", 197, [1.0, 0.03125, 0.0, -1.0], lambda t, j: torch.where(t == 3, 1000.0, 0.0)),
    # maximum in the first tile, every later score about 1000 lower: P underflows to exact 0 (alpha 1) or to 2^-90 (1/2)
    ("max_in_first_tile", 257, [1.0, 0.5, 0.0, 0.0078125], lambda t, j: torch.where(t == 0, 0.0, -1000.0)),
    # the only large score is token N-1, alone in the ragged last tile: 64 units (rescale), 32 (none), 256 (P of the rest 2^-46)
    ("max_at_last_token", 197, [1.0, 0.5, 4.0, 0.0], lambda t, j: torch.where(j == 196, 64.0, 0.0)),
]


@pytest.mark.parametrize("name,N,alphas,beta", CRAFTED, ids=[c[0] for c in CRAFTED])
def test_attention_crafted_softmax_matches_fp64(lib, name, N, alphas, beta):
    """Exact crafted scores with random v, at >= 3 items per CTA; out and lse2 within kernel_ref's bounds."""
    H = 2
    sm = sm_count()
    B = batch_for(N, H, 1)
    items, grid = attention_items(B, N, H, sm)
    assert items >= 3 * grid and grid == sm
    qkv = crafted_qkv(B, N, H, alphas, _tiles(N, beta), seed=N)
    check_attention(lib, qkv)
