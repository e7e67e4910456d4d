"""generate() with several prompts per image, without a GPU: the refusals of resolve_prompt_groups, the shared prefix length P,
and the per-row assembly (pred_boxes repeated per row, each row with its image's region count)."""
import pytest
import torch

from groma.model.groma import GromaModel, resolve_prompt_groups, rows_of_images, shared_prefix_len
from groma_b200 import ops as G


def test_one_row_per_image_is_the_plain_call():
    assert resolve_prompt_groups(4, 4) == 1
    # the plain call accepts what it accepted before, groups or not
    assert resolve_prompt_groups(3, 3, refer_boxes=[torch.zeros(1, 4)] * 3, kv_cache_dtype=torch.float8_e4m3fn, num_beams=4) == 1
    assert resolve_prompt_groups(6, 2) == 3


@pytest.mark.parametrize("rows,images", [(5, 2), (3, 4), (7, 3)])
def test_rows_not_a_multiple_of_images(rows, images):
    with pytest.raises(ValueError, match="not a multiple"):
        resolve_prompt_groups(rows, images)


def test_refusals():
    with pytest.raises(ValueError, match="refer_boxes / ground_boxes"):
        resolve_prompt_groups(4, 2, refer_boxes=[torch.zeros(1, 4)] * 4)
    with pytest.raises(ValueError, match="refer_boxes / ground_boxes"):
        resolve_prompt_groups(4, 2, ground_boxes=[torch.zeros(1, 4)] * 4)
    with pytest.raises(ValueError, match="bf16 KV cache"):
        resolve_prompt_groups(4, 2, kv_cache_dtype=torch.float8_e4m3fn)
    with pytest.raises(ValueError, match="limit of 64"):
        resolve_prompt_groups(65, 1)
    assert resolve_prompt_groups(64, 1) == 64
    with pytest.raises(ValueError, match="256 rows"):
        resolve_prompt_groups(320, 5)
    assert resolve_prompt_groups(256, 4) == 64
    with pytest.raises(NotImplementedError, match="num_beams > 1"):
        resolve_prompt_groups(4, 2, num_beams=2)
    assert resolve_prompt_groups(4, 2, num_beams=1) == 2
    assert G.GROUP_MAX_PROMPTS == 64


def test_limits_match_the_header():
    from groma_b200.lib import HEADER
    text = HEADER.read_text()
    assert "#define GROMA_GROUP_MAX_PROMPTS 64" in text
    assert "groma_decode_rope_attention_grouped" in text


PAD = 0


def test_prefix_of_identical_prompts_is_capped():
    ids = torch.tensor([[5, 6, 7, 8]] * 3 + [[5, 6, 9, 9]] * 3)
    # image 0: identical rows -> 4, capped at T - 1 = 3; image 1 likewise
    assert shared_prefix_len(ids, 3) == 3


def test_prefix_min_over_images():
    ids = torch.tensor([[5, 6, 7, 8, 1],
                        [5, 6, 7, 9, 1],
                        [5, 6, 1, 1, 1],
                        [5, 7, 1, 1, 1]])
    assert shared_prefix_len(ids, 2) == 1      # image 0 shares 3, image 1 shares 1
    assert shared_prefix_len(ids[:2], 2) == 3


def test_prefix_zero():
    ids = torch.tensor([[5, 6, 7], [4, 6, 7]])
    assert shared_prefix_len(ids, 2) == 0


def test_prompts_differing_only_in_padding():
    # row 1 is row 0 cut short: they agree up to row 1's first pad
    ids = torch.tensor([[5, 6, 7, 8, 9], [5, 6, 7, PAD, PAD]])
    assert shared_prefix_len(ids, 2) == 3
    # both padded the same way: identical rows, capped
    ids = torch.tensor([[5, 6, 7, PAD, PAD], [5, 6, 7, PAD, PAD]])
    assert shared_prefix_len(ids, 2) == 4




def _bare_model():
    """A GromaModel shell with the special token ids only: _assemble is host-side integer bookkeeping."""
    m = GromaModel.__new__(GromaModel)
    torch.nn.Module.__init__(m)
    m.pad_token_id, m.img_token_id, m.reg_token_id = PAD, 100, 101
    m.box_idx_token_ids = list(range(200, 240))
    return m


def test_assembled_rows_and_prefix_with_different_region_counts():
    m = _bare_model()
    n, n_img = 3, 4
    q = [[50, 51], [50, 52], [53, PAD]]
    rows = [[10, 11, 100, 12, 101, 13] + t for t in q] * 2
    ids = torch.tensor(rows)
    sel = [torch.zeros(2, 4), torch.zeros(5, 4)]
    counts = [len(sel[i // n]) for i in range(2 * n)]
    out, _ = m._assemble(ids.clone(), None, counts, n_img)
    # every row of image 0 carries 2 regions, of image 1 five; the rows are padded to the longest
    assert out.shape == (2 * n, 2 + n_img + 1 + 2 * 5 + 1 + 2)
    for i in range(2 * n):
        assert int((out[i] == 101).sum()) == counts[i]
    # image 0's rows diverge right after its 2 regions; image 1's after its 5: P is image 0's
    P = shared_prefix_len(out, n)
    assert P == 2 + n_img + 1 + 2 * 2 + 1
    assert shared_prefix_len(out[n:], n) == 2 + n_img + 1 + 2 * 5 + 1


def test_pred_boxes_repeat_per_row():
    """generate()'s hidden_states pred_boxes: row i gets image i // n's selection (the eval scripts index pred_boxes[row])."""
    sel = [torch.rand(3, 4), torch.rand(6, 4)]
    n = 4
    rows = rows_of_images(sel, n)
    assert len(rows) == 8
    assert all(rows[i] is sel[0] for i in range(4)) and all(rows[i] is sel[1] for i in range(4, 8))
