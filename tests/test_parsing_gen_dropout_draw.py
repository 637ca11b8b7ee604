"""CPU: the parsing generator's Dropout2d draw (parsing_gen_train.dropout2d_mask, used by ParsingGenTrainer and by the
FCNHead autograd node) is nn.Dropout2d's: under the same seed it drops the same channels as F.dropout2d."""
import pytest
import torch
import torch.nn.functional as F


@pytest.mark.parametrize("B,C,p", [(2, 8, 0.1), (8, 64, 0.1), (3, 5, 0.5)])
def test_dropout2d_mask_is_f_dropout2d_draw(B, C, p):
    from text2human_b200.parsing_gen_train import dropout2d_mask
    for seed in (0, 2021):
        torch.manual_seed(seed)
        mask = dropout2d_mask(B, C, p, "cpu")
        torch.manual_seed(seed)
        y = F.dropout2d(torch.ones((B, C, 3, 2)), p, training=True)
        want = (y[:, :, 0, 0] != 0).float()
        assert torch.equal(mask, want)
        assert torch.equal(y, (mask / (1.0 - p)).view(B, C, 1, 1).expand(B, C, 3, 2))
    g1, g2 = torch.Generator().manual_seed(5), torch.Generator().manual_seed(5)
    assert torch.equal(dropout2d_mask(B, C, p, "cpu", g1), dropout2d_mask(B, C, p, "cpu", g2))
