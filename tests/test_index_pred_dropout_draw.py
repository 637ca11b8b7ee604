"""CPU: the index-prediction heads' Dropout2d draws.  MultiHeadFCNHead calls ONE nn.Dropout2d module once per head, in
head order; the training node (index_pred_autograd) draws them as 18 successive parsing_gen_train.dropout2d_mask calls,
so that under the same seed it drops the channels the reference drops."""
import pytest
import torch
import torch.nn as nn


@pytest.mark.parametrize("B,C,p", [(2, 8, 0.1), (4, 64, 0.1)])
def test_eighteen_draws_are_one_dropout2d_applied_per_head(B, C, p):
    from text2human_b200.parsing_gen_train import dropout2d_mask
    drop = nn.Dropout2d(p).train()
    for seed in (0, 2021):
        torch.manual_seed(seed)
        masks = [dropout2d_mask(B, C, p, "cpu") for _ in range(18)]
        torch.manual_seed(seed)
        ys = [drop(torch.ones((B, C, 3, 2))) for _ in range(18)]
        for m, y in zip(masks, ys):
            assert torch.equal(m, (y[:, :, 0, 0] != 0).float())
            assert torch.equal(y, (m / (1.0 - p)).view(B, C, 1, 1).expand(B, C, 3, 2))
