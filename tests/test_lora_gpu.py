"""Sampling with a merged LoRA adapter (-m gpu): the merged model's native forward against the oracle on the merged weights,
exact merge of a zero adapter, bitwise unmerge, and the refusal of a forward with an unmerged adapter."""
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _merged_case():
    from oracle import pixart_oracle as po
    from pixart_sigma_b200 import PixArtMS
    cfg = po.OracleConfig(depth=2, input_size=32, pe_interpolation=0.5)
    sd = po.synthetic_state_dict(cfg, seed=0)
    with torch.device(DEV):
        m = PixArtMS(depth=2, input_size=32, pe_interpolation=0.5, model_max_length=300)
    m.load_state_dict(sd, strict=False)
    m = m.to(torch.bfloat16).eval()
    m.output_dtype = torch.float32
    x, t, y, mask = po.synthetic_inputs(cfg, 2, (32, 32), lens=[300, 77])
    return po, cfg, sd, m, (x.to(DEV), t.to(DEV), y.to(DEV), mask.to(DEV))


def test_merged_forward_matches_oracle_and_unmerge_restores():
    """The merged model's native forward against the oracle on the merged weights; a zero B merges to the base weights
    exactly (same forward, bit for bit); unmerge restores the weights bit for bit; an unmerged adapter makes the forward
    raise."""
    from pixart_sigma_b200 import lora
    po, cfg, sd, m, (x, t, y, mask) = _merged_case()
    with torch.no_grad():
        base = m(x, t, y, mask=mask)
    w_before = {k: v.clone() for k, v in m.state_dict().items()}
    lora.inject_lora(m, 16, generator=torch.Generator().manual_seed(4))
    with torch.no_grad(), pytest.raises(RuntimeError, match="merge_lora"):
        m(x, t, y, mask=mask)
    lora.merge_lora(m)                                       # B = 0 at init: the merge is exact
    with torch.no_grad():
        assert torch.equal(m(x, t, y, mask=mask), base)
    lora.unmerge_lora(m)
    with torch.no_grad():
        for mod in m.modules():
            if hasattr(mod, "lora_B"):
                mod.lora_B.normal_(std=0.02, generator=torch.Generator(DEV).manual_seed(5))
    lora.merge_lora(m)
    with torch.no_grad():
        got = m(x, t, y, mask=mask).cpu()
    msd = m.state_dict()
    merged = {k: (msd[k] if k in msd else v).to(torch.bfloat16).float().cpu() for k, v in sd.items()}
    want = po.forward(merged, cfg, x.cpu().to(torch.bfloat16).float(), t.cpu(), y.cpu().to(torch.bfloat16).float(),
                      mask=mask.cpu())
    err = po.rel_err(got, want)
    moved = po.rel_err(got, base.cpu())
    print(f"merged forward: rel_err vs oracle {err:.3e}; the adapter moved the output by {moved:.3e}")
    assert err < 1e-2 and moved > 10 * err
    lora.unmerge_lora(m)
    after = m.state_dict()
    assert all(torch.equal(after[k], v) for k, v in w_before.items())
    with torch.no_grad(), pytest.raises(RuntimeError, match="merge_lora"):
        m(x, t, y, mask=mask)


def test_graphed_forward_with_merged_adapter():
    """A GraphedForward captured on the base model refuses to replay once an unmerged adapter is attached, and after the
    merge its replays equal the eager merged forward."""
    from pixart_sigma_b200 import lora
    from pixart_sigma_b200.graph import GraphedForward
    _, _, _, m, (x, t, y, mask) = _merged_case()
    y, mask = y.to(torch.bfloat16), mask.long()              # the graph's static input dtypes
    gf = GraphedForward(m, "forward")
    with torch.no_grad():
        base = m(x, t, y, mask=mask)
    assert torch.equal(gf(x, t, y, mask), base)
    lora.inject_lora(m, 8, generator=torch.Generator().manual_seed(6))
    with pytest.raises(RuntimeError, match="merge_lora"):
        gf(x, t, y, mask)
    with torch.no_grad():
        for mod in m.modules():
            if hasattr(mod, "lora_B"):
                mod.lora_B.normal_(std=0.02, generator=torch.Generator(DEV).manual_seed(7))
    lora.merge_lora(m)
    with torch.no_grad():
        eager = m(x, t, y, mask=mask)
    assert not torch.equal(eager, base)
    assert torch.equal(gf(x, t, y, mask), eager) and torch.equal(gf(x, t, y, mask), eager)
