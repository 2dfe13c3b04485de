"""CPU tests of the CAME optimizer and gradient clipping: known answers of the plain-torch restatement (oracle/came_oracle.py),
the parameter table `FlatCAME` builds from a reducer at XL/2 size, the C-ABI structs, and the conversion to / from the
torch.optim checkpoint layout."""
import ctypes
import os
import subprocess
import tempfile

import pytest
import torch

from oracle import came_oracle as co
from pixart_sigma_b200 import PixArtMS_XL_2, lib
from pixart_sigma_b200.optim import FlatCAME, came_layout
from pixart_sigma_b200.parallel import GradBucketReducer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(p0, grads, steps=1, **kw):
    p = p0.clone()
    st = [{}]
    for k in range(steps):
        co.came_step([p], [grads[k % len(grads)].clone()], st, **kw)
    return p, st[0]


def test_rank_one_second_moment_factors_exactly():
    """For a rank-1 g^2 (g = a b^T) the factored estimate row[r] col[c] / mean(row) equals the unfactored second moment, so the
    first moment of a matrix equals that of the same values stepped as one 1-D parameter."""
    g = torch.Generator().manual_seed(0)
    a, b = torch.randn(7, 1, generator=g, dtype=torch.float64), torch.randn(1, 9, generator=g, dtype=torch.float64)
    grad = a * b
    p0 = torch.randn(7, 9, generator=g, dtype=torch.float64)
    _, st2 = _run(p0, [grad], eps=(0.0, 1e-16))
    _, st1 = _run(p0.flatten(), [grad.flatten()], eps=(0.0, 1e-16))
    assert torch.allclose(st2["exp_avg"].flatten(), st1["exp_avg"], rtol=1e-12, atol=0)


@pytest.mark.parametrize("shape", [(1, 11), (11, 1)])
def test_single_row_and_single_column_matrices_reduce_to_the_unfactored_rule(shape):
    """R = 1: row / mean(row) = 1; C = 1: rsqrt(row / mean row) rsqrt(col) = rsqrt(row).  Either way the second-moment part
    equals the 1-D rule, so exp_avg matches the flattened parameter over several steps; the update differs only by the
    factored instability statistics."""
    g = torch.Generator().manual_seed(1)
    grads = [torch.randn(shape, generator=g, dtype=torch.float64) for _ in range(3)]
    p0 = torch.randn(shape, generator=g, dtype=torch.float64)
    _, st2 = _run(p0, grads, steps=3)
    _, st1 = _run(p0.flatten(), [x.flatten() for x in grads], steps=3)
    assert torch.allclose(st2["exp_avg"].flatten(), st1["exp_avg"], rtol=1e-12, atol=0)
    assert st2["exp_avg_sq_row"].shape == shape[:1] and st2["exp_avg_sq_col"].shape == shape[1:]


def test_zero_gradient_gives_finite_state_and_no_update():
    for shape in [(5, 6), (6,), (3, 2, 2, 2)]:
        p0 = torch.randn(shape)
        p, st = _run(p0, [torch.zeros(shape)], steps=3)
        assert torch.equal(p, p0), shape
        for k, v in st.items():
            if torch.is_tensor(v):
                assert torch.isfinite(v).all(), (shape, k)


def test_four_d_parameter_factors_per_leading_index():
    """A (3, 2, 5, 7) parameter is 6 independent 5 x 7 matrices (the clip RMS, which spans the whole tensor, is switched off)."""
    g = torch.Generator().manual_seed(2)
    grads = [torch.randn(3, 2, 5, 7, generator=g, dtype=torch.float64) for _ in range(2)]
    p0 = torch.randn(3, 2, 5, 7, generator=g, dtype=torch.float64)
    p, st = _run(p0, grads, steps=2, clip_threshold=1e30, weight_decay=0.1, lr=1e-2)
    assert st["exp_avg_sq_row"].shape == (3, 2, 5) and st["exp_avg_res_col"].shape == (3, 2, 7)
    for i in range(3):
        for j in range(2):
            pm, sm = _run(p0[i, j], [x[i, j] for x in grads], steps=2, clip_threshold=1e30, weight_decay=0.1, lr=1e-2)
            assert torch.allclose(p[i, j], pm, rtol=1e-13, atol=0)
            for k in ("exp_avg", "exp_avg_sq_row", "exp_avg_sq_col", "exp_avg_res_row", "exp_avg_res_col"):
                assert torch.allclose(st[k][i, j], sm[k], rtol=1e-13, atol=0), k


@pytest.mark.parametrize("shape", [(64,), (16, 24)])
def test_update_clipping_engages_on_the_first_step(shape):
    """From zero state with b2 = 0.999 the normalised update is |g| / sqrt(1e-3 g^2) ~ 31.6 per element, so the RMS clip
    (threshold 1) engages and exp_avg = (1 - b1) * u with RMS(u) = 1."""
    g = torch.Generator().manual_seed(3)
    grad = torch.randn(shape, generator=g, dtype=torch.float64)
    _, st = _run(torch.zeros(shape, dtype=torch.float64), [grad])
    rms_u = (st["exp_avg"] / (1 - 0.9)).norm() / st["exp_avg"].numel() ** 0.5
    assert abs(rms_u.item() - 1.0) < 1e-9


@pytest.mark.parametrize("max_norm,grad_scale", [(0.01, 1.0), (1e6, 1.0), (0.5, 0.25), (1e6, 0.25)])
def test_clip_grad_norm_oracle_matches_torch(max_norm, grad_scale):
    g = torch.Generator().manual_seed(4)
    ps = [torch.nn.Parameter(torch.randn(s, generator=g)) for s in [(5, 7), (13,), (2, 3, 4)]]
    for p in ps:
        p.grad = torch.randn(p.shape, generator=g)
    mine = [p.grad.clone() for p in ps]
    for p in ps:
        p.grad.mul_(grad_scale)
    want = torch.nn.utils.clip_grad_norm_(ps, max_norm)
    got = co.clip_grad_norm(mine, max_norm, grad_scale)
    assert torch.allclose(got, want, rtol=1e-6)
    for a, p in zip(mine, ps):
        assert torch.allclose(a, p.grad, rtol=1e-6, atol=0)


def _meta_xl(**kw):
    return PixArtMS_XL_2(input_size=128, **kw).to("meta")


@pytest.mark.parametrize("kv", [False, True])
def test_parameter_table_over_the_xl_model(kv):
    kw = dict(kv_compress_config=dict(sampling="conv", scale_factor=2, kv_compress_layer=list(range(28)))) if kv else {}
    model = _meta_xl(**kw)
    red = GradBucketReducer(model)
    entries, tot = came_layout(red)
    params = [p for b in red.buckets for p in b["params"]]
    assert len(entries) == len(params) == sum(1 for p in model.parameters() if p.requires_grad)
    row = col = vec = 0
    for bi, b in enumerate(red.buckets):
        mine = [(e, p) for e, p in zip(entries, params) if e["bucket"] == bi]
        off = 0
        for e, p in mine:
            assert e["offset"] == off and e["numel"] == p.numel()                 # back to back, no overlap
            if p.dim() >= 2:
                assert (e["R"], e["C"]) == tuple(p.shape[-2:]) and e["lead"] * e["R"] * e["C"] == p.numel()
                assert e["sq_off"] == row and e["col_off"] == col
                row, col = row + e["lead"] * e["R"], col + e["lead"] * e["C"]
            else:
                assert (e["lead"], e["R"], e["C"]) == (1, 1, p.numel()) and e["sq_off"] == vec
                vec += p.numel()
            off += p.numel()
        assert off <= b["flat"].numel() < off + 4 and all(e["bucket_numel"] == b["flat"].numel() for e, _ in mine)
    assert tot == dict(n_row=row, n_col=col, n_vec=vec)
    shapes = {(e["lead"], e["R"], e["C"]) for e in entries if e["factored"]}
    assert {(4608, 2, 2), (1, 6, 1152), (1, 4608, 1152), (1, 1152, 4608), (1, 6912, 1152)} <= shapes
    assert ((1152, 2, 2) in shapes) == kv                                       # attn.sr.weight (1152, 1, 2, 2)

    # the library plans the table on the host (no device needed) and rejects an entry that overruns its bucket
    table = (lib.CameParam * len(entries))()
    for t, e in zip(table, entries):
        t.param = t.grad = t.exp_avg = 16 * (1 + e["offset"])
        for k in ("numel", "offset", "bucket_numel", "sq_off", "col_off", "lead", "R", "C", "factored"):
            setattr(t, k, e[k])
    args = lib.CameArgs(n_vec=vec, n_row=row, n_col=col)
    nbytes = lib.came_plan(args, table)
    assert nbytes > 0 and args.n_tiles > 0 and args.n_fin > 0 and args.ws_floats * 4 == nbytes
    begins = [t.tile_begin for t in table]
    assert begins == sorted(begins) and table[0].tile_begin == 0
    last = entries[-1]
    table[len(entries) - 1].numel = last["bucket_numel"] - last["offset"] + 1
    with pytest.raises(lib.PxaError, match="numel|overrun"):
        lib.came_plan(args, table)


def test_came_structs_match_header_sizes():
    src = ('#include <stdio.h>\n#include "pixart_sm100.h"\nint main(){printf("%zu %zu %zu %zu\\n", sizeof(PxaGradBucket), '
           'sizeof(PxaGradClipArgs), sizeof(PxaCameParam), sizeof(PxaCameArgs));return 0;}\n')
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "s.c"), "w").write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), os.path.join(d, "s.c"), "-o", os.path.join(d, "s")])
        sizes = [int(v) for v in subprocess.check_output([os.path.join(d, "s")]).split()]
    assert sizes == [ctypes.sizeof(lib.GradBucket), ctypes.sizeof(lib.GradClipArgs), ctypes.sizeof(lib.CameParam),
                     ctypes.sizeof(lib.CameArgs)]


class _Tiny(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.w = torch.nn.Parameter(torch.randn(5, 6))
        self.frozen = torch.nn.Parameter(torch.randn(3), requires_grad=False)
        self.conv = torch.nn.Parameter(torch.randn(4, 2, 2, 3))
        self.b = torch.nn.Parameter(torch.randn(7))


def _host_came(model):
    """A FlatCAME whose flat state lives on the CPU (the conversion is host code; the step itself needs the GPU)."""
    red = GradBucketReducer(model, bucket_of=lambda n: "all")
    red.flatten_params()
    opt = FlatCAME.__new__(FlatCAME)
    opt.reducer, opt.eps, opt.clip_threshold, opt.betas, opt.weight_decay = red, (1e-30, 1e-16), 1.0, (0.9, 0.999, 0.9999), 0.0
    opt.entries, tot = came_layout(red)
    opt.exp_avg = [torch.zeros_like(b["flat_param"]) for b in red.buckets]
    opt.exp_avg_sq, opt.sq_row, opt.res_row = torch.zeros(tot["n_vec"]), torch.zeros(tot["n_row"]), torch.zeros(tot["n_row"])
    opt.sq_col, opt.res_col, opt.rms = torch.zeros(tot["n_col"]), torch.zeros(tot["n_col"]), torch.zeros(len(opt.entries))
    opt._lr, opt._lr_host, opt.step_count = torch.tensor([2e-5]), 2e-5, 0
    return opt


def test_torch_state_dict_round_trip_and_index_order():
    torch.manual_seed(0)
    model = _Tiny()
    opt = _host_came(model)
    for t in opt.exp_avg + [opt.exp_avg_sq, opt.sq_row, opt.res_row, opt.sq_col, opt.res_col, opt.rms]:
        t.copy_(torch.rand_like(t))
    opt.exp_avg[0][sum(e["numel"] for e in opt.entries):] = 0          # the bucket padding holds no state
    opt.step_count, opt.lr = 7, 1.5e-5
    sd = opt.to_torch_state_dict(model)
    params = list(model.parameters())
    assert [g["params"] for g in sd["param_groups"]] == [[k] for k in range(len(params))]
    assert sd["param_groups"][1].get("requires_grad") is False and 1 not in sd["state"]
    assert all(g["lr"] == 1.5e-5 and g["betas"] == (0.9, 0.999, 0.9999) and g["eps"] == (1e-30, 1e-16) for g in sd["param_groups"])
    want_keys = {0: {"step", "exp_avg", "exp_avg_sq_row", "exp_avg_sq_col", "exp_avg_res_row", "exp_avg_res_col", "RMS"},
                 3: {"step", "exp_avg", "exp_avg_sq", "RMS"}}
    for k, keys in want_keys.items():
        assert set(sd["state"][k]) == keys and sd["state"][k]["step"] == 7
    assert sd["state"][2]["exp_avg_sq_row"].shape == (4, 2, 2) and sd["state"][2]["exp_avg_sq_col"].shape == (4, 2, 3)
    assert sd["state"][0]["exp_avg"].shape == (5, 6) and sd["state"][3]["exp_avg_sq"].shape == (7,)
    # exp_avg is the parameter's own slice of the flat state, in model.parameters() order
    assert torch.equal(sd["state"][2]["exp_avg"].flatten(), opt.exp_avg[0][30:78])
    assert float(sd["state"][3]["RMS"]) == float(opt.rms[2])

    # a torch.save / torch.load of the state dict loads back into a fresh optimizer
    model2 = _Tiny()
    opt2 = _host_came(model2)
    with tempfile.TemporaryDirectory() as d:
        torch.save({"optimizer": sd}, os.path.join(d, "ckpt.pth"))
        sd_loaded = torch.load(os.path.join(d, "ckpt.pth"))["optimizer"]
    opt2.load_torch_state_dict(model2, sd_loaded)
    assert opt2.step_count == 7 and opt2.lr == 1.5e-5
    for a, b in zip(opt.exp_avg + [opt.exp_avg_sq, opt.sq_row, opt.res_row, opt.sq_col, opt.res_col, opt.rms],
                    opt2.exp_avg + [opt2.exp_avg_sq, opt2.sq_row, opt2.res_row, opt2.sq_col, opt2.res_col, opt2.rms]):
        assert torch.equal(a, b)
    with pytest.raises(ValueError):
        opt2.load_torch_state_dict(model2, {"state": {}, "param_groups": sd["param_groups"][:2]})
