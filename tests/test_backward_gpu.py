"""GPU parity tests (-m gpu) of the training-backward kernels through the C-ABI, each against torch autograd of the
fp32 op on the same bf16-rounded inputs (the attention oracle is oracle.pixart_oracle's softmax(QK^T)V restatement).

Tolerances (normwise ||a-b||/||b||): bf16 outputs 4e-3 (attention gradients 1e-2: P and dS are rounded to bf16 before
the gradient MMAs, as in every flash-attention backward), fp32 outputs / atomically reduced sums 1e-3 or better.
"""
import pytest
import torch
import torch.nn.functional as F

from oracle import pixart_oracle as po

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from pixart_sigma_b200 import lib
DEV = "cuda"


def _randn(*shape, seed=0, scale=1.0, dtype=torch.bfloat16):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(dtype).to(DEV)


@pytest.mark.parametrize("R,C", [(64, 64), (300, 1152), (4096, 3456), (1152, 4608), (130, 72), (377, 1152), (65, 33)])
def test_transpose(R, C):
    a = _randn(R, C, seed=1)
    out = lib.transpose(a)
    assert torch.equal(out, a.t().contiguous())


def test_transpose_of_a_column_slice():
    a = _randn(512, 3456, seed=2)
    out = lib.transpose(a[:, 1152:2304])
    assert torch.equal(out, a[:, 1152:2304].t().contiguous())


def test_gelu_forward_and_backward():
    pre = _randn(1024, 4608, seed=3, scale=1.5)
    dh = _randn(1024, 4608, seed=4)
    h = lib.gelu_tanh(pre)
    x = pre.float().requires_grad_(True)
    want = F.gelu(x, approximate="tanh")
    assert po.rel_err(h.float(), want.detach()) < 4e-3
    want.backward(dh.float())
    dpre = lib.gelu_tanh(pre, dh=dh)
    assert po.rel_err(dpre.float(), x.grad) < 4e-3


@pytest.mark.parametrize("gated", [True, False])
def test_gate_residual_forward_and_backward(gated):
    B, N, C = 3, 160, 1152
    M = B * N
    x = _randn(M, C, seed=5, dtype=torch.float32)
    y = _randn(M, C, seed=6)
    mod = _randn(B, 6, C, seed=7, dtype=torch.float32)
    gate = mod[:, 2] if gated else None
    out = torch.empty_like(x)
    lib.gate_residual_fwd(x, y, gate, out, gate_batch_stride=mod.stride(0), rows_per_batch=N)
    g = (gate if gated else torch.ones(B, C, device=DEV)).detach().clone().requires_grad_(True)
    yf = y.float().requires_grad_(True)
    want = x.view(B, N, C) + g[:, None] * yf.view(B, N, C)
    assert po.rel_err(out, want.detach().view(M, C)) < 1e-6
    dout = _randn(M, C, seed=8, dtype=torch.float32)
    want.backward(dout.view(B, N, C))
    dy = torch.empty(M, C, dtype=torch.bfloat16, device=DEV)
    dgate = torch.zeros(B, C, dtype=torch.float32, device=DEV) if gated else None
    lib.gate_residual_bwd(dout, y if gated else None, gate, dy, dgate, gate_batch_stride=mod.stride(0), rows_per_batch=N)
    assert po.rel_err(dy.float(), yf.grad) < 4e-3
    if gated:
        assert po.rel_err(dgate, g.grad) < 1e-4


@pytest.mark.parametrize("B,N", [(2, 256), (3, 50), (1, 1024)])
def test_ln_modulate_backward(B, N):
    C, M = 1152, B * N
    x = _randn(M, C, seed=9, dtype=torch.float32) * 2 + 0.3
    mod = _randn(B, 6, C, seed=10, dtype=torch.float32, scale=0.5)
    dxn = _randn(M, C, seed=11)
    xr = x.clone().requires_grad_(True)
    sh = mod[:, 0].clone().requires_grad_(True)
    sc = mod[:, 1].clone().requires_grad_(True)
    xn = F.layer_norm(xr.view(B, N, C), (C,), eps=1e-6) * (1 + sc[:, None]) + sh[:, None]
    xn.backward(dxn.float().view(B, N, C))
    dx = torch.empty_like(x)
    dshift = torch.zeros(B, C, dtype=torch.float32, device=DEV)
    dscale = torch.zeros(B, C, dtype=torch.float32, device=DEV)
    lib.ln_modulate_bwd(x, dxn, mod[:, 1], dx, dshift, dscale, mod_batch_stride=mod.stride(0), rows_per_batch=N)
    assert po.rel_err(dx, xr.grad) < 1e-4
    assert po.rel_err(dshift, sh.grad) < 1e-4
    assert po.rel_err(dscale, sc.grad) < 1e-4


def test_colsum_accumulates():
    a = _randn(1000, 3456, seed=12)
    out = torch.ones(1152, dtype=torch.float32, device=DEV)
    lib.colsum(a[:, 1152:2304], out)
    assert po.rel_err(out, 1 + a[:, 1152:2304].float().sum(0)) < 1e-5


def test_linear_backward_on_the_forward_gemm():
    """dX = dY W (gemm on W^T) and dW += dY^T X (gemm on the transposes, fp32 reduce-add epilogue into the gradient)."""
    M, N, K = 2048, 1152, 4608
    x, w = _randn(M, K, seed=13), _randn(N, K, seed=14, scale=K ** -0.5)
    dy = _randn(M, N, seed=15)
    dx = torch.empty(M, K, dtype=torch.bfloat16, device=DEV)
    lib.gemm(dy, lib.transpose(w), None, dx)
    assert po.rel_err(dx.float(), dy.float() @ w.float()) < 4e-3
    dw = torch.full((N, K), 0.5, dtype=torch.float32, device=DEV)
    lib.gemm(lib.transpose(dy), lib.transpose(x), None, dw, epilogue=lib.EPI_BIAS_RESIDUAL, residual=dw)
    assert po.rel_err(dw - 0.5, dy.float().t() @ x.float()) < 2e-4


@pytest.mark.parametrize("rows,n_out,k_in,bn,ks", [
    (2048, 1152, 1152, 0, 0), (2048, 3456, 1152, 0, 1), (4096, 1152, 4608, 256, 0), (377, 2304, 1152, 0, 0),
    (1200, 1152, 4096, 128, 3), (16384, 1152, 1152, 192, 0), (64, 128, 64, 128, 0), (8192, 4608, 1152, 0, 5),
])
def test_gemm_weight_gradient_form(rows, n_out, k_in, bn, ks):
    """dW (n_out, k_in) += dY (rows, n_out)^T X (rows, k_in): MN-major operands straight from the activations, split-K."""
    dy, x = _randn(rows, n_out, seed=40), _randn(rows, k_in, seed=41)
    dw = torch.full((n_out, k_in), 0.25, dtype=torch.float32, device=DEV)
    lib.gemm_wgrad(dy, x, dw, block_n=bn, k_splits=ks)
    assert po.rel_err(dw - 0.25, dy.float().t() @ x.float()) < 2e-4
    dy3 = _randn(rows, 3 * n_out, seed=42)                      # operands may be column slices (row-strided views)
    dw.zero_()
    lib.gemm_wgrad(dy3[:, n_out:2 * n_out], x, dw, block_n=bn, k_splits=ks)
    assert po.rel_err(dw, dy3[:, n_out:2 * n_out].float().t() @ x.float()) < 2e-4


@pytest.mark.parametrize("K", [1152, 4608])
def test_gemm_residual_epilogue_keeps_the_branch_output(K):
    """Training forward of `x + gate * (a W^T + b)`: out-of-place fp32 residual epilogue whose bf16 aux output is the
    un-gated branch (needed by the gate's backward); K=1152 takes the TMA-streamed single-CTA kernel, 4608 the CTA pair."""
    B, N, C = 2, 1024, 1152
    M = B * N
    a, w, bias = _randn(M, K, seed=50), _randn(C, K, seed=51, scale=K ** -0.5), _randn(C, seed=52, scale=0.1)
    x = _randn(M, C, seed=53, dtype=torch.float32)
    mod = _randn(B, 6, C, seed=54, dtype=torch.float32)
    out = torch.empty_like(x)
    y = torch.empty(M, C, dtype=torch.bfloat16, device=DEV)
    x_before = x.clone()
    lib.gemm(a, w, bias, out, epilogue=lib.EPI_BIAS_RESIDUAL, residual=x, gate=mod[:, 2], gate_batch_stride=mod.stride(0),
             rows_per_batch=N, out_aux=y, aux_is_branch=True)
    branch = F.linear(a.float(), w.float(), bias.float())
    want = x_before.view(B, N, C) + mod[:, 2][:, None] * branch.view(B, N, C)
    assert torch.equal(x, x_before)                                  # the residual input is not touched
    assert po.rel_err(out, want.view(M, C)) < 2e-4
    assert po.rel_err(y.float(), branch) < 4e-3


@pytest.mark.parametrize("M,N,K", [(2048, 4608, 1152), (512, 256, 128), (1000, 4608, 1152)])
def test_gemm_gelu_epilogue_keeps_the_pre_activation(M, N, K):
    a, w, bias = _randn(M, K, seed=70), _randn(N, K, seed=71, scale=K ** -0.5), _randn(N, seed=72, scale=0.1)
    h = torch.full((M, N), float("nan"), dtype=torch.bfloat16, device=DEV)
    pre = torch.full((M, N), float("nan"), dtype=torch.bfloat16, device=DEV)
    lib.gemm(a, w, bias, h, epilogue=lib.EPI_BIAS_GELU_AUX, out_aux=pre)
    want = F.linear(a.float(), w.float(), bias.float())
    assert po.rel_err(pre.float(), want) < 4e-3
    assert po.rel_err(h.float(), F.gelu(want, approximate="tanh")) < 4e-3


@pytest.mark.parametrize("M,N,K", [(2048, 4608, 1152), (512, 256, 128), (1000, 4608, 1152)])
def test_gemm_dgelu_epilogue(M, N, K):
    """dgrad GEMM of the MLP's second layer with gelu'(pre) applied in the epilogue: out = (dy W) * gelu'(pre)."""
    dy, wt = _randn(M, K, seed=73), _randn(N, K, seed=74, scale=K ** -0.5)          # wt = W^T rows (N = hidden)
    pre = _randn(M, N, seed=75, scale=1.5)
    out = torch.full((M, N), float("nan"), dtype=torch.bfloat16, device=DEV)
    lib.gemm(dy, wt, None, out, epilogue=lib.EPI_MUL_DGELU, residual=pre)
    x = pre.float().requires_grad_(True)
    F.gelu(x, approximate="tanh").backward(F.linear(dy.float(), wt.float()))
    assert po.rel_err(out.float(), x.grad) < 5e-3


def _attn_ref(q, k, v, lens, scale):
    """fp32 autograd reference: q (B,Nq,H,D), k/v (B,Nk,H,D) padded, sample b sees keys < lens[b]."""
    outs = []
    for b in range(q.shape[0]):
        L = lens[b]
        s = torch.einsum("qhd,khd->hqk", q[b], k[b, :L]) * scale
        outs.append(torch.einsum("hqk,khd->qhd", s.softmax(-1), v[b, :L]))
    return torch.stack(outs)


@pytest.mark.parametrize("B,H,Nq,Nk,lens", [
    (1, 2, 128, 128, None), (2, 3, 256, 256, None), (1, 16, 1024, 1024, None), (2, 2, 256, 64, None),
    (2, 2, 128, 300, [300, 77]), (3, 4, 256, 300, [5, 130, 256]), (2, 2, 200, 200, None), (1, 3, 4032, 4032, None),
    (2, 2, 72, 300, [300, 41]), (2, 2, 201, 130, None), (1, 3, 1089, 1089, None),     # Nq % 4 != 0: no TMA copies of lse / delta
    # more (128-row tile, head, sample) CTAs than SMs, ragged key lengths whose samples end inside a key tile
    (2, 16, 1024, 1024, None), (4, 16, 640, 300, [300, 77, 65, 130]), (3, 16, 516, 516, None),
])
def test_flash_attn_backward(B, H, Nq, Nk, lens):
    D, C = 72, H * 72
    scale = D ** -0.5
    q, k, v = _randn(B * Nq, H, D, seed=20), _randn(B * Nk, H, D, seed=21), _randn(B * Nk, H, D, seed=22)
    d_o = _randn(B * Nq, C, seed=23)
    kv_len = None if lens is None else torch.tensor(lens, dtype=torch.int32, device=DEV)
    o = torch.empty(B * Nq, C, dtype=torch.bfloat16, device=DEV)
    lse = torch.empty(B, H, Nq, dtype=torch.float32, device=DEV)
    strides = (C, D)
    lib.flash_attn(q, k, v, o, B=B, H=H, Nq=Nq, Nk=Nk, kv_rows=B * Nk, kv_len=kv_len, q_strides=strides, k_strides=strides,
                   v_strides=strides, scale=scale, lse=lse)
    qf, kf, vf = (t.float().view(B, -1, H, D).requires_grad_(True) for t in (q, k, v))
    ll = lens or [Nk] * B
    want = _attn_ref(qf, kf, vf, ll, scale)
    assert po.rel_err(o.float().view(B, Nq, H, D), want.detach()) < 6e-3
    # lse: natural-log logsumexp of the scaled scores, times log2(e)
    s = torch.einsum("bqhd,bkhd->bhqk", qf.detach(), kf.detach()) * scale
    for b in range(B):
        want_lse = torch.logsumexp(s[b, :, :, :ll[b]], dim=-1) * 1.4426950408889634
        assert (lse[b] - want_lse).abs().max() < 2e-2
    want.backward(d_o.float().view(B, Nq, H, D))
    dq, dk, dv = (torch.full_like(t, float("nan")) for t in (q, k, v))
    lib.flash_attn_bwd(q, k, v, o, d_o, lse, dq, dk, dv, B=B, H=H, Nq=Nq, Nk=Nk, kv_rows=B * Nk, kv_len=kv_len,
                       q_strides=strides, k_strides=strides, v_strides=strides, dq_strides=strides, dk_strides=strides,
                       dv_strides=strides, scale=scale)
    assert po.rel_err(dq.float().view(B, Nq, H, D), qf.grad) < 1e-2
    for b in range(B):      # rows of keys >= kv_len[b] are not written
        L = ll[b]
        assert po.rel_err(dk.float().view(B, Nk, H, D)[b, :L], kf.grad[b, :L]) < 1e-2
        assert po.rel_err(dv.float().view(B, Nk, H, D)[b, :L], vf.grad[b, :L]) < 1e-2


def test_flash_attn_backward_interleaved_qkv_and_packed_cross_keys():
    """The layouts the block uses: q/k/v and dq/dk/dv are slices of (rows, 3, H, 72) buffers; cross-attention keys are
    packed (kv_off) rows of a (sum L, 2, H, 72) buffer."""
    B, H, N, D = 2, 16, 256, 72
    C = H * D
    scale = D ** -0.5
    qkv = _randn(B * N, 3, H, D, seed=30)
    d_o = _randn(B * N, C, seed=31)
    o = torch.empty(B * N, C, dtype=torch.bfloat16, device=DEV)
    lse = torch.empty(B, H, N, dtype=torch.float32, device=DEV)
    st = (3 * C, D)
    lib.flash_attn(qkv[:, 0], qkv[:, 1], qkv[:, 2], o, B=B, H=H, Nq=N, Nk=N, kv_rows=B * N, q_strides=st, k_strides=st,
                   v_strides=st, scale=scale, lse=lse)
    dqkv = torch.empty_like(qkv)
    lib.flash_attn_bwd(qkv[:, 0], qkv[:, 1], qkv[:, 2], o, d_o, lse, dqkv[:, 0], dqkv[:, 1], dqkv[:, 2], B=B, H=H, Nq=N,
                       Nk=N, kv_rows=B * N, q_strides=st, k_strides=st, v_strides=st, dq_strides=st, dk_strides=st,
                       dv_strides=st, scale=scale)
    f = qkv.float().view(B, N, 3, H, D).requires_grad_(True)
    want = _attn_ref(f[:, :, 0], f[:, :, 1], f[:, :, 2], [N] * B, scale)
    want.backward(d_o.float().view(B, N, H, D))
    assert po.rel_err(dqkv.float().view(B, N, 3, H, D), f.grad) < 1e-2

    lens = [77, 300]
    kv = _randn(sum(lens), 2, H, D, seed=32)
    q = _randn(B * N, C, seed=33)
    kv_len = torch.tensor(lens, dtype=torch.int32, device=DEV)
    kv_off = torch.tensor([0, 77], dtype=torch.int32, device=DEV)
    lib.flash_attn(q, kv[:, 0], kv[:, 1], o, B=B, H=H, Nq=N, Nk=300, kv_rows=sum(lens), kv_len=kv_len, kv_off=kv_off,
                   q_strides=(C, D), k_strides=(2 * C, D), v_strides=(2 * C, D), scale=scale, lse=lse)
    dq = torch.empty_like(q)
    dkv = torch.empty_like(kv)
    lib.flash_attn_bwd(q, kv[:, 0], kv[:, 1], o, d_o, lse, dq, dkv[:, 0], dkv[:, 1], B=B, H=H, Nq=N, Nk=300,
                       kv_rows=sum(lens), kv_len=kv_len, kv_off=kv_off, q_strides=(C, D), k_strides=(2 * C, D),
                       v_strides=(2 * C, D), dq_strides=(C, D), dk_strides=(2 * C, D), dv_strides=(2 * C, D), scale=scale)
    qf = q.float().view(B, N, H, D).requires_grad_(True)
    kvf = kv.float().requires_grad_(True)
    outs = []
    for b, (off, L) in enumerate(zip([0, 77], lens)):
        s = torch.einsum("qhd,khd->hqk", qf[b], kvf[off:off + L, 0]) * scale
        outs.append(torch.einsum("hqk,khd->qhd", s.softmax(-1), kvf[off:off + L, 1]))
    torch.stack(outs).backward(d_o.float().view(B, N, H, D))
    assert po.rel_err(dq.float().view(B, N, H, D), qf.grad) < 1e-2
    assert po.rel_err(dkv.float(), kvf.grad) < 1e-2


@pytest.mark.parametrize("B,H,W", [(2, 16, 16), (1, 8, 24)])
def test_kv_compress_backward(B, H, W):
    """Depthwise conv 2x2/s2 + LayerNorm(affine) backward vs torch autograd (fp32) of the same op on K and V."""
    C = 1152
    qkv = _randn(B * H * W, 3 * C, seed=60)
    conv_w = _randn(C, 1, 2, 2, seed=61, scale=0.5) + 0.25
    conv_b, ln_w, ln_b = _randn(C, seed=62, scale=0.1), _randn(C, seed=63, scale=0.2) + 1.0, _randn(C, seed=64, scale=0.1)
    n_out = (H // 2) * (W // 2)
    dkc, dvc = _randn(B * n_out, C, seed=65), _randn(B * n_out, C, seed=66)
    dqkv = torch.zeros_like(qkv)
    g = [torch.zeros(C, 1, 2, 2, device=DEV), torch.zeros(C, device=DEV), torch.zeros(C, device=DEV), torch.zeros(C, device=DEV)]
    lib.kv_compress_bwd(qkv[:, C:2 * C], qkv[:, 2 * C:], dkc, dvc, dqkv[:, C:2 * C], dqkv[:, 2 * C:], conv_w, conv_b, ln_w, *g,
                        B=B, H=H, W=W, ld_in=3 * C, ld_din=3 * C)
    f = qkv.float().requires_grad_(True)
    pw, pb, pg, pbeta = (t.float().requires_grad_(True) for t in (conv_w, conv_b, ln_w, ln_b))
    outs = []
    for i in (1, 2):
        img = f[:, i * C:(i + 1) * C].reshape(B, H, W, C).permute(0, 3, 1, 2)
        y = F.conv2d(img, pw, pb, stride=2, groups=C).reshape(B, C, -1).permute(0, 2, 1)
        outs.append(F.layer_norm(y, (C,), pg, pbeta, eps=1e-5).reshape(B * n_out, C))
    (outs[0] * dkc.float()).sum().add((outs[1] * dvc.float()).sum()).backward()
    assert float(dqkv[:, :C].abs().max()) == 0.0
    assert po.rel_err(dqkv[:, C:].float(), f.grad[:, C:]) < 4e-3
    for got, want in zip(g, (pw.grad, pb.grad, pg.grad, pbeta.grad)):
        assert po.rel_err(got, want) < 1e-3
