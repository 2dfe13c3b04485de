"""Stage-local float64 references for one training block (`autograd.BlockFn`, forward and backward): the ordered list of
kernel calls BlockFn makes, and for every call the float64 value of the mathematically correct operation with an
element-wise bound.  Shared by test_block_stages_cpu.py, which proves that the chain of references composes to float64
autograd of the oracle block and that wiring defects fail at their stage, and test_block_train_numerics_gpu.py, which
records the real kernel calls and checks each against its reference.

Roles.  `expected_trace` lists BlockFn's `lib` calls in order, each with the output arguments it writes and the role
(name) of each output.  A recorded trace is mapped to roles by position; the recorded trace must match the list exactly.
Every reference takes its inputs from the block's definition -- the test's weights (the bf16 values the kernels consume,
formed by the test from the parameters), `mod`, `dout`, the caption rows -- and from the recorded outputs of EARLIER stages
in their correct roles, never from the tensors the code passed.  So a wrong operand, modulation column, row grouping, scale
or a missing term fails at the stage where it happens, at that kernel's own rounding bound, instead of inside an end-to-end
tolerance.  Casts BlockFn does in torch between kernels (x1 -> bf16 for the cross-attention query, the qk-norm input
gradient -> bf16 in dqkv) are part of the references of the stages that consume them.

Bounds are those of the modules that own the kernels, reused, not re-derived:
  - GEMMs (forward epilogues, dgrad, MUL_DGELU, split-K weight gradients): gemm_bounds.py, the split count of
    `gemm_bounds.auto_splits`;
  - attention forward (bf16 P, or hi + lo P under fp32_attention) and backward: attn_bounds.py, given the recorded O / lse;
  - LN-modulate forward (2 ulp + the two-pass statistics, test_numerics_gpu._ln_slack), its backward and the per-sample
    column sums (test_backward_numerics_gpu._ln_bwd_slack and the 16-row-warp + atomic sums), layernorm_affine_ (same form);
  - gate_residual_bwd: dy = bf16(dout gate) (one fp32 product: u |dy|, then half a bf16 ulp) and dgate[b] += sum dout y
    (one fmaf per row in a 32-row CTA, then one atomic per CTA: (32 + W_b) u sum |terms|, W_b the CTAs touching sample b);
  - colsum: 16 rows per thread, 8 shared-memory partials, one atomic per 128-row slab: (24 + slabs) u (|pre| + sum |a|);
  - gate_residual_fwd without a gate (dx1 = dx2 + dxb): one fp32 rounding; gate_residual_bwd without a gate (dy2 =
    bf16(dx2)): one bf16 rounding.
Each output is held to c ulp(|ref| + slack) + slack (gemm_bounds.Tally) in its own dtype, with c = 1/2 for a final rounding,
1 for the GELU and attention outputs (their contracts) and 2 for the LayerNorm forwards (test_numerics_gpu's bound).
Bias statistics apply to bf16 outputs with the MAX_BIAS of the owning module (gemm_bounds for GEMMs and roundings,
attn_bounds for attention); fp32 outputs are held by the element-wise bound alone, as in gemm_bounds.
"""
import torch

import attn_bounds as ab
import gemm_bounds as gb
import norm_bounds as nb
from oracle.pixart_oracle import kv_downsample

U = gb.U
TAGS = ("qkv", "proj", "q", "kv", "cproj", "fc1", "fc2")
MODULE = dict(qkv="attn.qkv", proj="attn.proj", q="cross_attn.q_linear", kv="cross_attn.kv_linear", cproj="cross_attn.proj",
              fc1="mlp.fc1", fc2="mlp.fc2")    # the projection of each tag, as a name inside PixArtMSBlock


# ------------------------------------------------------------------------------------------------- the kernel trace
def _lin_bwd(tag, dx_role):
    """_linear_backward of projection `tag`: dgrad (when dx_role), weight gradient, bias column sum."""
    return ([("gemm", {3: dx_role})] if dx_role else []) + [("gemm_wgrad", {2: "dW." + tag}), ("colsum", {1: "db." + tag})]


def forward_trace(qk_norm=False, attention=True):
    """The `lib` calls of `_block_forward_kernels` (attention=False: the checkpoint recompute, which keeps O / lse)."""
    fa = lambda o, lse: [("flash_attn", {3: o, "lse": lse})] if attention else []
    qk = [("layernorm_affine_", {0: "qn"}), ("layernorm_affine_", {0: "kn"})] if qk_norm else []
    return ([("ln_modulate", {3: "xn1"}), ("gemm", {3: "qkv"})] + qk + fa("ao1", "lse1") +
            [("gemm", {3: "x1", "out_aux": "y1"}), ("gemm", {3: "qx"}), ("gemm", {3: "kv"})] + fa("ao2", "lse2") +
            [("gemm", {3: "x2"}), ("ln_modulate", {3: "xn2"}), ("gemm", {3: "h", "out_aux": "pre"}),
             ("gemm", {3: "x3", "out_aux": "y3"})])


def backward_trace(qk_norm=False):
    """The `lib` calls of `BlockFn.backward` after any recompute, in order (shadow transposes excluded: they are cache
    maintenance, and a wrong one fails the dgrad stage that reads it)."""
    qk = [("ln_modulate_bwd", {3: "dqn", 4: "db.q_norm", 5: "dw.q_norm"}),
          ("ln_modulate_bwd", {3: "dkn", 4: "db.k_norm", 5: "dw.k_norm"})] if qk_norm else []
    return ([("gate_residual_bwd", {3: "dy3", 4: "dm5"})] + _lin_bwd("fc2", None) + [("gemm", {3: "dpre"})] +
            _lin_bwd("fc1", "dxn2") + [("ln_modulate_bwd", {3: "dx2", 4: "dm3", 5: "dm4"}), ("gate_residual_bwd", {3: "dy2"})] +
            _lin_bwd("cproj", "dao2") + [("flash_attn_bwd", {6: "dq2", 7: "dk2", 8: "dv2"})] + _lin_bwd("q", "dxb") +
            _lin_bwd("kv", "dcond") + [("gate_residual_fwd", {3: "dx1"}), ("gate_residual_bwd", {3: "dy1", 4: "dm2"})] +
            _lin_bwd("proj", "dao1") + [("flash_attn_bwd", {6: "dq1", 7: "dk1", 8: "dv1"})] + qk + _lin_bwd("qkv", "dxn1") +
            [("ln_modulate_bwd", {3: "dx", 4: "dm0", 5: "dm1"})])


def expected_trace(qk_norm=False, ckpt=False):
    """[(lib function, {output argument (position or keyword): role})] of one BlockFn forward + backward.  Under
    activation checkpointing the backward starts with the forward again, without the attentions; its roles carry "rc."."""
    rc = [(n, {k: "rc." + r for k, r in outs.items()}) for n, outs in forward_trace(qk_norm, attention=False)] if ckpt else []
    return forward_trace(qk_norm) + rc + backward_trace(qk_norm)


# ------------------------------------------------------------------------------------------------- bounds helpers
class StageFailure(AssertionError):
    def __init__(self, stage, msg):
        super().__init__(f"stage {stage}: {msg}")
        self.stage = stage


class StageTally(gb.Tally):
    """gemm_bounds.Tally with the MAX_BIAS of the module that owns the bound (None: gemm_bounds' rule)."""

    def __init__(self, name, fp32=False, c=0.5, max_bias=None):
        super().__init__(name, fp32=fp32, c=c)
        self._max_bias = max_bias

    def max_bias(self):
        return 1.0 if self.fp32 else (self._max_bias if self._max_bias is not None else gb.MAX_BIAS)


def _ln_fwd(x, shift, scale, eps):
    """LN(x) (1 + scale) + shift, row-wise shift / scale (M, C), and the slack of the ln_modulate bound of
    test_numerics_gpu (norm_bounds.ln_slack + 2^-22 relative, at 2 ulp)."""
    xh, _, r = nb.ln_stats(x, eps)
    ref = xh * (1 + scale) + shift
    return ref, nb.ln_slack(x, r, (1 + scale).abs()) + 2.0 ** -22 * ref.abs()


def _ln_bwd(x, dxn, scale_rows, eps):
    """dx (without add_in) of the LN-modulate backward, xh, and the slack of dx and of the kernel's xh (e)."""
    xh, rstd, r = nb.ln_stats(x, eps)
    g = dxn * (1 + scale_rows)
    dx = rstd * (g - g.mean(-1, keepdim=True) - xh * (g * xh).mean(-1, keepdim=True))
    return dx, xh, nb.ln_bwd_slack(xh, rstd, g, r, 2.0 ** -19), 2.0 ** -18 * (1 + r) + 2.0 ** -19 * xh.abs()


def _sample_sum(terms, b_of, B, pre=None):
    out = torch.zeros(B, terms.shape[1], dtype=torch.float64, device=terms.device).index_add_(0, b_of, terms)
    return out if pre is None else out + pre


def _warps(B, rpb, M, rows, device):
    """Number of `rows`-row groups that touch each sample (one flush per group and sample)."""
    first = torch.arange(B, device=device) * rpb
    last = torch.clamp(first + rpb, max=M) - 1
    return (last // rows - first // rows + 1).double()[:, None]


# ------------------------------------------------------------------------------------------------- the stages
class BlockStages:
    """The stage references of one block.  `inp` (float64 tensors, on any device):
         x (M, C) fp32 values, cond (R, C) bf16 values, mod (B, 6, C), dout (M, C);
         W[tag] (N, K) / bias[tag] (N,): the bf16 values the kernels consume;
         qk: None or {"q": (w, b), "k": (w, b)} of q_norm / k_norm (bf16 values), qk_eps;
         B, N, H, keys = [(first row, count)] of each sample's valid caption rows in cond; ln_eps of norm1 / norm2;
         kv_pick: None or (sampling, sr, (H, W)) of a parameter-free KV compression ('uniform', 'ave', 'uniform_every');
         fp32_p: the self-attention forward's hi + lo P; pre[role]: what a gradient output held before its kernel
         (the bucket's pre-filled value, or 0); splits(M, N, K): the weight-gradient split count;
         cast: the bf16 rounding of a torch cast between kernels (identity for the exact chain of the CPU proof).
    `run(R, emulate=None)` walks the stages in order.  Checking: R holds the recorded outputs by role; each stage's
    reference is formed from `inp` and the roles of earlier stages and compared with R; the first stage outside its bound
    raises StageFailure.  Emulating (emulate = a function (ref, dtype) -> value): R is filled with each reference as the
    stage's output, which later stages then read."""

    def __init__(self, inp):
        self.i = inp
        self.tallies = {}

    def _out(self, stage, role, ref, slack, dtype, c=0.5, max_bias=None, exact_zero=None):
        if self.emulate is not None:
            v = self.emulate(ref, dtype)
            if exact_zero is not None:
                v = torch.where(exact_zero, torch.zeros_like(v), v)
            self.R[role] = v
            return
        got = self.R[role].double().reshape(ref.shape)
        t = self.tallies.setdefault(role, StageTally(f"{stage}: {role}", fp32=dtype == torch.float32, c=c, max_bias=max_bias))
        try:
            t.add(got, ref, slack)
        except AssertionError as e:
            raise StageFailure(stage, str(e))
        if exact_zero is not None and exact_zero.any():
            nz = (got[exact_zero] != 0).sum().item()
            if nz:
                raise StageFailure(stage, f"{role}: {nz} elements that must be exact zeros are not")
        if not t.ok():
            raise StageFailure(stage, f"{role}: {t.bad} elements outside the bound (e.g. got / want / bound {t.example}), "
                                      f"bias {t.bias:+.4f}")

    def r(self, role):
        return self.R[role].double()

    # -- projections
    def _gemm(self, a, w, bias=None):
        acc, s, _ = gb.accumulate(a, w)
        return gb.bias_out(acc, s, bias)

    def _wgrad(self, stage, role, dy, x):
        """dW += dY^T X into the pre-filled output: split-K accumulator, k reduce-adds."""
        ks = self.i["splits"](dy.shape[1], x.shape[1], dy.shape[0])
        acc, s, parts = gb.accumulate(dy.T, x.T, k_splits=ks)
        parts = acc.abs() if parts is None else parts
        pre = self.i["pre"][role]
        self._out(stage, role, pre + acc, s + ks * U * (pre.abs() + parts), torch.float32)

    def _colsum(self, stage, role, a):
        pre = self.i["pre"][role]
        slabs = -(-a.shape[0] // 128)
        self._out(stage, role, pre + a.sum(0), (24 + slabs) * U * (pre.abs() + a.abs().sum(0)), torch.float32)

    def _lin_bwd(self, stage, tag, dy, x, dx_role=None):
        if dx_role:
            y, s = self._gemm(dy, self.i["W"][tag].T)
            self._out(stage, dx_role, y, s, torch.bfloat16)
        self._wgrad(stage, "dW." + tag, dy, x)
        self._colsum(stage, "db." + tag, dy)

    # -- attention, one (sample, head) at a time
    def _attn_fwd(self, stage, q, k, v, keys, scale, split_p, o_role, lse_role):
        i = self.i
        B, N, H = i["B"], i["N"], i["H"]
        C = q.shape[1]
        D = C // H
        o, so = torch.zeros_like(q), torch.zeros_like(q)
        lse, sl = (torch.zeros(B, H, N, dtype=torch.float64, device=q.device) for _ in range(2))
        for b, (k0, L) in enumerate(keys):
            if L == 0:
                continue                                  # no keys: zero output, lse 0
            for h in range(H):
                cs = slice(h * D, (h + 1) * D)
                f = ab.forward(q[b * N:(b + 1) * N, cs], k[k0:k0 + L, cs], v[k0:k0 + L, cs], scale, split_p=split_p)
                o[b * N:(b + 1) * N, cs], so[b * N:(b + 1) * N, cs] = f["o"], f["slack_o"]
                lse[b, h], sl[b, h] = f["lse"], f["slack_lse"]
        self._out(stage, o_role, o, so, torch.bfloat16, c=1.0, max_bias=ab.MAX_BIAS)
        self._out(stage, lse_role, lse, sl, torch.float32, c=1.0)

    def _attn_bwd(self, stage, q, k, v, o, lse, do, keys, scale, roles):
        i = self.i
        B, N, H = i["B"], i["N"], i["H"]
        C = q.shape[1]
        D = C // H
        dq, sq = torch.zeros_like(q), torch.zeros_like(q)
        dk, sk, dv, sv = (torch.zeros_like(k) for _ in range(4))
        valid = torch.zeros(k.shape[0], dtype=torch.bool, device=k.device)
        for b, (k0, L) in enumerate(keys):
            valid[k0:k0 + L] = True
            if L == 0:
                continue                                  # no keys: dQ = 0
            for h in range(H):
                cs = slice(h * D, (h + 1) * D)
                rq, rk = slice(b * N, (b + 1) * N), slice(k0, k0 + L)
                g = ab.backward(q[rq, cs], k[rk, cs], v[rk, cs], do[rq, cs], o[rq, cs], lse[b, h], scale)
                dq[rq, cs], sq[rq, cs] = g["dq"], g["slack_dq"]
                dk[rk, cs], sk[rk, cs], dv[rk, cs], sv[rk, cs] = g["dk"], g["slack_dk"], g["dv"], g["slack_dv"]
        zero_rows = (~valid)[:, None].expand_as(dk)         # key rows no sample reads: no gradient at all
        self._out(stage, roles[0], dq, sq, torch.bfloat16, c=1.0, max_bias=ab.MAX_BIAS)
        self._out(stage, roles[1], dk, sk, torch.bfloat16, c=1.0, max_bias=ab.MAX_BIAS, exact_zero=zero_rows)
        self._out(stage, roles[2], dv, sv, torch.bfloat16, c=1.0, max_bias=ab.MAX_BIAS, exact_zero=zero_rows)

    # -- gate / residual / LN-modulate backward pieces
    def _gate_bwd(self, stage, dy_role, dg_role, dout, y, gate_col):
        i = self.i
        M, B, N = dout.shape[0], i["B"], i["N"]
        b_of = torch.arange(M, device=dout.device) // N
        g = i["mod"][:, gate_col][b_of]
        dy = dout * g
        # a zero gate (a sample drop path removed) gives an exact zero branch gradient
        self._out(stage, dy_role, dy, U * dy.abs(), torch.bfloat16, exact_zero=(g == 0))
        terms = dout * y
        wb = _warps(B, N, M, 32, dout.device)
        self._out(stage, dg_role, _sample_sum(terms, b_of, B), (32 + wb) * U * _sample_sum(terms.abs(), b_of, B),
                  torch.float32)

    def _ln_mod_bwd(self, stage, roles, x, dxn, scale, rpb, eps, add_in=None):
        """dx (+ add_in) and the per-sample column sums dshift = sum dxn, dscale = sum dxn xh of ln_modulate_bwd; scale
        (B', C) per sample of rpb rows."""
        M = x.shape[0]
        B = scale.shape[0]
        b_of = torch.arange(M, device=x.device) // rpb
        dx, xh, s_dx, e = _ln_bwd(x, dxn, scale[b_of], eps)
        if add_in is not None:
            dx = dx + add_in
        self._out(stage, roles[0], dx, s_dx, torch.float32, c=1.0)
        ssum = lambda t: _sample_sum(t, b_of, B)
        slack = lambda t: nb.sample_sum_slack(b_of, B, rpb, M, t, torch.zeros_like(scale))    # zero-filled sums
        self._out(stage, roles[1], ssum(dxn), slack(dxn), torch.float32)
        self._out(stage, roles[2], ssum(dxn * xh), slack(dxn * xh) + ssum(dxn.abs() * e), torch.float32)

    def _kv_rows(self, M):
        """The qkv rows a parameter-free KV compression keeps (inp["kv_pick"] = (sampling, sr, (H, W)), else None), from the
        oracle's downsample_2d applied to the row indices."""
        if self.i.get("kv_pick") is None:
            return None
        sampling, sr, (Hh, Ww) = self.i["kv_pick"]
        rows = torch.arange(M, dtype=torch.float64, device=self.i["x"].device).view(self.i["B"], -1, 1)
        return kv_downsample(None, "", rows, Hh, Ww, sr, sampling).reshape(-1).long()

    # -- the walk
    def run(self, R, emulate=None):
        self.R, self.emulate = R, emulate
        i = self.i
        x, cond, mod, dout, W, bias = i["x"], i["cond"], i["mod"], i["dout"], i["W"], i["bias"]
        B, N, H = i["B"], i["N"], i["H"]
        M, C = x.shape
        D = C // H
        cast = i["cast"]
        b_of = torch.arange(M, device=x.device) // N
        col = lambda j: mod[:, j][b_of]
        scale = D ** -0.5

        # ---------------- forward
        ref, s = _ln_fwd(x, col(0), col(1), i["ln_eps"])
        self._out("xn1", "xn1", ref, s, torch.bfloat16, c=2.0)
        y, s = self._gemm(self.r("xn1"), W["qkv"], bias["qkv"])
        self._out("qkv", "qkv", y, s, torch.bfloat16)
        qkv = self.r("qkv")
        q, k, v = qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:]
        if i["qk"] is not None:
            for j, (role, src) in enumerate((("qn", q), ("kn", k))):
                w, bb = i["qk"]["qk"[j]]
                ref, s = _ln_fwd(src, bb.expand_as(src), (w - 1).expand_as(src), i["qk_eps"])
                self._out("q/k norm", role, ref, s, torch.bfloat16, c=2.0)
            q, k = self.r("qn"), self.r("kn")
        pick = self._kv_rows(M)
        if pick is not None:                                           # parameter-free KV compression: a row pick (torch)
            k, v = k[pick], v[pick]
        Nk = k.shape[0] // B
        self_keys = [(b * Nk, Nk) for b in range(B)]
        self._attn_fwd("ao1/lse1", q, k, v, self_keys, scale, i["fp32_p"], "ao1", "lse1")
        acc, s_acc, _ = gb.accumulate(self.r("ao1"), W["proj"])
        y, s_y = gb.bias_out(acc, s_acc, bias["proj"])
        o, s = gb.residual_out(y, s_y, col(2), x)
        self._out("x1/y1", "x1", o, s, torch.float32)
        self._out("x1/y1", "y1", y, s_y, torch.bfloat16)
        xb = cast(self.r("x1"))                                        # xb: the bf16 cast of x1 (torch)
        y, s = self._gemm(xb, W["q"], bias["q"])
        self._out("qx", "qx", y, s, torch.bfloat16)
        y, s = self._gemm(cond, W["kv"], bias["kv"])
        self._out("kv", "kv", y, s, torch.bfloat16)
        kv = self.r("kv")
        self._attn_fwd("ao2/lse2", self.r("qx"), kv[:, :C], kv[:, C:], i["keys"], scale, False, "ao2", "lse2")
        y, s_y = self._gemm(self.r("ao2"), W["cproj"], bias["cproj"])
        o, s = gb.residual_out(y, s_y, torch.ones_like(y), self.r("x1"))
        self._out("x2", "x2", o, s, torch.float32)
        ref, s = _ln_fwd(self.r("x2"), col(3), col(4), i["ln_eps"])
        self._out("xn2", "xn2", ref, s, torch.bfloat16, c=2.0)
        y, s_y = self._gemm(self.r("xn2"), W["fc1"], bias["fc1"])
        g, s_g = gb.gelu_out(y, s_y)
        self._out("h/pre", "h", g, s_g, torch.bfloat16, c=1.0)
        self._out("h/pre", "pre", y, s_y, torch.bfloat16)
        y, s_y = self._gemm(self.r("h"), W["fc2"], bias["fc2"])
        o, s = gb.residual_out(y, s_y, col(5), self.r("x2"))
        self._out("x3/y3", "x3", o, s, torch.float32)
        self._out("x3/y3", "y3", y, s_y, torch.bfloat16)

        # ---------------- backward
        self._gate_bwd("dy3 + dm[5]", "dy3", "dm5", dout, self.r("y3"), 5)
        dy3 = self.r("dy3")
        self._wgrad("fc2 wgrad + colsum", "dW.fc2", dy3, self.r("h"))
        self._colsum("fc2 wgrad + colsum", "db.fc2", dy3)
        acc, s_acc, _ = gb.accumulate(dy3, W["fc2"].T)
        ref, s = gb.dgelu_out(acc, s_acc, self.r("pre"))
        self._out("dpre", "dpre", ref, s, torch.bfloat16)
        self._lin_bwd("fc1 dgrad/wgrad/colsum", "fc1", self.r("dpre"), self.r("xn2"), "dxn2")
        self._ln_mod_bwd("dx2 + dm[3,4]", ("dx2", "dm3", "dm4"), self.r("x2"), self.r("dxn2"), mod[:, 4], N, i["ln_eps"],
                         add_in=dout)
        self._out("dy2", "dy2", self.r("dx2"), 0.0, torch.bfloat16)
        self._lin_bwd("cproj", "cproj", self.r("dy2"), self.r("ao2"), "dao2")
        self._attn_bwd("cross-attention backward", self.r("qx"), kv[:, :C], kv[:, C:], self.r("ao2"), self.r("lse2"),
                       self.r("dao2"), i["keys"], scale, ("dq2", "dk2", "dv2"))
        dq2 = self.r("dq2").reshape(M, C)
        dkv = torch.cat([self.r("dk2").reshape(-1, C), self.r("dv2").reshape(-1, C)], 1)
        self._lin_bwd("q / kv dgrad + wgrad", "q", dq2, xb, "dxb")
        self._lin_bwd("q / kv dgrad + wgrad", "kv", dkv, cond, "dcond")
        self._out("dx1", "dx1", self.r("dx2") + self.r("dxb"), 0.0, torch.float32)
        self._gate_bwd("dy1 + dm[2]", "dy1", "dm2", self.r("dx1"), self.r("y1"), 2)
        self._lin_bwd("proj", "proj", self.r("dy1"), self.r("ao1"), "dao1")
        self._attn_bwd("self-attention backward", q, k, v, self.r("ao1"), self.r("lse1"), self.r("dao1"), self_keys, scale,
                       ("dq1", "dk1", "dv1"))
        dq1, dk1, dv1 = self.r("dq1").reshape(M, C), self.r("dk1").reshape(-1, C), self.r("dv1").reshape(-1, C)
        if pick is not None:                                           # scattered into the zero-filled dqkv (torch)
            dk1, dv1 = (torch.zeros_like(dq1).index_copy_(0, pick, d) for d in (dk1, dv1))
        if i["qk"] is not None:
            qkv_pre = self.r("qkv")
            for j, (roles, d) in enumerate(((("dqn", "db.q_norm", "dw.q_norm"), dq1), (("dkn", "db.k_norm", "dw.k_norm"), dk1))):
                w, _ = i["qk"]["qk"[j]]
                self._ln_mod_bwd("qk-norm backward", roles, qkv_pre[:, j * C:(j + 1) * C], d, (w - 1)[None], M, i["qk_eps"])
            dq1, dk1 = cast(self.r("dqn")), cast(self.r("dkn"))       # stored into the bf16 dqkv (torch)
        dqkv = torch.cat([dq1, dk1, dv1], 1)
        self._lin_bwd("qkv", "qkv", dqkv, self.r("xn1"), "dxn1")
        self._ln_mod_bwd("dx + dm[0,1]", ("dx", "dm0", "dm1"), x, self.r("dxn1"), mod[:, 1], N, i["ln_eps"], add_in=self.r("dx1"))
        return self.tallies


def roles_of(trace, expected):
    """{role: after-snapshot} of a recorded trace [(name, before, after)] against expected_trace; the names must match in
    order.  Also returns {role: before-snapshot}."""
    names = [t[0] for t in trace]
    want = [n for n, _ in expected]
    assert names == want, f"kernel trace differs from expected_trace:\n got  {names}\n want {want}"
    after, before = {}, {}
    for (name, bef, aft), (_, outs) in zip(trace, expected):
        for slot, role in outs.items():
            after[role], before[role] = aft[slot], bef[slot]
    return after, before


def round_to(ref, dtype):
    """The emulated kernel output: the float64 reference rounded once to the output dtype."""
    return ref.to(dtype).double()


def exact(ref, dtype):
    return ref
