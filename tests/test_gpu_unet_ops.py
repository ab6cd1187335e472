"""GPU: every op of the MDM_UNET engine's op lists (the forward, the guided forward and the fp16 input-VJP) against an fp64
reference of the same op on the inputs the op actually read.

Engine.test_unet_ops runs a real forward (or guided forward + input-VJP) and calls back around every op; before the op
the test reads its inputs from the engine's buffers, decoded the way the op reads them (bf16 hi + lo, hi alone, one fp16
plane, fp32), after it the output.  The reference of an op is the module its name points to (oracle/unet_ops.py, the
state-dict prefix; tests/test_unet_ops_reference.py shows those compose to the model), with the weights rounded the way
the engine rounds them -- not the op's own parameters, so a wrong tap, phase, weight or bias fails.  Every output's halo
rows (the zero padding the next 5-tap convolution reads) must be exactly 0.

Gates, elementwise, with |A| * |W| the same op on absolute values (the scale of the accumulation) and R the reference:
  bf16x3  GEMM  |E - R| <= 8 * 2^-18 * (|A| * |W| + |b| + |res|) + the output's rounding (hi + lo: 2^-16 |R|)
          GroupNorm-Mish: hi + lo within 2^-15 |R| + 2^-20 * max|R| of its group
  bf16    GEMM  over bf16(A), bf16(W): |E - R| <= 2^-20 * (|A| * |W| + ...) + the output's rounding (hi alone: half a
          bf16 ulp, + 1/16 ulp for the fp32 value it rounds)
          GroupNorm-Mish: as bf16x3 on hi + lo, and hi within half a bf16 ulp (+ 1/16)
  fp16    GEMM  R at autocast's rounding points: fp16(fp16(S) + fp16(b)) for a convolution, fp16(S + fp16(b)) for a
          linear layer, fp16(S) + res in fp32 for an input-VJP sum; E within two fp16 ulps of the larger of |S|, |R|
          plus 2^-20 |A| * |W| (the fp32 sum is one ulp off where it cancels; the second rounding can follow it)
          GroupNorm-Mish (and its backward): within one fp16 ulp of R plus 2^-20 * max|R| of the group; out_f32 at fp32
          and at most FRAC16 of an op's elements not exactly R (GEMMs, GroupNorm and its backward)
The ratio max(|E - R| / bound) of every op and its share off R are printed; the test fails above 1 or above FRAC16.
Worst measured on one H100 80 GB: bf16x3 GEMM 0.064, GroupNorm 0.25; bf16 GEMM 0.89, GroupNorm 0.89; fp16 GEMM 0.996
(forward) and 0.99 (input-VJP), GroupNorm and its backward 0.50; off R 1.1e-3.  The embedding builder is bit-exact from
the engine's own timestep-table row and text projection, each of which is checked against fp64 on its own.
"""
import pytest
import torch
import torch.nn.functional as F

import condmdi_b200 as C
from oracle import condmdi_oracle as O
from oracle import unet_ops as U

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
X3, BF, H = C.PRECISION_BF16X3, C.PRECISION_BF16, C.PRECISION_FP16
PNAME = {X3: "bf16x3", BF: "bf16", H: "fp16"}
ULP16_MIN = 2.0 ** -24


class _Arr:
    def __init__(self, ptr, n, typestr):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": typestr, "data": (ptr, False), "version": 3, "strides": None}


def raw(ptr, rows, cols, ld, dtype):
    """a [rows, cols] view with row pitch ld of engine memory, copied to fp64"""
    assert ptr, "null view"
    n = (rows - 1) * ld + cols
    ts = {torch.float32: "<f4", torch.float16: "<f2", torch.bfloat16: "<i2"}[dtype]
    t = torch.as_tensor(_Arr(ptr, n, ts), device=DEV)
    if dtype == torch.bfloat16:
        t = t.view(torch.bfloat16)
    return t.as_strided((rows, cols), (ld, 1)).to(torch.float64)


def planes(hi, lo, rows, cols, ld, mode):
    """mode 'x3': bf16 hi + lo, 'bf': hi alone, 'h': one fp16 plane"""
    if mode == "h":
        return raw(hi, rows, cols, ld, torch.float16)
    v = raw(hi, rows, cols, ld, torch.bfloat16)
    return v + raw(lo, rows, cols, ld, torch.bfloat16) if mode == "x3" else v


def lp(level):
    return 256 >> level


def interior(t, level, nseq):
    """level layout [nseq * Lp, C] -> [nseq, C, 224 >> level]"""
    return t.view(nseq, lp(level), -1)[:, 2:2 + (224 >> level)].transpose(1, 2)


def halo_max(t, level, nseq):
    v = t.view(nseq, lp(level), -1)
    return max(v[:, :2].abs().max().item(), v[:, 2 + (224 >> level):].abs().max().item())


def f16(t):
    return t.half().double()


def ulp16(t):
    """the fp16 spacing at |t| (subnormal spacing below 2^-14)"""
    a = t.abs().clamp_min(2.0 ** -14)
    return torch.exp2(torch.floor(torch.log2(a)) - 10).clamp_min(ULP16_MIN)


def ulpbf(t):
    a = t.abs().clamp_min(2.0 ** -126)
    return torch.exp2(torch.floor(torch.log2(a)) - 7)


def group_scale(r):
    """max |r| per (sequence, group of 8) broadcast back: [nseq, C, P]"""
    n, c, p = r.shape
    return r.abs().view(n, 8, c // 8 * p).amax(-1).repeat_interleave(c // 8, 1)[..., None]


# gate constants (the ratios they give on H100 are in the module docstring)
C_X3 = 8.0 * 2.0 ** -18
C_BF = 2.0 ** -20
C_GN = 2.0 ** -20
C_ACC16 = 2.0 ** -20
# fp16: the share of an op's elements that are not exactly autocast's value R (where an fp32 sum one ulp off from the
# exact one crosses an fp16 rounding boundary).  Measured on H100: at most 1.1e-3 for any GEMM, GroupNorm or backward op.
# A reference with one of autocast's rounding points left out is 2.3e-2 (the bias unrounded) .. 0.54 (SUM32's fp32 sum
# rounded) off R on every op it touches, while its ulp bound alone passes them at 0.50 .. 0.99.
FRAC16 = 4e-3


class Checker:
    """the hook: checks every op against its reference and records (list, name) -> ratio"""

    def __init__(self, sd, prec, cfg, B, x, xo, kf_mask, perturb=None):
        self.sd = {k: v.to(DEV, torch.float64) for k, v in sd.items()}
        self.prec, self.cfg, self.B, self.perturb = prec, cfg, B, perturb
        self.x, self.xo, self.kf_mask = x, xo, kf_mask
        self.ada_cols = U.ada_columns(sd)
        self.inputs, self.ratios, self.halo = {}, {}, {}
        self.ada_base = None
        self.block_in = {}
        self.off = {}        # fp16: (list, op, name) -> share of elements != R
        self.list_ops = {}   # list -> its length, as the engine reports it
        self.checked = {}    # list -> indices of the ops checked
        self.sum32 = set()

    # -------- weights as the engine holds them --------
    def wb(self, name):
        w, b = U.weight_bias(self.sd, name)
        if self.perturb == "tap" and w.dim() == 3 and w.shape[-1] == 5:
            w = torch.roll(w, 1, dims=-1)
        if self.perturb == "bias" and b is not None:
            b = b.clone()
            b[0] = 0.0
        if self.prec == BF:
            w = w.float().bfloat16().double()
        elif self.prec == H:
            w, b = f16(w), (b.float().double() if self.perturb == "bias_unrounded" else f16(b))
        else:
            w = w.float().double()
        return w, b.float().double() if self.prec != H else b

    def a_mode(self, info):
        return "h" if info.f16 else ("x3" if info.nsplit == 3 else "bf")

    def out_mode(self, info):
        return "h" if info.f16 else ("x3" if info.nsplit_out == 3 else "bf")

    def __call__(self, lst, i, phase, info):
        name = info.name.decode()
        key = (lst, i)
        nseq = info.num_seqs
        if phase == 0:
            self.inputs[key] = self.read_inputs(info, name, nseq)
            return
        ins = self.inputs.pop(key)
        handlers = {0: self.gemm, 1: self.gn, 2: self.input_builder, 3: self.emb, 4: self.gn_bwd, 5: self.input_grad}
        assert info.kind in handlers, f"{name}: op kind {info.kind} has no reference"
        self.cur = (lst, i, name)
        if info.kind == 0 and info.sum32:
            self.sum32.add(self.cur)
        self.ratios[self.cur] = handlers[info.kind](info, name, nseq, ins)
        assert self.list_ops.setdefault(lst, info.list_ops) == info.list_ops
        self.checked.setdefault(lst, set()).add(i)

    def note_off(self, e, r):
        """fp16: the share of elements of E that are not exactly R (R already at E's rounding)"""
        k = self.cur
        self.off[k] = max(self.off.get(k, 0.0), (e != r).double().mean().item())

    # -------- inputs --------
    def read_inputs(self, info, name, nseq):
        if info.kind == 0:
            w, _ = U.weight_bias(self.sd, name)
            tr = name.endswith("^T")
            up = U.is_upsample(name)
            if ".time_mlp." in name:
                return {"a": planes(info.in_hi, info.in_lo, nseq, w.shape[1], info.in_ld, self.a_mode(info)),
                        "res": None}
            cin = (w.shape[1] if up else w.shape[0]) if tr else (w.shape[0] if up else w.shape[1])
            cols = min(cin, info.in_ld)
            a = planes(info.in_hi, info.in_lo, nseq * lp(info.in_level), cols, info.in_ld, self.a_mode(info))
            res = raw(info.residual, nseq * lp(info.out_level), info.N, info.ld_res, torch.float32) if info.residual else None
            return {"a": a, "res": res}
        if info.kind == 1:
            rows = nseq * lp(info.level)
            d = {"y": raw(info.y, rows, info.C, info.ld_y, torch.float32), "ada": None, "res": None}
            if info.ada:
                d["ada"] = raw(info.ada, nseq, 2 * info.C, info.ld_ada, torch.float32)
            if info.res_f32:
                d["res"] = raw(info.res_f32, rows, info.C, info.ld_res_gn, torch.float32)
            elif info.res_hi:
                d["res"] = planes(info.res_hi, info.res_lo, rows, info.C, info.ld_res_gn,
                                  "h" if info.f16 else ("x3" if info.res_lo else "bf"))
            return d
        if info.kind == 4:
            rows = nseq * lp(info.level)
            d = {"y": raw(info.y, rows, info.C, info.ld_y, torch.float16),
                 "ada": raw(info.ada, nseq, 2 * info.C, info.ld_ada, torch.float32) if info.ada else None}
            d["dout"] = (raw(info.dout, rows, info.C, info.ld_dout, torch.float32) if info.dout
                         else raw(info.dout_h, rows, info.C, info.ld_dout, torch.float16))
            d["add"] = raw(info.dout_add, rows, info.C, info.ld_add, torch.float32) if info.dout_add else None
            return d
        if info.kind == 5:
            return {"xg": raw(info.in_f32, nseq * 256, self.x.shape[1], info.in_ld, torch.float32)}
        return {}

    def check_ada(self, info, name):
        pre = name.removesuffix("^T")[: -len("blocks.0.block1.2")]
        assert self.ada_base is not None
        assert info.ada == self.ada_base + 4 * self.ada_cols[pre], f"{name}: AdaGN reads another block's [scale | shift]"

    # -------- GEMMs --------
    def gemm(self, info, name, nseq, ins):
        tr = name.endswith("^T")
        base = name.removesuffix("^T")
        w, b = self.wb(base)
        a = ins["a"]
        if name == "*.time_mlp.1":
            self.ada_base = info.out_f32
        if ".time_mlp." in base:
            s, sa = F.linear(a, w), F.linear(a.abs(), w.abs())
            out_rows, lvl = nseq, None
        elif tr:
            in_len = 224 >> info.out_level
            dout = interior(a, info.in_level, nseq)
            if base == "unet.final_conv.1":
                dout = dout[:, : w.shape[0]]
            s = U.gemm_vjp(base, dout, w, in_len)
            sa = U.gemm_vjp(base, dout.abs(), w.abs(), in_len)
            b = None
            # the GEMM's N columns: the first D_pad input channels of downs.0.0 (x_t's share), or zero columns past C_in
            pad = 0 if base.endswith(".3.conv") else info.N - s.shape[1]  # (Downsample^T: N = 2C over pair rows)
            s, sa = (F.pad(s, (0, 0, 0, pad)), F.pad(sa, (0, 0, 0, pad))) if pad > 0 else (s[:, : info.N], sa[:, : info.N])
            lvl = info.out_level
        else:
            x = interior(a, info.in_level, nseq)
            s, sa = U.gemm_forward(base, x, w, None), U.gemm_forward(base, x.abs(), w.abs(), None)
            lvl = info.out_level
            if self.perturb == "phase" and base.startswith("unet.ups."):
                s = s.view(s.shape[0], s.shape[1], -1, 2).flip(-1).reshape(s.shape)
        bb = None if b is None else (b[:, None] if s.dim() == 3 else b)
        res = None
        if ins["res"] is not None:
            res = interior(ins["res"], lvl, nseq)
        if self.prec == H:
            s16 = f16(s)
            if tr or ".time_mlp." not in base:
                if self.perturb == "sum_unrounded":  # (teeth: the convolution's sum not rounded before its bias)
                    v = f16(s) if bb is None else f16(s + bb)
                else:
                    v = s16 if bb is None else f16(s16 + bb)
                if res is not None:
                    if info.sum32 and self.perturb != "sum32_rounded":
                        v = (s16 + res).float().double()   # fp16 dgrad + fp32 residual, not rounded again
                    else:
                        v = f16(v + res)
            else:
                v = f16(s + bb)
            if U.gemm_act(base):
                v = f16(F.mish(v))
            # two roundings (the sum, then sum + bias or after Mish), each of which an fp32 sum one ulp off can move
            bound = 2.0 * ulp16(torch.maximum(s.abs(), v.abs())) + C_ACC16 * sa
            ref = v
        else:
            v = s if bb is None else s + bb
            if res is not None:
                v = v + res
            scale = sa + (0 if bb is None else bb.abs()) + (0 if res is None else res.abs())
            ref = F.mish(v) if U.gemm_act(base) else v
            bound = (C_X3 if self.prec == X3 else C_BF) * scale * (1.1 if U.gemm_act(base) else 1.0)
        worst = 0.0
        outs = []
        if info.rowmap == 3:  # final_conv.1: frame-major model_out rows of the first L frames
            L, D = info.frames, w.shape[0]
            e = raw(info.out_f32, nseq * L, D, info.out_ld32, torch.float32).view(nseq, L, D).transpose(1, 2)
            outs.append((e, ref[..., :L], bound[..., :L], None))
        elif lvl is None:
            if info.out_f32:
                outs.append((raw(info.out_f32, nseq, info.N, info.out_ld32, torch.float32), ref, bound, None))
            if info.out_hi:
                m = self.out_mode(info)
                outs.append((planes(info.out_hi, info.out_lo, nseq, info.N, info.out_ld, m), ref,
                             bound + (0 if m == "h" else self.rnd(m, ref)), None))
        else:
            cout = ref.shape[1]
            rows = nseq * lp(lvl)
            if info.out_f32:
                full = raw(info.out_f32, rows, cout, info.out_ld32, torch.float32)
                outs.append((interior(full, lvl, nseq), ref, bound, full))
            if info.out_hi:
                m = self.out_mode(info)
                full = planes(info.out_hi, info.out_lo, rows, cout, info.out_ld, m)
                if m == "h":  # (a sum32 output's fp16 plane is the rounding of its fp32 value)
                    outs.append((interior(full, lvl, nseq), f16(ref) if info.sum32 else ref, bound + (ulp16(ref) if info.sum32 else 0), full))
                else:
                    outs.append((interior(full, lvl, nseq), ref, bound + self.rnd(m, ref), full))
        assert outs, name
        for e, r, bd, full in outs:
            k = min(e.shape[1], r.shape[1])
            worst = max(worst, ((e[:, :k] - r[:, :k]).abs() / bd[:, :k].clamp_min(1e-300)).max().item())
            if e.shape[1] > k:  # dgrad columns past the module's input channels (D_pad > njoints)
                assert e[:, k:].abs().max().item() == 0, name
            if full is not None:
                self.halo[(name, full.data_ptr())] = halo_max(full, lvl, nseq)
            if self.prec == H:
                self.note_off(e[:, :k], r[:, :k])
        return worst

    def rnd(self, mode, ref):
        # bf: half a bf16 ulp of the fp32 value, which is itself off R by the fp32 arithmetic (1/16 ulp of slack)
        return {"x3": 2.0 ** -16 * ref.abs(), "bf": ulpbf(ref) * 0.5625, "h": ulp16(ref)}[mode]

    # -------- GroupNorm -> AdaGN -> Mish -> + residual --------
    def gn(self, info, name, nseq, ins):
        lvl = info.level
        g, bt = self.sd[name + ".weight"], self.sd[name + ".bias"]
        y = interior(ins["y"], lvl, nseq)
        scale = shift = None
        if ins["ada"] is not None:
            self.check_ada(info, name)
            scale, shift = ins["ada"][:, : info.C], ins["ada"][:, info.C:]
        res = None if ins["res"] is None else interior(ins["res"], lvl, nseq)
        pre = name[: -len("blocks.1.block.2")]
        blk = self.block_in.pop(pre, None) if name.endswith("blocks.1.block.2") else None
        if blk is not None and pre + "residual_conv.weight" not in self.sd:
            # an identity residual is the block's input as its first convolution read it
            assert torch.equal(f16(res) if self.prec == H else res, blk), f"{name}: residual is not the block input"
        ops_round = f16 if self.prec == H and self.perturb != "scale_unrounded" else None
        ref = U.gn_mish(y, g.double(), bt.double(), scale, shift, res, one_plus_scale=ops_round)
        slack = C_GN * group_scale(ref)
        rows = nseq * lp(lvl)
        worst = 0.0
        if self.prec == H:
            e = raw(info.gn_out_hi, rows, info.C, info.ld_gn_out, torch.float16)
            worst = max(worst, ((interior(e, lvl, nseq) - ref).abs() / (ulp16(ref) + slack)).max().item())
            self.note_off(interior(e, lvl, nseq), f16(ref))
            self.halo[(name, e.data_ptr())] = halo_max(e, lvl, nseq)
            if info.gn_out_f32:
                e32 = raw(info.gn_out_f32, rows, info.C, info.ld_gn_out_f32, torch.float32)
                worst = max(worst, ((interior(e32, lvl, nseq) - ref).abs() / (2.0 ** -22 * ref.abs() + slack)).max().item())
                self.halo[(name + " f32", e32.data_ptr())] = halo_max(e32, lvl, nseq)
        else:
            e = planes(info.gn_out_hi, info.gn_out_lo, rows, info.C, info.ld_gn_out, "x3")
            worst = max(worst, ((interior(e, lvl, nseq) - ref).abs() / (2.0 ** -15 * ref.abs() + slack)).max().item())
            self.halo[(name, e.data_ptr())] = halo_max(e, lvl, nseq)
            if self.prec == BF:
                hi = interior(planes(info.gn_out_hi, None, rows, info.C, info.ld_gn_out, "bf"), lvl, nseq)
                worst = max(worst, ((hi - ref).abs() / (0.5625 * ulpbf(ref) + slack)).max().item())
        return worst

    def gn_bwd(self, info, name, nseq, ins):
        lvl = info.level
        base = name.removesuffix("^T")
        g, bt = self.sd[base + ".weight"], self.sd[base + ".bias"]
        y = interior(ins["y"], lvl, nseq)
        dout = ins["dout"]
        rows = nseq * lp(lvl)
        if ins["add"] is not None:
            total = (dout + ins["add"]).float().double()
            back = raw(info.dout, rows, info.C, info.ld_dout, torch.float32)
            assert torch.equal(back, total), f"{name}: dout + dout_add written back"
            dout = total
        scale = shift = None
        if ins["ada"] is not None:
            self.check_ada(info, name)
            scale, shift = ins["ada"][:, : info.C], ins["ada"][:, info.C:]
        ref = U.gn_mish_vjp(y, interior(dout, lvl, nseq), g.double(), bt.double(), scale, shift,
                            one_plus_scale=None if self.perturb == "scale_unrounded" else f16)
        e = raw(info.dy, rows, info.C, info.ld_dy, torch.float16)
        self.halo[(name, e.data_ptr())] = halo_max(e, lvl, nseq)
        self.note_off(interior(e, lvl, nseq), f16(ref))
        return ((interior(e, lvl, nseq) - ref).abs() / (ulp16(ref) + C_GN * group_scale(ref))).max().item()

    # -------- the builders and the input gradient: bit-exact --------
    def input_builder(self, info, name, nseq, ins):
        B, D, L = self.x.shape[0], self.x.shape[1], self.x.shape[-1]
        x = self.x.to(DEV).reshape(B, D, L).double()
        if self.xo is not None:
            m = self.kf_mask.to(DEV).reshape(B, D, L)
            x = torch.cat([torch.where(m, self.xo.to(DEV).reshape(B, D, L).double(), x), m.double()], 1)
        v = torch.zeros(nseq, 256, info.out_ld, dtype=torch.float64, device=DEV)
        v[:, 2:2 + L, : x.shape[1]] = x.repeat(nseq // B, 1, 1).transpose(1, 2)
        v = v.view(nseq * 256, -1)
        rows, ld = nseq * 256, info.out_ld
        if self.prec == H:
            assert torch.equal(raw(info.out_hi, rows, ld, ld, torch.float16), f16(v)), "input builder (fp16)"
        else:
            hi = v.float().bfloat16()
            assert torch.equal(raw(info.out_hi, rows, ld, ld, torch.bfloat16), hi.double()), "input builder (hi)"
            assert torch.equal(raw(info.out_lo, rows, ld, ld, torch.bfloat16), (v.float() - hi.float()).bfloat16().double()), \
                "input builder (lo)"
        return 0.0

    def emb(self, info, name, nseq, ins):
        """the embedding rows, bit-exact from the engine's timestep table row and text projection: fp32 sum split into bf16
        hi / lo, or at fp16 fp16(table + fp16(projection)); then the table row and the projection each against fp64"""
        sd, t, B = self.sd, self.t, self.B
        row = raw(info.temb_table + 4 * 512 * t, 1, 512, 512, torch.float32)[0]
        add = torch.zeros(nseq, 512, dtype=torch.float64, device=DEV)
        if info.cond_proj:
            proj = raw(info.cond_proj, B, 512, 512, torch.float32)
            unc = raw(info.uncond_proj, 1, 512, 512, torch.float32)[0]
            assert torch.equal(unc, sd["embed_text.bias"].float().double()), "embed_text(0) is not the bias"
            seqs = torch.arange(nseq, device=DEV)
            add = torch.where((seqs < info.n_cond_seqs)[:, None], proj[seqs % B], unc[None])
            assert info.n_cond_seqs == (0 if self.uncond else B)
            self.check_linear(proj, self.cond.to(DEV).double(), sd["embed_text.weight"], sd["embed_text.bias"], "embed_text")
        else:
            assert self.cond is None
        rows = nseq
        if self.prec == H:
            want = (row[None].float() + (add.half().float() if info.cond_proj else 0)).half().double().expand(nseq, 512)
            assert torch.equal(raw(info.out_hi, rows, 512, info.out_ld, torch.float16), want), "embedding builder (fp16)"
        else:
            v = (row[None].float() + add.float()) if info.cond_proj else row[None].float().expand(nseq, 512)
            hi = v.bfloat16()
            assert torch.equal(raw(info.out_hi, rows, 512, info.out_ld, torch.bfloat16), hi.double()), "embedding builder (hi)"
            assert torch.equal(raw(info.out_lo, rows, 512, info.out_ld, torch.bfloat16), (v - hi.float()).bfloat16().double()), \
                "embedding builder (lo)"
        return self.check_temb(row)

    def quant(self, t):
        return {X3: t.float().double(), BF: t.float().bfloat16().double(), H: f16(t)}[self.prec]

    def check_linear(self, e, x, w, b, what):
        """embed_text(cond) as the engine computes it: fp32 FMAs of the fp32 operands, or autocast's fp16 linear"""
        if self.prec == H:
            s_, sa = F.linear(f16(x), f16(w)), F.linear(f16(x).abs(), f16(w).abs())
            r = f16(s_ + f16(b))
            bound = 2.0 * ulp16(torch.maximum(s_.abs(), r.abs())) + C_ACC16 * sa
        else:
            r = F.linear(x, w, b)
            bound = 2.0 ** -17 * (F.linear(x.abs(), w.abs()) + b.abs())  # (K = 512 fp32 FMAs)
        ratio = ((e - r).abs() / bound).max().item()
        assert ratio <= 1.0, f"{what}: {ratio:.3f} of its bound"

    def check_temb(self, row):
        """the table row time_embed(pe[t]) (Linear -> SiLU -> Linear at the engine's precision) against fp64, each layer's
        operands rounded as the engine rounds them, the first layer's error carried through the second's |W|"""
        sd, q = self.sd, self.quant
        pe = sd["sequence_pos_encoder.pe"].reshape(5000, -1)[self.t]
        w0, b0 = sd["embed_timestep.time_embed.0.weight"], sd["embed_timestep.time_embed.0.bias"]
        w2, b2 = sd["embed_timestep.time_embed.2.weight"], sd["embed_timestep.time_embed.2.bias"]
        if self.prec == H:
            b0, b2 = f16(b0), f16(b2)
        u, rh = {X3: (C_X3, 2.0 ** -16), BF: (C_BF, 2.0 ** -8), H: (C_ACC16, 2.0 ** -10)}[self.prec]
        h = F.silu(q(w0) @ q(pe) + b0)
        dh = 1.1 * u * (q(w0).abs() @ q(pe).abs() + b0.abs()) + rh * h.abs() + (ulp16(h) if self.prec == H else 0)
        r = q(w2) @ q(h) + b2
        bound = q(w2).abs() @ dh + u * (q(w2).abs() @ q(h).abs() + b2.abs()) + (2.0 * ulp16(r) if self.prec == H else 0)
        return ((row - r).abs() / bound).max().item()

    def input_grad(self, info, name, nseq, ins):
        B, D, L = self.x.shape[0], self.x.shape[1], self.x.shape[-1]
        g = interior(ins["xg"], 0, nseq)[..., :L]
        if self.kf_mask is not None:
            g = g * (~self.kf_mask.to(DEV).reshape(B, D, L)).double().repeat(nseq // B, 1, 1)
        e = raw(info.out_f32, nseq * L, D, info.out_ld32, torch.float32).view(nseq, L, D).transpose(1, 2)
        assert torch.equal(e, g), "input gradient"
        return 0.0


# ------------------------------------------------------------------------------------------------------------------------
def model(mults, kf, text, feats):
    sd = O.random_unet_state_dict(seed=11, mults=mults, keyframe_conditioned=kf, text=text, feats=feats)
    m = C.MDM_UNET(dim_mults=mults, keyframe_conditioned=kf, njoints=feats,
                   **({"cond_mode": "text", "cond_mask_prob": 0.1} if text else {}))
    assert not any(m.load_state_dict(sd, strict=False))
    return m.to(DEV), sd


def inputs(B, D, L, seed, kf, text):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, D, 1, L, generator=g)
    xo = torch.randn(B, D, 1, L, generator=g) if kf else None
    lengths = torch.randint(max(L // 5, 2), L + 1, (B,), generator=g)
    if kf and D == 263:
        mask = C.get_keyframes_mask(torch.randn(B, D, 1, L, generator=g), lengths, "benchmark_sparse", trans_length=5)
    else:  # (other feature sets: random keyframe columns)
        mask = (torch.rand(B, 1, 1, L, generator=g) < 0.2).expand(B, D, 1, L).contiguous() if kf else None
    cond = torch.randn(B, 512, generator=g) if text else None
    scale = torch.full((B,), 2.5)
    return x, xo, mask, cond, scale


def run_ops(mults, kf, text, feats, L, B, cfg, prec, vjp=False, perturb=None, seed=3):
    m, sd = model(mults, kf, text, feats)
    eng = m.engine_for(DEV, max_batch=B, precision=prec, nframes=L)
    x, xo, mask, cond, scale = inputs(B, feats, L, seed, kf, text)
    chk = Checker(sd, prec, cfg, B, x, xo, mask, perturb)
    chk.cond, chk.uncond = cond, False
    t = chk.t = 500
    orig = chk.gemm

    def gemm(info, name, nseq, ins):  # remember each block's input as its first convolution read it
        if name.endswith("blocks.0.block1.0") and not name.endswith("^T"):
            # (in the encoding an identity residual reads: hi + lo also where the convolution reads hi alone)
            a = planes(info.in_hi, info.in_lo, nseq * lp(info.in_level), ins["a"].shape[1], info.in_ld, "h" if info.f16 else "x3")
            chk.block_in[name[: -len("blocks.0.block1.0")]] = interior(a, info.in_level, nseq)
        return orig(info, name, nseq, ins)

    chk.gemm = gemm
    kw = dict(cond_emb=cond, cfg=cfg, text_scale=scale if cfg else None, obs_x0=xo, obs_mask=mask)
    if vjp:
        g = torch.Generator().manual_seed(seed + 1)
        target = torch.randn(B, feats, 1, L, generator=g)
        imask = torch.rand(B, feats, 1, L, generator=g) < 0.4
        eng.test_unet_ops(chk, x, t, inpainted_motion=target, inpainting_mask=imask, **kw)
    else:
        eng.test_unet_ops(chk, x, t, **kw)
    torch.cuda.synchronize()
    return chk


def report(chk, what):
    lists = {0: "forward", 1: "guided", 2: "vjp"}
    kinds = {}
    offs = {}
    for key, r in sorted(chk.ratios.items(), key=lambda kv: (kv[0][0], kv[0][1])):
        lst, i, name = key
        print(f"[{what}] {lists[lst]:7s} {i:3d} {name:42s} max|E-R|/bound = {r:.3f}"
              + (f"  off R: {chk.off[key]:.2e}" if key in chk.off else ""))
        k = ("^T" if name.endswith("^T") else "") + ("gn" if U.is_gn(name) else "gemm")
        kinds[k] = max(kinds.get(k, 0.0), r)
        if key in chk.off:
            offs[k] = max(offs.get(k, 0.0), chk.off[key])
    print(f"[{what}] worst per kind: " + ", ".join(f"{k} {v:.3f}" for k, v in sorted(kinds.items()))
          + ("; off R: " + ", ".join(f"{k} {v:.2e}" for k, v in sorted(offs.items())) if offs else ""))
    return kinds


def failing(chk):
    """the ops outside their bound, or (fp16) off R in more than FRAC16 of their elements"""
    return {k: (r, chk.off.get(k)) for k, r in chk.ratios.items() if not (r <= 1.0 and chk.off.get(k, 0.0) <= FRAC16)}


def assert_all(chk, what):
    report(chk, what)
    # coverage: every op of every list the call ran was checked (an op without a reference fails inside the hook)
    assert not chk.inputs, f"ops read but never completed: {list(chk.inputs)}"
    for lst, n in chk.list_ops.items():
        assert chk.checked[lst] == set(range(n)), f"{what}: list {lst} has {n} ops, checked {sorted(chk.checked[lst])}"
    bad = failing(chk)
    assert not bad, f"{what}: ops outside their bound or off R: {bad}"
    halo = {k: v for k, v in chk.halo.items() if v != 0}
    assert not halo, f"{what}: non-zero halo rows: {halo}"


XL = ((2, 2, 2, 2), True, True, 263, 196)
CASES = {
    "xl-kf-text-B2-cfg": (XL, 2, True),
    "xl-kf-text-B64-cfg": (XL, 64, True),
    "111-nokf-B2": (((1, 1, 1), False, False, 263, 196), 2, False),
    "764x120-kf-B2": (((1, 1), True, False, 764, 120), 2, False),
}


@pytest.mark.parametrize("prec", [X3, BF, H], ids=PNAME.get)
@pytest.mark.parametrize("case", list(CASES))
def test_unet_forward_ops(case, prec):
    """every op of the forward list against its reference; no op of the list without one (coverage)"""
    if case == "764x120-kf-B2" and prec != H:
        pytest.skip("the 764 x 120 geometry is the fp16 one")
    cfg_, B, cfg = CASES[case]
    chk = run_ops(*cfg_, B, cfg, prec)
    assert_all(chk, f"{case} {PNAME[prec]}")
    assert set(chk.list_ops) == {0}


@pytest.mark.parametrize("case", ["xl-kf-text-B2-cfg", "xl-kf-text-B64-cfg", "111-nokf-B2", "764x120-kf-B2"])
def test_unet_fp16_guided_and_vjp_ops(case):
    """fp16: every op of the guided forward (its stash outputs included) and of the input-VJP, through the input gradient"""
    cfg_, B, cfg = CASES[case]
    chk = run_ops(*cfg_, B, cfg, H, vjp=True)
    assert_all(chk, f"{case} fp16 vjp")
    assert set(chk.list_ops) == {1, 2}
    assert any(name == "input^T" for _, _, name in chk.ratios)


@pytest.mark.parametrize("perturb", ["tap", "phase", "bias"])
@pytest.mark.parametrize("prec", [X3, H], ids=PNAME.get)
def test_reference_perturbations_fail_the_gates(perturb, prec):
    """teeth: with the kernels unchanged, a reference whose 5-tap weights are shifted by one tap, whose Upsample phases are
    swapped, or whose first output channel has no bias puts the ops it touches far outside their bounds"""
    chk = run_ops((1, 1, 1), False, False, 263, 196, 2, False, prec, perturb=perturb)
    touched = {"tap": lambda n: n.endswith("block1.0") or n.endswith("block.0"),
               "phase": lambda n: n.startswith("unet.ups.") and n.endswith(".3.conv"),
               "bias": lambda n: not U.is_gn(n) and n not in ("input", "emb")}[perturb]
    hit = {name: r for (_, _, name), r in chk.ratios.items() if touched(name)}
    print(f"[teeth {perturb} {PNAME[prec]}] smallest ratio of a perturbed op: {min(hit.values()):.1f}")
    assert hit and min(hit.values()) > 4.0


ROUNDING_POINTS = {
    # the convolution's sum rounded to fp16 before its fp16 bias is added (gemm_epilogue.cuh, F16 && num_taps > 0)
    "sum_unrounded": lambda n, info: not n.endswith("^T") and ".time_mlp." not in n and not U.is_gn(n) and n not in ("input", "emb"),
    # the bias rounded to fp16
    "bias_unrounded": lambda n, info: not n.endswith("^T") and not U.is_gn(n) and n not in ("input", "emb"),
    # linear2_f16_sum32_kernel: the fp16 dgrad plus the fp32 residual, not rounded again
    "sum32_rounded": lambda n, info: info,
    # AdaGN's 1 + scale rounded to fp16 (forward and backward)
    "scale_unrounded": lambda n, info: n.removesuffix("^T").endswith("blocks.0.block1.2"),
}


@pytest.mark.parametrize("perturb", list(ROUNDING_POINTS))
def test_fp16_reference_without_a_rounding_point_fails_the_gates(perturb):
    """teeth at fp16: a reference that leaves out one of autocast's rounding points makes every op it touches fail its
    gate, by its bound or by its share of elements off R"""
    chk = run_ops((1, 1, 1), False, True, 263, 196, 2, True, H, vjp=True, perturb=perturb)
    touched = [k for k in chk.ratios if ROUNDING_POINTS[perturb](k[2], k in chk.sum32)]
    fails = failing(chk)
    print(f"[teeth {perturb}] {len(touched)} ops touched; least off R: "
          f"{min(chk.off[k] for k in touched):.2e}, largest ratio {max(chk.ratios[k] for k in touched):.2f}")
    assert touched and all(k in fails for k in touched), [k for k in touched if k not in fails]


# ------------------------------------------------------------------------------------------------------------------------
def test_fp16_forward_and_vjp_do_not_depend_on_the_calls_before_them():
    """fp16: a forward and an input-VJP are bit-identical on a fresh engine and after a B = 64 CFG input-VJP, a guided
    sampling loop, an unconditional forward with other keyframes and a forward at another B"""
    m, sd = model(*XL[:3], 263)
    eng = m.engine_for(DEV, max_batch=64, precision=H, nframes=196)
    x, xo, mask, cond, scale = inputs(2, 263, 196, 1, True, True)
    x64, xo64, mask64, cond64, scale64 = inputs(64, 263, 196, 2, True, True)
    tgt = torch.randn(2, 263, 1, 196, generator=torch.Generator().manual_seed(5))
    imask = torch.rand(2, 263, 1, 196, generator=torch.Generator().manual_seed(6)) < 0.4

    def calls():
        f = eng.forward(x.to(DEV), 500, cond_emb=cond.to(DEV), cfg=True, text_scale=scale.to(DEV), obs_x0=xo.to(DEV),
                        obs_mask=mask.to(DEV))
        g = eng.test_input_vjp(x, 500, tgt, imask, cond_emb=cond, cfg=True, text_scale=scale, obs_x0=xo, obs_mask=mask)
        return f.clone(), g.clone()

    first = calls()
    eng.test_input_vjp(x64 * 3, 30, xo64, mask64, cond_emb=cond64, cfg=True, text_scale=scale64, obs_x0=xo64, obs_mask=mask64)
    d = C.create_gaussian_diffusion(timestep_respacing="ddim5")
    d.precision = H
    w = C.ClassifierFreeSampleModel(m)
    table = {str(i): cond64[i].to(DEV) for i in range(4)}
    m.encode_text = lambda texts: torch.stack([table[s] for s in texts])
    y = {"text": [str(i) for i in range(4)], "text_scale": scale64[:4].to(DEV), "inpainted_motion": xo64[:4].to(DEV),
         "inpainting_mask": mask64[:4].to(DEV), "reconstruction_guidance": True, "reconstruction_weight": 20.0,
         "gradient_schedule": None, "diffusion_steps": 1000, "stop_recguidance_at": 0,
         "mask": torch.ones(4, 1, 1, 196, dtype=torch.bool, device=DEV)}
    d.ddim_sample_loop(w, (4, 263, 1, 196), model_kwargs={"y": y, "obs_x0": xo64[:4].to(DEV), "obs_mask": mask64[:4].to(DEV)},
                       skip_timesteps=2, init_image=xo64[:4].to(DEV))
    eng.forward(x64[:5].to(DEV), 10, obs_x0=xo64[5:10].to(DEV), obs_mask=mask64[5:10].to(DEV))
    eng.forward(x64[:7].to(DEV), 700, cond_emb=cond64[:7].to(DEV), obs_x0=xo64[:7].to(DEV), obs_mask=mask64[:7].to(DEV))
    again = calls()
    for a, b, what in zip(first, again, ("forward", "input-VJP")):
        print(f"[fp16 {what} after other calls] max |diff| = {(a - b).abs().max().item():.3e}")
        assert torch.equal(a, b), what


def test_bf16x3_forward_does_not_depend_on_the_calls_before_it():
    """bf16x3: a CFG forward is bit-identical on a fresh engine and after a B = 64 CFG forward, a sampling loop, an
    unconditional forward with other keyframes and a forward at another B"""
    m, sd = model(*XL[:3], 263)
    eng = m.engine_for(DEV, max_batch=64, precision=X3, nframes=196)
    x, xo, mask, cond, scale = inputs(2, 263, 196, 1, True, True)
    x64, xo64, mask64, cond64, scale64 = inputs(64, 263, 196, 2, True, True)

    def call():
        return eng.forward(x.to(DEV), 500, cond_emb=cond.to(DEV), cfg=True, text_scale=scale.to(DEV), obs_x0=xo.to(DEV),
                           obs_mask=mask.to(DEV)).clone()

    first = call()
    eng.forward(x64.to(DEV) * 3, 30, cond_emb=cond64.to(DEV), cfg=True, text_scale=scale64.to(DEV), obs_x0=xo64.to(DEV),
                obs_mask=mask64.to(DEV))
    d = C.create_gaussian_diffusion(timestep_respacing="ddim5")
    w = C.ClassifierFreeSampleModel(m)
    table = {str(i): cond64[i].to(DEV) for i in range(4)}
    m.encode_text = lambda texts: torch.stack([table[s] for s in texts])
    y = {"text": [str(i) for i in range(4)], "text_scale": scale64[:4].to(DEV), "mask": torch.ones(4, 1, 1, 196, dtype=torch.bool, device=DEV)}
    d.ddim_sample_loop(w, (4, 263, 1, 196), model_kwargs={"y": y, "obs_x0": xo64[:4].to(DEV), "obs_mask": mask64[:4].to(DEV)},
                       skip_timesteps=2, init_image=xo64[:4].to(DEV))
    eng.forward(x64[:5].to(DEV), 10, obs_x0=xo64[5:10].to(DEV), obs_mask=mask64[5:10].to(DEV))
    eng.forward(x64[:7].to(DEV), 700, cond_emb=cond64[:7].to(DEV), obs_x0=xo64[:7].to(DEV), obs_mask=mask64[:7].to(DEV))
    again = call()
    print(f"[bf16x3 forward after other calls] max |diff| = {(again - first).abs().max().item():.3e}")
    assert torch.equal(again, first)
