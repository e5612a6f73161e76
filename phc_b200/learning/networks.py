"""Actor / critic / discriminator networks of the AMP agent on flat fp32 buckets, computed by libphc_b200.so.

Mirrors the module tree the reference builds with rl_games' builders so that checkpoints interchange:
  AMPBuilder.Network (phc/learning/amp_network_builder.py:13-249) on top of A2CBuilder.Network
  (phc/learning/network_builder.py:130-330): `actor_mlp` / `critic_mlp` / `_disc_mlp` are nn.Sequential(Linear, act, ...)
  so the Linear layers sit at even indices (`actor_mlp.0`, `actor_mlp.2`), heads are `mu`, `value`, `_disc_logits`,
  `sigma` is a fixed (requires_grad False) log-std initialised to -2.9 (im.yaml:22-27).
State-dict keys are `a2c_network.<name>.{weight,bias}` exactly as the reference's `model.state_dict()`.

Storage: every trainable tensor lives in ONE flat parameter bucket (and one flat gradient bucket of the same layout)
so that the per-minibatch all-reduce, the global-norm clip and Adam are single passes.  Weight rows are padded to a
multiple of 4 floats (934 -> 936) because the GEMM loads 16-byte chunks; pad columns stay exactly zero.
"""
from __future__ import annotations

import math
import os
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

import torch

from .. import _lib
from ..ops import _ptr, _stream


def round4(x: int) -> int:
    return (x + 3) & ~3


@dataclass
class LinearSpec:
    name: str          # e.g. "actor_mlp.0", "mu"
    in_dim: int
    out_dim: int
    w_off: int = 0     # offsets into the flat bucket (floats)
    b_off: int = 0
    img_fwd: int = 0   # offsets of the layer's weight images in AMPNetwork.images (floats)
    img_dx: int = 0

    @property
    def in_pad(self) -> int:
        return round4(self.in_dim)


class MLPStack:
    """One MLP = hidden Linear+act layers followed by a linear head."""

    def __init__(self, prefix: str, head: str, in_dim: int, units: Sequence[int], out_dim: int, head_relu: bool = False,
                 activation: str = "relu"):
        self.layers: List[LinearSpec] = []
        d = in_dim
        for i, u in enumerate(units):
            self.layers.append(LinearSpec(f"{prefix}.{2 * i}", d, u))
            d = u
        self.layers.append(LinearSpec(head, d, out_dim))
        self.in_dim, self.out_dim = in_dim, out_dim
        self.head_relu = head_relu          # MCP composer: the last Linear is followed by the activation too (ending_act;
                                            # the name is historical: it is the stack's own activation, relu or silu)
        assert activation in ("relu", "silu")
        self.activation = activation        # hidden activation: nn.ReLU (im.yaml) or nn.SiLU (im_big / im_pnn_big / im_mcp_big)

    @property
    def hidden(self) -> List[LinearSpec]:
        return self.layers[:-1]

    @property
    def head(self) -> LinearSpec:
        return self.layers[-1]


class AMPNetwork:
    """Parameter container (flat buckets + named views).  Compute lives in MLPEngine."""

    def __init__(self, obs_dim: int, action_dim: int, amp_dim: int, units: Sequence[int] = (1024, 512),
                 disc_units: Sequence[int] = (1024, 512), activation: str = "relu", sigma_init: float = -2.9,
                 device="cuda:0", seed: int = 0, kind: str = "amp", num_prim: int = 4, training_prim: int = 0, ending_act: bool = True):
        """kind: 'amp' (AMPBuilder, actor_mlp + mu), 'amp_pnn' (AMPPNNBuilder: `num_prim` independent actor columns
        `pnn.actors.K`, column `training_prim` is the one evaluated / trained -- pnn.py:11-131, amp_network_pnn_builder.py:23-87)
        or 'amp_mcp' (AMPMCPBuilder: `composer` MLP whose `action_dim` = num_prim outputs keep the final ReLU --
        amp_network_mcp_builder.py:23-91; ending_act False strips that ReLU, :58-59)."""
        if activation not in ("relu", "silu"):
            raise NotImplementedError(f"activation {activation!r}: the shipped configs use relu and silu")
        self.activation = activation        # mlp.activation; the discriminator is relu in every shipped config
        assert kind in ("amp", "amp_pnn", "amp_mcp")
        self.device = torch.device(device)
        self.kind, self.num_prim, self.training_prim = kind, num_prim, training_prim
        self.obs_dim, self.action_dim, self.amp_dim = obs_dim, action_dim, amp_dim
        n_h = len(units)
        if kind == "amp_pnn":
            self.pnn_actors = [MLPStack(f"pnn.actors.{k}", f"pnn.actors.{k}.{2 * n_h}", obs_dim, units, action_dim, activation=activation)
                               for k in range(num_prim)]
            self.actor = self.pnn_actors[training_prim]
            actor_stacks = self.pnn_actors
        elif kind == "amp_mcp":
            st = MLPStack("composer", f"composer.{2 * n_h}", obs_dim, units, action_dim, head_relu=ending_act, activation=activation)
            self.actor, actor_stacks = st, [st]
        else:
            self.actor = MLPStack("actor_mlp", "mu", obs_dim, units, action_dim, activation=activation)
            actor_stacks = [self.actor]
        self.actor_stacks = actor_stacks
        self.critic = MLPStack("critic_mlp", "value", obs_dim, units, 1, activation=activation)
        self.disc = MLPStack("_disc_mlp", "_disc_logits", amp_dim, disc_units, 1)
        off = 0
        for st in (*actor_stacks, self.critic, self.disc):
            for l in st.layers:
                l.w_off = off
                off += l.out_dim * l.in_pad
                l.b_off = off
                off += round4(l.out_dim)
        self.num_floats = off
        self.params = torch.zeros(off, dtype=torch.float32, device=self.device)
        self.grads = torch.zeros(off, dtype=torch.float32, device=self.device)
        # 3xTF32 operand split of the weights for the pre-split GEMM back end (refreshed after every optimiser step)
        self.params_hi = torch.zeros(off, dtype=torch.float32, device=self.device)
        self.params_lo = torch.zeros(off, dtype=torch.float32, device=self.device)
        self.sigma = torch.full((action_dim,), float(sigma_init), dtype=torch.float32, device=self.device)
        # weight images (include/phc_b200.h, PhcGemmDesc.B_img) of every layer in both of the GEMM's weight-side forms: the
        # forward (B = W: N = out, K = in) and dX (B = W read MN-major: N = in, K = out)
        lib, off, descs = _lib.load(), 0, []
        for l in self.all_layers():
            l.img_fwd = off
            off += lib.phc_gemm_image_floats(l.out_dim, l.in_dim)
            l.img_dx = off
            off += lib.phc_gemm_image_floats(l.in_dim, l.out_dim)
        self.images = torch.zeros(off, dtype=torch.float32, device=self.device)
        for l in self.all_layers():
            W = self.weight(l)
            descs += [_lib.PhcGemmImageDesc(W.data_ptr(), W.stride(0), 1, l.out_dim, l.in_dim, self.images[l.img_fwd:].data_ptr()),
                      _lib.PhcGemmImageDesc(W.data_ptr(), W.stride(0), 0, l.in_dim, l.out_dim, self.images[l.img_dx:].data_ptr())]
        self._image_descs = (_lib.PhcGemmImageDesc * len(descs))(*descs)
        self._images_of = None            # params._version the images were made from
        self._init_default(seed)
        self.refresh_images()

    # ---- views -------------------------------------------------------------------------------------------
    def weight(self, l: LinearSpec, grad: bool = False, part: Optional[str] = None) -> torch.Tensor:
        buf = self.grads if grad else {None: self.params, "hi": self.params_hi, "lo": self.params_lo}[part]
        return buf[l.w_off:l.w_off + l.out_dim * l.in_pad].view(l.out_dim, l.in_pad)

    def image(self, l: LinearSpec, kmajor: bool) -> torch.Tensor:
        """The weight image of layer l as the forward's B (kmajor) or dX's B; remade first if params was written through torch
        since the last refresh_images()."""
        if self._images_of != self.params._version:
            self.refresh_images()
        return self.images[l.img_fwd if kmajor else l.img_dx:]

    def refresh_images(self) -> None:
        """Remake every weight image from params, in one launch.  A stale image gives silently wrong products, so every writer
        of params calls this: construction, load_state_dict, the optimiser step (where the engine reads images) and the
        multi-GPU broadcast.  Writes through
        torch are also caught by image(), from the bucket's version counter; writes through raw pointers are not."""
        _lib.check(_lib.load().phc_gemm_make_images(self._image_descs, len(self._image_descs), _stream()), "phc_gemm_make_images")
        self._images_of = self.params._version

    def refresh_split(self) -> None:
        """hi = rna_tf32(W), lo = rna_tf32(W - hi) over the whole bucket (one streaming pass, 5.5 M floats)."""
        n = self.num_floats
        _lib.check(_lib.load().phc_split_tf32(self.params.data_ptr(), n, 1, n, self.params_hi.data_ptr(), self.params_lo.data_ptr(),
                                              n, _stream()), "phc_split_tf32")

    def bias(self, l: LinearSpec, grad: bool = False) -> torch.Tensor:
        buf = self.grads if grad else self.params
        return buf[l.b_off:l.b_off + l.out_dim]

    def all_layers(self) -> List[LinearSpec]:
        return [l for st in self.actor_stacks for l in st.layers] + self.critic.layers + self.disc.layers

    def load_actor_column(self, checkpoint_model: Dict[str, torch.Tensor], idx: int = 0) -> None:
        """PNN.load_actor (pnn.py:53-60): copy a single-policy checkpoint (actor_mlp.* / mu.*) into primitive column idx."""
        col = self.pnn_actors[idx]
        names = [f"a2c_network.actor_mlp.{2 * i}" for i in range(len(col.hidden))] + ["a2c_network.mu"]
        for l, n in zip(col.layers, names):
            self.set_layer(l, checkpoint_model[n + ".weight"], checkpoint_model[n + ".bias"])

    # ---- init: PyTorch's default nn.Linear init (`initializer: default`), disc biases zero, logits U(-1, 1) --------
    def _init_default(self, seed: int) -> None:
        g = torch.Generator().manual_seed(seed)
        for st in (*self.actor_stacks, self.critic, self.disc):
            for l in st.layers:
                bound = 1.0 / math.sqrt(l.in_dim)
                w = (torch.rand(l.out_dim, l.in_dim, generator=g) * 2 - 1) * bound     # kaiming_uniform(a=sqrt(5))
                b = (torch.rand(l.out_dim, generator=g) * 2 - 1) * bound
                if st is self.disc:
                    b.zero_()                                                          # amp_network_builder.py:240-244
                    if l is st.head:
                        w = torch.rand(l.out_dim, l.in_dim, generator=g) * 2 - 1       # DISC_LOGIT_INIT_SCALE = 1 (:246)
                self.set_layer(l, w, b)

    def set_layer(self, l: LinearSpec, w: torch.Tensor, b: torch.Tensor) -> None:
        W = self.weight(l)
        W.zero_()
        W[:, :l.in_dim] = w.to(self.device, torch.float32)
        self.bias(l).copy_(b.to(self.device, torch.float32))

    # ---- checkpoint interchange with the reference ----------------------------------------------------------------
    def state_dict(self, prefix: str = "a2c_network.") -> Dict[str, torch.Tensor]:
        sd = {prefix + "sigma": self.sigma.clone()}
        for l in self.all_layers():
            sd[f"{prefix}{l.name}.weight"] = self.weight(l)[:, :l.in_dim].clone()
            sd[f"{prefix}{l.name}.bias"] = self.bias(l).clone()
        return sd

    def load_state_dict(self, sd: Dict[str, torch.Tensor], prefix: str = "a2c_network.") -> None:
        for l in self.all_layers():
            self.set_layer(l, sd[f"{prefix}{l.name}.weight"], sd[f"{prefix}{l.name}.bias"])
        if prefix + "sigma" in sd:
            self.sigma.copy_(sd[prefix + "sigma"].to(self.device))
        self.refresh_images()

    def get_disc_logit_weights(self) -> torch.Tensor:
        return self.weight(self.disc.head)[:, :self.disc.head.in_dim].flatten()

    def get_disc_weights(self) -> List[torch.Tensor]:
        return [self.weight(l)[:, :l.in_dim].flatten() for l in self.disc.layers]


def _splits(tiles: int, K: int) -> int:
    """split-K factor for the weight-gradient GEMMs (M, N are layer widths, K is the batch)."""
    want = max(1, (4 * 132 + tiles - 1) // tiles)      # ~4 tiles per SM
    return int(max(1, min(want, K // 512, 64)))


def group_splits(K: int) -> int:
    """split-K factor of a weight-gradient problem inside a grouped launch (K = batch rows): about 32 k-blocks of 32 rows per
    split, so a dW tile costs about as much as a dX / forward tile of the same launch (the static tile striding then balances)."""
    env = os.environ.get("PHC_DW_KB_PER_SPLIT")
    per = int(env) if env else 32
    return int(max(1, min(64, round(((K + 31) // 32) / per))))


class MLPEngine:
    """Forward / backward of the MLP stacks through phc_gemm, with per-batch-size activation workspaces."""

    _mode_set = None       # the library's precision switch is process wide: remember what was set last

    def __init__(self, net: AMPNetwork, backend: Optional[str] = None, precision: str = "fp32"):
        """precision: "fp32" = 3xTF32, fp32-equivalent (default, the parity path); "tf32" = one tensor-core pass per product
        (PHC_GEMM_TF32_SINGLE_PASS, ~1e-3 relative, tc5s back end only): the reduced-precision mode of BASELINE.json configs[3]."""
        assert precision in ("fp32", "tf32")
        self.precision = precision
        self.net = net
        self.lib = _lib.load()
        self.dev = net.device
        self._ws: Dict[Tuple[str, int], Dict[str, torch.Tensor]] = {}
        # "tc5s" (default): grouped wgmma 3xTF32 with the operand split in shared memory (gemm_wgmma.cu);
        # "tc5": the same kernel with operands pre-split in global memory (phc_gemm_tc5); "mma": warp-level mma.sync 3xTF32
        # (gemm.cu).  The latter two stay as cross-check implementations (PHC_GEMM=tc5 | mma)
        self.backend = backend or os.environ.get("PHC_GEMM", "tc5s")
        assert self.backend in ("mma", "tc5", "tc5s")
        if precision == "tf32" and self.backend != "tc5s":
            raise ValueError("precision='tf32' (single tensor-core pass) exists on the tc5s back end only")
        self._companions: Dict[Tuple[int, Tuple[int, ...], Tuple[int, ...]], Tuple[torch.Tensor, torch.Tensor]] = {}
        self.gemm_flops = 0.0          # algorithmic fp32 FLOPs (2 M N K) of every grouped launch so far (bench.py reads it)
        # the weight images feed the grouped 3xTF32 launches; the single-pass kernel stages B itself and never reads them
        self.uses_images = self.backend == "tc5s" and precision == "fp32"
        # activation images, one buffer per (tensor, ld, rows, K, k-major): of the weight-gradient operands and the first layer's
        # input (remade by every launch that reads them), and of hidden outputs (written by the epilogue of the GEMM producing them)
        self._act_images: Dict[Tuple[int, int, int, int, bool], torch.Tensor] = {}
        if self.backend == "tc5":
            net.refresh_split()

    # -- operand split bookkeeping for the pre-split path --------------------------------------------------------------
    def companions(self, t: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        """(hi, lo) buffers that shadow activation tensor `t` (same shape / strides)."""
        key = (t.data_ptr(), tuple(t.shape), tuple(t.stride()))
        c = self._companions.get(key)
        if c is None:
            base_rows, ld = t.shape[0], t.stride(0)
            c = (torch.zeros(base_rows, ld, device=self.dev)[:, :t.shape[1]], torch.zeros(base_rows, ld, device=self.dev)[:, :t.shape[1]])
            self._companions[key] = c
        return c

    def split(self, t: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        hi, lo = self.companions(t)
        rc = self.lib.phc_split_tf32(t.data_ptr(), t.stride(0), t.shape[0], t.shape[1], hi.data_ptr(), lo.data_ptr(), hi.stride(0), _stream())
        if rc:
            _lib.check(rc, "phc_split_tf32")
        return hi, lo

    def _weight_parts(self, W: torch.Tensor) -> Optional[Tuple[torch.Tensor, torch.Tensor]]:
        """If W is a view into the parameter bucket, the matching views of the pre-split buckets."""
        p = self.net.params
        off = (W.data_ptr() - p.data_ptr()) // 4
        if 0 <= off < p.numel() and W.data_ptr() >= p.data_ptr():
            n = W.shape[0] * W.stride(0)
            return (self.net.params_hi[off:off + n].view(W.shape[0], W.stride(0))[:, :W.shape[1]],
                    self.net.params_lo[off:off + n].view(W.shape[0], W.stride(0))[:, :W.shape[1]])
        return None

    # -- raw GEMM ------------------------------------------------------------------------------------------------
    def gemm(self, A, a_k, B, b_k, C, M, N, K, alpha=1.0, bias=None, relu=False, mask=None, accumulate=False, k_splits=1,
             a_split=None, b_split=None, split_out: bool = False, act: Optional[int] = None):
        """act: PHC_ACT_* code (default: RELU if relu else NONE); mask: the epilogue's `aux` matrix (see include/phc_b200.h).
        a_split / b_split: already up-to-date (hi, lo) companions of the operand (skips the split pass);
        split_out: also produce C's companions in the epilogue (tc5 only)."""
        lda = A.stride(0)
        ldb = B.stride(0)
        if act is None:
            act = _lib.PHC_ACT_RELU if relu else _lib.PHC_ACT_NONE
        if self.backend == "tc5":
            Ah, Al = a_split or self._weight_parts(A) or self.split(A)
            Bh, Bl = b_split or self._weight_parts(B) or self.split(B)
            Ch = Cl = None
            if split_out and not accumulate:
                Ch, Cl = self.companions(C)
            rc = self.lib.phc_gemm_tc5(Ah.data_ptr(), Al.data_ptr(), lda, 1 if a_k else 0, Bh.data_ptr(), Bl.data_ptr(), ldb,
                                       1 if b_k else 0, C.data_ptr(), _ptr(Ch), _ptr(Cl), C.stride(0), M, N, K, alpha, _ptr(bias),
                                       act, _ptr(mask), mask.stride(0) if mask is not None else 0,
                                       1 if accumulate else 0, k_splits, _stream())
            if rc:
                _lib.check(rc, "phc_gemm_tc5")
            return (Ch, Cl) if Ch is not None else None
        if self.backend == "tc5s":
            self._set_mode()
        fn = self.lib.phc_gemm_tc5s if self.backend == "tc5s" else self.lib.phc_gemm
        rc = fn(A.data_ptr(), lda, 1 if a_k else 0, B.data_ptr(), ldb, 1 if b_k else 0, C.data_ptr(),
                               C.stride(0), M, N, K, alpha, _ptr(bias), act, _ptr(mask),
                               mask.stride(0) if mask is not None else 0, 1 if accumulate else 0, k_splits, _stream())
        if rc:
            _lib.check(rc, "phc_gemm")

    # -- grouped launches (tc5s only): one persistent kernel over the tiles of up to PHC_GEMM_GROUP_MAX independent GEMMs ------
    def image(self, l: LinearSpec, kmajor: bool) -> Optional[torch.Tensor]:
        """layer l's weight image for the forward (kmajor) or dX form, or None where the launches do not read images"""
        return self.net.image(l, kmajor) if self.uses_images else None

    def gdesc(self, A, a_k, B, b_k, C, M, N, K, alpha=1.0, bias=None, act=0, aux=None, accumulate=False, k_splits=1, B_img=None,
              A_img=None, C_img=None):
        """B_img: B's weight image for this N and K (AMPNetwork.image), or None to stage B from the fp32 operand.  A_img: A's image
        (act_image(A, M, K)); C_img: the buffer the epilogue writes C's image into (act_image(C, M, N))."""
        return _lib.PhcGemmDesc(A.data_ptr(), A.stride(0), 1 if a_k else 0, B.data_ptr(), B.stride(0), 1 if b_k else 0, C.data_ptr(),
                                C.stride(0), M, N, K, alpha, _ptr(bias), act, _ptr(aux), aux.stride(0) if aux is not None else 0,
                                1 if accumulate else 0, k_splits, None, _ptr(B_img), _ptr(A_img), _ptr(C_img))

    def act_image(self, t: torch.Tensor, rows: int, K: int, kmajor: bool = True) -> torch.Tensor:
        """The image buffer of activation t (rows x K, k-major or mn-major), allocated on first use."""
        key = (t.data_ptr(), t.stride(0), rows, K, kmajor)
        img = self._act_images.get(key)
        if img is None:
            img = torch.empty(self.lib.phc_gemm_image_floats(rows, K), dtype=torch.float32, device=self.dev)
            self._act_images[key] = img
        return img

    def _reads_image(self, st: MLPStack, li: int) -> bool:
        """Whether the forward and the dX of layer li take A from its image (on the pair loop).  Hidden layers do: the GEMM that
        produces their A writes the image from its epilogue, except the first layer's input, which run_group images once for
        the launch.  The heads stay on the image loop: their dY comes from the loss kernels, and with N = 69 or 1 their A would
        cost an image pass as large as the product."""
        return self.uses_images and li < len(st.hidden)

    def fwd_desc(self, st: MLPStack, li: int, x: torch.Tensor, ws: Dict[str, torch.Tensor]):
        """Layer li of the forward pass of stack st on batch x / workspace ws (the same epilogues as forward())."""
        net, l, B = self.net, st.layers[li], x.shape[0]
        inp = x if li == 0 else ws["h"][li - 1]
        silu = st.activation == "silu"
        if li < len(st.hidden):
            out = ws["h"][li]
            act = _lib.PHC_ACT_SILU if silu else (_lib.PHC_ACT_RELU_BITS if "hbits" in ws else _lib.PHC_ACT_RELU)
            aux = ws["z"][li] if silu else (ws["hbits"][li] if "hbits" in ws else None)
        else:
            out = ws["out"]
            act = _lib.PHC_ACT_NONE if not st.head_relu else (_lib.PHC_ACT_SILU if silu else (_lib.PHC_ACT_RELU_BITS if "obits" in ws else _lib.PHC_ACT_RELU))
            aux = None if not st.head_relu else (ws["z_out"] if silu else ws.get("obits"))
        d = self.gdesc(inp, True, net.weight(l), True, out, B, l.out_dim, l.in_dim, bias=net.bias(l), act=act, aux=aux,
                       B_img=self.image(l, True), C_img=self.act_image(out, B, l.out_dim) if self._reads_image(st, li + 1) else None)
        if self._reads_image(st, li) and li == 0:
            d.image_of = (("A_img", inp, B, True),)             # made by run_group; actor and critic share the input's image
        elif self._reads_image(st, li):
            d.A_img = self.act_image(inp, B, l.in_dim).data_ptr()
        return d

    def bwd_descs(self, st: MLPStack, li: int, x: torch.Tensor, ws: Dict[str, torch.Tensor], dx: Optional[torch.Tensor] = None):
        """(dW, dX) problems of layer li: dW[out, in] += dY^T X (split-K, reduce-add into the gradient bucket) and
        dX = (dY W) * act'(layer below).  dX is None for the first layer unless `dx` is given."""
        net, l, B = self.net, st.layers[li], x.shape[0]
        dY = ws["dout"] if li == len(st.layers) - 1 else ws["dh"][li]
        inp = x if li == 0 else ws["h"][li - 1]
        dw = self.dw_desc(dY, inp, net.weight(l, grad=True), l.out_dim, l.in_dim, B)
        dxd = None
        img = self.image(l, False)
        if li > 0:
            # A = dY: the image that the dX of the layer above wrote (hidden layers); C = dh[li - 1]: its image for the dX below
            dh = ws["dh"][li - 1]
            imgs = dict(B_img=img, A_img=self.act_image(dY, B, l.out_dim) if self._reads_image(st, li) else None,
                        C_img=self.act_image(dh, B, l.in_dim) if li > 1 and self._reads_image(st, li - 1) else None)
            if st.activation == "silu":
                dxd = self.gdesc(dY, True, net.weight(l), False, dh, B, l.in_dim, l.out_dim, act=_lib.PHC_ACT_SILU_BWD, aux=ws["z"][li - 1], **imgs)
            elif "hbits" in ws:
                dxd = self.gdesc(dY, True, net.weight(l), False, dh, B, l.in_dim, l.out_dim, act=_lib.PHC_ACT_MASK_BITS, aux=ws["hbits"][li - 1], **imgs)
            else:
                dxd = self.gdesc(dY, True, net.weight(l), False, dh, B, l.in_dim, l.out_dim, aux=ws["h"][li - 1], **imgs)
        elif dx is not None:
            dxd = self.gdesc(dY, True, net.weight(l), False, dx, B, l.in_dim, l.out_dim, B_img=img)
        return dw, dxd

    def dw_desc(self, dY: torch.Tensor, X: torch.Tensor, dW: torch.Tensor, M: int, N: int, K: int):
        """The weight-gradient problem dW[M, N] += dY[:K, :M]^T X[:K, :N], split-K, added into the gradient bucket.  Where the
        launches read images, it asks for images of dY (A) and X (B): run_group makes them right before the launch."""
        d = self.gdesc(dY, False, X, False, dW, M, N, K, accumulate=True, k_splits=group_splits(K))
        # An image costs one pass over its operand (fp32 read, hi / lo written) and saves the split and store of that operand in
        # every tile across the other dimension.  Timed on the bench minibatch (H100 SXM, 700 W), the layer-0 dW (8 x 8 and 8 x 16
        # tiles of 128 x 128) is faster with images and the 4 x 8-tile hidden layer and the heads are slower: images are asked for
        # from tiles_m * tiles_n >= 4 (tiles_m + tiles_n) on.
        tm, tn = -(-M // 128), -(-N // 128)
        if self.uses_images and tm * tn >= 4 * (tm + tn):
            d.image_of = (("A_img", dY, M, False), ("B_img", X, N, False))
        return d

    def make_images(self, descs):
        """Points the image fields of the descriptors that ask for activation images made before the launch (image_of: the
        weight gradient's operands, the first layer's input) at their buffers and returns the image jobs (PhcGemmImageDesc array,
        count), one per distinct (tensor, rows, K, order): actor and critic share the input's image."""
        jobs = {}
        for d in descs:
            srcs = getattr(d, "image_of", ())
            if not d.B_img and all(f == "A_img" for f, *_ in srcs):   # B staged from fp32 (its image cleared): so is A
                d.A_img = None
                continue
            for field, t, rows, kmajor in srcs:
                img = self.act_image(t, rows, d.K, kmajor)
                key = (t.data_ptr(), t.stride(0), rows, d.K, kmajor)
                if key not in jobs:
                    jobs[key] = _lib.PhcGemmImageDesc(t.data_ptr(), t.stride(0), 1 if kmajor else 0, rows, d.K, img.data_ptr())
                setattr(d, field, img.data_ptr())
        return (_lib.PhcGemmImageDesc * len(jobs))(*jobs.values()), len(jobs)

    def _set_mode(self) -> None:
        mode = _lib.PHC_GEMM_TF32_SINGLE_PASS if self.precision == "tf32" else _lib.PHC_GEMM_FP32_3XTF32
        if MLPEngine._mode_set != mode:
            _lib.check(self.lib.phc_gemm_set_precision(mode), "phc_gemm_set_precision")
            MLPEngine._mode_set = mode

    def run_group(self, descs) -> None:
        self._set_mode()
        descs = [d for d in descs if d is not None]
        for i in range(0, len(descs), _lib.PHC_GEMM_GROUP_MAX):
            part = descs[i:i + _lib.PHC_GEMM_GROUP_MAX]
            jobs, n = self.make_images(part)
            if n:
                _lib.check(self.lib.phc_gemm_make_images(jobs, n, _stream()), "phc_gemm_make_images")
            self.gemm_flops += sum(2.0 * d.M * d.N * d.K for d in part)
            arr = (_lib.PhcGemmDesc * len(part))(*part)
            rc = self.lib.phc_gemm_group(arr, len(part), _stream())
            if rc:
                _lib.check(rc, "phc_gemm_group")

    def forward_group(self, items) -> None:
        """items: [(stack, x, ws)]: the stacks advance layer by layer together, one grouped launch per layer index."""
        depth = max(len(st.layers) for st, _, _ in items)
        for li in range(depth):
            self.run_group([self.fwd_desc(st, li, x, ws) for st, x, ws in items if li < len(st.layers)])

    def colsum(self, X, M, N, out, alpha=1.0, accumulate=True):
        rc = self.lib.phc_colsum(X.data_ptr(), X.stride(0), M, N, alpha, out.data_ptr(), 1 if accumulate else 0, _stream())
        if rc:
            _lib.check(rc, "phc_colsum")

    def colsum_group(self, items) -> None:
        """items: [(X, M, N, out)] -- out[n] += sum_m X[m, n] for all of them in one launch (phc_colsum_group)."""
        for i in range(0, len(items), _lib.PHC_GEMM_GROUP_MAX):
            part = items[i:i + _lib.PHC_GEMM_GROUP_MAX]
            arr = (_lib.PhcColsumDesc * len(part))(*[_lib.PhcColsumDesc(X.data_ptr(), X.stride(0), M, N, 1.0, out.data_ptr()) for X, M, N, out in part])
            rc = self.lib.phc_colsum_group(arr, len(part), _stream())
            if rc:
                _lib.check(rc, "phc_colsum_group")

    # -- workspaces ----------------------------------------------------------------------------------------------
    def workspace(self, tag: str, st: MLPStack, batch: int) -> Dict[str, torch.Tensor]:
        key = (tag, batch)
        ws = self._ws.get(key)
        if ws is None:
            z = lambda *s: torch.zeros(*s, dtype=torch.float32, device=self.dev)
            ws = {"h": [z(batch, round4(l.out_dim)) for l in st.hidden], "out": z(batch, round4(st.out_dim)),
                  "dh": [z(batch, round4(l.out_dim)) for l in st.hidden], "dout": z(batch, round4(st.out_dim))}
            if st.activation == "relu" and self.backend == "tc5s":     # ReLU backward from 1 bit per element (PHC_ACT_RELU_BITS)
                ws["hbits"] = [torch.zeros(batch, (l.out_dim + 31) // 32, dtype=torch.int32, device=self.dev) for l in st.hidden]
                if st.head_relu:
                    ws["obits"] = torch.zeros(batch, (st.out_dim + 31) // 32, dtype=torch.int32, device=self.dev)
            if st.activation == "silu":          # SiLU backward needs the pre-activations
                ws["z"] = [z(batch, round4(l.out_dim)) for l in st.hidden]
                if st.head_relu:
                    ws["z_out"] = z(batch, round4(st.out_dim))
            self._ws[key] = ws
        return ws

    # -- forward: x is [B, in_pad] (zero padded) -------------------------------------------------------------------
    def forward(self, st: MLPStack, x: torch.Tensor, ws: Dict[str, torch.Tensor]) -> torch.Tensor:
        if self.backend == "tc5s":                          # the grouped launch, so that B comes from the weight images
            self.forward_group([(st, x, ws)])
            return ws["out"]
        net, B = self.net, x.shape[0]
        tc5 = self.backend == "tc5"
        cur, cur_split = x, (self.split(x) if tc5 else None)
        ws["x_split"] = cur_split
        ws["h_split"] = []
        silu = st.activation == "silu"
        bits = ws.get("hbits")
        for i, (l, h) in enumerate(zip(st.hidden, ws["h"])):
            cur_split = self.gemm(cur, True, net.weight(l), True, h, B, l.out_dim, l.in_dim, bias=net.bias(l),
                                  act=_lib.PHC_ACT_SILU if silu else (_lib.PHC_ACT_RELU_BITS if bits else _lib.PHC_ACT_RELU),
                                  mask=ws["z"][i] if silu else (bits[i] if bits else None), a_split=cur_split, split_out=True)
            ws["h_split"].append(cur_split)
            cur = h
        l = st.head
        head_act = _lib.PHC_ACT_NONE if not st.head_relu else (_lib.PHC_ACT_SILU if silu else _lib.PHC_ACT_RELU)
        self.gemm(cur, True, net.weight(l), True, ws["out"], B, l.out_dim, l.in_dim, bias=net.bias(l), a_split=cur_split,
                  act=head_act, mask=ws["z_out"] if (st.head_relu and silu) else None)
        return ws["out"]

    # -- backward: ws["dout"] holds d(loss)/d(out) [B, round4(out)]; accumulates into net.grads --------------------
    def backward(self, st: MLPStack, x: torch.Tensor, ws: Dict[str, torch.Tensor], dx: Optional[torch.Tensor] = None) -> None:
        net, B = self.net, x.shape[0]
        tc5 = self.backend == "tc5"
        acts = [x] + ws["h"]
        act_splits = ([ws.get("x_split")] + list(ws.get("h_split", []))) if tc5 else [None] * len(acts)
        dcur = ws["dout"]
        if st.head_relu:                                    # MCP composer: activation after the head (ending_act)
            silu = st.activation == "silu"
            aux = ws["z_out"] if silu else ws["out"]
            rc = self.lib.phc_act_backward(dcur.data_ptr(), dcur.stride(0), aux.data_ptr(), aux.stride(0), B, st.out_dim,
                                           _lib.PHC_ACT_SILU if silu else _lib.PHC_ACT_RELU, _stream())
            if rc:
                _lib.check(rc, "phc_act_backward")
        dsplit = self.split(dcur) if tc5 else None          # the loss kernels wrote dout: split it once for both GEMMs
        for li in range(len(st.layers) - 1, -1, -1):
            l = st.layers[li]
            a_in = acts[li]
            tiles = ((l.out_dim + 127) // 128) * ((l.in_dim + 127) // 128)
            # dW[out, in] += dY^T X
            self.gemm(dcur, False, a_in, False, net.weight(l, grad=True), l.out_dim, l.in_dim, B, accumulate=True,
                      k_splits=_splits(tiles, B), a_split=dsplit, b_split=act_splits[li])
            self.colsum(dcur, B, l.out_dim, net.bias(l, grad=True))
            if li > 0:
                # dX = dY W, times the derivative of the activation of the layer below (ReLU: its output > 0; SiLU: at z)
                if st.activation == "silu":
                    nsplit = self.gemm(dcur, True, net.weight(l), False, ws["dh"][li - 1], B, l.in_dim, l.out_dim,
                                       mask=ws["z"][li - 1], act=_lib.PHC_ACT_SILU_BWD, a_split=dsplit, split_out=True)
                elif ws.get("hbits"):
                    nsplit = self.gemm(dcur, True, net.weight(l), False, ws["dh"][li - 1], B, l.in_dim, l.out_dim,
                                       mask=ws["hbits"][li - 1], act=_lib.PHC_ACT_MASK_BITS)
                else:
                    nsplit = self.gemm(dcur, True, net.weight(l), False, ws["dh"][li - 1], B, l.in_dim, l.out_dim, mask=acts[li],
                                       a_split=dsplit, split_out=True)
                dcur, dsplit = ws["dh"][li - 1], nsplit
            elif dx is not None:
                self.gemm(dcur, True, net.weight(l), False, dx, B, l.in_dim, l.out_dim, a_split=dsplit)
