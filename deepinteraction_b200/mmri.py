"""MMRI encoder on libdi_b200: parameter holders with the reference's state_dict schema and the
kernel schedule of one forward pass.

Reference: projects/mmdet3d_plugin/models/necks/deepinteraction_encoder.py:8-85 and
models/utils/encoder_utils.py (ConvBNReLU :11-34, LocalContextAttentionBlock :84-135, BEVWarp
:137-199, MMRI_P2I :202-213, MMRI_I2P :216-320).

Differences from the reference schedule (results are unchanged, fp32):
  * feature maps live pixel-major (NHWC) between kernels; the NCHW inputs are consumed directly by
    the first 3x3 conv and the outputs are returned as NCHW-shaped channels-last views;
  * BatchNorm (eval) is folded into the 1x1 convs; each `cat + Conv+BN` pair is ONE 3-source GEMM;
  * the window logits/probabilities never leave the SM (fused similar/softmax/weighting);
  * the I2P single-head attention is folded (no per-key K/V projection, no (6,128,20P) gather tensor);
  * BEVWarp geometry (projection, depth scatter, depth completion, lifting) runs once per frame on
    the GPU and is shared by both layers; the reference recomputes it per layer with a CPU OpenCV
    round trip per camera;
  * no host synchronisation anywhere in the forward.
"""
import torch
import torch.nn as nn

from . import fold, geom, ops
from .graph import GraphCache

PC_RANGE = (-54.0, -54.0, -5.0, 54.0, 54.0, 3.0)     # hard-coded in the reference (encoder_utils.py:190)
POINT_CAP_MIN = 1 << 19      # staged point arrays: capacity = max(2^19, next power of two) rows per sample (graph.py)


def _pow2_cap(n, floor):
    """Capacity of a staged per-frame array: a power of two >= floor, so that ordinary frame-to-frame variation never
    crosses a capacity boundary (every boundary costs a graph re-capture)."""
    c = floor
    while c < n:
        c *= 2
    return c


# ------------------------------------------------------------------------------------------------
# parameter holders (names == reference state_dict keys; they never run torch math)
# ------------------------------------------------------------------------------------------------
class ConvBN(nn.Module):
    def __init__(self, cin, cout, k=1, norm=True, affine=True, dims=2):
        super().__init__()
        conv = nn.Conv2d if dims == 2 else nn.Conv1d
        self.conv = conv(cin, cout, k, padding=k // 2, bias=not norm)
        if norm:
            self.bn = (nn.BatchNorm2d if dims == 2 else nn.BatchNorm1d)(cout, affine=affine)


class LocalContextAttentionBlock(nn.Module):
    def __init__(self, cin, cout, kernel_size, last_affine=True):
        super().__init__()
        self.kernel_size = kernel_size
        self.query_project = nn.Sequential(ConvBN(cin, cout), ConvBN(cout, cout))
        self.key_project = nn.Sequential(ConvBN(cin, cout), ConvBN(cout, cout))
        self.value_project = ConvBN(cin, cout, affine=last_affine)
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.xavier_uniform_(m.weight)


class MMRI_I2P(nn.Module):
    def __init__(self, pts_channels, img_channels, dropout):
        super().__init__()
        self.pts_channels, self.img_channels, self.dropout = pts_channels, img_channels, dropout
        self.learnedAlign = nn.MultiheadAttention(pts_channels, 1, dropout=dropout, kdim=img_channels,
                                                  vdim=img_channels, batch_first=True)


class BEVWarp(nn.Module):
    pass


class MMRI_P2I(nn.Module):
    def __init__(self, cin, cout, kernel_size):
        super().__init__()
        self.Warp = BEVWarp()
        self.Local = LocalContextAttentionBlock(cin, cout, kernel_size)


class DeepInteractionEncoderLayer(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.I2P_block = MMRI_I2P(c, c, 0.1)
        self.P_IML = LocalContextAttentionBlock(c, c, 9)
        self.P_out_proj = ConvBN(2 * c, c)
        self.P_integration = ConvBN(2 * c, c)
        self.P2I_block = MMRI_P2I(c, c, 9)
        self.I_IML = LocalContextAttentionBlock(c, c, 9)
        self.I_out_proj = ConvBN(2 * c, c)
        self.I_integration = ConvBN(2 * c, c)


# ------------------------------------------------------------------------------------------------
# weight packs
# ------------------------------------------------------------------------------------------------
def _pack_lcab(blk, device):
    wq1, bq1 = fold.pointwise(blk.query_project[0])
    wq2, bq2 = fold.pointwise(blk.query_project[1])
    wk1, bk1 = fold.pointwise(blk.key_project[0])
    wk2, bk2 = fold.pointwise(blk.key_project[1])
    wv, bv = fold.pointwise(blk.value_project)
    d = lambda t: fold.dev(t, device)
    Wt = lambda t: fold.Weight(t, device)
    C = wq2.shape[0]
    return dict(C=C, ks=blk.kernel_size,
                w_self=Wt(torch.cat([wq1, wk1, wv], 0)), b_self=d(torch.cat([bq1, bk1, bv], 0)),
                w_q1=Wt(wq1), b_q1=d(bq1), w_kv1=Wt(torch.cat([wk1, wv], 0)), b_kv1=d(torch.cat([bk1, bv], 0)),
                w_q2=Wt(wq2), b_q2=d(bq2), w_k2=Wt(wk2), b_k2=d(bk2),
                w_2=Wt(torch.cat([wq2, wk2], 0)), b_2=d(torch.cat([bq2, bk2], 0)))


def lcab_forward(pk, target, source, N, H, W):
    """target/source: [N*H*W, C] pixel-major row views (same tensor object => self attention).
    Where the tensor-core path applies, the projections that feed the window kernel write its operand format
    directly (bf16 hi/mid words), so the window kernel has no conversion work."""
    C = pk['C']
    if ops.can_window_tc(N * H * W, C, pk['ks']):
        # one C-ABI call: the fused projections (lcab_proj.cu), then the planar window kernel; the rows go in through
        # their leading dimension, a view whose rows are not 16-byte aligned as a contiguous copy
        aligned = lambda x: x.stride(1) == 1 and x.stride(0) >= C and x.stride(0) % 4 == 0 and x.data_ptr() % 16 == 0
        t = target if aligned(target) else target.contiguous()
        s = t if source is target else source if aligned(source) else source.contiguous()
        return ops.lcab_forward_tc(t, s, pk['w_self'], pk['b_self'], pk['w_2'], pk['b_2'], N, H, W)
    pre = ops.can_presplit(N * H * W, C, pk['ks'])
    if target is source:
        if pre:
            t = ops.linear_split([source], pk['w_self'], pk['b_self'], ops.ACT_RELU, 2 * C, 2)    # q1 | k1 | v(split)
        else:
            t = ops.linear([source], pk['w_self'], pk['b_self'], ops.ACT_RELU)        # [M, 3C] = q1 | k1 | v
        q1, k1, v = t[:, :C], t[:, C:2 * C], t[:, 2 * C:]
    else:
        q1 = ops.linear([target], pk['w_q1'], pk['b_q1'], ops.ACT_RELU)
        if pre:
            t = ops.linear_split([source], pk['w_kv1'], pk['b_kv1'], ops.ACT_RELU, C, 2)          # k1 | v(split)
        else:
            t = ops.linear([source], pk['w_kv1'], pk['b_kv1'], ops.ACT_RELU)          # [M, 2C] = k1 | v
        k1, v = t[:, :C], t[:, C:]
    if pre:
        q = ops.linear_split([q1], pk['w_q2'], pk['b_q2'], ops.ACT_RELU, 0, 1)
        k = ops.linear_split([k1], pk['w_k2'], pk['b_k2'], ops.ACT_RELU, 0, 1)
        return ops.lcab_window_pre(q, k, v, N, H, W, C)
    q = ops.linear([q1], pk['w_q2'], pk['b_q2'], ops.ACT_RELU)
    k = ops.linear([k1], pk['w_k2'], pk['b_k2'], ops.ACT_RELU)
    return ops.lcab_window(q, k, v, N, H, W, C, pk['ks'])


class Geometry:
    """Per-frame geometry shared by both encoder layers (and by the decoder's projections)."""

    def __init__(self, img_metas, pts_metas, feat_hw, bev_hw, device, want_debug=False, side_stream=None,
                 cams=None, counts=None):
        """The depth maps / completion / lifting chain is latency-bound (one CTA per camera) and independent of
        the feature maps, so it is issued on `side_stream` and overlaps the shared convs and the BEV branch;
        consumers call wait() before the first BEV sampling.  cams = (proj, i2l) device tensors when the caller
        already uploaded the camera rows (graph replay), else they are derived from img_metas here.  counts: device
        int32 [1 + B] (live pillar count, live point count per sample) when the point arrays are capacity buffers."""
        self.in_hw = geom.input_hw(img_metas)
        self.proj, self.i2l = cams if cams is not None else geom.camera_rows(img_metas, device)   # (B,V,12), (B*V,12)
        B, V = self.proj.shape[:2]
        h, w = feat_hw
        main = torch.cuda.current_stream()
        side = side_stream if side_stream is not None else main
        pts_list = []
        for b in range(B):
            pts = pts_metas['pts'][b]
            if pts.device != self.proj.device or pts.dtype != torch.float32:
                pts = pts.to(device=device, dtype=torch.float32)
            pts_list.append(pts)
        if side is not main:
            side.wait_stream(main)
        with torch.cuda.stream(side), ops.module('BEVWarp_geometry (once per frame, side stream)',
                                                 12 * sum(int(p.shape[0]) for p in pts_list) + 3 * 4 * B * V * h * w):
            keys = torch.zeros(B * V, h, w, device=device, dtype=torch.int64)
            for b in range(B):
                ops.depth_scatter(pts_list[b], self.proj[b], keys[b * V:(b + 1) * V], self.in_hw,
                                  None if counts is None else counts[1 + b:2 + b])
            if want_debug:
                self.dense, self.sparse = ops.depth_complete(keys, want_sparse=True)
            else:
                self.dense = ops.depth_complete(keys)
            self.grid = ops.lift_grid(self.dense, self.i2l, self.in_hw, bev_hw, PC_RANGE)
            self.ready = torch.cuda.Event()
            self.ready.record(side)
        if side is not main and not torch.cuda.is_current_stream_capturing():
            # The buffers were allocated under the side stream but are read by kernels of the consumer stream: tell
            # the caching allocator, or a later frame's geometry could reuse a block while bev_sample of this frame is
            # still queued (eager path with several frames in flight).  Captured graphs own a private pool instead.
            for t in (keys, self.dense, self.grid, getattr(self, 'sparse', None)):
                if t is not None:
                    t.record_stream(main)
        self._side, self._main = side, main
        self.V = V

    def wait(self):
        if self._side is not self._main:
            torch.cuda.current_stream().wait_event(self.ready)


class DeepInteractionEncoder(nn.Module):
    """Drop-in for the reference ``DeepInteractionEncoder`` (NECKS): same constructor, same state_dict,
    same forward signature and return structure; inference (eval) only."""

    def __init__(self, num_layers=2, in_channels_img=64, in_channels_pts=128 * 3, hidden_channel=128,
                 bn_momentum=0.1, bias='auto'):
        super().__init__()
        use_bias = True if bias == 'auto' else bool(bias)
        self.shared_conv_pts = nn.Conv2d(in_channels_pts, hidden_channel, 3, padding=1, bias=use_bias)
        self.shared_conv_img = nn.Conv2d(in_channels_img, hidden_channel, 3, padding=1, bias=use_bias)
        self.num_layers = num_layers
        self.hidden_channel = hidden_channel
        self.fusion_blocks = nn.ModuleList(DeepInteractionEncoderLayer(hidden_channel) for _ in range(num_layers))
        self.bn_momentum = bn_momentum
        for m in self.modules():
            if isinstance(m, (nn.BatchNorm2d, nn.BatchNorm1d)):
                m.momentum = bn_momentum
        self._pack = None
        self._pack_key = None
        self.last_geometry = None
        self._side_streams = {}              # one geometry side stream per consumer stream (frames in flight)
        self._graphs = GraphCache()

    # -- packing -----------------------------------------------------------------------------------
    def _state_key(self):
        return tuple((p.data_ptr(), p._version) for p in list(self.parameters()) + list(self.buffers()))

    def pack(self, force=False):
        key = self._state_key()
        if self._pack is not None and key == self._pack_key and not force:
            return self._pack
        device = self.shared_conv_pts.weight.device
        if device.type != 'cuda':
            raise RuntimeError('DeepInteractionEncoder (libdi_b200) runs on CUDA only; move the module to a GPU')
        d = lambda t: fold.dev(t, device)
        Wt = lambda t: fold.Weight(t, device)
        pk = dict()
        for name in ('shared_conv_pts', 'shared_conv_img'):
            W, b = fold.conv_bn(getattr(self, name))
            pk[name] = (Wt(fold.pack_conv3x3(W)), d(b))
        layers = []
        for blk in self.fusion_blocks:
            M1, c1, M2, c2 = fold.i2p_fold(blk.I2P_block.learnedAlign)
            wp, bp = fold.fuse_pair(blk.P_out_proj, blk.P_integration)
            wi, bi = fold.fuse_pair(blk.I_out_proj, blk.I_integration)
            layers.append(dict(i2p=(Wt(M1), d(c1), Wt(M2), d(c2)), p_iml=_pack_lcab(blk.P_IML, device),
                               p2i=_pack_lcab(blk.P2I_block.Local, device), i_iml=_pack_lcab(blk.I_IML, device),
                               p_fuse=(Wt(wp), d(bp)), i_fuse=(Wt(wi), d(bi))))
        pk['layers'] = layers
        self._pack, self._pack_key = pk, key
        self._graphs.clear()                 # captured graphs hold pointers into the previous pack
        return pk

    # -- forward -----------------------------------------------------------------------------------
    def i2p(self, lp, pts_nhwc, img_nhwc, pts_metas, g, n_dev=None, dropout=None):
        """n_dev: device int32 [1] with the live pillar count when the pillar arrays are capacity buffers.  dropout = (p, seed):
        training-mode attention dropout (train.py only)."""
        B, Y, X, C = pts_nhwc.shape
        coors = pts_metas['pillar_coors']
        out = torch.zeros_like(pts_nhwc)
        if coors.shape[0] == 0:
            return out
        M1, c1, M2, c2 = lp['i2p']
        rows = ops.gather_rows(pts_nhwc, coors, n_dev)
        qk = ops.linear([rows], M1, c1)
        s, cnt = ops.i2p_attend(qk, pts_metas['pillars'], pts_metas['pillars_num_points'], coors, g.proj, img_nhwc,
                                g.V, g.in_hw, n_dev, dropout)
        o = ops.linear([s], M2, c2)
        return ops.scatter_rows(o, cnt, coors, out, n_dev)

    @staticmethod
    def _canon_pts_metas(pts_metas, device):
        """pts_metas without 'pillars' (or pillars=None): the pillars are generated on the GPU from pts_metas['pts']
        inside the schedule (ops.pillarize: the reference's 'pillar' voxelisation, detectors/deepinteraction.py:132-139)."""
        pm = dict(pts_metas)
        if pm.get('pillars') is None:
            pm['pillars'] = pm['pillar_coors'] = pm['pillars_num_points'] = None
            return pm
        pm['pillars'] = pm['pillars'].to(device=device, dtype=torch.float32).contiguous()
        pm['pillar_coors'] = pm['pillar_coors'].to(device=device, dtype=torch.int32).contiguous()
        pm['pillars_num_points'] = pm['pillars_num_points'].to(device=device, dtype=torch.int32).contiguous()
        return pm

    def forward_nhwc(self, img_feats, pts_feats, img_metas, pts_metas, debug=None):
        """-> img [B*V,h,w,C], pts_conv [B,Y,X,C], pts [B,Y,X,C]  (pixel-major, fp32).
        The kernel schedule is replayed from a CUDA graph once an input signature repeats (graph.py)."""
        if self.training:
            raise NotImplementedError('libdi_b200 DeepInteractionEncoder is forward/eval only (call .eval())')
        self.pack()
        dev_ = img_feats.device
        pm = self._canon_pts_metas(pts_metas, dev_)
        pts_list = [p.to(device=dev_, dtype=torch.float32) for p in pm['pts']]
        if debug is not None:
            return self._schedule(img_feats, pts_feats, img_metas, pm, pts_list, None, debug)
        proj_h, i2l_h = geom.camera_rows_host(img_metas)
        inputs = [img_feats.contiguous(), pts_feats.contiguous()]
        # per-frame arrays (row counts change every frame): staged at bucketed capacities, live counts via `consts`
        auto = pm['pillars'] is None                # generate the pillars on the GPU inside the schedule
        staged = ([] if auto else [pm['pillars'], pm['pillar_coors'], pm['pillars_num_points']]) + pts_list
        # pillars: at most one per BEV cell (the physical maximum) -> a capacity that never changes for a given map size
        B_, _, Y_, X_ = pts_feats.shape
        caps = ([] if auto else [_pow2_cap(pm['pillars'].shape[0], B_ * Y_ * X_)] * 3) + \
            [_pow2_cap(p.shape[0], POINT_CAP_MIN) for p in pts_list]
        counts_h = torch.tensor([0 if auto else pm['pillars'].shape[0]] + [p.shape[0] for p in pts_list], dtype=torch.int32)
        sig = (tuple(tuple(t.shape) for t in inputs), tuple(tuple(t.shape[1:]) for t in staged), auto,
               geom.input_hw(img_metas), id(self._pack))
        k0 = 0 if auto else 3

        def fn(ins, consts, st):
            pmx = dict(pillars=None, pillar_coors=None, pillars_num_points=None) if auto else \
                dict(pillars=st[0], pillar_coors=st[1], pillars_num_points=st[2])
            return self._schedule(ins[0], ins[1], img_metas, pmx, st[k0:], (consts[0], consts[1]), None, counts=consts[2])
        return self._graphs.run(sig, inputs, [proj_h, i2l_h, counts_h], fn, staged=staged, caps=caps)

    def _schedule(self, img_feats, pts_feats, img_metas, pm, pts_list, cams, debug, counts=None):
        pk = self._pack
        dev_ = img_feats.device
        C = self.hidden_channel
        BV, _, h, w = img_feats.shape
        B, _, Y, X = pts_feats.shape
        V = BV // B
        cur_id = torch.cuda.current_stream().cuda_stream
        if cur_id not in self._side_streams:
            self._side_streams[cur_id] = torch.cuda.Stream(device=dev_)
        pm = dict(pm)
        pm['pts'] = pts_list
        n_pil_dev = None if counts is None else counts[0:1]
        if pm['pillars'] is None:                   # (f1) pillars from the raw points, live count stays on the device
            pts_c = [p.contiguous() for p in pts_list]
            pm['pillars'], pm['pillar_coors'], pm['pillars_num_points'], n_pil_dev = ops.pillarize(
                pts_c, (Y, X), PC_RANGE, 20, None if counts is None else counts[1:1 + B])
        g = Geometry(img_metas, pm, (h, w), (Y, X), dev_, want_debug=debug is not None,
                     side_stream=self._side_streams[cur_id], cams=cams, counts=counts)
        self.last_geometry = g
        # module-boundary bytes of SURVEY.md 8(d) (fp32 maps: F_i image side, F_b BEV side) for bench.py's roofline table
        F_i, F_b = 4 * BV * h * w * C, 4 * B * Y * X * C
        n_pil, n_pts = pm['pillars'].shape[0], sum(int(p.shape[0]) for p in pts_list)
        with ops.module('shared_conv_img+pts', 4 * (img_feats.numel() + pts_feats.numel()) + F_i + F_b,
                        2 * 9 * C * (img_feats.numel() + pts_feats.numel())):
            img = ops.conv3x3(img_feats.contiguous(), *pk['shared_conv_img'], cout=C, x_nhwc=False)
            pts = ops.conv3x3(pts_feats.contiguous(), *pk['shared_conv_pts'], cout=C, x_nhwc=False)
        pts_conv = pts
        lcab_flops = lambda npx: 2 * npx * C * (5 * C + 2 * 81)
        for li, lp in enumerate(pk['layers']):
            img_r, pts_r = img.view(BV * h * w, C), pts.view(B * Y * X, C)
            with ops.module('MMRI_I2P', n_pil * (C * 4 + 20 * 12 + 16) + F_i + F_b):
                i2p = self.i2p(lp, pts, img, pm, g, n_pil_dev)
            with ops.module('LCAB_self_bev', 2 * F_b, lcab_flops(B * Y * X)):
                p2p = lcab_forward(lp['p_iml'], pts_r, pts_r, B, Y, X)
            with ops.module('P_out_proj+P_integration', 4 * F_b, 2 * B * Y * X * C * 3 * C):
                new_pts = ops.linear([i2p.view(-1, C), p2p, pts_r], *lp['p_fuse']).view(B, Y, X, C)
            if li == 0:
                g.wait()
            with ops.module('MMRI_P2I', 2 * F_i + F_b + 12 * n_pts, lcab_flops(BV * h * w)):
                warped = ops.bev_sample(pts, g.grid, V)
                p2i = lcab_forward(lp['p2i'], img_r, warped.view(-1, C), BV, h, w)
            with ops.module('LCAB_self_img', 2 * F_i, lcab_flops(BV * h * w)):
                i2i = lcab_forward(lp['i_iml'], img_r, img_r, BV, h, w)
            with ops.module('I_out_proj+I_integration', 4 * F_i, 2 * BV * h * w * C * 3 * C):
                new_img = ops.linear([p2i, i2i, img_r], *lp['i_fuse']).view(BV, h, w, C)
            if debug is not None:
                debug.append(dict(i2p=i2p, p2p=p2p.view(B, Y, X, C), warped=warped, p2i=p2i.view(BV, h, w, C),
                                  i2i=i2i.view(BV, h, w, C)))
            img, pts = new_img, new_pts
        return img, pts_conv, pts

    def forward(self, img_feats, pts_feats, img_metas, pts_metas):
        img, pts_conv, pts = self.forward_nhwc(img_feats, pts_feats, img_metas, pts_metas)
        # NCHW-shaped views of the pixel-major results (values identical to the reference's NCHW tensors)
        return img.permute(0, 3, 1, 2), [pts_conv.permute(0, 3, 1, 2), pts.permute(0, 3, 1, 2)]
