"""``DEVA`` - the network object the inference core drives (API of deva/model/network.py:18-190).

Holds the checkpoint tensors under the reference's own names (so ``state_dict()`` /
``load_state_dict()`` / ``load_weights()`` exchange checkpoints with the reference unchanged) and
runs inference through ``deva.model.native_engine.NativeEngine``.  Inference only: ``read_memory`` (the training-time twin of the
memory read) is provided forward-only on the same kernels; the ``need_aux`` heads and the ``forward(mode, ...)`` dispatch
used by DDP training are not part of the propagation hot path.
"""
from typing import Dict, Iterable, Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F

from deva.model.native_engine import NativeEngine
from deva.model.param_spec import checkpoint_spec, synthetic_state_dict


class _Node(nn.Module):
    """Anonymous container used to reproduce the dotted checkpoint names."""


class DEVA(nn.Module):
    def __init__(self, config: Dict, *, init_seed: int = 0):
        super().__init__()
        self.pix_feat_dim = config['pix_feat_dim']
        self.key_dim = config['key_dim']
        self.value_dim = config['value_dim']
        init = synthetic_state_dict(init_seed, self.key_dim, self.value_dim, self.pix_feat_dim)
        for name, (shape, role) in checkpoint_spec(self.key_dim, self.value_dim, self.pix_feat_dim).items():
            *path, leaf = name.split('.')
            node = self
            for part in path:
                if not hasattr(node, part):
                    node.add_module(part, _Node())
                node = getattr(node, part)
            if role in ('bn_mean', 'bn_var', 'bn_count'):
                node.register_buffer(leaf, init[name].clone())
            else:
                node.register_parameter(leaf, nn.Parameter(init[name].clone(), requires_grad=False))
        self._engine = None
        self._engine_key = None
        self.return_full_logits = True  # segment() also returns the up-sampled logits like the reference

    # ------------------------------------------------------------------ weights
    def load_weights(self, src_dict: Dict[str, torch.Tensor]) -> None:
        self.load_state_dict(src_dict)
        self._engine = None

    def _apply(self, fn, *args, **kwargs):  # .cuda() / .to() invalidate the folded tables
        self._engine = None
        return super()._apply(fn, *args, **kwargs)

    @property
    def engine(self) -> NativeEngine:
        probe = self.key_proj.key_proj.weight
        key = (probe.device, probe.data_ptr(), probe._version)
        if self._engine is None or self._engine_key != key:
            if probe.device.type != 'cuda':
                raise RuntimeError('deva_b200: the network runs on a CUDA device only (call .cuda()); '
                                   'there is no CPU fallback')
            with torch.no_grad():
                self._engine = NativeEngine({k: v.detach() for k, v in self.state_dict().items()})
            self._engine_key = key
        return self._engine

    # ------------------------------------------------------------------ reference API
    def aggregate(self, prob: torch.Tensor, dim: int) -> torch.Tensor:
        """Soft aggregation (network.py:33-40), always fp32."""
        prob = prob.float()
        full = torch.cat([torch.prod(1 - prob, dim=dim, keepdim=True), prob], dim).clamp(1e-7, 1 - 1e-7)
        return torch.log(full / (1 - full))

    @torch.no_grad()
    def encode_image(self, image: torch.Tensor) -> Tuple[Iterable[torch.Tensor], torch.Tensor]:
        return self.engine.encode_image(image.float())

    @torch.no_grad()
    def transform_key(self, feat: torch.Tensor, *, need_sk: bool = True, need_ek: bool = True):
        return self.engine.transform_key(feat, need_sk, need_ek)

    @torch.no_grad()
    def read_memory(self, query_key: torch.Tensor, query_selection: torch.Tensor, memory_key: torch.Tensor,
                    memory_shrinkage: torch.Tensor, memory_value: torch.Tensor) -> torch.Tensor:
        """The reference's training-time read (network.py:72-92 -> memory_utils.get_affinity / readout): full softmax
        over all memory tokens, no top-k.  query_key/selection [B,CK,H,W], memory_key [B,CK,T,H,W], memory_shrinkage
        [B,1,T,H,W], memory_value [B,K,CV,T,H,W] -> [B,K,CV,H,W].  Forward only (this engine carries no autograd), on the
        same kernels as MemoryManager.consolidation: similarity GEMM (split fp16x3) + row softmax + dense readout GEMM."""
        from deva import _native as nat
        b_sz, k = memory_value.shape[:2]
        cv, ck = memory_value.shape[2], query_key.shape[1]
        h, w = query_key.shape[-2:]
        q = h * w
        dev = query_key.device
        if cv % 128:
            raise RuntimeError(f'deva_b200: read_memory needs value_dim % 128 == 0 (got {cv})')
        out = torch.empty(b_sz, k * cv, q, dtype=torch.float32, device=dev)
        for b in range(b_sz):
            mk = memory_key[b].reshape(ck, -1).float().contiguous()
            n = mk.shape[1]
            ms = memory_shrinkage[b].reshape(-1).float().contiguous()
            k_hi = torch.zeros(n, 2 * ck, dtype=torch.float16, device=dev)
            k_lo = torch.zeros_like(k_hi)
            neg_s, raw_shr = torch.empty(n, device=dev), torch.empty(n, device=dev)
            raw_key = torch.empty(n, ck, device=dev)
            nat.pack_keys(mk, None, n, 1, ms, ck, n, k_hi, k_lo, neg_s, raw_key, None, raw_shr)
            ld = (n + 7) // 8 * 8
            vals = torch.zeros(k * cv, ld, dtype=torch.float16, device=dev)
            nat.append_values(memory_value[b].reshape(k * cv, n).float().contiguous(), n, vals, ld, k * cv, n)
            q_hi = torch.empty(q, 2 * ck, dtype=torch.float16, device=dev)
            q_lo = torch.empty_like(q_hi)
            bsq = torch.empty(q, device=dev)
            nat.pack_query(query_key[b].reshape(ck, q).float().contiguous(), query_selection[b].reshape(ck, q).float().contiguous(),
                           q, 1, ck, q, q_hi, q_lo, bsq)
            sim_ws = torch.empty(q, ld, dtype=torch.float32, device=dev)
            aff = torch.zeros(q, ld, dtype=torch.float16, device=dev)
            nat.sim_dense_softmax(k_hi, k_lo, neg_s, raw_shr, n, 0, q_hi, q_lo, bsq, q, ck, sim_ws, ld, aff, ld, None)
            for i in range(0, k, nat.MAX_GROUPS):
                rows = [j * cv for j in range(i, min(k, i + nat.MAX_GROUPS))]
                nat.readout(vals, ld, k * cv, rows, rows, cv, aff, ld, n, q, out[b], q)
        return out.view(b_sz, k, cv, h, w)

    @torch.no_grad()
    def encode_mask(self, image: torch.Tensor, ms_features: Iterable[torch.Tensor], h: torch.Tensor,
                    masks: torch.Tensor, *, is_deep_update: bool = True, chunk_size: int = -1):
        return self.engine.encode_mask(image.float(), ms_features, h, masks, deep_update=is_deep_update,
                                       chunk_size=chunk_size)

    @torch.no_grad()
    def segment(self, multi_scale_features, memory_readout, sensory, last_mask, *, selector=None,
                need_aux: bool = False, chunk_size: int = -1, update_sensory: bool = True,
                independent_objects: bool = False):
        """Returns (sensory, logits [1,K+1,H,W], prob [1,K+1,H,W]) like network.py:94-173 (inference branch)."""
        if need_aux:
            raise NotImplementedError('need_aux is a training-time head; this engine is inference only')
        sensory, logits = self.engine.decode(multi_scale_features, memory_readout, sensory, last_mask,
                                             update_sensory=update_sensory, chunk_size=chunk_size)
        if selector is None and not independent_objects:
            full_logits, prob = self.engine.probabilities(logits, want_logits=self.return_full_logits)
            return sensory, full_logits, prob
        logits = logits.float()
        prob = torch.sigmoid(logits)
        if selector is not None:
            prob = prob * selector
        if independent_objects:
            # per-object softmax against its own background (network.py:148-162); like the reference, the second
            # return value is the up-sampled aggregated LOGITS [K,2,H,W], not their softmax
            k, h, w = prob.shape[1:]
            each_logits = self.aggregate(prob.view(k, 1, h, w), dim=1)
            each_logits = F.interpolate(each_logits, scale_factor=4, mode='bilinear', align_corners=False)
            each = F.softmax(each_logits, dim=1)
            background = each[:, 0].min(dim=0)[0]
            prob = torch.cat([background.unsqueeze(0), each[:, 1]], dim=0).unsqueeze(0)
            return sensory, each_logits, prob
        logits = self.aggregate(prob, dim=1)
        logits = F.interpolate(logits, scale_factor=4, mode='bilinear', align_corners=False)
        return sensory, logits, F.softmax(logits, dim=1)
