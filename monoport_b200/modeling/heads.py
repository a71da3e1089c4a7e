"""Skip-MLP head: parameter container with the reference's state-dict layout
(`filters.{l}.weight [Cout,Cin,1]`, `filters.{l}.bias`; heads/SurfaceClassifier.py:7-37) plus the binding to the
packed-weight handle of the fused kernel.  In eval mode MonoPortNet.query never calls `forward`: the MLP runs
inside the fused sm_90a kernel."""
import ctypes

import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import _lib


class SurfaceClassifier(nn.Module):
    def __init__(self, filter_channels, num_views=1, no_residual=True, last_op=None):
        super().__init__()
        if num_views != 1:
            raise NotImplementedError("multi-view mean pooling (SurfaceClassifier.py:60-66) is not on the recon path")
        self.filter_channels = list(filter_channels)
        self.num_views = num_views
        self.no_residual = no_residual
        self.last_op = last_op
        self.filters = nn.ModuleList()
        c0 = filter_channels[0]
        for l in range(len(filter_channels) - 1):
            cin = filter_channels[l] + (c0 if (l > 0 and not no_residual) else 0)
            self.filters.append(nn.Conv1d(cin, filter_channels[l + 1], 1))
        self._handle = None
        self._handle_key = None
        # largest |feature| a frame may have for the tensor-core program to be used (None = the library default, by output
        # count and last op: 12 with Sigmoid, 8 for the colour head's Tanh, 4 for a 3-output head with no last op, 3 for a
        # 1-output head with Tanh or none; float("inf") disables the guard); larger frames take the exact fp32 kernel
        self.tc_feature_limit = None

    # ---- autograd / stand-alone module forward (training scaffolding, not the hot path) ----------------
    def forward(self, feature):
        y = feature
        for l, f in enumerate(self.filters):
            y = f(y if (l == 0 or self.no_residual) else torch.cat([y, feature], 1))
            if l != len(self.filters) - 1:
                y = F.leaky_relu(y)
        return self.last_op(y) if self.last_op else y

    # ---- fused-kernel weight handle -----------------------------------------------------------------------
    def last_op_code(self):
        if self.last_op is None:
            return _lib.LAST_NONE
        if isinstance(self.last_op, nn.Sigmoid):
            return _lib.LAST_SIGMOID
        if isinstance(self.last_op, nn.Tanh):
            return _lib.LAST_TANH
        raise NotImplementedError("last_op %r" % (self.last_op,))

    def _key(self):
        def ver(p):
            try:
                return p._version
            except RuntimeError:          # inference-mode tensors carry no version counter
                return None
        return tuple((p.data_ptr(), ver(p), p.device) for p in self.parameters())

    def handle(self):
        """mp_mlp_t* for the current parameters (rebuilt when they change: load_state_dict, .to(), optimizer step)."""
        key = self._key()
        if self._handle is not None and key == self._handle_key and not any(k[1] is None for k in key):
            return self._with_limit(self._handle)
        self.release()
        lib = _lib.load()
        dev = self.filters[0].weight.device
        if dev.type != "cuda":
            raise RuntimeError("monoport_b200: the head must live on a CUDA device (no CPU path); got %s" % dev)
        ws = [f.weight.detach().to(torch.float32).reshape(f.weight.shape[0], -1).contiguous() for f in self.filters]
        bs = [f.bias.detach().to(torch.float32).contiguous() for f in self.filters]
        n = len(ws)
        chans = (ctypes.c_int * (n + 1))(*self.filter_channels)
        wp = (ctypes.c_void_p * n)(*[w.data_ptr() for w in ws])
        bp = (ctypes.c_void_p * n)(*[b.data_ptr() for b in bs])
        h = ctypes.c_void_p()
        with torch.cuda.device(dev):
            torch.cuda.current_stream().synchronize()
            _lib.check(lib.mp_mlp_create(n, chans, wp, bp, 0 if self.no_residual else 1, self.last_op_code(), 1,
                                         ctypes.byref(h)), "mp_mlp_create")
        self._handle, self._handle_key = h, key
        self._applied_limit = None
        return self._with_limit(h)

    def _with_limit(self, h):
        if self.tc_feature_limit is not None and self.tc_feature_limit != self._applied_limit:
            _lib.check(_lib.load().mp_mlp_set_tc_feature_limit(h, ctypes.c_float(float(self.tc_feature_limit))),
                       "mp_mlp_set_tc_feature_limit")
            self._applied_limit = self.tc_feature_limit
        return h

    # native handles never travel with a copy: deepcopy / pickle / copy.copy drop them (rebuilt lazily on first use);
    # sharing the pointer would end in two mp_mlp_destroy calls on it
    def __getstate__(self):
        d = dict(self.__dict__)
        d["_handle"], d["_handle_key"] = None, None
        d.pop("_applied_limit", None)
        return d

    def tc_supported(self):
        return bool(_lib.load().mp_mlp_tc_supported(self.handle()))

    def release(self):
        if self._handle is not None:
            _lib.load().mp_mlp_destroy(self._handle)
            self._handle = None
            self._handle_key = None

    def __del__(self):
        try:
            self.release()
        except Exception:
            pass


def PIFuNetGMLP(*args, **kwargs):
    return SurfaceClassifier([257, 1024, 512, 256, 128, 1], 1, False, nn.Sigmoid())


def PIFuNetCMLP(*args, **kwargs):
    return SurfaceClassifier([513, 1024, 512, 256, 128, 3], 1, False, nn.Tanh())
