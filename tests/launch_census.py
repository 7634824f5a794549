"""Launch census of the benchmarked updates: every call of a public wrapper of speecht5_b200.kernels during one update,
reduced to a signature -- what the kernel sees apart from data and dropout seeds.

A signature holds the wrapper name and every argument:
  - scalars as they are, except seeds and dropout offsets (only whether the seed is device-resident is kept);
  - for each tensor: dtype, shape, strides, base address mod 16, and the storage it lives in (a per-call group id and
    the byte offset from the first operand seen in that storage), so `ln_bwd` with dx on top of ds or a shared
    reduce-add output stays visible;
  - for an st5_attn_args struct: its fields, each pointer described like a tensor argument (attn_args is wrapped too,
    to learn which tensor each pointer came from).
Calls that differ only in data pointers and seeds are one signature.

The wrappers are found by introspecting the module, so a kernel added later is recorded without a change here. The
workloads are built the way bench.py builds them, from its own shape constants. CUDA only."""
import ctypes
import gc
import inspect

import torch

# size helpers and struct builders: they launch nothing
EXCLUDED = ("attn_args", "dtype_id")
SEED_FLAG = 1 << 63


def wrapper_names(K):
    """Public launch wrappers of `K` (speecht5_b200.kernels)."""
    return sorted(n for n, f in vars(K).items()
                  if inspect.isfunction(f) and f.__module__ == K.__name__ and not n.startswith("_")
                  and n not in EXCLUDED and not n.endswith("_ws_floats"))


class _Call:
    """Describes the arguments of one call; tensors sharing a storage get one group id."""

    def __init__(self):
        self.groups = {}

    def tensor(self, t):
        st = t.untyped_storage().data_ptr()
        if st not in self.groups:
            self.groups[st] = (len(self.groups), t.data_ptr())
        gid, p0 = self.groups[st]
        return ("T", str(t.dtype).replace("torch.", ""), tuple(t.shape), tuple(t.stride()), t.data_ptr() % 16, gid,
                t.data_ptr() - p0)

    def value(self, v, origin=None):
        if isinstance(v, torch.Tensor):
            return self.tensor(v)
        if isinstance(v, (list, tuple)):
            return tuple(self.value(x) for x in v)
        if isinstance(v, dict):
            return tuple((k, self.value(x)) for k, x in sorted(v.items()))
        if isinstance(v, ctypes.Structure):
            return self.struct(v, origin or {})
        if v is None or isinstance(v, (bool, int, float, str)):
            return v
        return ("obj", type(v).__name__)

    def struct(self, s, origin):
        out = []
        seedflag = bool(getattr(s, "offset", 0) & SEED_FLAG)
        for name, ctype in s._fields_:
            v = getattr(s, name)
            if name == "seed":
                v = "device" if seedflag else "host"
            elif name == "offset":
                v = None
            elif ctype is ctypes.c_void_p:
                v = self.tensor(origin[name]) if name in origin else (None if not v else ("ptr",))
            elif isinstance(v, ctypes.Structure):
                v = self.struct(v, {})
            elif isinstance(v, float):
                v = float(ctypes.c_float(v).value)
            out.append((name, v))
        return ("S", type(s).__name__, tuple(out))


def signature(fn, name, args, kwargs, origins):
    ba = inspect.signature(fn).bind(*args, **kwargs)
    ba.apply_defaults()
    c = _Call()
    off = ba.arguments.get("offset")
    items = []
    for k, v in ba.arguments.items():
        if k == "seed":
            v = "device" if (isinstance(off, int) and off & SEED_FLAG) else "host"
        elif k == "offset":
            continue
        else:
            v = c.value(v, origins.get(id(v)))
        items.append((k, v))
    return (name, tuple(items))


class Recorder:
    """Context manager: wraps every public wrapper of speecht5_b200.kernels (pass-through) and collects signatures.
    `calls` counts launches through the wrappers, `sigs` maps each distinct signature to its number of calls."""

    def __init__(self):
        self.calls = 0
        self.sigs = {}
        self._saved = {}
        self._origins = {}

    def __enter__(self):
        from speecht5_b200 import kernels as K
        self._K = K
        for n in wrapper_names(K):
            self._saved[n] = getattr(K, n)
            setattr(K, n, self._wrap(n, self._saved[n]))
        self._saved["attn_args"] = K.attn_args
        K.attn_args = self._attn_args
        return self

    def __exit__(self, *exc):
        for n, f in self._saved.items():
            setattr(self._K, n, f)
        self._origins.clear()
        return False

    def _attn_args(self, **kw):
        a = self._saved["attn_args"](**kw)
        a._st5_src = {k: v for k, v in kw.items() if isinstance(v, torch.Tensor)}  # which tensor each pointer came from
        return a

    def _wrap(self, name, fn):
        def call(*args, **kwargs):
            origins = {id(a): a._st5_src for a in list(args) + list(kwargs.values()) if hasattr(a, "_st5_src")}
            sig = signature(fn, name, args, kwargs, origins)
            self.sigs[sig] = self.sigs.get(sig, 0) + 1
            self.calls += 1
            return fn(*args, **kwargs)
        call.__wrapped__ = fn
        return call

    def by_wrapper(self):
        out = {}
        for sig in self.sigs:
            out.setdefault(sig[0], []).append(sig)
        return out


def args_of(sig):
    """The described arguments of a signature as a dict (struct fields as a dict as well)."""
    d = dict(sig[1])
    for k, v in d.items():
        if isinstance(v, tuple) and v[:1] == ("S",):
            d[k] = dict(v[2])
    return d


# ------------------------------------------------------------------------------------------------ workloads
def _fresh(dtype, seed=1):
    from speecht5_b200.ops import RT
    RT.dtype = dtype
    RT.clear_static()
    RT.invalidate_shadows()
    RT.manual_seed(seed)
    RT.stage_callback = None
    RT.layer_keep = RT.layer_keep_host = None
    RT.wgrad_stream = None
    RT._side_keep.clear()


def record_tts(dev, dtype=torch.bfloat16, use_cuda_graph=True):
    """One update of bench.py's tts workload (its WORKLOAD shapes, model options and trainer options), recorded."""
    import bench
    from speecht5_b200.criterions import SpeechT5Criterion
    from speecht5_b200.data import synthetic_tts_batch
    from speecht5_b200.models import make_args
    from speecht5_b200.tasks import SpeechT5Task
    from speecht5_b200.trainer import B200Trainer, _to_device
    W = bench.WORKLOAD
    _fresh(dtype)
    torch.manual_seed(1337)
    margs = make_args(W["arch"], encoder_layerdrop=0.0, decoder_layerdrop=0.0, bert_init=True,
                      decoder_layers=W["decoder_layers"], share_input_output_embed=True, max_text_positions=600,
                      max_speech_positions=1876)
    task = SpeechT5Task(margs)
    model = task.build_model(margs).to(dev).train()
    trainer = B200Trainer(model, SpeechT5Criterion(task, use_guided_attn_loss=True), task, lr=1e-4, betas=(0.9, 0.98),
                          eps=1e-8, clip_norm=25.0, use_cuda_graph=use_cuda_graph)
    batch = _to_device(synthetic_tts_batch(W["batch_per_gpu"], W["text_len"], W["mel_frames"], seed=0), dev)
    with Recorder() as rec:
        trainer.train_step([batch])
        torch.cuda.synchronize()
    del trainer, model, task, batch
    _fresh(torch.bfloat16)
    gc.collect()
    torch.cuda.empty_cache()
    return rec


WORKLOADS = {"tts": record_tts}
