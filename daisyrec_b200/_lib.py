"""ctypes loader for libdaisyrec_b200.so -- the C ABI declared in include/daisyrec_b200.h.

The header is the one declaration of that ABI: the restype / argtypes of every drb_* entry point and the DRB_* constants
below are read from it, so a binding cannot drift from the prototype the compiler checks the definition against.
The product path has NO CPU fallback: if the shared object is missing (and cannot be built
because nvcc is absent) or a call fails, a RuntimeError is raised.
"""
import ctypes as C
import os
import re

from . import _build

_lib = None


class Hyper(C.Structure):
    """struct drb_hyper"""
    _fields_ = [("lr", C.c_float), ("reg_1", C.c_float), ("reg_2", C.c_float), ("opt", C.c_int32),
                ("beta1", C.c_float), ("beta2", C.c_float), ("eps", C.c_float), ("loss", C.c_int32)]


def _header():
    with open(_build.HEADER) as f:
        return f.read()


def defines(text):
    """name -> value of every `#define DRB_* <integer>` of the C text."""
    return {m[1]: int(m[2]) for m in re.finditer(r"^\s*#define\s+(DRB_\w+)\s+(-?\d+)\b", text, re.M)}


def prototypes(text):
    """name -> (return type, [parameter types]) of every drb_* prototype of the C text, the types as C spells them."""
    text = re.sub(r"/\*.*?\*/|//[^\n]*", " ", text, flags=re.S)          # comments
    text = re.sub(r"^\s*#[^\n]*", "", text, flags=re.M)                    # preprocessor lines
    out = {}
    for decl in re.split(r"[;{}]", text):
        m = re.fullmatch(r"\s*(.*?)\b(drb_\w+)\s*\((.*)\)\s*", decl, re.S)
        if m is None:
            continue
        ret, name, params = m.groups()
        params = [p.strip() for p in params.split(",")]
        params = [] if params == ["void"] else [re.sub(r"\w+$", "", p).strip() for p in params]     # drop the names
        out[name] = (ret.strip(), params)
    return out


_SCALARS = {"int": C.c_int, "int32_t": C.c_int32, "int64_t": C.c_int64, "uint32_t": C.c_uint32, "uint64_t": C.c_uint64,
            "uint8_t": C.c_uint8, "unsigned long long": C.c_ulonglong, "size_t": C.c_size_t, "float": C.c_float,
            "double": C.c_double}


def ctype(decl, fn, ret=False):
    """ctypes type of the C type ``decl`` in the signature of ``fn`` (its return type when ``ret``): the scalars by value,
    a returned `const char *` as c_char_p, `void **` as POINTER(c_void_p), `drb_hyper *` as POINTER(Hyper) and every other
    pointer as c_void_p.  ValueError for a type outside these."""
    stars = decl.count("*")
    base = " ".join(w for w in re.findall(r"\w+", decl) if w != "const")
    if stars == 0 and base in _SCALARS:
        return _SCALARS[base]
    if stars == 1 and base == "char" and ret:
        return C.c_char_p
    if stars == 2 and base == "void":
        return C.POINTER(C.c_void_p)
    if stars == 1 and base == "drb_hyper":
        return C.POINTER(Hyper)
    if stars and (base in _SCALARS or base in ("void", "char", "drb_hyper")):
        return C.c_void_p
    raise ValueError(f"{fn}: unknown C type '{decl}' in include/daisyrec_b200.h")


def signatures(text):
    """name -> (restype, argtypes) of every drb_* prototype of the C text."""
    return {name: (ctype(ret, name, ret=True), [ctype(p, name) for p in params])
            for name, (ret, params) in prototypes(text).items()}


_DEFINES = defines(_header())
DRB_OK = _DEFINES["DRB_OK"]
globals().update((k, v) for k, v in _DEFINES.items() if k.startswith("DRB_ERR_"))     # DRB_ERR_INVALID, DRB_ERR_CUDA, ...
OPT_KIND = {k.removeprefix("DRB_OPT_").lower(): v for k, v in _DEFINES.items() if k.startswith("DRB_OPT_")}
OPT_SGD, OPT_ADAM = OPT_KIND["sgd"], OPT_KIND["adam"]
LOSS_KIND = {k.removeprefix("DRB_LOSS_"): v for k, v in _DEFINES.items() if k.startswith("DRB_LOSS_")}
KPI_NAMES = tuple(k.removeprefix("DRB_KPI_").lower() for k in sorted(_DEFINES, key=_DEFINES.get)
                  if k.startswith("DRB_KPI_") and k != "DRB_KPI_COUNT")                 # DRB_KPI_* order


def so_path():
    # DRB_LIB_PATH: developer override used by scripts/tune_variants.sh to A/B kernel builds
    return os.environ.get("DRB_LIB_PATH") or _build.SO


def _cuda_device_count():
    """Devices the driver reports, without touching the runtime of this process (0 when there is no driver)."""
    try:
        cu = C.CDLL("libcuda.so.1")
        n = C.c_int(0)
        if cu.cuInit(0) != 0 or cu.cuDeviceGetCount(C.byref(n)) != 0:
            return 0
        return n.value
    except OSError:
        return 0


_CANARY = r"""
import ctypes, sys
l = ctypes.CDLL(sys.argv[1])
l.drb_mf_step_variant.argtypes = [ctypes.c_int32, ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p]
l.drb_mt19937_stream_variant.argtypes = [ctypes.c_int64]
a = l.drb_mf_step_variant(64, 0, None, None)                 # step-kernel selection, tables inside L2
b = l.drb_mf_step_variant(128, 1 << 20, None, None)          # ... streamed from HBM
c = l.drb_mt19937_stream_variant(3 << 20)                    # segmented MT19937 kernel's device check
print("CANARY OK", a, b, c, flush=True)
"""


def _canary(path):
    """The kernels that select themselves on the device (lean step instantiations, segmented MT19937) first run in a sacrificial
    child process: if that child crashes or does not come back, this process keeps the kernels that have a GPU record
    (DRB_NO_LEAN / DRB_MT_SEQUENTIAL are set before the library reads them).  Skipped without a device and under DRB_NO_CANARY."""
    if os.environ.get("DRB_NO_CANARY") or os.environ.get("DRB_NO_LEAN") or _cuda_device_count() == 0:
        return
    import subprocess
    import sys
    env = dict(os.environ)
    local = int(env.get("LOCAL_RANK", "0") or 0)
    vis = [v for v in env.get("CUDA_VISIBLE_DEVICES", "").split(",") if v.strip()]
    env["CUDA_VISIBLE_DEVICES"] = vis[local] if local < len(vis) else (vis[0] if vis else str(local))
    ok = False
    try:
        r = subprocess.run([sys.executable, "-c", _CANARY, path], env=env, capture_output=True, text=True, timeout=90)
        ok = r.returncode == 0 and "CANARY OK" in r.stdout
        why = (r.stdout + r.stderr)[-300:]
    except Exception as e:  # noqa: BLE001  (timeout, spawn failure)
        why = repr(e)
    if not ok:
        os.environ["DRB_NO_LEAN"] = "1"
        os.environ["DRB_MT_SEQUENTIAL"] = "1"
        sys.stderr.write(f"[daisyrec_b200] canary run of the self-selecting kernels failed ({why!r}): keeping the general step "
                         "kernel and the one-CTA MT19937 kernel in this process\n")


def lib():
    """Load (building first if the .so is absent and nvcc is present).  Fails loudly otherwise."""
    global _lib
    if _lib is not None:
        return _lib
    path = so_path()
    if not os.path.exists(path):
        try:
            _build.build()
        except Exception as e:  # noqa: BLE001
            raise RuntimeError(
                f"libdaisyrec_b200.so is missing ({path}) and could not be built: {e}. "
                "The GPU path has no CPU fallback; run `python -c 'import __graft_entry__ as g; g.build()'`.") from e
    L = C.CDLL(path)
    for name, (res, args) in signatures(_header()).items():
        fn = getattr(L, name)          # AttributeError here == header and library out of sync
        fn.restype, fn.argtypes = res, args
    _canary(path)
    _lib = L
    return L


class DrbError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"[libdaisyrec_b200 rc={code}] {msg}")
        self.code = code


# the errors the reference raises for these conditions (AbstractRecommender.py:122-123; numpy's choice() on an empty population;
# BatchNorm1d given one row in training mode)
NAN_LOSS_MESSAGE = "Loss=Nan or Infinity: current settings does not fit the recommender"
EMPTY_SET_MESSAGE = "'a' cannot be empty unless no samples are taken"
BATCHNORM_MESSAGE = "Expected more than 1 value per channel"


def check(rc):
    if rc == DRB_OK:
        return
    if rc == DRB_ERR_NAN_LOSS:
        raise ValueError(NAN_LOSS_MESSAGE)
    if rc == DRB_ERR_EMPTY_SET:
        raise ValueError(EMPTY_SET_MESSAGE)
    msg = (lib().drb_last_error() or b"").decode(errors="replace")
    if rc == DRB_ERR_NOT_PD:
        import numpy as np
        raise np.linalg.LinAlgError(msg)
    if rc == DRB_ERR_INVALID and msg.startswith(BATCHNORM_MESSAGE):
        raise ValueError(msg)
    raise DrbError(rc, msg)
