"""Cached-feature input pipeline of the matcher (SURVEY.md section 8f row 3): extractor outputs exported once
(`gluefactory/scripts/export_megadepth.py:105-141`, fp16 on disk) are read back per batch, padded to a fixed
keypoint count, and fed to the matcher -- the reference's `models/cache_loader.py:13-41, 59-144`.

Drop-in surface: `CacheLoader(conf)(data) -> pred` with the reference's conf keys (`path`, `data_keys`, `scale`,
`padding_fn` ("pad_local_features"), `padding_length`, `numeric_type`, `collate`, `device`) and the same padding rules
(`pad_local_features`: keypoints padded with per-coordinate uniform noise inside the detected keypoints' bounding
box -- `random_c` --, descriptors with uniform noise between their min and max -- `random` --, scores / scales / oris /
depths with zeros; models/utils/misc.py:18-55).  Padding keypoints are real inputs of the matcher (they are NOT
masked, SURVEY Appendix C.9), so only the distributions matter, not the random stream.

What is different on an H100 feeding thousands of pairs per second:
  * storage back end `FeaturePack`: one flat little-endian file per export + a JSON index, memory-mapped; a record is the
    fp16 arrays of one image laid out back to back, so assembling a batch is B memcpys into a PINNED staging buffer
    (no per-key Python objects, no HDF5 chunk decoding).  `FeaturePack.write` builds it from any mapping
    name -> {key: array} (e.g. an h5py file where h5py exists; it is not installed in this image -- the HDF5 back end
    below is used automatically when it is).
  * the batch crosses PCIe as fp16 (what is on disk): the up-cast to `numeric_type`, the multiplication of keypoints by
    the view's `scales` and the padding all run on the device, on the copy stream's consumer side -- half the H2D bytes
    of the reference (which up-casts on the host, cache_loader.py:109-119).
"""
import json
import os
import string

import numpy as np
import torch

_PAD_MODES = {"keypoints": "random_c", "keypoint_scores": "zeros", "descriptors": "random", "scales": "zeros",
              "oris": "zeros", "depth_keypoints": "zeros", "valid_depth_keypoints": "zeros"}
_PAD_DIMS = {"keypoints": -2, "descriptors": -2}  # everything else pads its last dim


def pad_to_length(x, length, pad_dim=-2, mode="zeros", bounds=(None, None)):
    """models/utils/misc.py:18-55 (same modes; the noise is drawn on x's device)."""
    d = x.shape[pad_dim]
    assert d <= length, (d, length)
    if d == length:
        return x
    shape = list(x.shape)
    shape[pad_dim] = length - d
    low, high = bounds
    if mode == "zeros":
        xn = torch.zeros(*shape, device=x.device, dtype=x.dtype)
    elif mode == "ones":
        xn = torch.ones(*shape, device=x.device, dtype=x.dtype)
    elif mode == "random":
        low = low if low is not None else x.min()
        high = high if high is not None else x.max()
        xn = torch.empty(*shape, device=x.device, dtype=x.dtype).uniform_(float(low), float(high))
    elif mode == "random_c":
        cols = []
        for i in range(shape[-1]):
            lo = x[..., i].min() if d > 0 else low
            hi = x[..., i].max() if d > 0 else high
            cols.append(torch.empty(*shape[:-1], 1, device=x.device, dtype=x.dtype).uniform_(float(lo), float(hi)))
        xn = torch.cat(cols, -1)
    else:
        raise ValueError(mode)
    return torch.cat([x, xn], pad_dim)


def pad_local_features(pred, seq_l):
    """models/cache_loader.py:13-41."""
    for k, mode in _PAD_MODES.items():
        if k in pred:
            pred[k] = pad_to_length(pred[k], seq_l, _PAD_DIMS.get(k, -1), mode=mode)
    return pred


class FeaturePack:
    """Flat, memory-mapped feature store: `<path>` (raw bytes) + `<path>.json` (index).

    index = {"records": {name: {key: [offset_bytes, dtype, shape]}}}.  Arrays are stored in the dtype they were written
    with (exports use float16, export_megadepth.py:140 `as_half=True`), 64-byte aligned."""

    def __init__(self, path):
        self.path = path
        with open(path + ".json") as f:
            self.index = json.load(f)["records"]
        self.mm = np.memmap(path, dtype=np.uint8, mode="r")

    def __contains__(self, name):
        return name in self.index

    def keys(self, name):
        return list(self.index[name].keys())

    def read(self, name, key):
        off, dt, shape = self.index[name][key]
        n = int(np.prod(shape)) * np.dtype(dt).itemsize
        return np.frombuffer(self.mm, dtype=np.dtype(dt), count=int(np.prod(shape)), offset=off).reshape(shape) if n else \
            np.zeros(shape, dtype=np.dtype(dt))

    @staticmethod
    def write(path, records):
        """records: mapping name -> {key: array-like}.  Returns the number of bytes written."""
        index, off = {}, 0
        with open(path, "wb") as f:
            for name, rec in records.items():
                index[name] = {}
                for key, arr in rec.items():
                    a = np.ascontiguousarray(np.asarray(arr))
                    pad = (-off) % 64
                    f.write(b"\0" * pad)
                    off += pad
                    index[name][key] = [off, a.dtype.str, list(a.shape)]
                    f.write(a.tobytes())
                    off += a.nbytes
        with open(path + ".json", "w") as f:
            json.dump({"records": index}, f)
        return off


def _open_store(fpath):
    if os.path.exists(fpath + ".json"):
        return FeaturePack(fpath)
    try:
        import h5py  # the reference's format, when h5py is available
    except ImportError as e:
        raise FileNotFoundError(f"{fpath}: no FeaturePack index ({fpath}.json) and h5py is not installed") from e
    return _H5Store(h5py.File(fpath, "r"))


class _H5Store:
    def __init__(self, f):
        self.f = f

    def __contains__(self, name):
        return name in self.f

    def keys(self, name):
        return list(self.f[name].keys())

    def read(self, name, key):
        return self.f[name][key].__array__()


class CacheLoader(torch.nn.Module):
    default_conf = {
        "name": None,
        "path": "???",            # may be a format string like exports/{scene}.pack
        "data_keys": None,        # None: every key of the record
        "device": None,           # None: the device of the tensors in `data` (cpu if there are none)
        "trainable": False,
        "add_data_path": True,
        "data_root": None,        # plugin-only: root joined in front of `path` when add_data_path (settings.DATA_PATH)
        "collate": True,
        "scale": ["keypoints", "lines", "orig_lines"],
        "padding_fn": None,       # "pad_local_features"
        "padding_length": None,   # required for batching
        "numeric_type": "float32",
        "pin_memory": True,       # plugin-only: stage batches in pinned memory and copy asynchronously
    }
    required_data_keys = ["name"]

    def __init__(self, conf=None):
        super().__init__()
        self.conf = dict(self.default_conf, **(dict(conf) if conf else {}))
        fn = self.conf["padding_fn"]
        assert fn in (None, "pad_local_features"), f"unknown padding_fn {fn}"
        self.padding_fn = pad_local_features if fn else None
        self.numeric_dtype = {None: None, "float16": torch.float16, "float32": torch.float32,
                              "float64": torch.float64}[self.conf["numeric_type"]]
        self._stores = {}
        self._staging = {}

    def _store(self, fpath):
        if fpath not in self._stores:
            self._stores[fpath] = _open_store(fpath)
        return self._stores[fpath]

    def _device(self, data):
        if self.conf["device"]:
            return torch.device(self.conf["device"])
        devs = {v.device for v in data.values() if isinstance(v, torch.Tensor)}
        assert len(devs) <= 1
        return devs.pop() if devs else torch.device("cpu")

    def _stage(self, key, arrays, device):
        """Stack the per-image arrays of one key (ragged in their first dim) into one staging buffer in the STORED dtype,
        pinned when the target is a CUDA device, and start its (asynchronous) copy.  Returns the device tensor and the
        per-image lengths."""
        lens = [a.shape[0] for a in arrays]
        tail = arrays[0].shape[1:]
        total = sum(lens)
        dt = torch.from_numpy(np.zeros(1, dtype=arrays[0].dtype)).dtype
        buf = self._staging.get((key, dt))
        need = total * int(np.prod(tail)) if tail else total
        if buf is None or buf.numel() < need:
            buf = torch.empty(max(need, 1), dtype=dt)
            if device.type == "cuda" and self.conf["pin_memory"]:
                buf = buf.pin_memory()
            self._staging[(key, dt)] = buf
        view = buf[:need].view(total, *tail)
        o = 0
        npv = view.numpy()
        for a, n in zip(arrays, lens):
            npv[o:o + n] = a
            o += n
        return view.to(device, non_blocking=True), lens

    def forward(self, data):
        conf = self.conf
        device = self._device(data)
        var_names = [x[1] for x in string.Formatter().parse(conf["path"]) if x[1]]
        names = list(data["name"])
        per_key = {}
        for i, name in enumerate(names):
            fpath = conf["path"].format(**{k: data[k][i] for k in var_names})
            if conf["add_data_path"] and conf["data_root"]:
                fpath = os.path.join(conf["data_root"], fpath)
            store = self._store(fpath)
            assert name in store, f"{name} not found in {fpath}"
            for k in (conf["data_keys"] if conf["data_keys"] is not None else store.keys(name)):
                per_key.setdefault(k, []).append(store.read(name, k))
        preds = [dict() for _ in names]
        for k, arrays in per_key.items():
            flat, lens = self._stage(k, arrays, device)       # one H2D copy per key, in the stored (fp16) dtype
            if flat.is_floating_point() and self.numeric_dtype is not None:
                flat = flat.to(self.numeric_dtype)            # up-cast on the device
            o = 0
            for i, n in enumerate(lens):
                preds[i][k] = flat[o:o + n]
                o += n
        for i, pred in enumerate(preds):
            for k in list(pred.keys()):
                for pattern in conf["scale"]:
                    if k.startswith(pattern):
                        view_idx = k.replace(pattern, "")
                        scales = data["scales"] if len(view_idx) == 0 else data[f"view{view_idx}"]["scales"]
                        pred[k] = pred[k] * scales[i].to(pred[k])
            if self.padding_fn is not None:
                preds[i] = self.padding_fn(pred, conf["padding_length"])
        if conf["collate"]:
            return {k: torch.stack([p[k] for p in preds], 0) for k in preds[0]}
        assert len(preds) == 1
        return preds[0]

    def loss(self, pred, data):
        raise NotImplementedError


__main_model__ = CacheLoader
