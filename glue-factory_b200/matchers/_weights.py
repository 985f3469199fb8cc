"""Pretrained weights by name, from local files only: the GlueStick and LightGlue plugins resolve a `weights` name the way
the reference matchers look for it on disk (gluestick.py:114-130, lightglue.py:365-382), but where the reference would
download the file, they raise FileNotFoundError listing every path they tried."""
import os
from pathlib import Path

import torch


def data_path():
    """glue-factory's DATA_PATH when `gluefactory.settings` imports, else None.  Imported on call, so that the plugins
    do not depend on glue-factory at import time."""
    try:
        from gluefactory.settings import DATA_PATH
    except ImportError:
        return None
    return Path(DATA_PATH)


def hub_checkpoint(file_name):
    """The file torch.hub.load_state_dict_from_url(url, file_name=file_name) reads from its cache."""
    return Path(torch.hub.get_dir()) / "checkpoints" / file_name


def load_weights(weights, candidates, plugin):
    """torch.load (on the CPU) the first existing file of `weights` itself, taken as a path, then `candidates`."""
    tried = [str(weights)] + [str(c) for c in candidates]
    for path in tried:
        if os.path.isfile(path):
            return torch.load(path, map_location="cpu")
    raise FileNotFoundError(f"gluefactory_b200 {plugin}: weights {str(weights)!r} not found; tried: {', '.join(tried)} "
                            "(this plugin never downloads; place the file at one of these paths or pass weights=None)")
