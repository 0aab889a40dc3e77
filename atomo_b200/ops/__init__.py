"""sm_90a ops: host-side planning (``plan``) and the native extension loader."""
from . import plan
from ._ext import load as load_ext, available as ext_available
