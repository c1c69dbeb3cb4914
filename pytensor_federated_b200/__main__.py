"""``python -m pytensor_federated_b200 [info|build|serve-demo]`` — small operator CLI.

* ``info``  — version, native library, graph backend, visible GPUs, TLS / metrics configuration.
* ``build`` — compile ``libb200fed.so`` for sm_90a (same as ``python -m pytensor_federated_b200.build``).
"""
from __future__ import annotations

import argparse
import json
import os
import sys


def collect_info() -> dict:
    from . import __version__
    from ._graph_backend import BACKEND
    from .config import get_config, tls_from_env
    from .ops import native

    info = {"version": __version__, "graph_backend": BACKEND, "python": sys.version.split()[0]}
    lib = native.LIB_PATH
    info["native_library"] = {"path": str(lib), "built": lib.exists()}
    if lib.exists():
        try:
            handle = native.load(build_if_missing=False)
            info["native_library"]["cuda_devices"] = int(handle.b200_device_count())
        except native.NativeError as ex:
            info["native_library"]["error"] = str(ex)
    try:
        import torch

        info["torch"] = torch.__version__
        info["gpus"] = [torch.cuda.get_device_name(i) for i in range(torch.cuda.device_count())]
    except ImportError:
        info["torch"] = None
    cfg = get_config()
    info["config"] = {k: getattr(cfg, k) for k in ("comm", "multicast", "glm_kernel", "timeout", "idle_timeout", "serve_ahead", "speculative_us")}
    tls = tls_from_env()
    info["tls"] = None if tls is None else {"ca": bool(tls.ca), "cert": bool(tls.cert), "mutual": tls.mutual,
                                            "server_name": tls.server_name}
    info["metrics_port"] = os.environ.get("B200FED_METRICS_PORT")
    return info


def main(argv=None) -> int:
    parser = argparse.ArgumentParser(prog="python -m pytensor_federated_b200")
    sub = parser.add_subparsers(dest="command")
    sub.add_parser("info", help="print the installation / configuration summary as JSON")
    b = sub.add_parser("build", help="compile the native library for sm_90a")
    b.add_argument("--force", action="store_true")
    args = parser.parse_args(argv)
    if args.command == "build":
        from . import build as native_build

        print(native_build.build(force=args.force))
        return 0
    print(json.dumps(collect_info(), indent=2))
    return 0


if __name__ == "__main__":
    sys.exit(main())
