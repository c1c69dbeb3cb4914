"""Checks that the .proto sources, the runtime descriptors and the hand-written
codec agree, and (when ``protoc`` exists) regenerates stock ``*_pb2.py`` files.

Counterpart of ``protobufs/generate.py`` — but the package does
not depend on generated code, so this is a verification tool, not a build step.
"""
import pathlib
import shutil
import subprocess
import sys

HERE = pathlib.Path(__file__).parent
sys.path.insert(0, str(HERE.parent))


def main() -> int:
    from pytensor_federated_b200.protocol import build_file_descriptors

    nd, sv = build_file_descriptors()
    for fd, path in ((nd, HERE / "npproto" / "ndarray.proto"), (sv, HERE / "service.proto")):
        text = path.read_text()
        for msg in fd.message_type:
            assert f"message {msg.name}" in text, (path, msg.name)
            for field in msg.field:
                assert f"{field.name} = {field.number};" in text, (path, msg.name, field.name)
        for svc in fd.service:
            for method in svc.method:
                assert f"rpc {method.name}(" in text, (path, method.name)
        print(f"{path.relative_to(HERE.parent)}: matches runtime descriptor")
    protoc = shutil.which("protoc")
    if protoc:
        out = HERE / "_generated"
        out.mkdir(exist_ok=True)
        subprocess.check_call(
            [protoc, "-I", str(HERE), f"--python_out={out}", "service.proto", "npproto/ndarray.proto"]
        )
        print(f"protoc output written to {out}")
    else:
        print("protoc not found: skipped *_pb2 generation (not needed by the package)")
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
