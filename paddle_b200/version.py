"""paddle.version."""
# API level of the reference this build tracks (what paddle.utils.require_version checks); the framework's own version is b200_version
full_version = "3.0.0"
major, minor, patch, rc = "3", "0", "0", "0"
b200_version = "0.1.0"
cuda_version = "12.9"
cudnn_version = "none (hand-written sm_90a kernels)"
istaged = True
commit = "paddle_b200"
with_pip_cuda_libraries = "OFF"


def show():
    print(f"full_version: {full_version}\ncuda: {cuda_version}\ncudnn: {cudnn_version}\ntarget: sm_90a")


def cuda():
    return cuda_version


def cudnn():
    return cudnn_version


def nccl():
    import torch

    try:
        return ".".join(str(v) for v in torch.cuda.nccl.version())
    except Exception:
        return "0"
