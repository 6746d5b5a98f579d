#!/usr/bin/env bash
# Builds libvqcuda.so for sm_90a IN-TREE (vqengine_b200/libvqcuda.so). No GPU needed (cross-compile).
set -euo pipefail
here="$(cd "$(dirname "$0")" && pwd)"
out="${VQ_OUT:-$here/../libvqcuda.so}"
NVCC="${NVCC:-/usr/local/cuda/bin/nvcc}"
FLAGS=(-gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 --shared -Xcompiler -fPIC,-fvisibility=hidden
       -Xptxas -v --expt-relaxed-constexpr -t 0)
"$NVCC" "${FLAGS[@]}" -o "$out" "$here"/vq_context.cu "$here"/vq_post.cu "$here"/vq_forward.cu "$here"/vq_ibl.cu "$here"/vq_host.cu "$here"/vq_surface.cu "$here"/vq_frame.cu "$here"/vq_shadow.cu "$here"/vq_group.cu "$@"
echo "built $out"
