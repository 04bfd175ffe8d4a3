#!/bin/bash
# the documented runtime switches still work on the final tree: model + DP tests under the stream and fusion switches
set -u
O=gpurun_out; mkdir -p $O
run() { # name, env..., -- pytest args
  name=$1; shift
  envs=()
  while [ "$1" != "--" ]; do envs+=("$1"); shift; done; shift
  env "${envs[@]}" timeout 200 python -m pytest -q -x -m gpu -p no:cacheprovider "$@" > $O/sw_$name.out 2>&1; echo "$name rc=$? $(tail -1 $O/sw_$name.out)"
}
run overlap0 AVC_OVERLAP=0 AVC_INFER_GRAPH=0 -- tests/test_gpu_model.py tests/test_gpu_dp.py
run wgstream1 AVC_WGRAD_STREAM=1 -- tests/test_gpu_model.py tests/test_gpu_dp.py tests/test_gpu_properties.py
run wgstream0 AVC_WGRAD_STREAM=0 -- tests/test_gpu_model.py -k "solver or graph"
run normbwd AVC_NORM_BWD_FUSED=1 -- tests/test_gpu_model.py -k "solver or graph or forward_backward"
