#!/bin/bash
# Host-side robustness run (no GPU): the file readers, the container quantiser, the tokenizer / samplers and the image decoders are compiled
# stand-alone with AddressSanitizer + UndefinedBehaviorSanitizer and fed damaged inputs.     bash tools/asan_fuzz.sh [iterations-scale]
set -e
cd "$(dirname "$0")/.."
S=${1:-1}; W=/tmp/mg4fuzz; mkdir -p $W
C=minigpt4_cpp_b200/csrc
CXX="g++ -std=c++17 -O1 -g -fsanitize=address,undefined -fno-sanitize-recover=all -I$C -I/usr/local/cuda/include"
CUDART="-L/usr/local/cuda/lib64 -lcudart_static -ldl -lrt -lpthread"
python - <<PY
import numpy as np
from PIL import Image
from minigpt4_cpp_b200 import modelgen as mg
rng = np.random.default_rng(0)
yy, xx = np.mgrid[0:48, 0:64]
arr = (np.stack([128 + 100 * np.sin(xx / 7.0), 128 + 90 * np.cos(yy / 5.0), (xx * 3 + yy * 5) % 256], -1) + rng.normal(0, 10, (48, 64, 3))).clip(0, 255).astype(np.uint8)
Image.fromarray(arr).save("$W/good.png"); Image.fromarray(arr[..., 0]).convert("P").save("$W/pal.png")
Image.fromarray(arr).save("$W/b.jpg", quality=80, subsampling=2); Image.fromarray(arr).save("$W/p.jpg", quality=80, subsampling=1, progressive=True)
Image.fromarray(arr).save("$W/r.jpg", quality=80, subsampling=2, restart_marker_blocks=2)
mg.write_llama_ggjt("$W/l.bin", mg.LlamaSpec(n_vocab=300, n_embd=128, n_head=1, n_layer=1, wtype="q4_1"))
mg.write_minigpt4("$W/v.bin", mg.VisionSpec(n_blocks=1, n_qformer_layers=1, n_embd_llm=4096))
PY
$CXX tools/fuzz/fuzz_png.cpp $C/image.cpp $C/jpeg.cpp -lz -lpthread -o $W/fuzz_png
$CXX tools/fuzz/fuzz_jpeg.cpp $C/jpeg.cpp $C/image.cpp -lpthread -o $W/fuzz_jpeg
$CXX tools/fuzz/fuzz_resize.cpp $C/image.cpp $C/jpeg.cpp -lpthread -o $W/fuzz_resize
$CXX tools/fuzz/fuzz_readers.cpp $C/formats.cpp $CUDART -o $W/fuzz_readers
$CXX tools/fuzz/fuzz_text.cpp $C/text.cpp $C/formats.cpp $CUDART -o $W/fuzz_text
$CXX tools/fuzz/fuzz_quantize.cpp $C/quantize.cpp $C/formats.cpp $CUDART -o $W/fuzz_quantize
echo "== PNG decoder (mutated chunks, checksums re-computed)"; $W/fuzz_png $W/good.png 1 $((20000*S)); $W/fuzz_png $W/pal.png 2 $((20000*S))
echo "== JPEG decoder (baseline / progressive / restart intervals)"; $W/fuzz_jpeg $W/b.jpg 1 $((20000*S)); $W/fuzz_jpeg $W/p.jpg 2 $((20000*S)); $W/fuzz_jpeg $W/r.jpg 3 $((20000*S))
echo "== bicubic resize, degenerate shapes"; $W/fuzz_resize | tail -3
echo "== ggjt v3 reader"; $W/fuzz_readers l $W/l.bin 5 $((4000*S))
echo "== MiniGPT-4 container reader"; $W/fuzz_readers v $W/v.bin 6 $((300*S))
echo "== container quantiser"; $W/fuzz_quantize $W/v.bin 3 $((60*S))
echo "== tokenizer + sampler chain (NaN / inf logits, wild parameters)"; $W/fuzz_text
echo "clean"
