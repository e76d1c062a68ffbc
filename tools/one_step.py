"""Three warm-up steps then exactly ONE step of the bench workload (yolov5s_city_seg, batch 16 x 512 x 1024, half mode: forward + NMS + seg
argmax) for Nsight Compute captures.  Prints, last line, the number of kernels of that one step.
    --skip-count: only print how many conv_tc launches precede the measured step (for `ncu -s`)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import bench
from multiyolov5_b200 import _lib
from multiyolov5_b200.models.yolo import Model
from multiyolov5_b200.utils.general import non_max_suppression, seg_argmax
WARM = 3
if "--skip-count" in sys.argv:
    m = Model("yolov5s_city_seg.yaml")
    from multiyolov5_b200.plan import build_plan
    pb = build_plan(m, 16, 512, 1024)
    n_tc = sum(1 for o in pb.ops if o.kind == _lib.OP_CONV and o.out.w >= 8 and o.out.h >= 2 and o.out.w * o.out.h >= 128)
    print(WARM * n_tc)
    sys.exit(0)
yml, cfg, sd = bench.make_weights("s_psp")
model = Model(yml)
model.load_state_dict(sd)
model.cuda().eval().half()
x = torch.rand(16, 3, 512, 1024, device="cuda").half()
for i in range(WARM + 1):
    (z, _), seg = model(x)
    non_max_suppression(z, 0.25, 0.45, return_padded=True)
    seg_argmax(seg, (512, 1024))
    torch.cuda.synchronize()
print(model.engine().launches() + 3)
