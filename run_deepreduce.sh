#!/usr/bin/env bash
# Launch recipes mirroring the reference's run_deepreduce.sh (OpenMPI/TCP, 1 GPU per host) on one 8-GPU H100 box:
# one process per GPU via torchrun, NCCL bootstrap, fused P2P exchange.  Data is synthetic.
N=${N:-8}
RUN="python -m torch.distributed.run --nnodes=1 --nproc-per-node $N --master-addr 127.0.0.1 --master-port ${PORT:-29400} -m deepreduce_b200.cli"

### ResNet-20 / CIFAR-shape: data volume and micro-benchmark (reference run_deepreduce.sh:26-35)
$RUN -a resnet20 --batch-size 256 --steps 50 --log_volume \
  --grace_config="{'compressor': 'topk', 'memory': 'residual', 'communicator': 'allgather', 'compress_ratio': 0.01, 'deepreduce':'index', 'index':'bloom', 'micro-benchmark':True}"

### ResNet-50 / ImageNet-shape, bloom index and 'both'
$RUN -a resnet50 --batch-size 256 --steps 50 --log_volume --log_time \
  --grace_config="{'compressor': 'topk', 'memory': 'residual', 'communicator': 'allgather', 'compress_ratio': 0.01, 'deepreduce':'index', 'index':'bloom'}"
$RUN -a resnet50 --batch-size 256 --steps 50 --log_volume --log_time \
  --grace_config="{'compressor': 'topk', 'memory': 'residual', 'communicator': 'allgather', 'compress_ratio': 0.01, 'deepreduce':'both', 'index':'bloom', 'value':'polyfit'}"

### NCF (MovieLens-20M shapes): dense baseline, inherently-sparse threshold variants (reference :37-74)
$RUN -a ncf --batch-size 131072 --steps 20 --weak_scaling --log_volume \
  --grace_config="{'compressor': 'none', 'memory': 'none', 'communicator': 'allreduce'}"
$RUN -a ncf --batch-size 131072 --steps 20 --weak_scaling --log_volume \
  --grace_config="{'compressor': 'threshold', 'memory': 'none', 'communicator': 'allgather', 'threshold': 0.0, 'deepreduce':'index', 'index':'bloom', 'policy':'p0', 'fpr':0.01}"
$RUN -a ncf --batch-size 131072 --steps 20 --weak_scaling --log_volume \
  --grace_config="{'compressor': 'threshold', 'memory': 'none', 'communicator': 'allgather', 'threshold': 0.0, 'deepreduce':'both', 'index':'bloom', 'policy':'random', 'fpr':0.01, 'value':'qsgd', 'bucket_size':512, 'quantum_num': 32}"

### NCF time breakdown with gradient accumulation (reference :92-107)
$RUN -a ncf --batch-size 131072 --steps 30 --weak_scaling --grads_accumulated=10 --log_time \
  --grace_config="{'compressor': 'topk', 'memory': 'residual', 'communicator': 'allgather', 'compress_ratio': 0.1, 'deepreduce':'index', 'index':'bloom'}"
