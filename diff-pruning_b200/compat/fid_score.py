"""`python -m fid_score <path> <path>` as in the reference README §4 (pytorch-fid's command line), on diff_pruning_b200.fid:
images are decoded on the host with PIL, the Inception pass and the feature moments run on the GPU, the Fréchet distance on the host.

    python -m fid_score --save-stats data/cifar10_images run/fid_stats_cifar10.npz --device cuda:0 --batch-size 256
    python -m fid_score run/sample/ddpm_cifar10_pruned run/fid_stats_cifar10.npz --device cuda:0 --batch-size 256

Not covered (NotImplementedError): --res / --dataset_name crop transforms, --num-workers > 1 (decoding stays in this process), CPU
devices."""
from argparse import ArgumentDefaultsHelpFormatter, ArgumentParser

from diff_pruning_b200.fid import (  # noqa: F401
    IMAGE_EXTENSIONS, InceptionV3, calculate_activation_statistics, calculate_fid_given_paths, calculate_frechet_distance,
    compute_statistics_of_path, get_activations, save_fid_stats,
)

parser = ArgumentParser(formatter_class=ArgumentDefaultsHelpFormatter)
parser.add_argument("--batch-size", type=int, default=50, help="Batch size to use")
parser.add_argument("--dataset_name", type=str, default=None)
parser.add_argument("--num-workers", type=int, help="Number of processes to use for data loading (only 1 is implemented)")
parser.add_argument("--device", type=str, default=None, help="Device to use, like cuda or cuda:0")
parser.add_argument("--dims", type=int, default=2048, choices=list(InceptionV3.BLOCK_INDEX_BY_DIM),
                    help="Dimensionality of Inception features to use. By default, uses pool3 features")
parser.add_argument("--num_samples", type=int, default=None, help="Number of samples for FID estimation")
parser.add_argument("--res", type=int, default=None, help="Resolutions of samples for FID estimation")
parser.add_argument("--save-stats", action="store_true",
                    help="Generate an npz archive from a directory of samples. The first path is used as input and the second as output.")
parser.add_argument("path", type=str, nargs=2, help="Paths to the generated images or to .npz statistic files")


def check_args(args):
    """The options the port does not cover, refused before any work is done; returns the torch device string."""
    if args.res is not None or args.dataset_name is not None:
        raise NotImplementedError("--res / --dataset_name crop transforms are not implemented")
    if args.num_workers is not None and args.num_workers > 1:
        raise NotImplementedError("--num-workers > 1: images are decoded with PIL in this process")
    device = args.device or "cuda"
    if not device.startswith("cuda"):
        raise NotImplementedError("the Inception feature pass runs on a CUDA device only")
    return device


def main(argv=None):
    args = parser.parse_args(argv)
    device = check_args(args)
    import torch
    if ":" in device:
        torch.cuda.set_device(torch.device(device))
    if args.save_stats:
        save_fid_stats(args.path, args.batch_size, device, args.dims, num_samples=args.num_samples)
        return
    fid_value = calculate_fid_given_paths(args.path, args.batch_size, device, args.dims, num_samples=args.num_samples)
    print("FID: ", fid_value)


if __name__ == "__main__":
    main()
