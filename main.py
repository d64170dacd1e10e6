"""CLI of the H100-native video-feature engine: the flags of the reference's main.py (main.py:93-149), same names,
defaults and choices.  ``--device_ids`` starts one process per GPU (reference: one thread per GPU); ``--cpu`` is
refused -- the reference's CPU path is what ``bench.py --impl reference`` times, the engine itself has no CPU path.
Beyond the reference: ``--gather_features`` (one all-gather of every GPU's features into one .npz) and the ``s3d``
feature type (torchvision's S3D, the Kinetics-400 clip feature upstream video_features added later), the first choice
outside the reference's list, and the ``CLIP-ViT-L/14`` / ``CLIP-ViT-L/14@336px`` feature types (openai's largest
released ViT, 768-d features), which the reference does not offer either; ``--model_name`` selects upstream's IG65M
R(2+1)D-34 models for ``r21d_rgb``; ``swin3d_t`` / ``swin3d_s`` / ``swin3d_b`` are torchvision's Swin3D video
transformers and ``mvit_v1_b`` / ``mvit_v2_s`` its Multiscale Vision Transformers (Kinetics-400 clip features);
``dinov2_vit{s,b,l,g}14`` and their ``_reg`` variants are DINOv2's self-supervised ViTs (per-frame features, the hub
model's class token after its final norm); ``videomae_vit{s,b,l}16`` are the Kinetics-400 fine-tuned VideoMAE models in
Hugging Face's layout (clip features, the classifier's input).
``--show_pred`` on the CLIP feature types is upstream video_features' zero-shot prediction: every frame's image feature
against the text features of ``--pred_texts`` (default: "a photo of {name}" for the Kinetics-400 classes).
"""
import argparse
import functools

import numpy  # noqa: F401  (kept first, as in the reference)
import torch  # noqa: F401

from video_features_b200.utils import form_list_from_user_input, sanity_check

SUPPORTED = ['i3d', 'raft', 'pwc', 'CLIP-ViT-B/32', 'CLIP-ViT-B/16', 'CLIP4CLIP-ViT-B-32', 'resnet18', 'resnet34', 'resnet50',
             'resnet101', 'resnet152', 'r21d_rgb', 'vggish_torch', 's3d', 'CLIP-ViT-L/14', 'CLIP-ViT-L/14@336px',
             'swin3d_t', 'swin3d_s', 'swin3d_b', 'mvit_v1_b', 'mvit_v2_s', 'dinov2_vits14', 'dinov2_vitb14',
             'dinov2_vitl14', 'dinov2_vitg14', 'dinov2_vits14_reg', 'dinov2_vitb14_reg', 'dinov2_vitl14_reg',
             'dinov2_vitg14_reg', 'videomae_vits16', 'videomae_vitb16', 'videomae_vitl16']


def build_extractor(args):
    """feature_type -> extractor (main.py:15-41)."""
    if args.feature_type in ['CLIP-ViT-B/32', 'CLIP-ViT-B/16', 'CLIP4CLIP-ViT-B-32', 'CLIP-ViT-L/14', 'CLIP-ViT-L/14@336px']:
        from video_features_b200.extract.extract_clip import ExtractCLIP
        return ExtractCLIP(args)
    if args.feature_type == 'i3d':
        from video_features_b200.extract.extract_i3d import ExtractI3D
        return ExtractI3D(args)
    if args.feature_type == 'raft':
        from video_features_b200.extract.extract_raft import ExtractRAFT
        return ExtractRAFT(args)
    if args.feature_type == 'pwc':
        from video_features_b200.extract.extract_pwc import ExtractPWC
        return ExtractPWC(args)
    if args.feature_type in ['resnet18', 'resnet34', 'resnet50', 'resnet101', 'resnet152']:
        from video_features_b200.extract.extract_resnet import ExtractResNet
        return ExtractResNet(args)
    if args.feature_type == 'r21d_rgb':
        from video_features_b200.extract.extract_r21d import ExtractR21D
        return ExtractR21D(args)
    if args.feature_type == 's3d':
        from video_features_b200.extract.extract_s3d import ExtractS3D
        return ExtractS3D(args)
    if args.feature_type in ['swin3d_t', 'swin3d_s', 'swin3d_b']:
        from video_features_b200.extract.extract_swin3d import ExtractSwin3D
        return ExtractSwin3D(args)
    if args.feature_type in ['mvit_v1_b', 'mvit_v2_s']:
        from video_features_b200.extract.extract_mvit import ExtractMViT
        return ExtractMViT(args)
    if args.feature_type.startswith('dinov2_'):
        from video_features_b200.extract.extract_dinov2 import ExtractDINOv2
        return ExtractDINOv2(args)
    if args.feature_type in ['videomae_vits16', 'videomae_vitb16', 'videomae_vitl16']:
        from video_features_b200.extract.extract_videomae import ExtractVideoMAE
        return ExtractVideoMAE(args)
    if args.feature_type == 'vggish_torch':
        from video_features_b200.extract.extract_vggish import ExtractVGGish
        return ExtractVGGish(args)
    if args.feature_type == 'vggish':
        raise NotImplementedError('vggish: the TF1 VGGish (a TF .ckpt, PCA and 8-bit quantisation) is not built; '
                                  'use vggish_torch')
    raise NotADirectoryError                      # main.py:41


def _pin_path_list(args):
    """Resolve the user's listing ONCE, here in the parent: every worker then sees the same list in the same order (a
    directory glob is unordered, and shard r is only meaningful against one enumeration).  Returns the list."""
    paths = form_list_from_user_input(args)
    if paths and isinstance(paths[0], tuple):
        args.video_paths, args.flow_paths = [p[0] for p in paths], [p[1] for p in paths]
    else:
        args.video_paths, args.flow_paths = list(paths), None
    args.file_with_video_paths = args.video_dir = args.flow_dir = None
    return paths


def _save_gathered(target, blocks):
    """--gather_features: every video's feature block, list order, in one .npz (rows + per-video row counts)."""
    import numpy as np
    rows = np.concatenate([b.numpy() for b in blocks]) if blocks else np.zeros((0, 0), np.float32)
    np.savez(target, features=rows, rows_per_video=np.array([b.shape[0] for b in blocks], dtype=np.int64))
    print(f'gathered {len(blocks)} feature blocks ({rows.shape[0]} rows) -> {target}')


def parallel_feature_extraction(args):
    from video_features_b200.dispatch import parallel_feature_extraction as run
    video_paths = _pin_path_list(args)
    gather = getattr(args, 'gather_features', None)
    key = {'i3d': (args.streams or ['rgb'])[0]}.get(args.feature_type, args.feature_type)
    run(functools.partial(build_extractor, args), len(video_paths), args.device_ids,
        gather_key=key if gather else None, on_gathered=functools.partial(_save_gathered, gather) if gather else None)


_FEATURE_TYPES = ('i3d vggish r21d_rgb resnet18 resnet34 resnet50 resnet101 resnet152 raft pwc CLIP-ViT-B/32 CLIP-ViT-B/16 '
                  'CLIP4CLIP-ViT-B-32 vggish_torch s3d CLIP-ViT-L/14 CLIP-ViT-L/14@336px swin3d_t swin3d_s swin3d_b mvit_v1_b mvit_v2_s '
                  'dinov2_vits14 dinov2_vitb14 dinov2_vitl14 dinov2_vitg14 dinov2_vits14_reg dinov2_vitb14_reg '
                  'dinov2_vitl14_reg dinov2_vitg14_reg videomae_vits16 videomae_vitb16 videomae_vitl16').split()

# (flag, argparse keywords): names, types, defaults, choices and dests are the reference's (main.py:93-149)
_FLAGS = [
    ('--feature_type', dict(required=True, choices=_FEATURE_TYPES, help='which extractor to run')),
    ('--video_paths', dict(nargs='+', help='videos to process')),
    ('--flow_paths', dict(nargs='+', help='folders of precomputed flow images, one per video (I3D --flow_type flow)')),
    ('--file_with_video_paths', dict(help='text file, one video path per line')),
    ('--video_dir', dict(type=str, help='directory whose files are all processed')),
    ('--flow_dir', dict(type=str, help='root of <video id>/flow_{x,y}_NNNNNN.jpg trees')),
    ('--device_ids', dict(type=int, nargs='+', help='GPUs to use: one process per id')),
    ('--cpu', dict(action='store_true', help='accepted for compatibility; refused at run time')),
    ('--tmp_path', dict(default='./tmp', help='scratch folder')),
    ('--keep_tmp_files', dict(dest='keep_tmp_files', action='store_true', default=False, help='keep the scratch files')),
    ('--on_extraction', dict(default='print', choices=['print', 'save_numpy', 'save_pickle'], help='sink of the features')),
    ('--output_path', dict(default='./output', help='root of the saved features')),
    ('--output_direct', dict(action='store_true', help='save as <output_path>/<video stem>.npy')),
    ('--extraction_fps', dict(type=float, help='resample to this frame rate first (I3D)')),
    ('--extract_method', dict(type=str, help='frame sampler: uni_N or fix_N')),
    # upstream video_features' model choice for r21d_rgb; None means r2plus1d_18_16_kinetics, so that sanity_check can
    # refuse the flag for other feature types
    ('--model_name', dict(choices=['r2plus1d_18_16_kinetics', 'r2plus1d_34_32_ig65m_ft_kinetics',
                                   'r2plus1d_34_8_ig65m_ft_kinetics'], default=None,
                          help='r21d_rgb network (default r2plus1d_18_16_kinetics; the R(2+1)D-34 IG65M models default '
                               'to 32 / 32 and 8 / 8 frame stacks)')),
    ('--stack_size', dict(type=int, help='frames per I3D / R(2+1)D / S3D / Swin3D stack (MViT: 16 only)')),
    ('--step_size', dict(type=int, help='frames between I3D / R(2+1)D / S3D / Swin3D / MViT stacks')),
    ('--streams', dict(nargs='+', choices=['flow', 'rgb'], help='I3D streams (default: both)')),
    ('--flow_type', dict(choices=['raft', 'pwc', 'flow'], default='pwc', help='optical flow feeding the I3D flow stream')),
    ('--batch_size', dict(type=int, default=1, help='frame pairs per RAFT call')),
    ('--resize_to_larger_edge', dict(dest='resize_to_smaller_edge', action='store_false', default=True,
                                    help='--side_size applies to the larger edge instead of the smaller one')),
    ('--side_size', dict(type=int, help='RAFT: resize frames to this edge length first')),
    ('--show_pred', dict(dest='show_pred', action='store_true', default=False,
                         help='print the top-5 classes of every feature (I3D, R(2+1)D, S3D, Swin3D, MViT: Kinetics-400; ResNet: '
                              'ImageNet; CLIP: zero-shot over --pred_texts; not DINOv2, whose checkpoints have no '
                              'classifier)')),
    ('--pred_texts', dict(nargs='+', default=None,
                          help='CLIP --show_pred: the prompts each frame is compared with (default: "a photo of {name}" '
                               'for the 400 Kinetics-400 classes; needs the BPE vocabulary bpe_simple_vocab_16e6.txt.gz '
                               'in $VF_CLIP_BPE, extract/checkpoints/ or ~/.cache/clip/)')),
    # not in the reference: after extraction, ONE all-gather (NCCL over NVLink) returns every rank's feature blocks and
    # rank 0 writes them, list order, to this .npz
    ('--gather_features', dict(type=str, default=None, help='also all-gather the features of all GPUs into this .npz')),
]


def make_parser():
    parser = argparse.ArgumentParser(description='H100-native video feature extraction')
    for flag, kw in _FLAGS:
        parser.add_argument(flag, **kw)
    return parser


if __name__ == "__main__":
    args = make_parser().parse_args()
    if args.on_extraction != 'print':
        print(f'features -> {args.output_path}')
    if args.keep_tmp_files:
        print(f'scratch files stay in {args.tmp_path}')
    sanity_check(args)
    if args.show_pred and args.feature_type in ('raft', 'pwc'):
        # the reference shows the flow in a cv2.imshow window; this engine ships headless OpenCV
        print(f'--show_pred: ignored for {args.feature_type} (the reference shows flow in a GUI window)')
    if args.cpu:
        raise SystemExit('--cpu: this engine has no CPU path (the reference CPU flow is timed by '
                         '`python bench.py --impl reference`); pass --device_ids')
    if not args.device_ids:
        args.device_ids = [0]
    parallel_feature_extraction(args)
