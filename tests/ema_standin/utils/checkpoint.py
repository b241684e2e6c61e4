"""utils/checkpoint.py:16-23, 85-106, 109-137 restated: the torch.amp branch (loss_scaler is not None) of save_model and
auto_load_model, with the EMA entry 'model_ema' = get_state_dict(model_ema), and _load_checkpoint_for_ema."""
import glob
import io
import os
from pathlib import Path

import torch

from .model import get_state_dict


def _load_checkpoint_for_ema(model_ema, checkpoint):
    buf = io.BytesIO()
    torch.save(checkpoint, buf)
    buf.seek(0)
    model_ema._load_checkpoint(buf)


def save_model(args, epoch, model, model_without_ddp, optimizer, loss_scaler, loss_balancer=None, model_ema=None):
    to_save = {'model': model_without_ddp.state_dict(), 'optimizer': optimizer.state_dict(), 'epoch': epoch,
               'scaler': loss_scaler.state_dict(), 'args': args}
    if loss_balancer is not None:
        to_save['loss_balancer'] = loss_balancer.state_dict()
    if model_ema is not None:
        to_save['model_ema'] = get_state_dict(model_ema)
    torch.save(to_save, Path(args.output_dir) / ('checkpoint-%s.pth' % epoch))


def auto_load_model(args, model, model_without_ddp, optimizer, loss_scaler, model_ema=None):
    if args.auto_resume and len(args.resume) == 0:
        found = [ckpt.split('-')[-1].split('.')[0] for ckpt in glob.glob(os.path.join(args.output_dir, 'checkpoint-*.pth'))]
        latest = max([int(t) for t in found if t.isdigit()], default=-1)
        if latest >= 0:
            args.resume = os.path.join(args.output_dir, 'checkpoint-%d.pth' % latest)
        print("Auto resume checkpoint: %s" % args.resume)
    if args.resume:
        checkpoint = torch.load(args.resume, map_location='cpu')
        model_without_ddp.load_state_dict(checkpoint['model'])
        print("Resume checkpoint %s" % args.resume)
        if 'optimizer' in checkpoint and 'epoch' in checkpoint:
            optimizer.load_state_dict(checkpoint['optimizer'])
            args.start_epoch = checkpoint['epoch'] + 1
            if hasattr(args, 'model_ema') and args.model_ema:
                _load_checkpoint_for_ema(model_ema, checkpoint['model_ema'])
            if 'scaler' in checkpoint:
                loss_scaler.load_state_dict(checkpoint['scaler'])
            print("With optim & sched!")
