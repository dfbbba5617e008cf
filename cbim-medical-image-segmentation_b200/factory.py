"""``get_model(args, pretrain=False)`` with the reference's dispatch (model/utils.py:6-125) for the
models of the hot path.  Anything the H100 path does not implement is a hard ValueError — never a
silent hand-off to stock PyTorch."""


def get_model(args, pretrain=False):
    if args.dimension == '3d':
        if args.model in ('unet', 'resunet'):
            from .unet3d import UNet
            if pretrain and args.model == 'resunet':
                raise ValueError('No pretrain model available')   # model/utils.py:77-78
            return UNet(args.in_chan, args.base_chan, num_classes=args.classes, scale=args.down_scale,
                        norm=args.norm, kernel_size=args.kernel_size, block=args.block)
        if args.model == 'unet++':
            from .unetpp import UNetPlusPlus
            if pretrain:
                raise ValueError('No pretrain model available')   # model/utils.py:14-17
            return UNetPlusPlus(args.in_chan, args.base_chan, num_classes=args.classes, scale=args.down_scale,
                                norm=args.norm, kernel_size=args.kernel_size, block=args.block)   # :87
        if args.model == 'attention_unet':
            from .attention_unet import AttentionUNet       # the 3d branch has no pretrain check (model/utils.py:88-90)
            return AttentionUNet(args.in_chan, args.base_chan, num_classes=args.classes, scale=args.down_scale,
                                 norm=args.norm, kernel_size=args.kernel_size, block=args.block)
        if args.model == 'medformer':
            from .medformer import MedFormer
            if pretrain:
                raise ValueError('No pretrain model available')   # model/utils.py:92-93
            return MedFormer(args.in_chan, args.classes, args.base_chan, map_size=args.map_size,
                             conv_block=args.conv_block, conv_num=args.conv_num, trans_num=args.trans_num,
                             num_heads=args.num_heads, fusion_depth=args.fusion_depth, fusion_dim=args.fusion_dim,
                             fusion_heads=args.fusion_heads, expansion=args.expansion, attn_drop=args.attn_drop,
                             proj_drop=args.proj_drop, proj_type=args.proj_type, norm=args.norm, act=args.act,
                             kernel_size=args.kernel_size, scale=args.down_scale, aux_loss=args.aux_loss)   # :95
        if args.model == 'swin_unetr':
            from .swin_unetr import SwinUNETR
            if getattr(args, 'pretrain', False) or pretrain:
                raise ValueError('No pretrain model available')   # model/utils.py:113-115 loads a site-local file
            return SwinUNETR(args.window_size, args.in_chan, args.classes, feature_size=args.base_chan)   # :111
        if args.model == 'unetr':
            from .unetr import UNETR                        # no pretrain check, as in the reference
            return UNETR(args.in_chan, args.classes, args.training_size, feature_size=16, hidden_size=768, mlp_dim=3072,
                         num_heads=12, pos_embed='perceptron', norm_name='instance', res_block=True)
        raise ValueError("model %r (3d) is not implemented by the H100 path" % (args.model,))
    if args.dimension == '2d':
        if args.model in ('unet', 'resunet'):
            from .unet2d import UNet2D
            if pretrain:
                raise ValueError('No pretrain model available')   # model/utils.py:11-12
            return UNet2D(args.in_chan, args.classes, args.base_chan, block=args.block)
        raise ValueError("model %r (2d) is not implemented by the H100 path (2d: unet, resunet)" % (args.model,))
    raise ValueError("Invalid dimension, should be '2d' or '3d'")
