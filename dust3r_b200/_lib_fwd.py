"""ctypes mirror of the forward-path structures and epilogue flags of include/dust3r_b200.h ("Path 1"); the prototypes are
in _lib.PROTOTYPES."""
import ctypes as C

F_BIAS, F_GELU, F_RELU, F_OUT_F32, F_RESID_INPLACE = 1, 2, 4, 8, 16
F_ADD0, F_ADD1, F_OUT2_RELU, F_ROPE, F_OUT2_BF16 = 32, 64, 128, 256, 2048


class Linear(C.Structure):
    _fields_ = [('w', C.c_void_p), ('b', C.c_void_p)]


class Norm(C.Structure):
    _fields_ = [('g', C.c_void_p), ('b', C.c_void_p)]


class EncBlock(C.Structure):
    _fields_ = [('norm1', Norm), ('norm2', Norm), ('qkv', Linear), ('proj', Linear), ('fc1', Linear), ('fc2', Linear)]


class DecBlock(C.Structure):
    _fields_ = [('norm1', Norm), ('norm2', Norm), ('norm3', Norm), ('norm_y', Norm),
                ('qkv', Linear), ('proj', Linear), ('projq', Linear), ('projkv', Linear), ('cproj', Linear),
                ('fc1', Linear), ('fc2', Linear)]


class Fusion(C.Structure):
    _fields_ = [('rcu1_conv1', Linear), ('rcu1_conv2', Linear), ('rcu2_conv1', Linear), ('rcu2_conv2', Linear),
                ('out_conv', Linear)]


class DptHead(C.Structure):
    _fields_ = [('act_conv', Linear * 4), ('act0_up', Linear), ('act1_up', Linear), ('act3_down', Linear),
                ('layer_rn', Linear * 4), ('refine', Fusion * 4), ('head0', Linear), ('head2', Linear),
                ('head4_w', C.c_void_p), ('head4_b', C.c_void_p)]


class Model(C.Structure):
    _fields_ = [('enc_dim', C.c_int32), ('enc_depth', C.c_int32), ('enc_heads', C.c_int32), ('dec_dim', C.c_int32),
                ('dec_depth', C.c_int32), ('dec_heads', C.c_int32), ('mlp_ratio', C.c_int32), ('patch', C.c_int32),
                ('head_type', C.c_int32), ('nch', C.c_int32), ('depth_mode', C.c_int32), ('conf_mode', C.c_int32),
                ('conf_min', C.c_float), ('conf_max', C.c_float), ('ln_eps', C.c_float),
                ('hooks', C.c_int32 * 4), ('rope_max_pos', C.c_int32),
                ('rope_cos', C.c_void_p), ('rope_sin', C.c_void_p),
                ('patch_embed', Linear), ('enc', C.POINTER(EncBlock)), ('enc_norm', Norm), ('decoder_embed', Linear),
                ('dec1', C.POINTER(DecBlock)), ('dec2', C.POINTER(DecBlock)), ('dec_norm', Norm),
                ('dpt', C.POINTER(DptHead) * 2), ('lin_head', Linear * 2)]

