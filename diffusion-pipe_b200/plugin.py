"""The part of the reference's model-plugin API (models/base.py:348-445, SURVEY.md 8b B-py.1) that lies OUTSIDE the hot
path, with the reference's own default behaviour, so that the unmodified driver (train.py, utils/saver.py,
utils/dataset.py) can call every method it calls on a plugin.  The hot-path methods (`prepare_inputs`, `to_layers`,
`get_loss_fn`, `configure_adapter`, `save_adapter`, `save_model`, `load_adapter_weights`, `get_param_groups`) live in the
model files."""


class PluginSurface:
    framerate = None
    pixels_round_to_multiple = 16

    def _noise_on_device(self, latents):
        """`device_prepare_inputs = true` under [model] (SURVEY.md 8(f)4): prepare_inputs draws the timesteps and the noise
        from the HOST generator exactly as the reference does (same stream, same order: bit-identical micro-batches) and
        leaves the flow-matching mix, the target and the packing to one device kernel (csrc/step_tail.cu: noise_pack) fed
        through pinned memory.  Only for host-resident latents and a CUDA model device."""
        import torch
        dev = torch.device(getattr(self, 'device', 'cpu'))
        return bool(self.model_config.get('device_prepare_inputs', False)) and dev.type == 'cuda' and latents.device.type == 'cpu'

    # ---- block swapping (models/base.py:438-445): not needed on 80 GB parts; the driver calls the prepare_* hooks
    #      around every evaluation (train.py:230-241), so they exist and do nothing, as in BasePipeline ----
    def enable_block_swap(self, blocks_to_swap):
        raise NotImplementedError('Block swapping is not implemented for this model')

    def prepare_block_swap_training(self):
        pass

    def prepare_block_swap_inference(self, disable_block_swap=False):
        pass

    # ---- latent / text-embedding caching (utils/cache.py and the VAE / text-encoder loaders stay the reference's: the
    #      north star leaves them unchanged; this engine trains from the cached tensors) ----
    def load_diffusion_model(self):
        pass

    def get_vae(self):
        raise NotImplementedError('the VAE is part of the latent-caching stage, which stays the reference\'s (utils/cache.py)')

    def get_text_encoders(self):
        raise NotImplementedError('text encoders are part of the embedding-caching stage, which stays the reference\'s')

    def get_call_vae_fn(self, vae):
        raise NotImplementedError('latent caching stays the reference\'s (utils/cache.py)')

    def get_call_text_encoder_fn(self, text_encoder):
        raise NotImplementedError('text-embedding caching stays the reference\'s (utils/cache.py)')

    def get_preprocess_media_file_fn(self):
        raise NotImplementedError('media preprocessing belongs to the caching stage, which stays the reference\'s')

    def free_vae_and_te(self):
        pass

    def load_and_fuse_adapter(self, path):
        raise NotImplementedError()

    def model_specific_dataset_config_validation(self, dataset_config):
        pass

    def get_param_groups(self, parameters):
        return [{'params': parameters}]
