#include "awm_engine.hh"
#include "awm_params.hh"
#include "awm_util.hh"

#include <string.h>

namespace {
awm_ctx *g_ctx = nullptr;
bool     g_failed = false;
struct SlotInfo { std::vector<unsigned char> key; size_t payload_size; int frames_per_bit; bool mix; };
std::vector<SlotInfo> g_slots;
/* the FrameMod table currently on the device */
std::vector<unsigned char> g_embed_key;
std::vector<int>           g_embed_bits;
int                        g_embed_fpb_mix = -1;
/* the role table currently on the device (batched embed) */
SlotInfo                   g_roles;
bool                       g_roles_valid = false;
}

awm_ctx *
Engine::ctx()
{
  if (!g_ctx && !g_failed)
    {
      const int rc = awm_create (Params::gpu_device, &g_ctx);
      if (rc != 0 || !g_ctx)
        {
          g_failed = true;
          g_ctx = nullptr;
          error ("audiowmark: cannot create GPU context on device %d (rc=%d): a CUDA device is required, there is no CPU fallback\n",
                 Params::gpu_device, rc);
        }
    }
  return g_ctx;
}

void
Engine::shutdown()
{
  if (g_ctx)
    awm_destroy (g_ctx);
  g_ctx = nullptr;
  g_failed = false;
  g_slots.clear();
  g_embed_key.clear();
  g_embed_bits.clear();
  g_roles_valid = false;
}

std::string
Engine::last_error()
{
  return g_ctx ? awm_last_error (g_ctx) : "no GPU context";
}

int
Engine::key_slot (const Key& key)
{
  awm_ctx *c = ctx();
  if (!c)
    return -1;
  const std::vector<unsigned char> kb (key.aes_key(), key.aes_key() + Key::SIZE);
  for (size_t i = 0; i < g_slots.size(); i++)
    if (g_slots[i].key == kb && g_slots[i].payload_size == Params::payload_size && g_slots[i].frames_per_bit == Params::frames_per_bit && g_slots[i].mix == Params::mix)
      return int (i);
  if (g_slots.size() >= AWM_MAX_KEYS)
    g_slots.clear();                               // recycle: tables are cheap to rebuild
  const int slot = int (g_slots.size());
  for (int mode : { AWM_MODE_BLOCK, AWM_MODE_CLIP })
    {
      const SyncTable t = gen_sync_table (key, mode);
      if (awm_set_sync_tables (c, slot, mode, t.entries.data(), int (t.entries.size()), t.bit_offsets.data(), int (t.bit_offsets.size()) - 1))
        {
          error ("audiowmark: %s\n", awm_last_error (c));
          return -1;
        }
    }
  const std::vector<MixEntry> mix = gen_mix_entries (key);
  std::vector<awm_mix_entry> me (mix.size());
  for (size_t i = 0; i < mix.size(); i++)
    {
      me[i].frame = mix[i].frame;
      me[i].up = mix[i].up;
      me[i].down = mix[i].down;
    }
  const size_t n_coded = code_size (ConvBlockType::a, Params::payload_size);
  const std::vector<unsigned> order = bit_order (key, n_coded);
  std::vector<uint16_t> order16 (order.begin(), order.end());
  if (awm_set_mix_tables (c, slot, me.data(), int (me.size()), order16.data(), int (n_coded), Params::frames_per_bit, int (frames_per_block())))
    {
      error ("audiowmark: %s\n", awm_last_error (c));
      return -1;
    }
  g_slots.push_back ({ kb, Params::payload_size, Params::frames_per_bit, Params::mix });
  return slot;
}

bool
Engine::set_embed_tables (const Key& key, const std::vector<int>& bitvec)
{
  awm_ctx *c = ctx();
  if (!c)
    return false;
  const std::vector<unsigned char> kb (key.aes_key(), key.aes_key() + Key::SIZE);
  const int sig = int (frames_per_block()) * 2 + (Params::mix ? 1 : 0);
  if (kb == g_embed_key && bitvec == g_embed_bits && sig == g_embed_fpb_mix)
    return true;                                  // same key + payload as the previous `add`: table is already uploaded
  const std::vector<uint8_t> fm = gen_frame_mod_ab (key, bitvec);
  if (fm.empty())
    return false;
  if (awm_set_embed_tables (c, fm.data(), int (frames_per_block())))
    {
      error ("audiowmark: %s\n", awm_last_error (c));
      return false;
    }
  g_embed_key = kb;
  g_embed_bits = bitvec;
  g_embed_fpb_mix = sig;
  return true;
}

bool
Engine::set_embed_roles (const Key& key)
{
  awm_ctx *c = ctx();
  if (!c)
    return false;
  const std::vector<unsigned char> kb (key.aes_key(), key.aes_key() + Key::SIZE);
  const SlotInfo sig { kb, Params::payload_size, Params::frames_per_bit, Params::mix };
  if (g_roles_valid && g_roles.key == sig.key && g_roles.payload_size == sig.payload_size && g_roles.frames_per_bit == sig.frames_per_bit &&
      g_roles.mix == sig.mix)
    return true;                                  // same key and layout as the previous batch: roles are already uploaded
  const std::vector<uint16_t> roles = gen_embed_roles (key);
  if (roles.empty())
    return false;
  if (awm_set_embed_roles (c, roles.data(), int (frames_per_block()), int (code_size (ConvBlockType::a, Params::payload_size))))
    {
      error ("audiowmark: %s\n", awm_last_error (c));
      return false;
    }
  g_roles = sig;
  g_roles_valid = true;
  return true;
}

bool
Engine::is_device_pointer (const void *p)
{
  return p && awm_is_device_pointer (p) != 0;
}
