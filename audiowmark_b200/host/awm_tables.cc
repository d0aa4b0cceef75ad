#include "awm_tables.hh"
#include "awm_params.hh"
#include "awm_util.hh"
#include "../csrc/awm_roles.hh"

#include <algorithm>
#include <assert.h>

size_t
mark_data_frame_count()
{
  return code_size (ConvBlockType::a, Params::payload_size) * Params::frames_per_bit;
}

size_t
mark_sync_frame_count()
{
  return Params::sync_bits * Params::sync_frames_per_bit;
}

void
UpDownGen::get (int f, UpDownArray& up, UpDownArray& down)
{
  std::vector<int> bands (Params::max_band - Params::min_band + 1);
  for (size_t i = 0; i < bands.size(); i++)
    bands[i] = Params::min_band + i;
  m_random.seed (f, m_stream);              // one reseed per frame
  m_random.shuffle (bands);
  for (size_t i = 0; i < Params::bands_per_frame; i++)
    {
      up[i] = bands[i];
      down[i] = bands[Params::bands_per_frame + i];
    }
}

BitPosGen::BitPosGen (const Key& key)
{
  m_pos.resize (frames_per_block());
  for (size_t i = 0; i < m_pos.size(); i++)
    m_pos[i] = i;
  Random random (key, 0, Random::Stream::frame_position);
  random.shuffle (m_pos);
}

std::vector<MixEntry>
gen_mix_entries (const Key& key)
{
  const int frame_count = mark_data_frame_count();
  std::vector<MixEntry> entries;
  entries.reserve (frame_count * Params::bands_per_frame);
  UpDownGen up_down_gen (key, Random::Stream::data_up_down);
  BitPosGen bit_pos_gen (key);
  for (int f = 0; f < frame_count; f++)
    {
      UpDownArray up, down;
      up_down_gen.get (f, up, down);
      for (size_t i = 0; i < up.size(); i++)
        entries.push_back ({ bit_pos_gen.data_frame (f), up[i], down[i] });
    }
  /* --linear (src/wmget.cc:110-152): the same (frame, up, down) triples in generation order, no mixing */
  if (Params::mix)
    {
      Random random (key, 0, Random::Stream::mix);
      random.shuffle (entries);
    }
  return entries;
}

std::vector<unsigned>
bit_order (const Key& key, size_t n)
{
  std::vector<unsigned> order (n);
  for (size_t i = 0; i < n; i++)
    order[i] = i;
  Random random (key, 0, Random::Stream::bit_order);
  random.shuffle (order);
  return order;
}

/* bit_order of the last key asked for: a batch encodes every payload with the same key */
static const std::vector<unsigned>&
cached_bit_order (const Key& key, size_t n)
{
  static std::vector<unsigned char> c_key;
  static std::vector<unsigned> c_order;
  const std::vector<unsigned char> kb (key.aes_key(), key.aes_key() + Key::SIZE);
  if (kb != c_key || c_order.size() != n)
    {
      c_order = bit_order (key, n);
      c_key = kb;
    }
  return c_order;
}

SyncTable
gen_sync_table (const Key& key, int mode)
{
  SyncTable tab;
  const int first_block_end = frames_per_block();
  const int block_count = mode == AWM_MODE_CLIP ? 2 : 1;    // a "long" block repeats the sync pattern with up/down swapped
  UpDownGen up_down_gen (key, Random::Stream::sync_up_down);
  BitPosGen bit_pos_gen (key);
  tab.bit_offsets.push_back (0);
  for (int bit = 0; bit < Params::sync_bits; bit++)
    {
      std::vector<awm_sync_entry> bit_entries;
      for (int f = 0; f < Params::sync_frames_per_bit; f++)
        {
          const int sf = f + bit * Params::sync_frames_per_bit;
          UpDownArray up, down;
          up_down_gen.get (sf, up, down);
          for (int block = 0; block < block_count; block++)
            {
              awm_sync_entry e;
              e.frame = bit_pos_gen.sync_frame (sf) + block * first_block_end;
              const UpDownArray& u = block == 0 ? up : down;
              const UpDownArray& d = block == 0 ? down : up;
              for (size_t i = 0; i < u.size(); i++)
                {
                  e.up[i] = u[i] - Params::min_band;
                  e.down[i] = d[i] - Params::min_band;
                }
              std::sort (e.up, e.up + AWM_BANDS_PER_FRAME);
              std::sort (e.down, e.down + AWM_BANDS_PER_FRAME);
              bit_entries.push_back (e);
            }
        }
      std::sort (bit_entries.begin(), bit_entries.end(), [] (const awm_sync_entry& a, const awm_sync_entry& b) { return a.frame < b.frame; });
      tab.entries.insert (tab.entries.end(), bit_entries.begin(), bit_entries.end());
      tab.bit_offsets.push_back (tab.entries.size());
    }
  return tab;
}

std::vector<uint16_t>
gen_embed_roles (const Key& key)
{
  const size_t fpb = frames_per_block(), n_bins = Params::max_band + 1;
  std::vector<uint16_t> roles (fpb * n_bins, 0);
  bool collision = false;
  /* an up band carries the bit, a down band its inverse (init_frame_mod_vec, src/wmadd.cc:61-84) */
  auto set = [&] (int frame, int bin, bool down, bool sync, int index)
    {
      uint16_t& r = roles[frame * n_bins + bin];
      collision |= r != 0;
      r = AWM_ROLE_MARK | (down ? AWM_ROLE_DOWN : 0) | (sync ? AWM_ROLE_SYNC : 0) | (index << AWM_ROLE_SHIFT);
    };
  BitPosGen bit_pos_gen (key);
  UpDownGen sync_gen (key, Random::Stream::sync_up_down);
  for (int f = 0; f < int (mark_sync_frame_count()); f++)
    {
      UpDownArray up, down;
      sync_gen.get (f, up, down);
      for (size_t i = 0; i < up.size(); i++)
        {
          set (bit_pos_gen.sync_frame (f), up[i], false, true, f / Params::sync_frames_per_bit);
          set (bit_pos_gen.sync_frame (f), down[i], true, true, f / Params::sync_frames_per_bit);
        }
    }
  /* data frames: with mixing the coded bit of an entry follows from its position after the shuffle, not from its frame */
  const std::vector<MixEntry> entries = gen_mix_entries (key);
  for (size_t e = 0; e < entries.size(); e++)
    {
      const int bit = e / Params::bands_per_frame / Params::frames_per_bit;
      set (entries[e].frame, entries[e].up, false, false, bit);
      set (entries[e].frame, entries[e].down, true, false, bit);
    }
  if (collision)
    {
      /* sync and data frames are distinct positions of one BitPosGen permutation and up / down bands of a frame are disjoint,
       * so no entry can carry two bits; a table that does would not embed what the reference embeds */
      error ("audiowmark: embed roles: a (frame, bin) entry is assigned twice\n");
      return {};
    }
  return roles;
}

std::vector<uint8_t>
gen_coded_bits (const Key& key, const std::vector<int>& bitvec)
{
  std::vector<uint8_t> out;
  for (ConvBlockType t : { ConvBlockType::a, ConvBlockType::b })
    {
      const std::vector<int> coded = code_encode (t, bitvec);
      const std::vector<unsigned>& order = cached_bit_order (key, coded.size());
      for (size_t i = 0; i < coded.size(); i++)
        out.push_back (coded[order[i]]);                  // randomize_bit_order (encode)
    }
  return out;
}

std::vector<uint8_t>
gen_coded_bits (const std::vector<unsigned>& order, const std::vector<int>& bitvec)
{
  std::vector<uint8_t> out;
  for (ConvBlockType t : { ConvBlockType::a, ConvBlockType::b })
    {
      const std::vector<int> coded = code_encode (t, bitvec);
      assert (coded.size() == order.size());
      for (size_t i = 0; i < coded.size(); i++)
        out.push_back (coded[order[i]]);                  // randomize_bit_order (encode)
    }
  return out;
}

awm_role_layout
embed_role_layout()
{
  awm_role_layout l;
  l.sync_frames = int (mark_sync_frame_count());
  l.sync_frames_per_bit = Params::sync_frames_per_bit;
  l.data_frames = int (mark_data_frame_count());
  l.frames_per_bit = Params::frames_per_bit;
  l.mix = Params::mix ? 1 : 0;
  l.n_coded_bits = int (code_size (ConvBlockType::a, Params::payload_size));
  return l;
}

std::vector<uint8_t>
gen_frame_mod_ab (const Key& key, const std::vector<int>& bitvec)
{
  const size_t fpb = frames_per_block(), n_bins = Params::max_band + 1;
  const std::vector<uint16_t> roles = gen_embed_roles (key);
  if (roles.empty())
    return {};
  const std::vector<uint8_t> coded = gen_coded_bits (key, bitvec);
  const size_t n_coded = coded.size() / 2;
  std::vector<uint8_t> tab (2 * fpb * n_bins);
  for (int ab = 0; ab < 2; ab++)
    for (size_t i = 0; i < fpb * n_bins; i++)
      tab[ab * fpb * n_bins + i] = role_frame_mod (roles[i], ab, &coded[ab * n_coded]);
  return tab;
}

std::vector<int>
parse_payload (const std::string& bits)
{
  std::vector<int> bitvec = bit_str_to_vec (bits);
  if (bitvec.empty())
    {
      error ("audiowmark: cannot parse bits '%s'\n", bits.c_str());
      return {};
    }
  if ((Params::payload_short || Params::strict) && bitvec.size() != Params::payload_size)
    {
      error ("audiowmark: number of message bits must match payload size (%zd bits)\n", Params::payload_size);
      return {};
    }
  if (bitvec.size() > Params::payload_size)
    {
      error ("audiowmark: number of bits in message '%s' larger than payload size\n", bits.c_str());
      return {};
    }
  if (bitvec.size() < Params::payload_size)
    {
      /* short messages are repeated cyclically (disabled by --strict) */
      std::vector<int> expanded (Params::payload_size);
      for (size_t i = 0; i < expanded.size(); i++)
        expanded[i] = bitvec[i % bitvec.size()];
      bitvec = expanded;
    }
  return bitvec;
}
