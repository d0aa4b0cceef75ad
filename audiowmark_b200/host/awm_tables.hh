// awm_tables.hh -- key / payload derived tables, built on the host and uploaded through the C ABI.
// Reference: UpDownGen (src/wmcommon.hh:91-123), BitPosGen (src/wmcommon.cc:143-165), gen_mix_entries
// (:179-202), randomize_bit_order (src/wmcommon.hh:165-185), SyncFinder::get_sync_bits
// (src/syncfinder.cc:30-77), init_frame_mod_vec (src/wmadd.cc:49-162).
#pragma once
#include <array>
#include <vector>
#include "awm_random.hh"
#include "awm_code.hh"
#include "../../include/awm_b200.h"

size_t mark_data_frame_count();
size_t mark_sync_frame_count();
inline size_t frames_per_block() { return mark_data_frame_count() + mark_sync_frame_count(); }

typedef std::array<int, 30> UpDownArray;

class UpDownGen
{
  Random::Stream m_stream;
  Random         m_random;
public:
  UpDownGen (const Key& key, Random::Stream stream) : m_stream (stream), m_random (key, 0, stream) {}
  void get (int f, UpDownArray& up, UpDownArray& down);
};

class BitPosGen
{
  std::vector<int> m_pos;
public:
  explicit BitPosGen (const Key& key);
  int sync_frame (int f) const { return m_pos[f]; }
  int data_frame (int f) const { return m_pos[f + mark_sync_frame_count()]; }
};

struct MixEntry { int frame, up, down; };
std::vector<MixEntry> gen_mix_entries (const Key& key);

/* permutation used by randomize_bit_order: encode out[i] = in[order[i]], decode out[order[i]] = in[i] */
std::vector<unsigned> bit_order (const Key& key, size_t n);
template<class T> std::vector<T>
randomize_bit_order (const Key& key, const std::vector<T>& v, bool encode)
{
  const std::vector<unsigned> order = bit_order (key, v.size());
  std::vector<T> out (v.size());
  for (size_t i = 0; i < v.size(); i++)
    if (encode) out[i] = v[order[i]]; else out[order[i]] = v[i];
  return out;
}

struct SyncTable            // get_sync_bits flattened bit-major for awm_set_sync_tables
{
  std::vector<awm_sync_entry> entries;
  std::vector<int>            bit_offsets;
};
SyncTable gen_sync_table (const Key& key, int mode /* AWM_MODE_* */);

/* role table [frames_per_block][101] for awm_set_embed_roles (codes: include/awm_b200.h); empty (with an error message) if an
 * entry would be assigned twice */
std::vector<uint16_t> gen_embed_roles (const Key& key);
/* coded data bits [2 (A, B)][n_coded] of one payload: randomize_bit_order (code_encode (A | B, bitvec)) */
std::vector<uint8_t> gen_coded_bits (const Key& key, const std::vector<int>& bitvec);
/* the same with the key's permutation given: order = bit_order (key, n_coded) */
std::vector<uint8_t> gen_coded_bits (const std::vector<unsigned>& order, const std::vector<int>& bitvec);
/* what gen_embed_roles depends on besides the key, under the current Params (awm_set_embed_roles_keys) */
awm_role_layout embed_role_layout();
/* FrameMod table [2][frames_per_block][101] for awm_set_embed_tables: 0 keep, 1 up, 2 down; roles x coded bits (empty on error) */
std::vector<uint8_t> gen_frame_mod_ab (const Key& key, const std::vector<int>& bitvec);

std::vector<int> parse_payload (const std::string& bits);   // src/wmcommon.cc:210-238
