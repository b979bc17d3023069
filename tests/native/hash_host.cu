/* Host build of the hash functions the kernels inline (cloudberry_b200/csrc/common.cuh, the __host__ __device__ ones: the same
 * source text nvcc compiles into every join / aggregate / Motion kernel).  Test harness only: compiled by
 * tests/test_device_hash_source.py with nvcc (host side of the translation unit) and compared with the reference's own
 * hashfunc.c / varchar.c / cdbhash.c / hashfn.h as compiled into oracle/_ref/libexec_ref.so.  The join table's slot format
 * helpers (ht_*) are the same kind of source and are tested here too. */
#include "../../cloudberry_b200/csrc/common.cuh"

extern "C" {
uint32_t	hh_hash_uint32(uint32_t k) { return pg_hash_uint32(k); }
uint32_t	hh_hashint8(int64_t v) { return pg_hashint8(v); }
uint32_t	hh_hashfloat8(uint64_t bits) { return pg_hashfloat8(bits); }
uint32_t	hh_hash_bpchar1(uint8_t ch) { return pg_hash_bpchar1(ch); }
uint32_t	hh_hash_bytes(const unsigned char *k, int len) { return pg_hash_bytes_host(k, len); }
uint32_t	hh_murmurhash32(uint32_t h) { return pg_murmurhash32(h); }
uint32_t	hh_hash_combine(uint32_t acc, uint32_t h, int isnull) { return pg_hash_combine(acc, h, isnull != 0); }
int32_t		hh_jump_consistent_hash(uint64_t key, int32_t nseg) { return pg_jump_consistent_hash(key, nseg); }
uint32_t	hh_jh_int8(int64_t v) { return jh_int8(v); }
uint32_t	hh_jh_mix32(uint32_t x) { return jh_mix32(x); }
int			hh_key_in_domain(int32_t keyslot, int64_t key) { return ht_key_in_domain(keyslot, key); }
uint32_t	hh_probe_tag(int32_t keyslot, uint32_t hash, int64_t key0) { return ht_probe_tag(keyslot, hash, key0); }
uint64_t	hh_slot_entry(uint32_t tag, uint32_t row) { return ht_slot_entry(tag, row); }
int			hh_slot_empty(uint64_t e) { return ht_slot_empty(e); }
uint32_t	hh_slot_row(uint64_t e) { return ht_slot_row(e); }
int			hh_tag_match(uint64_t e, uint32_t tag) { return ht_tag_match(e, tag); }
int64_t		hh_group_key(int type, int64_t v) { return agg_group_key(type, v); }
uint32_t	hh_group_hash(int n, const int32_t *types, const uint32_t *const *dicts, const int64_t *keys, uint32_t knull)
{ return agg_group_hash(n, types, dicts, keys, knull); }
int32_t		hh_cdb_route(int n, const int32_t *types, const uint32_t *const *dicts, const int64_t *keys, uint32_t knull, int32_t nsegs)
{ return cdb_route(n, types, dicts, keys, knull, nsegs); }
int64_t		hh_add_ovf(int64_t x, int64_t y, int *ovf) { bool o; int64_t r = i64_add_ovf(x, y, &o); *ovf = o; return r; }
int64_t		hh_sub_ovf(int64_t x, int64_t y, int *ovf) { bool o; int64_t r = i64_sub_ovf(x, y, &o); *ovf = o; return r; }
int64_t		hh_mul_ovf(int64_t x, int64_t y, int *ovf) { bool o; int64_t r = i64_mul_ovf(x, y, &o); *ovf = o; return r; }
}
