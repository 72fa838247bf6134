"""CPU: the vector side's field filter keeps only bits of indexed lexical fields (vector.rs:1228-1231 builds field_filter_set from the
lexical fields alone): indices past them name no field, and a filter left empty filters nothing."""
from seekstorm_b200.index import vector_field_mask


def test_bits_of_lexical_fields_are_kept():
    assert vector_field_mask(0b10, 2) == 0b10
    assert vector_field_mask(0b11, 3) == 0b11


def test_indices_past_the_lexical_fields_are_dropped():
    assert vector_field_mask(1 << 5, 2) == 0                 # field_filter=[5] on a 2-field schema: no filter, not "no row"
    assert vector_field_mask((1 << 5) | 0b01, 2) == 0b01
    assert vector_field_mask(0b1, 0) == 0                    # no lexical fields: the reference's filter set is empty


def test_bits_beyond_a_32_bit_mask_never_overflow():
    m = vector_field_mask((1 << 40) | (1 << 31) | 1, 64)
    assert m == (1 << 31) | 1 and m < 2 ** 32
