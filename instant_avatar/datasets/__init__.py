"""alias of the dataset modules (instantavatar_b200.data)"""
